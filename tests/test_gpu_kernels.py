"""Per-kernel parity on the H100: each C-ABI kernel against the CPU oracle / an fp64 torch reference."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from oracle import diffsound_oracle as O  # noqa: E402
from tests import sampler_reference as R  # noqa: E402
from tests.helpers import load_golden, sampler_case_inputs  # noqa: E402


@pytest.fixture(scope="module")
def G():
    from tests import gpu_common
    return gpu_common


def test_device_is_hopper(G):
    sms, major, minor = G.ops.device_info()
    assert (major, minor) == (9, 0), f"expected sm_90, got sm_{major}{minor}"
    assert sms >= 100


def test_round_tf32_and_silu(G):
    x = torch.randn(100003, device="cuda") * 3
    assert torch.equal(G.ops.round_tf32(x.clone()), G.tf32_round_ref(x))
    x = torch.randn(4096, device="cuda")
    assert (G.ops.silu(x) - F.silu(x)).abs().max() < 1e-6


def test_embed_tokens_matches_oracle(G):
    sd = O.make_transformer_state_dict(K=32, D=128, n_layer=1, n_head=2, cond_dim=64)
    ids = torch.randint(0, 33, (3, 265))
    ref = O.content_embedding(sd, "transformer.content_emb.", ids, (5, 53))
    p = "transformer.content_emb."
    out = G.ops.embed_tokens(ids.cuda(), sd[p + "emb.weight"].cuda(), sd[p + "height_emb.weight"].cuda(), sd[p + "width_emb.weight"].cuda())
    assert torch.equal(out.cpu(), ref)  # exact: same three-term fp32 sum in the reference's order


def test_layernorm_and_adaln_match_oracle(G):
    D, B, L, T = 256, 3, 265, 100
    sd = O.make_transformer_state_dict(K=32, D=D, n_layer=1, n_head=4, cond_dim=64)
    x = torch.randn(B, L, D) * 2 + 0.3
    g, b = sd["transformer.blocks.0.ln2.weight"], sd["transformer.blocks.0.ln2.bias"]
    ref = F.layer_norm(x, (D,), g, b)
    out = G.ops.layernorm(x.cuda(), g.cuda(), b.cuda())
    assert G.relerr(out, ref) < 2e-6
    t = torch.tensor([99, 0, 41])
    ref = O.ada_layer_norm(sd, "transformer.blocks.0.ln1.", x, t)
    p = "transformer.blocks.0.ln1."
    table = F.linear(F.silu(sd[p + "emb.weight"]), sd[p + "linear.weight"], sd[p + "linear.bias"])
    out = G.ops.ada_layernorm(x.cuda(), table.cuda(), t.cuda())
    assert G.relerr(out, ref) < 2e-6
    # the table itself through the set-up kernels (SiLU + exact fp32 GEMM)
    tab2 = G.ops.gemm_f32(G.ops.silu(sd[p + "emb.weight"].cuda()), sd[p + "linear.weight"].cuda(), sd[p + "linear.bias"].cuda())
    assert G.relerr(tab2, table) < 2e-6


@pytest.mark.parametrize("M,N,K", [(100, 2048, 1024), (530, 96, 200), (64, 64, 16)])
def test_gemm_f32_exact_mode(G, M, N, K):
    a, w, bias, res = torch.randn(M, K), torch.randn(N, K) * 0.05, torch.randn(N), torch.randn(M, N)
    ref = (a.double() @ w.double().T + bias.double())
    ref = ref * torch.sigmoid(1.702 * ref) + res.double()
    out = G.ops.gemm_f32(a.cuda(), w.cuda(), bias.cuda(), res.cuda(), gelu=True)
    assert G.relerr(out, ref) < 5e-6


@pytest.mark.parametrize("B,H,Lq,Lk", [(2, 2, 265, 265), (3, 16, 265, 77), (1, 1, 16, 5), (2, 4, 70, 130)])
def test_attention_matches_fp64(G, B, H, Lq, Lk):
    D = H * 64
    q, k, v = torch.randn(B * Lq, D), torch.randn(B * Lk, D), torch.randn(B * Lk, D)
    qh = q.view(B, Lq, H, 64).transpose(1, 2).double()
    kh = k.view(B, Lk, H, 64).transpose(1, 2).double()
    vh = v.view(B, Lk, H, 64).transpose(1, 2).double()
    att = torch.softmax(qh @ kh.transpose(-1, -2) / 8.0, dim=-1)
    ref = (att @ vh).transpose(1, 2).reshape(B * Lq, D)
    out = torch.full((B * Lq, D), float("nan"), device="cuda")
    G.ops.attention(q.cuda(), k.cuda(), v.cuda(), out, B=B, H=H, Lq=Lq, Lk=Lk, scale=0.125)
    assert torch.isfinite(out).all()
    assert G.relerr(out, ref) < 2e-3  # TF32 operands for QK^T and PV (max-abs error over the tensor, relative to its max)


def test_attention_strided_qkv_view(G):
    B, H, L = 2, 2, 265
    D = H * 64
    qkv = torch.randn(B * L, 3 * D, device="cuda")
    out = torch.empty(B * L, D, device="cuda")
    G.ops.attention(qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:], out, B=B, H=H, Lq=L, Lk=L, scale=0.125)
    q, k, v = (t.view(B, L, H, 64).transpose(1, 2).double() for t in (qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:]))
    ref = (torch.softmax(q @ k.transpose(-1, -2) / 8.0, -1) @ v).transpose(1, 2).reshape(B * L, D)
    assert G.relerr(out, ref) < 1e-3


@pytest.mark.parametrize("case", range(5))
@pytest.mark.parametrize("trunc", ["top0.85r", None, "top20p"])
def test_posterior_sampler_matches_oracle_and_reference_golden(G, case, trunc):
    """model_log_prob: every element within the bound of tests/sampler_reference.posterior, against the restatement and (twice the
    bound) against the oracle.  Token ids: equal to the oracle's and to the reference-generated golden's, except where the two ids'
    scores lie within the Gumbel and posterior rounding bounds of each other.  Columns whose truncation boundary falls inside a group
    of equal log-probs are left out: the reference's order of equal values is unspecified (tests/test_cpu_sampler_reference.py)."""
    logits, x_t, t, u = sampler_case_inputs(case)
    sched = O.schedule_buffers(100, 257)
    table = R.sched_table(sched, 100)
    nxt_ref, post_ref, _ = O.posterior_sample_step(sched, logits, x_t, t, u, T=100, truncation=trunc)
    mode, r, kk = (0, 0.0, 0) if trunc is None else ((1, float(trunc[3:-1]), 0) if trunc.endswith("r") else (2, 0.0, int(trunc[3:-1])))
    lpo = torch.full((2, 257, 265), float("nan"), device="cuda")
    nxt = G.ops.posterior_sample(logits.permute(0, 2, 1).contiguous().cuda(), x_t.cuda(), t.cuda(), u.cuda(), table.cuda(), T=100,
                                 trunc_mode=mode, trunc_r=r, trunc_k=kk, log_prob_out=lpo).cpu()
    _, post, bound, val, gb, excl, tie = R.sample_step(logits, x_t, t, u, table, 100, trunc)
    ok = ~(excl | tie).unsqueeze(1)
    lpo = lpo.cpu().double()
    assert bool((((lpo - post).abs() <= bound) | ~ok).all())
    assert bool((((lpo - post_ref.double()).abs() <= 2 * bound) | ~ok).all())
    _, gold = load_golden("sampler_cases.npz")
    gref = torch.from_numpy(gold[f"c{case}_{ {'top0.85r': 'nuc', None: 'raw', 'top20p': 'topk'}[trunc] }_next"]).long()
    for ref in (nxt_ref, gref):
        wrong, _ = R.id_check(nxt, val, gb, extra=bound, ref=ref)
        assert int((wrong & ok.squeeze(1)).sum()) == 0, f"{int(wrong.sum())} id mismatches beyond the rounding bounds"


def test_posterior_sampler_k512_and_t_post(G):
    B, K, L, T = 2, 512, 265, 100
    gen = torch.Generator().manual_seed(3)
    logits = torch.randn(B, K, L, generator=gen) * 3
    u = torch.rand(B, K + 1, L, generator=gen)
    x_t = torch.where(torch.rand(B, L, generator=gen) < 0.5, torch.full((B, L), K), torch.randint(0, K, (B, L), generator=gen))
    t = torch.tensor([60, 7])
    tp = torch.tensor([58, 7])  # sample_fast: q_posterior at t - skip_step (diffusion_transformer.py:799-802)
    sched = O.schedule_buffers(T, K + 1)
    ref, post, _ = O.posterior_sample_step(sched, logits, x_t, t, u, T=T, truncation="top0.85r", t_posterior=tp)
    nxt = G.ops.posterior_sample(logits.permute(0, 2, 1).contiguous().cuda(), x_t.cuda(), t.cuda(), u.cuda(), R.sched_table(sched, T).cuda(), T=T, t_post=tp.cuda())
    assert int((nxt.cpu() != ref).sum()) <= 1


@pytest.mark.parametrize("B,H,Lq,Lk", [(2, 2, 265, 265), (3, 16, 265, 77), (1, 1, 16, 5), (2, 4, 70, 130)])
def test_attention_f16_matches_fp64(G, B, H, Lq, Lk):
    D = H * 64
    gen = torch.Generator().manual_seed(B * 100 + Lk)
    qkv = torch.randn(B * Lq, 3 * D, generator=gen).half()
    kv = torch.randn(B * Lk, 2 * D, generator=gen).half()
    q = qkv[:, :D]
    k, v = (kv[:, :D], kv[:, D:])
    qh = q.double().view(B, Lq, H, 64).transpose(1, 2)
    kh = k.double().view(B, Lk, H, 64).transpose(1, 2)
    vh = v.double().view(B, Lk, H, 64).transpose(1, 2)
    ref = (torch.softmax(qh @ kh.transpose(-1, -2) / 8.0, dim=-1) @ vh).transpose(1, 2).reshape(B * Lq, D)
    qkv_d, kv_d = qkv.cuda(), kv.cuda()
    out = torch.full((B * Lq, D), float("nan"), device="cuda", dtype=torch.float16)
    G.ops.attention(qkv_d[:, :D], kv_d[:, :D], kv_d[:, D:], out, B=B, H=H, Lq=Lq, Lk=Lk, scale=0.125)
    assert torch.isfinite(out).all()
    assert G.relerr(out.float(), ref) < 1.5e-3  # fp16 P and fp16 output rounding
    out32 = torch.empty(B * Lq, D, device="cuda")
    G.ops.attention(qkv_d[:, :D], kv_d[:, :D], kv_d[:, D:], out32, B=B, H=H, Lq=Lq, Lk=Lk, scale=0.125)
    assert G.relerr(out32, ref) < 1e-3


@pytest.mark.parametrize("pipelined", [False, True])
@pytest.mark.parametrize("B,H,Lq,Lk", [(2, 2, 265, 265), (3, 16, 265, 77), (1, 1, 16, 5), (2, 4, 70, 130), (1, 2, 128, 272), (16, 16, 265, 265)])
def test_attention_tcgen05_matches_fp64(G, B, H, Lq, Lk, pipelined):
    """Tensor-core attention (S = Q K^T and O = P V with mma.sync, K / V staged by TMA in SWIZZLE_128B tiles) through both C entry points
    (dsb_attention_tc and dsb_attention_tc2, `pipelined`), which launch the same kernel; repeated launches included."""
    D = H * 64
    gen = torch.Generator().manual_seed(B * 1000 + Lq + Lk)
    qkv = torch.randn(B * Lq, 3 * D, generator=gen).half()
    kv = torch.randn(B * Lk, 2 * D, generator=gen).half()
    qh = qkv[:, :D].double().view(B, Lq, H, 64).transpose(1, 2)
    kh = kv[:, :D].double().view(B, Lk, H, 64).transpose(1, 2)
    vh = kv[:, D:].double().view(B, Lk, H, 64).transpose(1, 2)
    ref = (torch.softmax(qh @ kh.transpose(-1, -2) / 8.0, dim=-1) @ vh).transpose(1, 2).reshape(B * Lq, D)
    qkv_d, kv_d = qkv.cuda(), kv.cuda()
    for _ in range(3):
        out = torch.full((B * Lq, D), float("nan"), device="cuda", dtype=torch.float16)
        G.ops.attention_tc(qkv_d[:, :D], kv_d[:, :D], kv_d[:, D:], out, B=B, H=H, Lq=Lq, Lk=Lk, scale=0.125, pipelined=pipelined)
        assert torch.isfinite(out).all()
        assert G.relerr(out.float(), ref) < 1.5e-3


def test_philox_replay_matches_torch_rand_bit_for_bit():
    """The fused sampling loop draws its own uniforms; they must be the very numbers torch.rand_like would have produced from the default CUDA
    generator (reference diffusion_transformer.py:360), for any tensor size (ATen's launch geometry changes with numel) and any offset."""
    import _pkg
    _pkg.load()
    from diffsound_b200 import ops
    gen = torch.cuda.default_generators[torch.cuda.current_device()]
    for seed, n in ((1234, 16 * 257 * 265), (7, 257 * 265), (2 ** 40 + 3, 1000), (99, 512 * 513 * 265 // 4), (5, 3)):
        torch.manual_seed(seed)
        assert gen.initial_seed() == seed and gen.get_offset() == 0
        a = torch.rand(n, device="cuda")
        off1 = gen.get_offset()
        nthreads, counter_offset = ops.aten_rand_geometry(n)
        assert off1 == counter_offset, (off1, counter_offset)          # the offset bookkeeping the loop relies on
        assert torch.equal(ops.aten_uniform(n, seed, 0), a), (seed, n)
        b = torch.rand(n, device="cuda")                                # second draw: offset advanced by counter_offset
        assert torch.equal(ops.aten_uniform(n, seed, off1), b), (seed, n)
    x = torch.rand(2, 257, 265, device="cuda")                          # rand_like of a (B, K+1, L) tensor = the flat stream in memory order
    torch.manual_seed(11)
    y = torch.rand_like(x)
    assert torch.equal(ops.aten_uniform(x.numel(), 11, 0).view_as(y), y)


def test_sampling_loop_kernel_equals_explicit_uniforms():
    """dsb_posterior_sample_loop (in-kernel RNG, in-place ids, device-side schedule) == dsb_posterior_sample fed torch.rand's tensor, step by
    step, for K = 63, 256 and 1055 without truncation, with nucleus 0.85 and with top-20.  After every step the loop state is read back: the
    RNG offset advanced by exactly one increment, the step counted, the CTA ticket back to 0, the next step's t and t_post written to every
    batch row, and after the last step t and t_post left as they were."""
    import _pkg
    _pkg.load()
    from diffsound_b200 import ops
    from oracle import diffsound_oracle as O
    B, L, T = 3, 265, 100
    steps, post = [99, 98, 60, 60, 3, 0], [99, 97, 60, 58, 3, 0]
    n = len(steps)
    for K in (63, 256, 1055):
        sched = R.sched_table(O.schedule_buffers(T, K + 1), T).cuda()
        g = torch.Generator().manual_seed(K)
        logits = [(torch.randn(B, L, K, generator=g) * 3).cuda() for _ in steps]
        x0 = torch.full((B, L), K, dtype=torch.long, device="cuda")
        for mode, r, k in ((0, 0.0, 0), (1, 0.85, 0), (2, 0.0, 20)):
            tr = dict(trunc_mode=mode, trunc_r=r, trunc_k=k)
            seed = 4242 + K + mode
            torch.manual_seed(seed)
            refs, ref = [], x0.clone()
            for lg, ti, tp in zip(logits, steps, post):
                u = torch.rand(B, K + 1, L, device="cuda")
                ref = ops.posterior_sample(lg, ref, torch.full((B,), ti, device="cuda"), u, sched, T=T, t_post=torch.full((B,), tp, device="cuda"), **tr)
                refs.append(ref.clone())
            nthreads, inc = ops.aten_rand_geometry(B * (K + 1) * L)
            ctrl = torch.tensor([seed, 0, inc, nthreads, 0, n, 0, 0], dtype=torch.int64, device="cuda")
            t_s, tp_s = torch.tensor(steps, device="cuda"), torch.tensor(post, device="cuda")
            t = torch.full((B,), steps[0], device="cuda")
            tpb = torch.full((B,), post[0], device="cuda")
            x = x0.clone()
            for i, lg in enumerate(logits):
                ops.posterior_sample_loop(lg, x, t, tpb, sched, ctrl, t_s, tp_s, T=T, **tr)
                torch.cuda.synchronize()
                what = (K, mode, i)
                assert torch.equal(x, refs[i]), what
                assert ctrl.tolist() == [seed, inc * (i + 1), inc, nthreads, i + 1, n, 0, 0], (what, ctrl.tolist())
                j = min(i + 1, n - 1)
                assert t.tolist() == [steps[j]] * B and tpb.tolist() == [post[j]] * B, (what, t.tolist(), tpb.tolist())
