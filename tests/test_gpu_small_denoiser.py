"""Diffsound's small denoiser (caps_small_transformer.yaml: 18 layers, n_embd 512, 16 heads of 32) on the H100: the head_dim-32 split-fp16 and
fp32 attention cores against fp64, the full small config against the fp32 oracle (teacher-forced logits and free-running token ids), the public
sample(), DALLE -> decoder -> MelGAN, and the refusals of the modes that have no head_dim-32 form."""
import os

import pytest
import torch

from oracle import diffsound_oracle as O
from tests.helpers import ROOT, build_dt, rel_err

pytestmark = pytest.mark.gpu

K, D, NL, NH, CD, L, HD = 256, 512, 18, 16, 512, 265, 32
SHAPES = [(1, 1), (9, 33), (63, 64), (65, 65), (77, 77), (265, 77), (265, 265), (128, 300), (265, 700)]


@pytest.fixture(scope="module")
def ops():
    from tests import gpu_common
    return gpu_common.ops


def _pair(p, C, lo=None):
    return p[:, :C].double() + p[:, (C if lo is None else lo):(C if lo is None else lo) + C].double()


def _heads(x, B, Lx, H):
    return x.reshape(B, Lx, H, HD).permute(0, 2, 1, 3)


def _ref(q, k, v, B, H, Lq, Lk):
    """fp64 softmax(Q K^T / sqrt(32)) V of fp64 (B*L, H*32) matrices."""
    s = _heads(q, B, Lq, H) @ _heads(k, B, Lk, H).transpose(-1, -2) / 32 ** 0.5
    return (torch.softmax(s, -1) @ _heads(v, B, Lk, H)).permute(0, 2, 1, 3).reshape(B * Lq, H * HD)


def _inputs(B, H, Lq, Lk, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    C = H * HD
    return (torch.randn(B * Lq, C, device="cuda", generator=g) * 1.5, torch.randn(B * Lk, C, device="cuda", generator=g) * 1.5,
            torch.randn(B * Lk, C, device="cuda", generator=g))


def _split_run(ops, B, H, Lq, Lk, seed):
    C = H * HD
    q, k, v = _inputs(B, H, Lq, Lk, seed)
    qp, kp, vp = ops.split_f16(q), ops.split_f16(k), ops.split_f16(v)
    out = torch.full((B * Lq, 2 * C), float("nan"), dtype=torch.float16, device="cuda")
    ops.attention_tc_split(qp[:, :C], kp[:, :C], vp[:, :C], out[:, :C], q_lo=C, k_lo=C, v_lo=C, o_lo=C, B=B, H=H, Lq=Lq, Lk=Lk,
                           scale=HD ** -0.5, head_dim=HD)
    return out, _ref(_pair(qp, C), _pair(kp, C), _pair(vp, C), B, H, Lq, Lk)


def _check(got, ref, tol=3e-6):
    assert torch.isfinite(got).all()
    err = float((got - ref).abs().max() / ref.abs().max())
    assert err < tol, err


@pytest.mark.parametrize("Lq,Lk", SHAPES)
def test_split_hd32_against_fp64(ops, Lq, Lk):
    """Query-tile and key-chunk edges, the model's 265 / 77, and a long key stream; B * H * pairs below the SM count."""
    out, ref = _split_run(ops, 2, 3, Lq, Lk, seed=Lq * 1000 + Lk)
    _check(_pair(out, 3 * HD), ref)


@pytest.mark.parametrize("B,H,Lq,Lk", [(37, 5, 265, 265), (64, 16, 265, 77), (16, 16, 265, 265)])
def test_split_hd32_more_units_than_ctas(ops, B, H, Lq, Lk):
    out, ref = _split_run(ops, B, H, Lq, Lk, seed=B)
    _check(_pair(out, H * HD), ref)


def test_split_hd32_engine_packed_views(ops):
    """The engine's calls at D = 512: self-attention off qkv = [Qh Kh Vh | Ql Kl Vl] (lo at 3D) and cross-attention of q2 = [Qh | Ql] against
    the last layer's K / V columns of kv_all = [every layer's Kh Vh | every layer's Kl Vl] (lo at n_layer * 2D)."""
    B, Lc = 3, 77
    g = torch.Generator(device="cuda").manual_seed(11)
    qkv = ops.split_f16(torch.randn(B * L, 3 * D, device="cuda", generator=g))
    att = torch.full((B * L, 2 * D), float("nan"), dtype=torch.float16, device="cuda")
    ops.attention_tc_split(qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:3 * D], att[:, :D], q_lo=3 * D, k_lo=3 * D, v_lo=3 * D, o_lo=D,
                           B=B, H=NH, Lq=L, Lk=L, scale=HD ** -0.5, head_dim=HD)
    ref = _ref(_pair(qkv, D, 3 * D), _pair(qkv[:, D:], D, 3 * D), _pair(qkv[:, 2 * D:], D, 3 * D), B, NH, L, L)
    _check(_pair(att, D), ref)
    q2 = ops.split_f16(torch.randn(B * L, D, device="cuda", generator=g))
    kv_all = ops.split_f16(torch.randn(B * Lc, NL * 2 * D, device="cuda", generator=g))
    kv_lo, li = NL * 2 * D, NL - 1
    kv = kv_all[:, li * 2 * D:]
    ops.attention_tc_split(q2[:, :D], kv[:, :D], kv[:, D:2 * D], att[:, :D], q_lo=D, k_lo=kv_lo, v_lo=kv_lo, o_lo=D, B=B, H=NH, Lq=L, Lk=Lc,
                           scale=HD ** -0.5, head_dim=HD)
    ref = _ref(_pair(q2, D), _pair(kv, D, kv_lo), _pair(kv[:, D:], D, kv_lo), B, NH, L, Lc)
    _check(_pair(att, D), ref)


def test_split_hd32_bits_repeat_graph_and_sentinels(ops):
    """Three launches and a CUDA-graph replay give the same bits; rows past B * Lq and the columns between and after the written hi / lo
    blocks keep their sentinel."""
    B, H, Lq, Lk = 3, 16, 265, 265
    C = H * HD
    q, k, v = _inputs(B, H, Lq, Lk, 5)
    qp, kp, vp = ops.split_f16(q), ops.split_f16(k), ops.split_f16(v)
    buf = torch.full((B * Lq + 7, 2 * C + 16), 1234.0, dtype=torch.float16, device="cuda")
    o_lo = C + 8

    def launch():
        ops.attention_tc_split(qp[:, :C], kp[:, :C], vp[:, :C], buf[:, :C], q_lo=C, k_lo=C, v_lo=C, o_lo=o_lo, B=B, H=H, Lq=Lq, Lk=Lk,
                               scale=HD ** -0.5, head_dim=HD)

    outs = []
    for _ in range(3):
        launch()
        outs.append(buf.clone())
    assert all(torch.equal(outs[0], o) for o in outs[1:])
    _check(_pair(outs[0][:B * Lq], C, o_lo), _ref(_pair(qp, C), _pair(kp, C), _pair(vp, C), B, H, Lq, Lk))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        launch()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        launch()
    buf.fill_(1234.0)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(buf, outs[0]), "CUDA-graph replay changed the bits"
    assert bool((buf[B * Lq:] == 1234.0).all())
    assert bool((buf[:, C:o_lo] == 1234.0).all()) and bool((buf[:, o_lo + C:] == 1234.0).all())


@pytest.mark.parametrize("Lq,Lk", [(1, 1), (63, 64), (77, 77), (265, 77), (265, 265), (128, 300)])
def test_fp32_attention_hd32_against_fp64(ops, Lq, Lk):
    """The attention core of the 'fp32' / 'tf32' modes (fp32 in and out, TF32 mma.sync for Q K^T and P V): the bound of its head_dim-64 form in
    test_gpu_kernels.py.  Rows past B * Lq and the columns after the heads keep their sentinel."""
    B, H = 2, 4
    q, k, v = _inputs(B, H, Lq, Lk, Lq + Lk)
    buf = torch.full((B * Lq + 3, H * HD + 8), 1234.0, device="cuda")
    ops.attention(q, k, v, buf[:B * Lq, :H * HD], B=B, H=H, Lq=Lq, Lk=Lk, scale=HD ** -0.5, head_dim=HD)
    _check(buf[:B * Lq, :H * HD].double(), _ref(q.double(), k.double(), v.double(), B, H, Lq, Lk), tol=2e-3)
    assert bool((buf[B * Lq:] == 1234.0).all()) and bool((buf[:, H * HD:] == 1234.0).all())


# ------------------------------------------------------------------ the full small config against the fp32 oracle
@pytest.fixture(scope="module")
def small_sd():
    torch.set_num_threads(min(16, torch.get_num_threads()))
    return O.make_transformer_state_dict(K=K, D=D, n_layer=NL, n_head=NH, cond_dim=CD, seed=0)


def _cond(B, g):
    c = torch.randn(B, 77, CD, generator=g)
    return c / c.norm(dim=-1, keepdim=True)


@pytest.mark.parametrize("precision,tol", [("f16x3", 3e-5), ("fp32", 3e-4), ("tf32", 2e-3)])
def test_small_config_teacher_forced_logits(ops, small_sd, precision, tol):
    B = 2
    g = torch.Generator().manual_seed(3)
    cond = _cond(B, g)
    x = torch.randint(0, K + 1, (B, L), generator=g)
    t = torch.tensor([99, 37])
    ref = O.transformer_forward(small_sd, x, cond, t, n_layer=NL, n_head=NH, spatial=(5, 53))
    m = build_dt(K, D, NL, NH, CD, small_sd, precision=precision)
    eng = m.transformer.engine
    out = eng.forward(x.cuda(), eng.encode_condition(cond.cuda()), t.cuda(), 77).permute(0, 2, 1).cpu()
    assert eng.head_dim == HD
    err = rel_err(out, ref)
    assert err < tol, err


def _run_chain(m, cond, us, steps):
    """Fused step on supplied uniforms (no torch RNG): the token grid after `steps` steps from all-[MASK]."""
    eng = m.transformer.engine
    B = cond.shape[0]
    kv = eng.encode_condition(cond)
    x = torch.full((B, L), K, dtype=torch.long, device="cuda")
    mode, r, k = m._trunc()
    sample = m._sampler_ops()[0]
    for i, ti in enumerate(range(99, 99 - steps, -1)):
        t = torch.full((B,), ti, dtype=torch.long, device="cuda")
        x = sample(eng.forward(x, kv, t, cond.shape[1]), x, t, us[i], m._sched(), T=100, trunc_mode=mode, trunc_r=r, trunc_k=k)
    return x


@pytest.fixture(scope="module")
def chain_b1(small_sd):
    """The oracle's 100-step top0.85r chain at B = 1 on stored uniforms."""
    g = torch.Generator().manual_seed(21)
    cond = _cond(1, g)
    us = [torch.rand(1, K + 1, L, generator=g) for _ in range(100)]
    ref = O.sample(small_sd, cond, lambda i: us[i], n_layer=NL, n_head=NH, spatial=(5, 53))
    return cond, us, ref


@pytest.mark.parametrize("precision", ["f16x3", "fp32"])
def test_small_config_100_steps_b1_token_ids_equal_oracle(ops, small_sd, chain_b1, precision):
    cond, us, ref = chain_b1
    m = build_dt(K, D, NL, NH, CD, small_sd, precision=precision)
    m.truncation = "top0.85r"
    got = _run_chain(m, cond.cuda(), [u.cuda() for u in us], 100).cpu()
    assert int((ref == K).sum()) == 0
    assert torch.equal(got, ref), f"{int((got != ref).sum())} of {ref.numel()} token ids differ"


def test_small_config_10_steps_b16_token_ids_equal_oracle(ops, small_sd):
    B, steps = 16, 10
    g = torch.Generator().manual_seed(22)
    cond = _cond(B, g)
    us = [torch.rand(B, K + 1, L, generator=g) for _ in range(steps)]
    ref = O.sample(small_sd, cond, lambda i: us[i], n_layer=NL, n_head=NH, spatial=(5, 53), steps=list(range(99, 99 - steps, -1)))
    m = build_dt(K, D, NL, NH, CD, small_sd, precision="f16x3")
    m.truncation = "top0.85r"
    got = _run_chain(m, cond.cuda(), [u.cuda() for u in us], steps).cpu()
    assert int((ref != K).sum()) > 0
    assert torch.equal(got, ref), f"{int((got != ref).sum())} of {ref.numel()} token ids differ"


def test_small_config_public_sample(ops):
    """sample() at B = 16 (torch RNG): the CUDA-graph loop, the eager loop and the stage-by-stage reference-named methods give the same tokens, in
    [0, K) with no [MASK] left; on supplied uniforms, clip j gets the same tokens alone as inside the batch."""
    torch.manual_seed(0)
    m = build_dt(K, D, NL, NH, CD, precision="f16x3")
    m.truncation = "top0.85r"
    g = torch.Generator().manual_seed(9)
    B = 16
    cond = _cond(B, g).cuda()
    toks = []
    for mode in ("graph", "graph", "eager", "unfused"):
        m.use_cuda_graph = mode == "graph"
        if mode == "unfused":
            m.p_sample = m.p_sample
        torch.manual_seed(1234)
        toks.append(m.sample(None, None, cond, filter_ratio=0, batch_size=B)["content_token"].cpu())
    del m.__dict__["p_sample"]
    m.use_cuda_graph = True
    tok = toks[0]
    assert tok.shape == (B, L) and int(tok.min()) >= 0 and int(tok.max()) < K
    assert torch.equal(toks[0], toks[1]), "two sample() runs differ"
    assert torch.equal(toks[1], toks[2]), "CUDA-graph replay changed the sampled tokens"
    assert torch.equal(toks[2], toks[3]), "fused and stage-by-stage paths disagree"
    steps = 12
    us = [torch.rand(B, K + 1, L, generator=g).cuda() for _ in range(steps)]
    full = _run_chain(m, cond, us, steps)
    for j in (0, 7, 15):
        solo = _run_chain(m, cond[j:j + 1], [u[j:j + 1].contiguous() for u in us], steps)
        assert torch.equal(solo[0], full[j]), f"clip {j} depends on its batch neighbours"


def test_small_dalle_to_wav(ops):
    """A DALLE built like caps_small_transformer.yaml (builders.DALLE_CONFIGS) -> SpecVQGAN decoder -> MelGAN: a finite waveform."""
    import _pkg
    _pkg.load()
    from diffsound_b200 import pipeline
    from diffsound_b200.utils.builders import DALLE_CONFIGS, build_dalle, build_vocoder
    dalle = build_dalle(**DALLE_CONFIGS["caps_small_transformer"], seed=0)
    assert dalle.transformer.transformer.engine.precision == "f16x3"
    voc = build_vocoder(os.path.join(ROOT, "oracle", "_ref", "best_netG.pt"))
    cond = _cond(2, torch.Generator().manual_seed(4)).cuda()
    out = pipeline.synthesize(dalle, voc, cond, sample_type="top0.85r", seed=1234)
    assert dalle.transformer.transformer.engine.head_dim == HD
    assert out["tokens"].shape == (2, L) and int(out["tokens"].max()) < K
    assert out["wav"].shape == (2, 1, 217088) and bool(torch.isfinite(out["wav"]).all()) and float(out["wav"].abs().max()) > 0


def test_f16_precision_refused_at_head_dim_32(ops):
    m = build_dt(K, D, 1, NH, CD, precision="f16")
    with pytest.raises(RuntimeError, match=r"precision 'f16' has no head_dim-32 attention"):
        m.transformer.engine.repack()


def test_training_forward_refused_at_head_dim_32(ops):
    from tests.gpu_common import run_loss_and_grads
    m = build_dt(K, D, 1, NH, CD, precision="f16x3")
    m.train()
    B = 2
    x0 = torch.randint(0, K, (B, L), device="cuda")
    cond = _cond(B, torch.Generator().manual_seed(5)).cuda()
    t = torch.tensor([10, 60], device="cuda")
    pt = torch.full((B,), 0.01, device="cuda")
    with pytest.raises(RuntimeError, match=r"training kernels need head_dim 64"):
        run_loss_and_grads(m, x0, x0.clone(), cond, t, pt)


def test_other_head_dims_still_refused(ops):
    m = build_dt(K, 256, 1, 16, CD, precision="f16x3")  # head_dim 16
    with pytest.raises(RuntimeError, match="head_dim 64 and 32"):
        m.transformer.engine.repack()
