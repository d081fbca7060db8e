"""Denoiser + diffusion-loop parity on the H100 through the drop-in nn.Module API."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import diffsound_oracle as O  # noqa: E402
from tests.helpers import build_dt, load_golden, rel_err  # noqa: E402,F401  (build_dt: also imported from here by other test modules)


@pytest.fixture(scope="module")
def G():
    from tests import gpu_common
    return gpu_common


def test_state_dict_keys_match_reference_golden(G):
    sd, g = load_golden("xf_tiny.npz")
    K, D, NL, NH, CD, B, L = [int(v) for v in g["__cfg"]]
    m = build_dt(K, D, NL, NH, CD)
    mine = set(m.state_dict().keys())
    assert set(sd.keys()) <= mine
    assert all("attn2.mask" in k for k in mine - set(sd.keys()))
    for n in ("log_at", "log_cumprod_bt", "log_1_min_cumprod_ct"):
        assert torch.equal(m.state_dict()[n].cpu(), sd[n])  # schedule is bit-identical to the reference's buffers


def test_tiny_denoiser_and_stage_methods_match_reference_golden(G):
    """Reference-generated golden (2 layers, D=128): logits within 1e-3 relative; log_pred / posterior within 2e-3 absolute."""
    sd, g = load_golden("xf_tiny.npz")
    K, D, NL, NH, CD, B, L = [int(v) for v in g["__cfg"]]
    m = build_dt(K, D, NL, NH, CD, sd)
    cond, x_t, t = torch.from_numpy(g["in_cond"]).cuda(), torch.from_numpy(g["in_x_t"]).long().cuda(), torch.from_numpy(g["in_t"]).cuda()
    logits = m.transformer(x_t, cond, t)
    assert logits.shape == (B, K, L)
    assert rel_err(logits.cpu(), torch.from_numpy(g["out_logits"])) < 2e-3  # 11-bit-significand operands, 2 layers
    log_x = O.index_to_log_onehot(x_t.cpu(), K + 1).cuda()
    m.truncation = "top0.85r"
    lp = m.predict_start(log_x, cond, t).cpu()
    ref_lp = torch.from_numpy(g["out_lp"])
    flipped = ((lp == -70) != (ref_lp == -70)).float().mean()
    assert flipped < 2e-3  # nucleus boundary flips caused by TF32 logits
    same = (lp == -70) == (ref_lp == -70)
    assert float((lp - ref_lp)[same].abs().max()) < 2e-3
    post = m.q_posterior(torch.from_numpy(g["out_lp"]).cuda(), log_x, t).cpu()
    assert float((post - torch.from_numpy(g["out_post"])).abs().max()) < 2e-5  # same log_pred in -> posterior kernel is fp32-exact


def test_fused_graph_and_unfused_paths_agree(G):
    sd, g = load_golden("xf_tiny.npz")
    K, D, NL, NH, CD, B, L = [int(v) for v in g["__cfg"]]
    m = build_dt(K, D, NL, NH, CD, sd)
    m.truncation = "top0.85r"
    cond = torch.from_numpy(g["in_cond"]).cuda()
    toks = []
    for mode in ("graph", "eager", "unfused"):
        m.use_cuda_graph = mode == "graph"
        if mode == "unfused":  # re-bind a stage method the way the reference DALLE does -> stage-by-stage path
            m.p_sample = m.p_sample
        torch.manual_seed(1234)
        toks.append(m.sample(None, None, cond, filter_ratio=0, batch_size=B)["content_token"].cpu())
    assert toks[0].shape == (B, L) and toks[0].dtype == torch.int64
    assert int(toks[0].max()) < K  # no [MASK] survives t=0
    assert torch.equal(toks[0], toks[1]), "CUDA-graph replay changed the sampled tokens"
    assert torch.equal(toks[1], toks[2]), "fused and stage-by-stage paths disagree"
    # same seed again through the cached graph
    m.use_cuda_graph = True
    del m.__dict__["p_sample"]
    torch.manual_seed(1234)
    again = m.sample(None, None, cond, filter_ratio=0, batch_size=B)["content_token"].cpu()
    assert torch.equal(again, toks[0])


@pytest.mark.parametrize("precision,tol", [("f16x3", 3e-5), ("f16", 2e-3), ("tf32", 2e-3), ("fp32", 3e-4)])
def test_teacher_forced_steps_match_oracle_full_width(G, precision, tol):
    """D=1024 / 16 heads / K=256 (4 layers to keep the CPU oracle fast): feed the oracle's x_t each step (SURVEY 7.2 ladder ii).
    Logit tolerance (max|err| / max|ref|): 2e-3 for 11-bit-significand tensor-core operands (f16 / tf32), 3e-4 with exact fp32
    GEMMs (the attention core keeps TF32 operands); sampled ids must agree on >= 98 % of positions given the same uniforms."""
    K, D, NL, NH, CD, B, L = 256, 1024, 4, 16, 512, 2, 265
    sd = O.make_transformer_state_dict(K=K, D=D, n_layer=NL, n_head=NH, cond_dim=CD, seed=0)
    m = build_dt(K, D, NL, NH, CD, sd, precision=precision)
    g = torch.Generator().manual_seed(5)
    cond = torch.randn(B, 77, CD, generator=g)
    cond = cond / cond.norm(dim=-1, keepdim=True)
    sched = {k: sd[k] for k in sd if k.startswith("log_")}
    x = torch.full((B, L), K, dtype=torch.long)
    eng = m.transformer.engine
    kv = eng.encode_condition(cond.cuda())
    mism = 0
    for ti in (99, 80, 50, 20, 0):
        t = torch.full((B,), ti, dtype=torch.long)
        ref_logits = O.transformer_forward(sd, x, cond, t, n_layer=NL, n_head=NH, spatial=(5, 53))
        logits = eng.forward(x.cuda(), kv, t.cuda(), 77)
        err = rel_err(logits.permute(0, 2, 1).cpu(), ref_logits)
        print(f"[{precision}] t={ti} logits rel err {err:.2e}")
        assert err < tol, f"t={ti}"
        u = torch.rand(B, K + 1, L, generator=g)
        ref_next, _, _ = O.posterior_sample_step(sched, ref_logits, x, t, u, T=100)
        nxt = G.ops.posterior_sample(logits, x.cuda(), t.cuda(), u.cuda(), m._sched(), T=100).cpu()
        mism += int((nxt != ref_next).sum())
        x = torch.where(torch.rand(B, L, generator=g) < 0.3, ref_next, x)  # progressively unmask along the oracle's trajectory
    assert mism <= 0.02 * 5 * B * L, f"{mism} token mismatches under teacher forcing"


def test_free_running_full_size_tokens_vs_oracle(G):
    """SURVEY 7.2 ladder (iii): the real configuration (19 layers, D=1024, K=256, 100 steps, top0.85r), B=1, free-running, same
    weights and the same uniforms as the fp32 CPU oracle.  precision='fp32' (exact FFMA GEMMs) must reproduce every token id;
    the default f16 tensor-core mode must agree on >= 97 % of the final grid (measured 99.6 %, first flip at step 67)."""
    K, D, NL, NH, CD, B, L = 256, 1024, 19, 16, 512, 1, 265
    torch.set_num_threads(min(16, torch.get_num_threads()))
    sd = O.make_transformer_state_dict(K=K, D=D, n_layer=NL, n_head=NH, cond_dim=CD, seed=0)
    g = torch.Generator().manual_seed(5)
    cond = torch.randn(B, 77, CD, generator=g)
    cond = cond / cond.norm(dim=-1, keepdim=True)
    us = [torch.rand(B, K + 1, L, generator=g) for _ in range(100)]
    ref = O.sample(sd, cond, lambda i: us[i], n_layer=NL, n_head=NH, spatial=(5, 53))
    for prec, floor in (("f16x3", 1.0), ("fp32", 1.0), ("f16", 0.97)):
        m = build_dt(K, D, NL, NH, CD, sd, precision=prec)
        eng = m.transformer.engine
        kv = eng.encode_condition(cond.cuda())
        x = torch.full((B, L), K, dtype=torch.long, device="cuda")
        for i, ti in enumerate(range(99, -1, -1)):
            t = torch.full((B,), ti, dtype=torch.long, device="cuda")
            x = G.ops.posterior_sample(eng.forward(x, kv, t, 77), x, t, us[i].cuda(), m._sched(), T=100)
        agree = float((x.cpu() == ref).float().mean())
        print(f"[{prec}] free-running final token agreement {agree:.4f}")
        assert agree >= floor, f"{prec}: {agree}"
        del m, eng
        torch.cuda.empty_cache()


def _run_chain(m, cond, us, steps):
    """Fused step on supplied uniforms (no torch RNG): returns the token grid after `steps` diffusion steps."""
    eng = m.transformer.engine
    B = cond.shape[0]
    K, L = m.num_classes - 1, m.shape
    kv = eng.encode_condition(cond)
    x = torch.full((B, L), K, dtype=torch.long, device="cuda")
    mode, r, k = m._trunc()
    for i, ti in enumerate(range(99, 99 - steps, -1)):
        t = torch.full((B,), ti, dtype=torch.long, device="cuda")
        x = G_ops().posterior_sample(eng.forward(x, kv, t, cond.shape[1]), x, t, us[i], m._sched(), T=100, trunc_mode=mode, trunc_r=r, trunc_k=k)
    return x


def G_ops():
    from tests import gpu_common
    return gpu_common.ops


def test_full_config_batch_invariance_and_properties(G):
    """BASELINE configs[1] shape (19 layers, D=1024, K=256, B=16): properties that do not need the CPU oracle at full size.
    (1) batch invariance: clip j sampled inside a batch of 16 gets exactly the tokens it gets alone (same per-clip uniforms) -- every
        kernel on the path reduces each row in an order that does not depend on the other rows;
    (2) determinism: two runs are bit-identical;  (3) after the full 100 steps no [MASK] id survives and ids < K;
    (4) the public sample() (CUDA graph, torch RNG) returns the same shape / range at B=16 and B=64."""
    K, D, NL, NH, CD, L = 256, 1024, 19, 16, 512, 265
    torch.manual_seed(0)
    m = build_dt(K, D, NL, NH, CD)
    m.truncation = "top0.85r"
    g = torch.Generator().manual_seed(9)
    B = 16
    cond = torch.randn(B, 77, CD, generator=g)
    cond = (cond / cond.norm(dim=-1, keepdim=True)).cuda()
    steps = 12
    us = [torch.rand(B, K + 1, L, generator=g).cuda() for _ in range(steps)]
    full = _run_chain(m, cond, us, steps)
    again = _run_chain(m, cond, us, steps)
    assert torch.equal(full, again)
    for j in (0, 7, 15):
        solo = _run_chain(m, cond[j:j + 1], [u[j:j + 1].contiguous() for u in us], steps)
        assert torch.equal(solo[0], full[j]), f"clip {j} depends on its batch neighbours"
    for Bs in (16, 64):
        c = torch.randn(Bs, 77, CD, generator=g)
        c = (c / c.norm(dim=-1, keepdim=True)).cuda()
        torch.manual_seed(1234)
        tok = m.sample(None, None, c, filter_ratio=0, batch_size=Bs)["content_token"]
        assert tok.shape == (Bs, L) and int(tok.min()) >= 0 and int(tok.max()) < K


def test_k512_codebook_config_runs(G):
    """caps_512.yaml's codebook (BASELINE configs[4]): K=512 logits head + K+1=513-class sampler (NJ=17 instantiation), 2 layers."""
    K, D, NL, NH, CD, B, L = 512, 1024, 2, 16, 512, 4, 265
    sd = O.make_transformer_state_dict(K=K, D=D, n_layer=NL, n_head=NH, cond_dim=CD, seed=2)
    m = build_dt(K, D, NL, NH, CD, sd)
    g = torch.Generator().manual_seed(4)
    cond = torch.randn(B, 77, CD, generator=g)
    cond = cond / cond.norm(dim=-1, keepdim=True)
    x = torch.where(torch.rand(B, L, generator=g) < 0.5, torch.full((B, L), K), torch.randint(0, K, (B, L), generator=g))
    t = torch.tensor([80, 40, 10, 0])
    ref_logits = O.transformer_forward(sd, x, cond, t, n_layer=NL, n_head=NH, spatial=(5, 53))
    eng = m.transformer.engine
    logits = eng.forward(x.cuda(), eng.encode_condition(cond.cuda()), t.cuda(), 77)
    assert rel_err(logits.permute(0, 2, 1).cpu(), ref_logits) < 2e-3
    u = torch.rand(B, K + 1, L, generator=g)
    sched = {k: sd[k] for k in sd if k.startswith("log_")}
    ref_next, _, _ = O.posterior_sample_step(sched, ref_logits, x, t, u, T=100)
    nxt = G.ops.posterior_sample(logits, x.cuda(), t.cuda(), u.cuda(), m._sched(), T=100).cpu()
    assert (nxt != ref_next).float().mean() < 0.02
    m.truncation = "top0.85r"
    tok = m.sample(None, None, cond.cuda(), filter_ratio=0, batch_size=B)["content_token"]
    assert int(tok.max()) < K


def _chain_vs_oracle(K, B, steps, seed=3, precision="f16x3"):
    """Free-running chain at the real denoiser size (19 layers, D=1024) against the fp32 CPU oracle on the same weights / caption embeddings / uniforms."""
    D, NL, NH, CD, L = 1024, 19, 16, 512, 265
    torch.set_num_threads(min(16, torch.get_num_threads()))
    sd = O.make_transformer_state_dict(K=K, D=D, n_layer=NL, n_head=NH, cond_dim=CD, seed=0)
    g = torch.Generator().manual_seed(seed)
    cond = torch.randn(B, 77, CD, generator=g)
    cond = cond / cond.norm(dim=-1, keepdim=True)
    us = [torch.rand(B, K + 1, L, generator=g) for _ in range(steps)]
    ts = list(range(99, 99 - steps, -1))
    ref = O.sample(sd, cond, lambda i: us[i], n_layer=NL, n_head=NH, spatial=(5, 53), steps=ts)
    m = build_dt(K, D, NL, NH, CD, sd, precision=precision)
    m.truncation = "top0.85r"
    got = _run_chain(m, cond.cuda(), [u.cuda() for u in us], steps).cpu()
    return ref, got


def test_configs1_batch16_short_chain_token_ids_equal_oracle(G):
    """BASELINE configs[1] shape (B=16, K=256, 19 layers), 10 free-running steps from all-[MASK]: every token id of every clip equals the oracle's
    in the parity-grade 'f16x3' mode (42 400 Gumbel-argmax decisions)."""
    ref, got = _chain_vs_oracle(K=256, B=16, steps=10)
    assert int((ref != 256).sum()) > 0  # some positions have been unmasked: the comparison is not vacuous
    assert torch.equal(got, ref), f"{int((got != ref).sum())} of {ref.numel()} token ids differ"


def test_configs4_k512_codebook_19_layers_token_ids_equal_oracle(G):
    """BASELINE configs[4]'s codebook (K=512, 513-class sampler) at full depth: B=4, 10 free-running steps, token ids equal the oracle's."""
    ref, got = _chain_vs_oracle(K=512, B=4, steps=10, seed=8)
    assert int((ref != 512).sum()) > 0
    assert torch.equal(got, ref), f"{int((got != ref).sum())} of {ref.numel()} token ids differ"


def test_f16_modes_under_activation_range_stress(G):
    """Exponent-range stress for the fp16 containers (ADVICE r1): the same network with its weights rescaled so that intermediate activations are
    64x larger (LayerNorm affine / MLP / value / projection weights x4 each way) -- mathematically a different but equally valid model.  The
    parity-grade 'f16x3' mode must keep fp32-class logits against the oracle run on the SAME rescaled weights; the single-pass 'f16' mode is
    measured too (its error is relative to the 11-bit operands, not the range, as long as nothing overflows)."""
    K, D, NL, NH, CD, B, L = 256, 1024, 4, 16, 512, 2, 265
    sd = O.make_transformer_state_dict(K=K, D=D, n_layer=NL, n_head=NH, cond_dim=CD, seed=0)
    for k in list(sd.keys()):
        if k.endswith("mlp.0.weight") or k.endswith("attn1.value.weight") or k.endswith("attn2.value.weight"):
            sd[k] = sd[k] * 64.0          # hidden / value activations 64x larger
        if k.endswith("mlp.2.weight") or k.endswith("attn1.proj.weight") or k.endswith("attn2.proj.weight"):
            sd[k] = sd[k] / 64.0          # ... folded back so the residual stream keeps its scale (GELU2 is not homogeneous: a different model)
    g = torch.Generator().manual_seed(5)
    cond = torch.randn(B, 77, CD, generator=g)
    cond = cond / cond.norm(dim=-1, keepdim=True)
    x = torch.where(torch.rand(B, L, generator=g) < 0.5, torch.full((B, L), K), torch.randint(0, K, (B, L), generator=g))
    t = torch.tensor([70, 20])
    ref = O.transformer_forward(sd, x, cond, t, n_layer=NL, n_head=NH, spatial=(5, 53))
    for prec, tol in (("f16x3", 3e-5), ("f16", 4e-3)):
        m = build_dt(K, D, NL, NH, CD, sd, precision=prec)
        eng = m.transformer.engine
        logits = eng.forward(x.cuda(), eng.encode_condition(cond.cuda()), t.cuda(), 77)
        err = rel_err(logits.permute(0, 2, 1).cpu(), ref)
        print(f"[{prec}] range-stressed logits rel err {err:.2e}")
        assert torch.isfinite(logits).all() and err < tol, (prec, err)


@pytest.mark.parametrize("B", [32, 128])
def test_large_batch_kernel_selection_keeps_parity(G, B):
    """Batches between the headline's 16 and configs[4]'s 512 land on other tile shapes / kernels of dsb_gemm_ex (M = 8 480 / 33 920 rows: the wave
    heuristic once sent the N = 3072 / 4096 layers to narrower, slower tiles there).  Whatever is selected, f16x3 logits must agree with the
    exact-fp32 GEMM mode of the same engine on the same weights to the f16x3 tolerance, at full width (D=1024, 16 heads), partly unmasked input."""
    K, D, NL, NH, CD, L = 256, 1024, 2, 16, 512, 265
    sd = O.make_transformer_state_dict(K=K, D=D, n_layer=NL, n_head=NH, cond_dim=CD, seed=1)
    g = torch.Generator().manual_seed(B)
    cond = torch.randn(B, 77, CD, generator=g)
    cond = (cond / cond.norm(dim=-1, keepdim=True)).cuda()
    x = torch.where(torch.rand(B, L, generator=g) < 0.5, torch.randint(0, K, (B, L), generator=g), torch.full((B, L), K)).cuda()
    t = torch.randint(0, 100, (B,), generator=g).cuda()
    outs = {}
    for precision in ("fp32", "f16x3"):
        eng = build_dt(K, D, NL, NH, CD, sd, precision=precision).transformer.engine
        outs[precision] = eng.forward(x, eng.encode_condition(cond), t, 77).float().clone()
        del eng
        torch.cuda.empty_cache()
    err = rel_err(outs["f16x3"].cpu(), outs["fp32"].cpu())
    print(f"B={B}: f16x3 vs exact-fp32 GEMM mode, logits rel err {err:.2e}")
    assert err < 3e-4  # the fp32 mode's own distance to the oracle (its attention core keeps TF32 operands) bounds this comparison
