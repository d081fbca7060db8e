"""A13 (training) parity on the H100: the training-side kernels against torch autograd references, and the whole
forward + loss + backward of the drop-in DiffusionTransformer against (i) the reference's own loss / gradients (tests/golden/train_tiny.npz,
made by oracle/gen_golden.py from the unmodified reference) and (ii) torch autograd through the oracle at a larger config."""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import diffsound_oracle as O  # noqa: E402
from tests.helpers import build_dt, load_golden, portable_uniform  # noqa: E402

SCHED_ROWS = ["log_at", "log_bt", "log_ct", "log_1_min_ct", "log_cumprod_at", "log_cumprod_bt", "log_cumprod_ct", "log_1_min_cumprod_ct"]


@pytest.fixture(scope="module")
def G():
    from tests import gpu_common
    return gpu_common


@pytest.fixture(scope="module")
def TO():
    from tests import gpu_common  # noqa: F401  (loads the package)
    from diffsound_b200 import train_ops
    return train_ops


def sched8(K, T=100):
    s = O.schedule_buffers(T, K + 1)
    out = torch.zeros(8, T + 1)
    for i, n in enumerate(SCHED_ROWS):
        out[i, : s[n].numel()] = s[n]
    return s, out


ACT = [torch.float32, torch.bfloat16]


def _tol(dt, f32, bf16):
    return f32 if dt == torch.float32 else bf16


# ------------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("dt", ACT)
def test_transpose_heads_colsum(G, TO, dt):
    x = torch.randn(3, 265, 72, device="cuda").to(dt)
    out = torch.full((3, 72, 272), 7.0, device="cuda", dtype=dt)
    TO.transpose(x, out)
    assert torch.equal(out[:, :, :265], x.transpose(1, 2))
    assert bool((out[:, :, 265:] == 7.0).all())  # padding columns untouched
    x2 = torch.randn(795, 200, device="cuda").to(dt)
    o2 = torch.empty(200, 800, device="cuda", dtype=dt)
    TO.transpose(x2[:, :136], o2[:136])
    assert torch.equal(o2[:136, :795], x2[:, :136].t())
    B, H, L = 3, 4, 77
    tok = torch.randn(B * L, 3 * H * 64, device="cuda").to(dt)
    heads = torch.empty(B * H, L, 64, device="cuda", dtype=dt)
    TO.heads_split(tok[:, H * 64:2 * H * 64], heads, B, H, L)
    ref = tok[:, H * 64:2 * H * 64].reshape(B, L, H, 64).permute(0, 2, 1, 3).reshape(B * H, L, 64)
    assert torch.equal(heads, ref)
    back = torch.zeros_like(tok)
    TO.heads_merge(heads, back[:, H * 64:2 * H * 64], B, H, L)
    assert torch.equal(back[:, H * 64:2 * H * 64], tok[:, H * 64:2 * H * 64]) and float(back[:, :H * 64].abs().max()) == 0.0
    cs = torch.empty(200, device="cuda")
    TO.colsum(x2, cs)
    assert torch.allclose(cs, x2.float().sum(0), rtol=1e-4, atol=1e-3)


@pytest.mark.parametrize("dt", ACT)
def test_gelu2_and_softmax_passes(G, TO, dt):
    u = (torch.randn(1000, 512, device="cuda") * 2).to(dt)
    a = torch.empty_like(u)
    TO.gelu2_fwd(u, a)
    uf = u.float().requires_grad_(True)
    ref = uf * torch.sigmoid(1.702 * uf)
    assert G.relerr(a.float(), ref.detach()) < _tol(dt, 1e-3, 8e-3)
    da = torch.randn_like(uf).to(dt)
    du = torch.empty_like(u)
    TO.gelu2_bwd(u, da, du)
    ref.backward(da.float())
    assert G.relerr(du.float(), uf.grad) < _tol(dt, 1e-3, 8e-3)
    rows, n, ld = 640, 265, 272
    S = torch.randn(rows, ld, device="cuda") * 3
    P = torch.zeros(rows, ld, device="cuda", dtype=dt)
    TO.softmax_fwd(S, P, n)
    Sr = S[:, :n].clone().requires_grad_(True)
    Pr = torch.softmax(Sr, -1)
    assert G.relerr(P[:, :n].float(), Pr.detach()) < _tol(dt, 1e-3, 8e-3)
    dP = torch.randn(rows, ld, device="cuda")
    dS = torch.zeros(rows, ld, device="cuda", dtype=dt)
    TO.softmax_bwd(P, dP, dS, n, 0.125)
    # reference uses the kernel's (rounded) P so that only the backward formula is under test
    Pk = P[:, :n].float()
    ref_dS = 0.125 * Pk * (dP[:, :n] - (dP[:, :n] * Pk).sum(-1, keepdim=True))
    assert G.relerr(dS[:, :n].float(), ref_dS) < _tol(dt, 1e-3, 8e-3)


@pytest.mark.parametrize("D", [128, 1024])
def test_layernorm_backward_plain_and_ada(G, TO, D):
    B, L = 3, 265
    x = torch.randn(B, L, D, device="cuda") * 1.5 + 0.3
    dy = torch.randn(B, L, D, device="cuda")
    gamma = (1 + 0.1 * torch.randn(D, device="cuda"))
    beta = 0.1 * torch.randn(D, device="cuda")
    xr, gr, br = x.clone().requires_grad_(True), gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
    torch.nn.functional.layer_norm(xr, (D,), gr, br).backward(dy)
    dx = torch.randn(B, L, D, device="cuda")
    dx0 = dx.clone()
    dg, db = torch.zeros(D, device="cuda"), torch.zeros(D, device="cuda")
    dxa = torch.empty(B, L, D, device="cuda", dtype=torch.bfloat16)
    TO.layernorm_bwd(x, dy, dx, gamma, dg, db, dx_act=dxa)
    assert G.relerr(dx - dx0, xr.grad) < 1e-4
    assert torch.equal(dxa, dx.bfloat16())  # the fused activation-dtype copy of the updated stream gradient
    assert G.relerr(dg, gr.grad) < 1e-4 and G.relerr(db, br.grad) < 1e-4
    # AdaLN: y = LN(x) (1 + scale[idx[b]]) + shift[idx[b]]; rows of the table selected by idx, two batch elements share a row
    table = 0.2 * torch.randn(4, 2 * D, device="cuda")
    idx = torch.tensor([2, 0, 2], device="cuda")
    xr, tr = x.clone().requires_grad_(True), table.clone().requires_grad_(True)
    sel = tr[idx]
    (torch.nn.functional.layer_norm(xr, (D,)) * (1 + sel[:, None, :D]) + sel[:, None, D:]).backward(dy)
    dx = torch.zeros(B, L, D, device="cuda")
    dtab = torch.zeros_like(table)
    dxa = torch.empty(B, L, D, device="cuda")
    TO.ada_layernorm_bwd(x, dy, dx, table, idx, dtab, dx_act=dxa)
    assert G.relerr(dx, xr.grad) < 1e-4
    assert torch.equal(dxa, G.tf32_round_ref(dx.cpu()).cuda())
    assert G.relerr(dtab, tr.grad) < 1e-4


def test_embedding_backward_and_row_gather_scatter(G, TO):
    B, L, D, H, W, NE = 3, 265, 128, 5, 53, 33
    ids = torch.randint(0, NE, (B, L), device="cuda")
    emb, he, we = [torch.randn(n, D, device="cuda", requires_grad=True) for n in (NE, H, W)]
    pos = (he[:, None, :] + we[None, :, :]).reshape(1, H * W, D)
    dxx = torch.randn(B, L, D, device="cuda")
    (torch.nn.functional.embedding(ids, emb) + pos[:, :L]).backward(dxx)
    de, dh, dw = torch.zeros(NE, D, device="cuda"), torch.zeros(H, D, device="cuda"), torch.zeros(W, D, device="cuda")
    TO.embed_bwd(ids, dxx, de, dh, dw)
    assert G.relerr(de, emb.grad) < 1e-5 and G.relerr(dh, he.grad) < 1e-5 and G.relerr(dw, we.grad) < 1e-5
    table = torch.randn(100, D, device="cuda")
    t = torch.tensor([5, 99, 5, 0], device="cuda")
    out = torch.empty(4, D, device="cuda")
    TO.gather_rows(table, t, out)
    assert torch.equal(out, table[t])
    acc = torch.zeros_like(table)
    TO.scatter_add_rows(acc, t, out)
    ref = torch.zeros_like(table).index_add_(0, t, out)
    assert torch.allclose(acc, ref, rtol=1e-6, atol=1e-6)
    x = torch.randn(4, D, device="cuda", requires_grad=True)
    dyy = torch.randn(4, D, device="cuda")
    torch.nn.functional.silu(x).backward(dyy)
    dxs = torch.empty(4, D, device="cuda")
    TO.silu_bwd(x.detach(), dyy, dxs)
    assert G.relerr(dxs, x.grad) < 1e-5


# K + 1 on both sides of every register-tile boundary of train_loss_kernel<NJ> (NJ = 2, 5, 9, 17, 33 columns of 32 classes per lane)
@pytest.mark.parametrize("K", [32, 63, 64, 159, 160, 256, 287, 288, 512, 543, 544, 1055])
def test_q_sample_and_fused_loss_match_oracle(G, TO, K):
    """q_sample ids bit-exact vs the oracle (same uniforms); loss terms, log_model_prob and d loss/d logits vs torch autograd through the oracle."""
    B, L, T = 5, 265, 100
    sched, s8 = sched8(K, T)
    x0 = (portable_uniform(1, (B, L)) * K).long().clamp(max=K - 1)
    t = torch.tensor([57, 0, 99, 1, 20])
    pt = torch.tensor([0.013, 0.004, 0.01, 0.02, 0.01])
    u = portable_uniform(2, (B, K + 1, L))
    x_t_ref = O.q_sample_ids(sched, x0, t, u, T=T, num_classes=K + 1)
    x_t = TO.q_sample(x0.cuda(), t.cuda(), u.cuda(), s8.cuda(), T)
    assert torch.equal(x_t.cpu(), x_t_ref)
    out = ((portable_uniform(3, (B, K, L)) - 0.5) * 6.0)
    out[:, :, :9] += 12.0 * torch.nn.functional.one_hot(x0[:, :9], K).permute(0, 2, 1)
    out.requires_grad_(True)
    ref = O.train_loss_from_logits(sched, out, x0, x_t_ref, t, pt, T=T, aux_weight=5e-4, adaptive_aux=True, mask_weight=(0.8, 1.2))
    ref["loss"].backward()
    logits = out.detach().permute(0, 2, 1).contiguous().cuda()
    dlog = torch.empty_like(logits)
    prob = torch.empty(B, K + 1, L, device="cuda")
    hits = torch.empty(B, L, 2, dtype=torch.int32, device="cuda")
    hist, cnt = torch.zeros(T, device="cuda"), torch.zeros(T, device="cuda")
    hist[57] = 3.0
    res = TO.train_loss(logits, x0.cuda(), x_t, t.cuda(), pt.cuda(), s8.cuda(), T, aux_weight=5e-4, adaptive=True, mask_weight=(0.8, 1.2), dlogits=dlog,
                        log_model_prob=prob, hits=hits, lt_history=hist, lt_count=cnt)
    assert abs(float(res["loss"]) - float(ref["loss"].detach())) <= 2e-5 * abs(float(ref["loss"].detach()))
    assert torch.allclose(res["kl_loss"].cpu(), ref["kl_loss"].detach(), rtol=5e-5, atol=1e-4)
    assert torch.allclose(res["vb_loss"].cpu(), ref["vb_loss"].detach(), rtol=5e-5, atol=1e-2)
    assert float((prob.cpu() - ref["log_model_prob"].detach()).abs().max()) < 5e-5
    g = out.grad.permute(0, 2, 1)
    assert float((dlog.cpu() - g).abs().max()) <= 3e-4 * float(g.abs().max())
    assert torch.equal(hits[..., 0].cpu().bool(), ref["x0_recon"] == x0) and torch.equal(hits[..., 1].cpu().bool(), ref["xt_1_recon"] == x_t_ref)
    kl = ref["kl_loss"].detach()
    exp_hist = torch.zeros(T); exp_hist[57] = 3.0
    new = 0.1 * kl ** 2 + 0.9 * exp_hist[t]
    exp_hist[t] = new
    assert torch.allclose(hist.cpu(), exp_hist, rtol=1e-4) and torch.equal(cnt.cpu(), torch.zeros(T).index_add_(0, t, torch.ones(B)))


# ------------------------------------------------------------------------------------------------ whole model
def _grad_report(tag, grads, ref_of, tol, loose=None):
    """Per-parameter max-abs error relative to that parameter's reference gradient scale.  Parameters whose true gradient is zero
    (attention key biases: softmax is invariant to a shift common to all keys) only carry rounding noise in the reference, so the scale
    is floored at 1e-4 of the largest gradient in the model.  loose = [(name fragments, tolerance), ...]: a parameter whose name contains one
    of a group's fragments is held to the first such group's tolerance instead of tol.  Returns the worst error."""
    refs = {n: ref_of(n) for n in grads}
    gmax = max(float(r.abs().max()) for r in refs.values())
    rows = []
    for n, gr in grads.items():
        r = refs[n]
        assert gr is not None and gr.shape == r.shape, n
        abs_err = float((gr.detach().cpu() - r).abs().max())
        rows.append((abs_err / max(float(r.abs().max()), 1e-4 * gmax), n, float(r.abs().max()), abs_err))
    rows.sort(reverse=True)
    for e, n, rm, ae in rows[:6]:
        print(f"[{tag}] {n}: rel {e:.3e} (ref max {rm:.3e}, abs err {ae:.3e})")
    if tol is not None:
        for e, n, rm, ae in rows:
            t_n = next((lt for frags, lt in (loose or ()) if any(f in n for f in frags)), tol)
            assert e < t_n, (n, e, t_n)
    return rows[0][0]


# (loss, gradient, log_model_prob): 4x the errors measured on an H100 80GB HBM3 (700 W) -- tf32 loss 2.3e-6, prob 1.4e-5, gradient 1.6e-3;
# bf16 loss 8.0e-6, prob 9.7e-5, gradient 8.5e-2 -- where that is tighter than the parametrised bound (prob: 5e-3 tf32, 5e-2 bf16)
TINY_MEASURED_TOL = {"tf32": (9.2e-6, 6.5e-3, 5.6e-5), "bf16": (3.2e-5, 3.4e-1, 3.9e-4)}


@pytest.mark.parametrize("precision,tol_loss,tol_grad", [("tf32", 2e-3, 2e-2), ("bf16", 2e-2, 1.2e-1)])
def test_tiny_training_step_matches_reference_loss_and_gradients(G, TO, precision, tol_loss, tol_grad):
    """Reference golden (unmodified DiffusionTransformer.forward(return_loss=True) + autograd, 2 layers, D=128)."""
    m_loss, m_grad, m_prob = TINY_MEASURED_TOL[precision]
    tol_prob = min(5e-3 if precision == "tf32" else 5e-2, m_prob)
    lt_rtol = 10 * tol_loss
    tol_loss, tol_grad = min(tol_loss, m_loss), min(tol_grad, m_grad)
    sd, gx = load_golden("xf_tiny.npz")
    _, g = load_golden("train_tiny.npz")
    K, D, NL, NH, CD, B, L = [int(v) for v in gx["__cfg"]]
    m = build_dt(K, D, NL, NH, CD, sd=sd)
    m.transformer.train_engine.__init__(m.transformer, precision=precision)
    x0 = torch.from_numpy(g["in_x0"]).long().cuda()
    t, pt = torch.from_numpy(g["in_t"]).cuda(), torch.from_numpy(g["in_pt"]).cuda()
    x_t = TO.q_sample(x0, t, torch.from_numpy(g["in_uniform"]).cuda(), m._sched(), 100)
    loss, prob, grads = G.run_loss_and_grads(m, x0, x_t, torch.from_numpy(g["in_cond"]).cuda(), t, pt)
    ref_loss = float(g["out_loss"])
    e_loss = abs(float(loss) - ref_loss) / abs(ref_loss)
    e_prob = float((prob.cpu() - torch.from_numpy(g["out_probs"])).abs().max())
    e_grad = _grad_report(precision, grads, lambda n: torch.from_numpy(g["grad.transformer." + n]), None)
    print(f"MEASURED tiny-{precision}: loss {float(loss):.6f} vs reference {ref_loss:.6f}, rel {e_loss:.3e}; prob {e_prob:.3e}; worst gradient rel {e_grad:.3e}")
    assert e_loss <= tol_loss and e_prob <= tol_prob and e_grad <= tol_grad
    assert torch.allclose(m.Lt_history.cpu(), torch.from_numpy(g["out_Lt_history"]), rtol=lt_rtol, atol=1e-3)


def test_midsize_training_step_matches_oracle_autograd(G, TO):
    """D=256 / 4 heads / 3 layers / K=64, B=4: every parameter gradient vs torch autograd through the oracle (CPU fp32).
    Tolerances: 4x the errors measured on an H100 80GB HBM3 (700 W): loss 3.7e-6 (was 2e-3), gradient 3.1e-3 (was 2e-2)."""
    _oracle_step(G, TO, "midsize", 64, 256, 3, 4, 96, torch.tensor([3, 0, 77, 99]), torch.tensor([0.01, 0.02, 0.005, 0.01]), "tf32", 1.5e-5, 1.25e-2)


# bf16 full width, per parameter group, 4x the worst error measured in the group on an H100 80GB HBM3 (700 W).  The attention query and key
# parameters get their gradients only through dS = scale P (dP - Delta), and with near-uniform scores at initialisation dP - Delta is a small
# difference of bf16-rounded terms.  The key biases have exactly zero gradient (their error is over the 1e-4 floor): measured 0.45.  The query
# weights / biases and key weights: 0.19.  Every other parameter: 8.1e-3, so an entirely wrong or zeroed gradient (error 1) fails.
FULL_BF16_GROUPS = [((".key.bias",), 1.8), ((".query.", ".key.weight"), 0.77)]
FULL_BF16_REST = 3.3e-2


@pytest.mark.parametrize("precision,tol_loss,tol_grad", [("tf32", 6.2e-6, 5e-2), ("bf16", 3.4e-5, 1.8)])
def test_full_width_training_step_matches_oracle_autograd(G, TO, precision, tol_loss, tol_grad):
    """The width the benchmark trains: D=1024 / 16 heads / hidden 4096 / 2 layers / K=256, B=2, 77 condition tokens.
    Tolerances: 4x the errors measured on an H100 80GB HBM3 (700 W): tf32 loss 1.5e-6, every gradient 1.2e-2; bf16 loss 8.5e-6, gradients
    per parameter group (FULL_BF16_GROUPS; the parametrised 1.8 is the key-bias group's bound)."""
    loose = None
    if precision == "bf16":
        assert FULL_BF16_GROUPS[0][1] == tol_grad
        loose, tol_grad = FULL_BF16_GROUPS, FULL_BF16_REST
    _oracle_step(G, TO, f"full-{precision}", 256, 1024, 2, 16, 512, torch.tensor([3, 77]), torch.tensor([0.01, 0.005]), precision, tol_loss, tol_grad,
                 loose=loose)


def _oracle_step(G, TO, tag, K, D, NL, NH, CD, t, pt, precision, tol_loss, tol_grad, loose=None):
    B, L = t.numel(), 265
    sd = O.make_transformer_state_dict(K=K, D=D, n_layer=NL, n_head=NH, cond_dim=CD, seed=3)
    gen = torch.Generator().manual_seed(5)
    for k in sd:
        if k.endswith("bias") or "ln2.weight" in k or "to_logits.0.weight" in k:
            sd[k] = sd[k] + 0.05 * torch.randn(sd[k].shape, generator=gen)
    m = build_dt(K, D, NL, NH, CD, sd=sd)
    m.transformer.train_engine.__init__(m.transformer, precision=precision)
    cond = torch.randn(B, 77, CD, generator=gen)
    cond = cond / cond.norm(dim=-1, keepdim=True)
    x0 = torch.randint(0, K, (B, L), generator=gen)
    u = portable_uniform(9, (B, K + 1, L))
    names = [n for n in sd if n.startswith("transformer.") and "attn2.mask" not in n]
    leaf = {k: (v.clone().requires_grad_(True) if k in names else v) for k, v in sd.items()}
    sched = {k: sd[k] for k in sd if k.startswith("log_")}
    ref = O.train_loss(leaf, sched, x0, cond, t, pt, u, n_layer=NL, n_head=NH, spatial=(5, 53), T=100, aux_weight=5e-4, adaptive_aux=True)
    ref["loss"].backward()
    x_t = TO.q_sample(x0.cuda(), t.cuda(), u.cuda(), m._sched(), 100)
    assert torch.equal(x_t.cpu(), ref["x_t"])
    loss, prob, grads = G.run_loss_and_grads(m, x0.cuda(), x_t, cond.cuda(), t.cuda(), pt.cuda())
    rl = float(ref["loss"].detach())
    e_loss = abs(float(loss) - rl) / abs(rl)
    e_grad = _grad_report(tag, grads, lambda n: leaf["transformer." + n].grad, None)
    if loose is not None:  # per-parameter tolerances; the worst-error print above is the record
        _grad_report(tag, grads, lambda n: leaf["transformer." + n].grad, tol_grad, loose=loose)
        tol_grad = float("inf")
    print(f"MEASURED {tag}: loss {float(loss):.6f} vs oracle {rl:.6f}, rel {e_loss:.3e}; worst gradient rel {e_grad:.3e}")
    assert e_loss <= tol_loss and e_grad <= tol_grad


def test_module_forward_backward_and_optimizer_steps(G, TO):
    """The reference-facing call: forward({'content_token', 'condition_embed_token'}, return_loss=True) -> loss.backward() -> AdamW on the
    parameter groups of parameters(name=...); on a fixed batch the loss must go down, and validation mode must not need gradients."""
    K, D, NL, NH, CD, B, L = 64, 256, 2, 4, 96, 4, 265
    m = build_dt(K, D, NL, NH, CD)
    m.train()
    for p in m.parameters():
        p.requires_grad_(True)
    groups = m.parameters(name="transformer")
    assert len(groups) == 2 and sum(len(g["params"]) for g in groups) == len(list(m.transformer.parameters()))
    opt = torch.optim.AdamW(groups, lr=3e-4, betas=(0.9, 0.96))
    gen = torch.Generator().manual_seed(0)
    batch = {"content_token": torch.randint(0, K, (B, L), generator=gen).cuda(), "condition_embed_token": torch.randn(B, 77, CD, generator=gen).cuda()}
    losses = []
    for it in range(12):
        torch.manual_seed(100)  # same (t, x_t) draw every iteration: isolates the optimisation effect
        out = m(batch, return_loss=True)
        assert out["logits"].shape == (B, K + 1, L) and out["loss"].dim() == 0
        opt.zero_grad()
        out["loss"].backward()
        assert all(p.grad is not None and torch.isfinite(p.grad).all() for p in m.transformer.parameters())
        opt.step()
        losses.append(float(out["loss"].detach()))
    print("losses", [round(v, 4) for v in losses])
    assert losses[-1] < losses[0]
    assert float(m.Lt_count.sum()) == 12 * B
    with torch.no_grad():
        out = m(batch, return_loss=True, return_logits=False)
    assert "logits" not in out and math.isfinite(float(out["loss"]))


def test_content_conditioned_sampling_runs(G, TO):
    """sample(filter_ratio>0): q_sample to t = start-1, then the fused loop from there (diffusion_transformer.py:647-655)."""
    K, D, NL, NH, CD, B, L = 64, 256, 2, 4, 96, 2, 265
    m = build_dt(K, D, NL, NH, CD)
    m.truncation = "top0.85r"
    tok = torch.randint(0, K, (B, L)).cuda()
    cond = torch.randn(B, 77, CD).cuda()
    run = lambda: m.sample(condition_token=None, condition_mask=None, condition_embed=cond, content_token=tok, filter_ratio=0.3, batch_size=B)["content_token"]
    torch.manual_seed(77)
    fused = run()
    assert fused.shape == (B, L) and int(fused.max()) < K and int(fused.min()) >= 0
    m.p_sample = m.p_sample  # re-bound instance attribute -> the stage-by-stage path (what a monkey-patching caller triggers)
    torch.manual_seed(77)
    staged = run()
    assert torch.equal(fused, staged)
    # the start state really is q_sample at t = 29: with the same seed the first RNG draw is q_sample's
    torch.manual_seed(77)
    x29 = m.q_sample(O.index_to_log_onehot(tok.cpu(), K + 1).cuda(), torch.full((B,), 29, device="cuda", dtype=torch.long), return_index=True)
    frac_masked = float((x29 == K).float().mean())
    assert 0.15 < frac_masked < 0.40 and float((x29[x29 != K] == tok[x29 != K]).float().mean()) > 0.9


@pytest.mark.parametrize("B,H,Lq,Lk", [(2, 4, 265, 265), (3, 2, 265, 77), (1, 1, 100, 64), (2, 3, 64, 130)])
def test_fused_attention_forward_backward_match_autograd(G, TO, B, H, Lq, Lk):
    """csrc/attention_train.cu on strided token-major views (as the engine calls it) vs torch autograd on the same bf16-rounded inputs."""
    g = torch.Generator().manual_seed(B * 1000 + Lq + Lk)
    D = H * 64
    qkv = (torch.randn(B * Lq, 3 * D + 8, generator=g) * 1.5).bfloat16().cuda()       # q lives in a wider buffer, like the QKV GEMM output
    kv = (torch.randn(B * Lk, 2 * D, generator=g) * 1.5).bfloat16().cuda()
    dout = torch.randn(B * Lq, D, generator=g).bfloat16().cuda()
    q, k, v = qkv[:, 8:8 + D], kv[:, :D], kv[:, D:]
    o = torch.empty(B * Lq, D, dtype=torch.bfloat16, device="cuda")
    lse = torch.empty(B * H, Lq, device="cuda")
    TO.attention_train_fwd(q, k, v, o, lse, B, H, Lq, Lk, 0.125)
    heads = lambda x, L: x.float().reshape(B, L, H, 64).permute(0, 2, 1, 3).detach().clone().requires_grad_(True)
    qr, kr, vr = heads(q, Lq), heads(k, Lk), heads(v, Lk)
    s = (qr @ kr.transpose(-1, -2)) * 0.125
    oref = torch.softmax(s, -1) @ vr
    unheads = lambda x, L: x.permute(0, 2, 1, 3).reshape(B * L, D)
    assert G.relerr(o.float(), unheads(oref, Lq).detach()) < 1e-2
    assert float((lse.reshape(B, H, Lq) - torch.logsumexp(s, -1).detach() * 1.4426950408889634).abs().max()) < 2e-3
    oref.backward(heads(dout, Lq).detach())
    dq = torch.zeros(B * Lq, 3 * D + 8, dtype=torch.bfloat16, device="cuda")
    dkv = torch.zeros(B * Lk, 2 * D, dtype=torch.bfloat16, device="cuda")
    delta = torch.empty(B * H, Lq, device="cuda")
    TO.attention_train_bwd(q, k, v, o, dout, lse, delta, dq[:, 8:8 + D], dkv[:, :D], dkv[:, D:], B, H, Lq, Lk, 0.125)
    e_q = G.relerr(dq[:, 8:8 + D].float(), unheads(qr.grad, Lq))
    e_k = G.relerr(dkv[:, :D].float(), unheads(kr.grad, Lk))
    e_v = G.relerr(dkv[:, D:].float(), unheads(vr.grad, Lk))
    print(f"fused attention B={B} H={H} Lq={Lq} Lk={Lk}: dq {e_q:.2e} dk {e_k:.2e} dv {e_v:.2e}")
    assert e_q < 1.5e-2 and e_k < 1.5e-2 and e_v < 1.5e-2
    assert float(dq[:, :8].float().abs().max()) == 0.0 and float(dq[:, 8 + D:].float().abs().max()) == 0.0   # nothing outside the head columns
