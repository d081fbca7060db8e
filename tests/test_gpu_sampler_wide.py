"""The CTA-per-column posterior sampler (dsb_posterior_sample_wide / _wide_loop, csrc/sampler.cu) per element against a restatement of its
contract, for codebooks up to K = 4095.

The contract is the warp kernel's (tests/test_gpu_sampler.py states it), and the order-independent parts of tests/sampler_reference.py are
used as they are: top-k keep-set, truncation, the posterior formula, Gumbel scores and the id check.  Two things depend on the reduction
order and are restated here for the wide kernel's order (block_ctx.cuh): element k = tid + 256 j; each thread adds its elements in
ascending j, a warp xor butterfly 16 ... 1 adds lane pairs, then the 8 warp partials are added in ascending warp order, starting from warp
0's.  That fixes
  * log_pred's fp64 sum of exp (block_sum below: bit for bit);
  * the tree depth in the nucleus and posterior error bounds: CAP + 5 + (8 - 1) roundings instead of the warp kernel's NJ + 5.
K covers both sides of every CAP instantiation (K + 1 <= 512, 1024, 2304, 4096), the warp kernel's limit 1055 / 1056 and the ceiling."""
import math

import pytest
import torch

from oracle import diffsound_oracle as O
from tests import sampler_reference as R
from tests.test_gpu_sampler import POST_SCALE, REGIMES, SENTINEL, TRUNCS, check_ids, make_inputs

pytestmark = pytest.mark.gpu

T = 100
NT, NW = 256, 8
MAX_K = 4095
KS = [1, 31, 255, 256, 510, 511, 512, 1022, 1023, 1024, 1055, 1056, 1087, 2047, 2048, 2302, 2303, 2304, 4094, 4095]
SHAPES = [(1, 1), (1, 7), (3, 9), (16, 8), (3, 265)]


@pytest.fixture(scope="module")
def ops():
    from tests import gpu_common
    return gpu_common.ops


def cap_of(C):
    return (C + NT - 1) // NT


def block_sum(x):
    """fp64 sum over the last dim in the wide kernel's order (see the module docstring).  The last dim is padded with zeros to CAP * NT;
    adding an exact zero changes nothing, so the padding reproduces the threads that hold no element."""
    n = x.shape[-1]
    cap = cap_of(n)
    v = torch.zeros(*x.shape[:-1], cap * NT, dtype=torch.float64)
    v[..., :n] = x
    v = v.reshape(*x.shape[:-1], cap, NT)
    s = torch.zeros(v.shape[:-2] + (NT,), dtype=torch.float64)
    for j in range(cap):
        s = s + v[..., j, :]
    s = s.reshape(*x.shape[:-1], NW, 32)
    for o in (16, 8, 4, 2, 1):
        s = s[..., :o] + s[..., o:2 * o]
    s = s[..., 0]
    r = s[..., 0]
    for w in range(1, NW):
        r = r + s[..., w]
    return r


def log_pred_wide(logits):
    """sampler_reference.log_pred with the wide kernel's summation order; same near-midpoint rule."""
    B, K, L = logits.shape
    x = logits.permute(0, 2, 1).float()
    d = x.double() - x.max(dim=-1, keepdim=True).values.double()
    lse = torch.log(block_sum(torch.exp(d))).unsqueeze(-1)
    v64 = d - lse
    f = v64.float()
    mid = ((d - lse * (1 + 2.0 ** -45)).float() != (d - lse * (1 - 2.0 ** -45)).float()) & (v64 > -70.001)
    pad = lambda t, val: torch.cat((t.permute(0, 2, 1), torch.full((B, 1, L), val, dtype=t.dtype)), dim=1)
    return pad(f.clamp(-70, 0), -70.0), pad(mid, False)


def near_midpoint_across_orders(logits, eps=2.0 ** -45):
    """(B, K+1, L) mask of log-probs whose fp32 rounding can differ between two summation orders of the fp64 sum s = sum exp(d).  Both sums
    hold every term to within (depth + 1) 2^-53 s (positive terms: the tree depth bounds the relative error, one more for fp64 exp), so
    their lse = log s differ by at most (NJ + 5 + CAP + 5 + NW + 2) 2^-53 absolute: below 2^-47 for every K this file compares.  The
    same-order window of log_pred_wide is relative to lse, which is too narrow here when one logit dominates and lse is tiny; this one is
    absolute: d - lse -+ eps round to different fp32 values."""
    B, K, L = logits.shape
    x = logits.permute(0, 2, 1).float()
    d = x.double() - x.max(dim=-1, keepdim=True).values.double()
    v64 = d - torch.log(block_sum(torch.exp(d))).unsqueeze(-1)
    near = ((v64 - eps).float() != (v64 + eps).float()) & (v64 > -70.001)
    return torch.cat((near.permute(0, 2, 1), torch.zeros(B, 1, L, dtype=torch.bool)), dim=1)


def keep_nucleus_wide(lp, r):
    """sampler_reference.keep_nucleus with the wide kernel's tree depth: CAP + 5 + NW roundings along its sum instead of NJ + 5."""
    B, C, L = lp.shape
    sv, idx = R.order(lp)
    e = torch.exp(sv.double()).float().double()
    Tc = torch.cumsum(e, dim=1) - e
    T_nz = torch.cumsum(e * (sv != 0), dim=1) - e * (sv != 0)
    n = torch.arange(C, dtype=torch.float64).view(1, C, 1)
    delta = 5 * R.U32 * T_nz + (cap_of(C) + 5 + NW + n) * R.U64 * Tc
    fr = float(torch.tensor(r, dtype=torch.float32))
    keep_s = Tc.float() < fr
    keep_s[:, 0] = True
    amb_s = ((Tc - delta).float() < fr) != ((Tc + delta).float() < fr)
    amb_s[:, 0] = False
    return R._unsort(keep_s, idx), R._unsort(amb_s, idx), R._tie_at_boundary(sv, keep_s.sum(1))


def posterior_wide(lp, x_t, t_post, sched):
    """sampler_reference.posterior with the wide kernel's tree depth.  Its logsumexp error term counts NJ + 5 summation roundings; the wide
    kernel's sum has CAP + 5 + NW.  That term enters the bound linearly and twice (directly, and through qn into the last lae with weight
    1), so the bound moves by 2 (CAP + NW - NJ) u."""
    C = lp.shape[1]
    post, bound = R.posterior(lp, x_t, t_post, sched, T)
    return post, bound + 2 * (cap_of(C) + NW - (C + 31) // 32) * R.U32


def reference_keep_wide(logits, mode, r, k):
    lp, mid = log_pred_wide(logits)
    B, C, L = lp.shape
    amb = torch.zeros_like(lp, dtype=torch.bool)
    tie = torch.zeros(B, L, dtype=torch.bool)
    lpt = lp
    if mode == 1:
        keep, amb, tie = keep_nucleus_wide(lp, r)
        lpt = R.truncate(lp, keep)
    elif mode == 2:
        keep, tie = R.keep_topk(lp, k)
        lpt = R.truncate(lp, keep)
    return lp, lpt, mid.any(1, keepdim=True), amb, tie


def run_stages(ops, fn, logits, x_t, tp, u, sched, tr, with_tp, seed):
    """The five stage combinations of the library on one case; returns (log-probs, ids) of each, on the host."""
    B, K, L = logits.shape
    C = K + 1
    dev = lambda t: t.contiguous().cuda()
    blk, u_d, x_d, s_d = dev(logits.permute(0, 2, 1)), dev(u), dev(x_t), dev(sched)
    t_d = dev(torch.randint(0, T, (B,), generator=torch.Generator().manual_seed(seed)) if with_tp else tp)
    tp_d = dev(tp) if with_tp else None
    nan = lambda: torch.full((B, C, L), math.nan, device="cuda")
    sentinel = lambda: torch.full((B, L), SENTINEL, dtype=torch.long, device="cuda")
    IN, NOPOST, NOSAMP = ops.STAGE_INPUT_LOGPROB, ops.STAGE_SKIP_POSTERIOR, ops.STAGE_SKIP_SAMPLE
    out = {}
    lp, x = nan(), sentinel()
    fn(blk, None, None, None, None, T=T, **tr, x_next=x, log_prob_out=lp, stage=NOPOST | NOSAMP)
    out["ps"] = (lp, x)
    lp, x = nan(), sentinel()
    fn(blk, None, None, u_d, None, T=T, **tr, x_next=x, log_prob_out=lp, stage=NOPOST)
    out["ts"] = (lp, x)
    lp, x = nan(), sentinel()
    fn(out["ps"][0], x_d, t_d, None, s_d, T=T, trunc_mode=0, t_post=tp_d, x_next=x, log_prob_out=lp, stage=IN | NOSAMP)
    out["qp"] = (lp, x)
    lp, x = nan(), sentinel()
    fn(out["qp"][0], None, None, u_d, None, T=T, trunc_mode=0, x_next=x, log_prob_out=lp, stage=IN | NOPOST)
    out["ls"] = (lp, x)
    lp, x = nan(), sentinel()
    fn(blk, x_d, t_d, u_d, s_d, T=T, **tr, t_post=tp_d, x_next=x, log_prob_out=lp, stage=0)
    out["f"] = (lp, x)
    return {k: (a.cpu(), b.cpu()) for k, (a, b) in out.items()}


def case_inputs(K, regime, it, seed):
    mode, r, k = TRUNCS[it]
    C = K + 1
    if mode == 2:
        k = {-1: C - 1, 0: C}.get(k, k)
    B, L = SHAPES[(KS.index(K) + REGIMES.index(regime) + it) % len(SHAPES)] if K in KS else SHAPES[(K + it) % len(SHAPES)]
    logits, x_t, tp, u = make_inputs(K, B, L, regime, seed)
    sched = R.sched_table(O.schedule_buffers(T, C), T)
    return dict(trunc_mode=mode, trunc_r=r, trunc_k=k), logits, x_t, tp, u, sched


def run_case(ops, K, regime, it, seed, stats):
    tr, logits, x_t, tp, u, sched = case_inputs(K, regime, it, seed)
    B, _, L = logits.shape
    mode, r, k = tr["trunc_mode"], tr["trunc_r"], tr["trunc_k"]
    o = run_stages(ops, ops.posterior_sample_wide, logits, x_t, tp, u, sched, tr, seed % 2 == 0, seed)
    (lp_ps, x_ps), (lp_ts, x_ts), (lp_qp, x_qp), (lp_ls, x_ls), (lp_f, x_f) = (o[s] for s in ("ps", "ts", "qp", "ls", "f"))
    what = f"K={K} B={B} L={L} {regime} trunc={(mode, r, k)}"

    _, lpt, mid, amb, tie = reference_keep_wide(logits, mode, r, k)
    differ = lp_ps != lpt
    bad = differ & ~mid & ~amb
    assert not bad.any(), f"{what}: predict_start differs at {bad.nonzero()[:4].tolist()}: {lp_ps[bad][:4].tolist()} vs {lpt[bad][:4].tolist()}"
    assert bool((x_ps == SENTINEL).all()) and bool((x_qp == SENTINEL).all()), f"{what}: a SKIP_SAMPLE launch wrote x_next"
    stats["midpoint_columns"] += int(mid.sum())
    stats["ambiguous"] += int(amb.sum())
    stats["ambiguous_differ"] += int((differ & amb).sum())
    stats["tie_at_boundary"] += int(tie.sum())

    assert torch.equal(lp_ts, lp_ps), what
    stats["near_tie"] += check_ids(x_ts, lp_ts, u, what + " truncate-then-sample")

    post, bound = posterior_wide(lp_ps, x_t, tp, sched)
    err = (lp_qp.double() - post).abs()
    over = ~(err <= POST_SCALE * bound)
    assert not over.any(), f"{what}: posterior error {err[over][:4].tolist()} over bound {bound[over][:4].tolist()} at {over.nonzero()[:4].tolist()}"
    key = f"CAP={cap_of(K + 1)}"
    stats["post_err"][key] = max(stats["post_err"].get(key, 0.0), float(err.max()))
    stats["post_ratio"][key] = max(stats["post_ratio"].get(key, 0.0), float((err / bound).max()))

    assert torch.equal(lp_ls, lp_qp), what
    stats["near_tie"] += check_ids(x_ls, lp_qp, u, what + " log_sample_categorical")

    assert torch.equal(lp_f, lp_qp) and torch.equal(x_f, x_ls), f"{what}: fused launch differs from the staged launches"
    stats["cases"] += 1


def new_stats():
    return dict(cases=0, midpoint_columns=0, ambiguous=0, ambiguous_differ=0, tie_at_boundary=0, near_tie=0, post_err={}, post_ratio={})


def test_block_sum_restates_the_order_it_documents():
    """block_sum is not a plain sum: the fp64 results of a sequential sum and of the kernel's order differ on some rows (this guards against
    the restatement silently degenerating to torch.sum)."""
    g = torch.Generator().manual_seed(3)
    x = torch.exp(torch.randn(64, 2049, generator=g, dtype=torch.float64) * 4)
    seq = x.cumsum(-1)[:, -1]
    assert not torch.equal(block_sum(x), seq)
    assert torch.allclose(block_sum(x), seq, rtol=1e-13, atol=0)


@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("K", KS)
def test_wide_sampler_stages_match_restatement(ops, K, regime):
    stats = new_stats()
    for it in range(len(TRUNCS)):
        run_case(ops, K, regime, it, seed=1000 * K + 10 * REGIMES.index(regime) + it + 7, stats=stats)
    print(f"\nWIDE SAMPLER K={K} {regime}: {stats}")
    if regime == "quantised" and K >= 31:
        assert stats["tie_at_boundary"] > 0


@pytest.mark.parametrize("K", [1, 31, 256, 1023, 1055])
def test_wide_equals_warp_kernel(ops, K):
    """Same inputs through both kernels: predict_start log-probs bit-identical except in near-midpoint columns (their fp64 sums run in
    different orders), posteriors within the bound, and fused ids equal except at near ties of the Gumbel scores."""
    stats = dict(mid_columns=0, near_tie=0)
    for regime in REGIMES:
        for it in range(len(TRUNCS)):
            seed = 77 * K + 10 * REGIMES.index(regime) + it
            tr, logits, x_t, tp, u, sched = case_inputs(K, regime, it, seed)
            wide = run_stages(ops, ops.posterior_sample_wide, logits, x_t, tp, u, sched, tr, False, seed)
            warp = run_stages(ops, ops.posterior_sample, logits, x_t, tp, u, sched, tr, False, seed)
            what = f"K={K} {regime} trunc={tuple(tr.values())}"
            mid = near_midpoint_across_orders(logits)
            amb = torch.zeros_like(mid)
            if tr["trunc_mode"] == 1:  # either kernel's nucleus decision may rest on the last bits of its own sum
                lp_w, _ = log_pred_wide(logits)
                lp_p, _, _ = R.log_pred(logits)
                amb = keep_nucleus_wide(lp_w, tr["trunc_r"])[1] | R.keep_nucleus(lp_p, tr["trunc_r"])[1]
            near_col = mid.any(1, keepdim=True) | amb.any(1, keepdim=True)
            differ = wide["ps"][0] != warp["ps"][0]
            assert not (differ & ~near_col).any(), f"{what}: predict_start differs outside near-midpoint columns"
            stats["mid_columns"] += int((differ.any(1, keepdim=True) & near_col).sum())
            same_col = ~differ.any(1)
            post, bound = posterior_wide(warp["ps"][0], x_t, tp, sched)
            for s in ("qp", "f"):
                e = (wide[s][0].double() - warp[s][0].double()).abs()
                assert bool(((e <= 2 * bound) | ~same_col.unsqueeze(1)).all()), f"{what}: stage {s} posteriors differ beyond twice the bound"
            _, _, val, gb = R.gumbel_ids(warp["f"][0], u)
            wrong, near = R.id_check(wide["f"][1], val, gb, extra=2 * bound, ref=warp["f"][1])
            wrong &= same_col
            assert not wrong.any(), f"{what}: {int(wrong.sum())} fused ids differ beyond a near tie"
            stats["near_tie"] += int((near & same_col).sum())
    print(f"\nWIDE vs WARP K={K}: {stats}")


def test_wide_gumbel_exact_ties_pick_the_lowest_index(ops):
    """K = 2048: equal log-probs and equal uniforms across lanes of one warp, across warps, within one thread (k and k + 256), and with the
    mask class K (thread 0, slot 8).  The lowest index must win, with no allowance."""
    K = 2048
    groups = [(5, 37), (3, 40, 300), (10, 266), (37, 293, 40), (7, K), (K - 1, K), (0, K), (300, 1800, K), (255, 256), (1000, 2000),
              (31, 32), (1792, 2047)]
    B, L, C = 2, len(groups), K + 1
    g = torch.Generator().manual_seed(K)
    lp = -40.0 - 20.0 * torch.rand(B, C, L, generator=g)
    u = torch.rand(B, C, L, generator=g)
    for l, gr in enumerate(groups):
        for b in range(B):
            lp[b, list(gr), l] = -0.25 - b
            u[b, list(gr), l] = 0.625
    want = torch.tensor([min(gr) for gr in groups]).expand(B, L)
    _, _, val, _ = R.gumbel_ids(lp, u)
    assert torch.equal(val.argmax(1), want)
    x = torch.full((B, L), SENTINEL, dtype=torch.long, device="cuda")
    ops.posterior_sample_wide(lp.cuda(), None, None, u.cuda(), None, T=T, trunc_mode=0, x_next=x,
                              stage=ops.STAGE_INPUT_LOGPROB | ops.STAGE_SKIP_POSTERIOR)
    assert torch.equal(x.cpu(), want), (x.cpu().tolist(), groups)


def test_wide_loop_kernel_equals_explicit_uniforms(ops):
    """dsb_posterior_sample_wide_loop == dsb_posterior_sample_wide fed torch.rand's tensor, step by step, for K = 1056 and 2048 without
    truncation, with nucleus 0.85 and with top-20, over 6 steps with t_post != t.  After every step the loop state is read back as in the warp
    kernel's loop test."""
    B, L = 3, 265
    steps, post = [99, 98, 60, 60, 3, 0], [99, 97, 60, 58, 3, 0]
    n = len(steps)
    for K in (1056, 2048):
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
                ref = ops.posterior_sample_wide(lg, ref, torch.full((B,), ti, device="cuda"), u, sched, T=T,
                                                t_post=torch.full((B,), tp, device="cuda"), **tr)
                refs.append(ref.clone())
            nthreads, inc = ops.aten_rand_geometry(B * (K + 1) * L)
            ctrl = torch.tensor([seed, 0, inc, nthreads, 0, n, 0, 0], dtype=torch.int64, device="cuda")
            t_s, tp_s = torch.tensor(steps, device="cuda"), torch.tensor(post, device="cuda")
            t = torch.full((B,), steps[0], device="cuda")
            tpb = torch.full((B,), post[0], device="cuda")
            x = x0.clone()
            for i, lg in enumerate(logits):
                ops.posterior_sample_wide_loop(lg, x, t, tpb, sched, ctrl, t_s, tp_s, T=T, **tr)
                torch.cuda.synchronize()
                what = (K, mode, i)
                assert torch.equal(x, refs[i]), what
                assert ctrl.tolist() == [seed, inc * (i + 1), inc, nthreads, i + 1, n, 0, 0], (what, ctrl.tolist())
                j = min(i + 1, n - 1)
                assert t.tolist() == [steps[j]] * B and tpb.tolist() == [post[j]] * B, (what, t.tolist(), tpb.tolist())


def test_in_kernel_uniforms_at_k2048_equal_torch_rand(ops):
    """The Philox replay at the sampling loop's size for the 2048-code codebook, (16, 2049, 265), is torch.rand bit for bit."""
    shape = (16, 2049, 265)
    n = shape[0] * shape[1] * shape[2]
    torch.manual_seed(2049)
    a = torch.rand(*shape, device="cuda")
    assert torch.equal(ops.aten_uniform(n, 2049, 0).view(shape), a)


def test_wide_sampler_refuses_bad_arguments(ops):
    """K above the ceiling and trunc_mode = 3 are refused by both wide entry points before anything is launched."""
    sched = R.sched_table(O.schedule_buffers(T, 33), T).cuda()
    for K, mode, msg in ((MAX_K + 1, 1, "too large"), (2048, 3, "trunc_mode")):
        logits = torch.zeros(1, 3, K, device="cuda")
        lpo = torch.full((1, K + 1, 3), math.nan, device="cuda")
        with pytest.raises(RuntimeError, match=msg):
            ops.posterior_sample_wide(logits, None, None, None, None, T=T, trunc_mode=mode, log_prob_out=lpo,
                                      stage=ops.STAGE_SKIP_POSTERIOR | ops.STAGE_SKIP_SAMPLE)
        x = torch.full((1, 3), SENTINEL, dtype=torch.long, device="cuda")
        t = torch.full((1,), 50, device="cuda")
        ctrl = torch.tensor([1, 0, 4, 256, 0, 1, 0, 0], device="cuda")
        with pytest.raises(RuntimeError, match=msg):
            ops.posterior_sample_wide_loop(logits, x, t, t.clone(), sched, ctrl, t, t.clone(), T=T, trunc_mode=mode)
        torch.cuda.synchronize()
        assert bool(lpo.isnan().all()) and bool((x == SENTINEL).all()) and ctrl.tolist() == [1, 0, 4, 256, 0, 1, 0, 0]
