"""The posterior sampler kernel (csrc/sampler.cu) per column against the CPU restatement of its contract (tests/sampler_reference.py).

Every element is compared; nothing is summarised by a tensor maximum.  K covers every NJ template and both sides of each dispatch
boundary (C = K + 1 on and off a multiple of 32, up to K = 1055 with every lane full); L covers a tail CTA of 1 ... 8 warps; B has a
different t_post per row, t = 0 and t = T - 1 among them.  Each case runs the five stage combinations the library uses:
  predict_start (SKIP_POSTERIOR | SKIP_SAMPLE), truncate-then-sample (SKIP_POSTERIOR), q_posterior (INPUT_LOGPROB | SKIP_SAMPLE) on
  the kernel's own truncated log-probs, log_sample_categorical (INPUT_LOGPROB | SKIP_POSTERIOR) on its own posterior, and fused (0).
What must hold:
  * predict_start log-probs and keep-set: bit-identical to log_pred + keep (+-0 equal), except near-midpoint columns and ambiguous
    nucleus decisions, which are counted and printed (run with -s);
  * posterior: every element within POST_SCALE times the bound derived in sampler_reference.posterior;
  * ids: the argmax of the fp64 scores of the kernel's own log_prob_out, except a near-tie within the Gumbel rounding bound (counted);
  * the fused launch equals the staged launches bit for bit, and stages that skip sampling leave x_next untouched."""
import math

import pytest
import torch

from oracle import diffsound_oracle as O
from tests import sampler_reference as R

pytestmark = pytest.mark.gpu

T = 100
KS = [1, 31, 32, 63, 64, 159, 160, 255, 256, 287, 288, 543, 544, 1023, 1055]
SHAPES = [(3, 265), (16, 9), (1, 7), (3, 8), (1, 1), (16, 8), (1, 265), (3, 9)]
REGIMES = ["scale1", "scale12", "scale40", "scale1e3", "quantised"]
# (trunc_mode, r, k); k = -1 and 0 stand for C - 1 and C
TRUNCS = [(0, 0.0, 0)] + [(1, r, 0) for r in (0.85, 1e-6, 0.5, 1.0, 1.5)] + [(2, 0.0, k) for k in (1, 2, 20, 32, 33, -1, 0)]
# Posterior tolerance as a fraction of the bound derived in sampler_reference.posterior.  Measured on an H100 80GB HBM3 (700 W): the
# largest error / bound was 0.64 at K = 1 and at most 0.27 for every other K (largest absolute error 7.9e-6, bounds up to 6.3e-5).
# Four times the measurement is above the derivation, so the derivation itself is the tolerance.
POST_SCALE = 1.0
SENTINEL = -7


@pytest.fixture(scope="module")
def ops():
    from tests import gpu_common
    return gpu_common.ops


def make_inputs(K, B, L, regime, seed):
    """logits (B, K, L), x_t (B, L), t_post (B,), uniforms (B, K+1, L) for one case."""
    g = torch.Generator().manual_seed(seed)
    if regime == "quantised":  # small integers: equal log-probs, so nucleus and top-k boundaries fall inside tie groups
        logits = torch.randint(-3, 4, (B, K, L), generator=g).float()
    else:                      # at 1e3 most entries clamp to -70 and the top is 0
        logits = torch.randn(B, K, L, generator=g) * {"scale1": 1.0, "scale12": 12.0, "scale40": 40.0, "scale1e3": 1e3}[regime]
    if regime == "scale1e3" and K > 1:
        # column (0, 0): log-probs exactly 0 (index K - 1) and -40 (index 0), the rest -70.  With r = 1 the prefix sum before index 0 is
        # expf(0) = 1 exactly, so index 0 is dropped (1 < 1 is false), with no rounding to hide behind.
        logits[0, :, 0] = -1000.0
        logits[0, K - 1, 0] = 5.0
        logits[0, 0, 0] = -35.0
    u = torch.rand(B, K + 1, L, generator=g)
    u.view(-1)[torch.randint(0, u.numel(), (max(1, u.numel() // 500),), generator=g)] = 0.0  # ATen maps a uniform of 1 to 0
    ids = torch.randint(0, K, (B, L), generator=g)
    rows = []
    for b in range(B):  # all masked, none masked, mixed
        p = (b + seed) % 3
        rows.append(torch.rand(L, generator=g) < 0.5 if p == 2 else torch.full((L,), p == 0))
    x_t = torch.where(torch.stack(rows), torch.full_like(ids, K), ids)
    tp = torch.randint(0, T, (B,), generator=g)
    tp[0] = (0, T - 1)[seed % 2]
    if B > 1:
        tp[1] = (T - 1, 0)[seed % 2]
    return logits, x_t, tp, u


def reference_keep(logits, mode, r, k):
    """(log_pred, truncated log_pred, near-midpoint columns (B, 1, L), ambiguous elements, tie-at-boundary columns)."""
    lp, _, mid = R.log_pred(logits)
    B, C, L = lp.shape
    amb = torch.zeros_like(lp, dtype=torch.bool)
    tie = torch.zeros(B, L, dtype=torch.bool)
    lpt = lp
    if mode == 1:
        keep, amb, tie = R.keep_nucleus(lp, r)
        lpt = R.truncate(lp, keep)
    elif mode == 2:
        keep, tie = R.keep_topk(lp, k)
        lpt = R.truncate(lp, keep)
    return lp, lpt, mid.any(1, keepdim=True), amb, tie


def check_ids(x, values, u, what):
    """ids from the kernel against gumbel_ids of the values it sampled from; returns the near-tie count."""
    _, _, val, gb = R.gumbel_ids(values, u)
    wrong, near = R.id_check(x, val, gb)
    assert not wrong.any(), f"{what}: {int(wrong.sum())} ids differ beyond the Gumbel rounding bound, first at {wrong.nonzero()[0].tolist()}"
    return int(near.sum())


def run_case(ops, K, regime, it, seed, stats):
    mode, r, k = TRUNCS[it]
    C = K + 1
    if mode == 2:
        k = {-1: C - 1, 0: C}.get(k, k)
    B, L = SHAPES[(KS.index(K) + REGIMES.index(regime) + it) % len(SHAPES)]
    logits, x_t, tp, u = make_inputs(K, B, L, regime, seed)
    sched = R.sched_table(O.schedule_buffers(T, C), T)
    dev = lambda t: t.contiguous().cuda()
    blk, u_d, x_d, s_d = dev(logits.permute(0, 2, 1)), dev(u), dev(x_t), dev(sched)
    # every other case passes t_post (and a t the kernel must ignore), the others pass t alone
    with_tp = seed % 2 == 0
    t_d = dev(torch.randint(0, T, (B,)) if with_tp else tp)
    tp_d = dev(tp) if with_tp else None
    nan = lambda: torch.full((B, C, L), math.nan, device="cuda")
    sentinel = lambda: torch.full((B, L), SENTINEL, dtype=torch.long, device="cuda")
    IN, NOPOST, NOSAMP = ops.STAGE_INPUT_LOGPROB, ops.STAGE_SKIP_POSTERIOR, ops.STAGE_SKIP_SAMPLE
    tr = dict(trunc_mode=mode, trunc_r=r, trunc_k=k)
    lp_ps, x_ps = nan(), sentinel()
    ops.posterior_sample(blk, None, None, None, None, T=T, **tr, x_next=x_ps, log_prob_out=lp_ps, stage=NOPOST | NOSAMP)
    lp_ts, x_ts = nan(), sentinel()
    ops.posterior_sample(blk, None, None, u_d, None, T=T, **tr, x_next=x_ts, log_prob_out=lp_ts, stage=NOPOST)
    lp_qp, x_qp = nan(), sentinel()
    ops.posterior_sample(lp_ps, x_d, t_d, None, s_d, T=T, trunc_mode=0, t_post=tp_d, x_next=x_qp, log_prob_out=lp_qp, stage=IN | NOSAMP)
    lp_ls, x_ls = nan(), sentinel()
    ops.posterior_sample(lp_qp, None, None, u_d, None, T=T, trunc_mode=0, x_next=x_ls, log_prob_out=lp_ls, stage=IN | NOPOST)
    lp_f, x_f = nan(), sentinel()
    ops.posterior_sample(blk, x_d, t_d, u_d, s_d, T=T, **tr, t_post=tp_d, x_next=x_f, log_prob_out=lp_f, stage=0)
    lp_ps, lp_ts, lp_qp, lp_ls, lp_f = (t.cpu() for t in (lp_ps, lp_ts, lp_qp, lp_ls, lp_f))
    x_ps, x_ts, x_qp, x_ls, x_f = (t.cpu() for t in (x_ps, x_ts, x_qp, x_ls, x_f))
    what = f"K={K} B={B} L={L} {regime} trunc={(mode, r, k)}"

    # predict_start: log_pred + keep-set, bit for bit
    _, lpt, mid, amb, tie = reference_keep(logits, mode, r, k)
    differ = lp_ps != lpt
    bad = differ & ~mid & ~amb
    assert not bad.any(), f"{what}: predict_start differs at {bad.nonzero()[:4].tolist()}: {lp_ps[bad][:4].tolist()} vs {lpt[bad][:4].tolist()}"
    assert bool((x_ps == SENTINEL).all()) and bool((x_qp == SENTINEL).all()), f"{what}: a SKIP_SAMPLE launch wrote x_next"
    stats["midpoint_columns"] += int(mid.sum())
    tag = "_r1" if (mode, r) == (1, 1.0) else ""
    stats["ambiguous" + tag] += int(amb.sum())
    stats["ambiguous_differ" + tag] += int((differ & amb).sum())
    stats["tie_at_boundary"] += int(tie.sum())

    # truncate-then-sample: the same log-probs, ids from them
    assert torch.equal(lp_ts, lp_ps), what
    stats["near_tie"] += check_ids(x_ts, lp_ts, u, what + " truncate-then-sample")

    # q_posterior on the kernel's own truncated log-probs
    post, bound = R.posterior(lp_ps, x_t, tp, sched, T)
    err = (lp_qp.double() - post).abs()
    over = ~(err <= POST_SCALE * bound)
    assert not over.any(), f"{what}: posterior error {err[over][:4].tolist()} over bound {bound[over][:4].tolist()} at {over.nonzero()[:4].tolist()}"
    key = f"NJ={(C + 31) // 32}"
    stats["post_err"][key] = max(stats["post_err"].get(key, 0.0), float(err.max()))
    stats["post_ratio"][key] = max(stats["post_ratio"].get(key, 0.0), float((err / bound).max()))
    stats["post_bound"][key] = max(stats["post_bound"].get(key, 0.0), float(bound.max()))

    # log_sample_categorical passes the log-probs through and samples from them
    assert torch.equal(lp_ls, lp_qp), what
    stats["near_tie"] += check_ids(x_ls, lp_qp, u, what + " log_sample_categorical")

    # fused == predict_start -> q_posterior -> log_sample_categorical, bit for bit
    assert torch.equal(lp_f, lp_qp) and torch.equal(x_f, x_ls), f"{what}: fused launch differs from the staged launches"
    stats["cases"] += 1


@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("K", KS)
def test_sampler_stages_match_restatement(ops, K, regime):
    stats = dict(cases=0, midpoint_columns=0, ambiguous=0, ambiguous_differ=0, ambiguous_r1=0, ambiguous_differ_r1=0, tie_at_boundary=0,
                 near_tie=0, post_err={}, post_ratio={}, post_bound={})
    for it in range(len(TRUNCS)):
        run_case(ops, K, regime, it, seed=1000 * K + 10 * REGIMES.index(regime) + it, stats=stats)
    print(f"\nSAMPLER K={K} {regime}: {stats}")
    if regime == "quantised" and K >= 31:
        assert stats["tie_at_boundary"] > 0  # the boundary did fall inside tie groups


@pytest.mark.parametrize("K", [63, 256, 1055])
def test_gumbel_exact_ties_pick_the_lowest_index(ops, K):
    """Equal log-probs and equal uniforms at chosen indices: the same lane at different j, different lanes, the mask class K.  The kernel
    keeps the first maximum within a lane (strict >) and the lower index across lanes; the lowest index must win, with no allowance."""
    groups = [(5, 37), (3, 40, 101), (10, 33), (37, 69, 40), (7, K), (K - 1, K), (0, K), (40, 101, K)]
    groups = [gr for gr in groups if max(gr) <= K]
    B, L, C = 2, len(groups), K + 1
    g = torch.Generator().manual_seed(K)
    lp = -40.0 - 20.0 * torch.rand(B, C, L, generator=g)  # every other score stays below -23
    u = torch.rand(B, C, L, generator=g)
    for l, gr in enumerate(groups):
        for b in range(B):
            lp[b, list(gr), l] = -0.25 - b
            u[b, list(gr), l] = 0.625
    want = torch.tensor([min(gr) for gr in groups]).expand(B, L)
    _, _, val, _ = R.gumbel_ids(lp, u)
    assert torch.equal(val.argmax(1), want)
    x = torch.full((B, L), SENTINEL, dtype=torch.long, device="cuda")
    ops.posterior_sample(lp.cuda(), None, None, u.cuda(), None, T=T, trunc_mode=0, x_next=x,
                         stage=ops.STAGE_INPUT_LOGPROB | ops.STAGE_SKIP_POSTERIOR)
    assert torch.equal(x.cpu(), want), (x.cpu().tolist(), groups)


def test_sampler_refuses_bad_arguments(ops):
    """K = 1056 (C > 32 * 33) and trunc_mode = 3 are refused by the C-ABI before anything is launched."""
    sched = R.sched_table(O.schedule_buffers(T, 33), T).cuda()
    for K, mode, msg in ((1056, 1, "too large"), (32, 3, "trunc_mode")):
        logits = torch.zeros(1, 3, K, device="cuda")
        lpo = torch.full((1, K + 1, 3), math.nan, device="cuda")
        with pytest.raises(RuntimeError, match=msg):
            ops.posterior_sample(logits, None, None, None, None, T=T, trunc_mode=mode, log_prob_out=lpo,
                                 stage=ops.STAGE_SKIP_POSTERIOR | ops.STAGE_SKIP_SAMPLE)
        x = torch.full((1, 3), SENTINEL, dtype=torch.long, device="cuda")
        t = torch.full((1,), 50, device="cuda")
        ctrl = torch.tensor([1, 0, 4, 256, 0, 1, 0, 0], device="cuda")
        with pytest.raises(RuntimeError, match="bad shape" if K > 1055 else "trunc_mode"):
            ops.posterior_sample_loop(logits, x, t, t.clone(), sched, ctrl, t, t.clone(), T=T, trunc_mode=mode)
        torch.cuda.synchronize()
        assert bool(lpo.isnan().all()) and bool((x == SENTINEL).all()) and ctrl.tolist() == [1, 0, 4, 256, 0, 1, 0, 0]
