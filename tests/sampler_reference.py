"""CPU restatement of the contract of csrc/sampler.cu (the fused p_sample tail), one function per stage.

Plain torch, fp64 where the kernel computes in fp64.  Nothing here comes from the CUDA package or from the oracle's sampler functions.
The oracle follows the reference op by op, and the reference leaves the order of equal log-probs unspecified: torch.sort without
stable=True and torch.topk return tie members in no defined order.  The kernel defines one, and this module states it:
  * order: value descending, equal values by lower index (the kernel's key is the orderable value bits, then 0xFFFF - index);
  * nucleus keeps element k iff fl32(fp64 sum of expf(v_i) over the elements before k) < fl32(r); the first element is always kept;
  * top-k keeps the first k elements of that order;
  * Gumbel-argmax: of equal values the lowest index wins.
Layouts are the reference's: logits (B, K, L), log-probs (B, K+1, L), ids (B, L).
"""
import math

import torch

U32 = 2.0 ** -24                                                         # fp32 unit roundoff
U64 = 2.0 ** -53                                                         # fp64 unit roundoff
LOGZ = float(torch.tensor(-69.07755279, dtype=torch.float32))            # log(1e-30) as the fp32 value the kernel uses
EPS30 = float(torch.tensor(1e-30, dtype=torch.float32))                  # the 1e-30f of the Gumbel transform
SCHED_ROWS = ("log_at", "log_bt", "log_ct", "log_1_min_ct", "log_cumprod_at", "log_cumprod_bt", "log_cumprod_ct", "log_1_min_cumprod_ct")


def sched_table(sched, T):
    """The (8, T+1) fp32 schedule table dsb_posterior_sample reads, rows in SCHED_ROWS order, zero past each buffer's length."""
    s = torch.zeros(8, T + 1)
    for i, n in enumerate(SCHED_ROWS):
        s[i, : sched[n].numel()] = sched[n]
    return s


def warp_sum(x):
    """fp64 sum over the last dim (length NJ * 32, element k = lane + 32 j) in the kernel's order: each lane adds its elements in
    ascending j, then the xor butterfly (offsets 16 ... 1) adds lane pairs.  fp addition commutes, so both lanes of a pair hold the same
    sum and keeping the lower half at each level reproduces every lane's result bit for bit."""
    nj = x.shape[-1] // 32
    v = x.reshape(*x.shape[:-1], nj, 32)
    s = torch.zeros(v.shape[:-2] + (32,), dtype=torch.float64)
    for j in range(nj):
        s = s + v[..., j, :]
    for o in (16, 8, 4, 2, 1):
        s = s[..., :o] + s[..., o:2 * o]
    return s[..., 0]


def log_pred(logits):
    """predict_start tail: fp64 log_softmax over K, cast to fp32, clamped to [-70, 0]; the mask row K is -70.

    The sum of exp runs in the kernel's order (warp_sum).  A sequential fp64 sum is not enough: when one logit dominates, lse is tiny,
    and the top element's log-prob is -lse, so the fp64 rounding of a sum near 1 moves it by many fp32 ulps.  In the same order the
    kernel and this function compute the same d = x - max exactly and differ only in lse = log(sum exp d), through fp64 exp and log
    at 1 ulp each: by at most 2^-51 lse (exp(0) = 1 exactly, and the other terms' errors sum to at most 2^-52 (1 - 1/s) <= 2^-52 lse),
    then one more fp64 rounding of d - lse.  So the fp32 results can differ only for a value within about 2^-50 lse of an fp32 rounding
    midpoint.  Returns (lp fp32, the fp64 value before the cast, near-midpoint mask: d - lse * (1 -+ 2^-45) round to different fp32
    values; with lse = 0 the value is d itself on both sides and nothing is near).  Values below -70 clamp either way."""
    B, K, L = logits.shape
    x = logits.permute(0, 2, 1).float()
    d = x.double() - x.max(dim=-1, keepdim=True).values.double()
    nj = (K + 1 + 31) // 32
    e = torch.zeros(B, L, nj * 32, dtype=torch.float64)
    e[..., :K] = torch.exp(d)
    lse = torch.log(warp_sum(e)).unsqueeze(-1)
    v64 = d - lse
    f = v64.float()
    mid = ((d - lse * (1 + 2.0 ** -45)).float() != (d - lse * (1 - 2.0 ** -45)).float()) & (v64 > -70.001)
    pad = lambda t, val: torch.cat((t.permute(0, 2, 1), torch.full((B, 1, L), val, dtype=t.dtype)), dim=1)
    return pad(f.clamp(-70, 0), -70.0), pad(v64, -70.0), pad(mid, False)


def order(lp):
    """The kernel's total order along dim 1: value descending, equal values by lower index.  -0 and +0 are equal."""
    return torch.sort(lp + 0.0, dim=1, descending=True, stable=True)


def _unsort(sorted_mask, idx):
    return torch.zeros_like(sorted_mask).scatter_(1, idx, sorted_mask)


def _tie_at_boundary(sv, n_keep):
    """Columns whose kept prefix ends inside a group of equal values: there the reference's choice of members is unspecified."""
    C = sv.shape[1]
    last = sv.gather(1, (n_keep - 1).clamp(0, C - 1).unsqueeze(1)).squeeze(1)
    nxt = sv.gather(1, n_keep.clamp(max=C - 1).unsqueeze(1)).squeeze(1)
    return (n_keep < C) & (last == nxt)


def keep_nucleus(lp, r):
    """'top{r}r' keep-set.  Returns (keep, ambiguous, tie_at_boundary (B, L)).

    The terms here are exp(v) rounded once to fp32, summed in fp64 in sequence.  The kernel adds (double)expf(v) in tree order, and
    CUDA's expf is within 2 ulp of exp, so within 2.5 ulp (5 * 2^-24 relative) of these terms; expf(0) is exactly 1.  Its sum
    therefore lies within delta = 5 * 2^-24 * (sum of the terms with v != 0) + (NJ + 5 + n) * 2^-53 * T of this one (NJ + 5
    roundings along the kernel's tree, n along this cumsum).  An element is ambiguous when the decision fl32(T) < fl32(r) differs
    between T - delta and T + delta.  With r near 1 the boundary moves into the tail, where the decision rests on the last bits of
    the sum of all terms: there many elements are ambiguous."""
    B, C, L = lp.shape
    sv, idx = order(lp)
    e = torch.exp(sv.double()).float().double()
    T = torch.cumsum(e, dim=1) - e
    T_nz = torch.cumsum(e * (sv != 0), dim=1) - e * (sv != 0)
    n = torch.arange(C, dtype=torch.float64).view(1, C, 1)
    delta = 5 * U32 * T_nz + ((C + 31) // 32 + 5 + n) * U64 * T
    fr = float(torch.tensor(r, dtype=torch.float32))
    keep_s = T.float() < fr
    keep_s[:, 0] = True
    amb_s = ((T - delta).float() < fr) != ((T + delta).float() < fr)
    amb_s[:, 0] = False
    return _unsort(keep_s, idx), _unsort(amb_s, idx), _tie_at_boundary(sv, keep_s.sum(1))


def keep_topk(lp, k):
    """'top{k}p' keep-set: the first k elements of the order.  Returns (keep, tie_at_boundary (B, L))."""
    B, C, L = lp.shape
    sv, idx = order(lp)
    keep_s = (torch.arange(C).view(1, C, 1) < k).expand(B, C, L).clone()
    return _unsort(keep_s, idx), _tie_at_boundary(sv, torch.full((B, L), min(k, C), dtype=torch.long))


def truncate(lp, keep):
    return torch.where(keep, lp, torch.full_like(lp, -70.0))


def _lae(a, b, ea, eb):
    """log_add_exp (diffusion_transformer.py:28-30) in fp64, and the error bound of the kernel's fp32 lae on inputs carrying errors
    ea, eb.  The kernel computes m = max(a, b), d = a - m (the other difference is 0), expf(d), expf(0) = 1, s = sum, logf(s), m + log.
    Input errors pass with weight <= 1 (the weights are the softmax of (a, b)).  Rounding d: u|d| e^d <= u/e; expf at 2 ulp = 4u of a
    term that is at most half of s: 2u; the sum: u; logf at 1 ulp of log(s) in [0, ln 2]: u; the last add: u|result|."""
    m = torch.maximum(a, b)
    res = m + torch.log(torch.exp(a - m) + torch.exp(b - m))
    return res, torch.maximum(ea, eb) + 5 * U32 + U32 * res.abs()


def posterior(lp, x_t, t_post, sched, T):
    """q_posterior closed form (diffusion_transformer.py:293-339) in fp64 from the fp32 log-probs lp (B, K+1, L) and the fp32 table
    sched (8, T+1); t - 1 wraps to T at t = 0 (q_pred's (t + T + 1) % (T + 1)).  Returns (clamped output, per-element error bound of
    the kernel's fp32 evaluation).

    Bound, first order in u = 2^-24, from the kernel's steps (CUDA expf <= 2 ulp, logf <= 1 ulp):
      lqt = lae(oh + cA, cB), l1 = lae(oh + la, lb): the add u|oh + .| when oh = log(1e-30), then _lae.  Masked and mask-class
          entries are table values, exact.
      qv = lp - lqt:                        E_qv  = E_lqt + u|qv|
      slse = logf(sum expf(qv - qmax)) + qmax (logsumexp is 1-Lipschitz):
                                            E_lse = max E_qv + u sum p|qv - qmax| + 4u (expf) + (NJ + 5)u (sum: NJ per lane, 5 levels)
                                                    + 2u|log ssum| (logf) + u|slse|
      qn = qv - slse:                       E_qn  = E_qv + E_lse + u|qn|
      r = lae(qn + pA, pB) (k < K), lae(qn + pC1, pC) (k = K): the add u|qn + p|, then _lae
      out = (r + l1) + slse, clamped:       E_out = E_r + E_l1 + E_lse + u|r + l1| + u|out|"""
    B, C, L = lp.shape
    K = C - 1
    u = U32
    s = sched.double()
    tp = t_post.long()
    tm1 = (tp - 1 + (T + 1)) % (T + 1)
    row = lambda i, t: s[i, t].view(B, 1, 1)
    la, lb, lc, cA, cB, cC = row(0, tp), row(1, tp), row(2, tp), row(4, tp), row(5, tp), row(6, tp)
    pA, pB, pC, pC1 = row(4, tm1), row(5, tm1), row(6, tm1), row(7, tm1)
    k = torch.arange(C).view(1, C, 1)
    xt = x_t.view(B, 1, L)
    masked = xt == K
    is_cls = k < K
    oh = torch.where(k == xt, 0.0, LOGZ).double()
    zero = torch.zeros(B, C, L, dtype=torch.float64)
    a1 = oh + cA
    lqt_n, e_lqt_n = _lae(a1, cB.expand_as(a1), u * a1.abs() * (oh != 0), zero)
    a2 = oh + la
    l1_n, e_l1_n = _lae(a2, lb.expand_as(a2), u * a2.abs() * (oh != 0), zero)
    mask_val = torch.where(masked, 0.0, LOGZ).double().expand(B, C, L)
    lqt = torch.where(is_cls, torch.where(masked, cC.expand(B, C, L), lqt_n), mask_val)
    l1 = torch.where(is_cls, torch.where(masked, lc.expand(B, C, L), l1_n), mask_val)
    e_lqt = torch.where(is_cls & ~masked, e_lqt_n, zero)
    e_l1 = torch.where(is_cls & ~masked, e_l1_n, zero)

    qv = lp.double() - lqt
    e_qv = e_lqt + u * qv.abs()
    qmax = qv.max(dim=1, keepdim=True).values
    d = qv - qmax
    ssum = torch.exp(d).sum(dim=1, keepdim=True)
    p = torch.exp(d) / ssum
    slse = torch.log(ssum) + qmax
    nj = (C + 31) // 32
    e_lse = (e_qv.max(dim=1, keepdim=True).values + u * (p * d.abs()).sum(dim=1, keepdim=True) + (4 + nj + 5) * u
             + 2 * u * torch.log(ssum).abs() + u * slse.abs())
    qn = qv - slse
    e_qn = e_qv + e_lse + u * qn.abs()
    a3 = qn + torch.where(is_cls, pA, pC1)
    r, e_r = _lae(a3, torch.where(is_cls, pB, pC).expand_as(a3), e_qn + u * a3.abs(), zero)
    s1 = r + l1
    out = s1 + slse
    bound = e_r + e_l1 + e_lse + u * s1.abs() + u * out.abs()
    return out.clamp(-70, 0), bound


def gumbel_ids(values, u):
    """log_sample_categorical with the uniforms given: argmax over dim 1 of -log(-log(u + 1e-30) + 1e-30) + values in fp64, first index
    on a tie.  Returns (ids, top-two margin, the fp64 scores, per-element error bound of the kernel's fp32 score).

    Kernel: y = -logf(u + 1e-30f) (the add is exact for every u the generator makes; logf 1 ulp = relative 2u of y), then
    g = -logf(y + 1e-30f): 2u from y, 1 ulp of |g| = 2u|g|; score g + v: u|score|.  Bound u (2 + 2|g| + |score|)."""
    g = -torch.log(-torch.log(u.double() + EPS30) + EPS30)
    val = g + values.double()
    ids = val.argmax(dim=1)
    top2 = val.topk(2, dim=1).values if val.shape[1] > 1 else torch.cat((val, val - math.inf), dim=1)
    return ids, top2[:, 0] - top2[:, 1], val, U32 * (2 + 2 * g.abs() + val.abs())


def id_check(ids, val, bound, extra=None, ref=None):
    """Compare sampled ids (B, L) with ref (default: the argmax of the fp64 scores val (B, C, L)), where each implementation's score
    is within bound (+ extra, an error on the values themselves) of val.  Returns (wrong, near_tie): near_tie marks a different id
    whose score lies within the two bounds of ref's, which rounding can reach; wrong marks any other difference, or an id outside
    [0, C)."""
    e = bound if extra is None else bound + extra
    ref = val.argmax(dim=1) if ref is None else ref
    valid = (ids >= 0) & (ids < val.shape[1])
    idc = torch.where(valid, ids, ref)
    diff = ids != ref
    g = lambda t, i: t.gather(1, i.unsqueeze(1)).squeeze(1)
    reach = valid & ((g(val, idc) - g(val, ref)).abs() <= g(e, idc) + g(e, ref))
    return diff & ~reach, diff & reach


def sample_step(logits, x_t, t, u, sched, T, trunc):
    """The whole p_sample tail on logits (B, K, L) with truncation given as the reference writes it ('top0.85r', 'top20p' or None).
    Returns (lp after truncation, posterior, its bound, Gumbel scores, their bound, columns with an ambiguous nucleus decision or a
    log-prob near a midpoint, columns whose truncation boundary falls inside a group of equal values)."""
    B, K, L = logits.shape
    lp, _, mid = log_pred(logits)
    amb = torch.zeros_like(lp, dtype=torch.bool)
    tie = torch.zeros(B, L, dtype=torch.bool)
    if trunc is not None and trunc.endswith("r"):
        keep, amb, tie = keep_nucleus(lp, float(trunc[3:-1]))
        lp = truncate(lp, keep)
    elif trunc is not None:
        keep, tie = keep_topk(lp, int(trunc[3:-1]))
        lp = truncate(lp, keep)
    post, bound = posterior(lp, x_t, t, sched, T)
    _, _, val, gb = gumbel_ids(post, u)
    return lp, post, bound, val, gb, mid.any(1) | amb.any(1), tie
