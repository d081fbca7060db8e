"""The denoiser's training kernels (csrc/train.cu, csrc/attention_train.cu), each against a plain torch restatement of the same operation on
the same rounded inputs, evaluated in fp64.

Data-movement kernels (transpose, heads split / merge, cast_scale, gather_rows) must match bit for bit.  Arithmetic kernels get a per-element
bound derived from their own arithmetic, stated beside each check.  Units used throughout:
  u = 2^-24   fp32 unit roundoff;  gamma(n) = n u / (1 - n u) bounds an fp32 sum of depth n, relative to the sum of |terms|;
  half an ulp of the output type for the final store: tf32 keeps 11 significant bits (cvt.rna: at most 2^-11 relative), bf16 keeps 8 (RNE: at
  most 2^-8 relative).  The per-element checks use the half ulp of the stored value itself, which is never larger than those relative figures;
  the attention and ladder bounds, which need the rounding of values that are not stored, use the relative figures.
Where a bound keeps only first-order terms, the neglected products of two first-order terms are covered by the stated (1 + 2^-6) factor: every
first-order relative term is below 2^-6.
Buffers around the operands are NaN, and outputs outside the written region are sentinels that must come back unchanged."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
SECOND_ORDER = 1 + 2.0 ** -6


@pytest.fixture(scope="module")
def G():
    from tests import gpu_common
    return gpu_common


@pytest.fixture(scope="module")
def TO():
    from tests import gpu_common  # noqa: F401  (loads the package)
    from diffsound_b200 import train_ops
    return train_ops


ACT = [torch.float32, torch.bfloat16]
DT_ID = {torch.float32: "tf32", torch.bfloat16: "bf16"}


def gamma(n):
    return n * U / (1 - n * U)


def _bits(t):
    """Integer view on the CPU: equal bits, not merely equal values (-0.0 != +0.0, NaN payloads compare)."""
    t = t.contiguous().cpu()
    return t.view({torch.float32: torch.int32, torch.bfloat16: torch.int16, torch.float16: torch.int16, torch.float64: torch.int64}[t.dtype])


def _assert_bitwise(got, ref, what=""):
    assert got.shape == ref.shape and got.dtype == ref.dtype, (what, got.shape, ref.shape, got.dtype, ref.dtype)
    bad = _bits(got) != _bits(ref)
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} of {ref.numel()} elements differ, first at {bad.nonzero()[0].tolist()}"


def _store_ref(G, x32, dt):
    """The kernels' store of an fp32 value: cvt.rna to tf32, or RNE to bf16."""
    return G.tf32_round_ref(x32) if dt == torch.float32 else x32.bfloat16()


def _half_ulp(out, dt):
    """Half an ulp of each stored value (fp64, CPU), from its exponent: tf32 2^(E-138), bf16 2^(E-135); zero and subnormals take E = 1."""
    e = (_bits(out.float()) >> 23) & 0xFF
    return torch.pow(2.0, (e.clamp(min=1) - (138 if dt == torch.float32 else 135)).double())


def _assert_within(got, ref, bound, what=""):
    """Per element |got - ref| <= bound (fp64, CPU); got must be finite."""
    got, ref, bound = got.double().cpu(), ref.double().cpu(), bound.double().cpu()
    assert bool(torch.isfinite(got).all()), f"{what}: non-finite output"
    err = (got - ref).abs()
    bad = err > bound
    if bool(bad.any()):
        j = int((err - bound).flatten().argmax())
        raise AssertionError(f"{what}: {int(bad.sum())} of {ref.numel()} elements outside the bound; worst: got {got.flatten()[j].item()!r} "
                             f"ref {ref.flatten()[j].item()!r} err {err.flatten()[j].item():.3e} bound {bound.flatten()[j].item():.3e}")


def _nan_like(shape, dtype):
    return torch.full(shape, float("nan"), dtype=dtype, device="cuda")


# ================================================================================================ fused attention (bf16)
LS = [1, 63, 64, 65, 77, 129, 265]
ATTN_CASES = ([(2, 2, lq, lk, "uniform") for lq in LS for lk in LS]
              + [(2, 2, lq, lk, "random") for lq in LS for lk in LS]
              + [(2, 2, lq, lk, r) for r in ("saturated", "lastmax", "equal") for lq, lk in ((77, 77), (265, 265), (265, 77), (65, 129), (1, 265), (129, 1))]
              + [(2, 16, 265, 265, "random"), (2, 16, 265, 77, "uniform"), (3, 16, 77, 265, "lastmax")])


def _attn_inputs(B, H, Lq, Lk, regime, seed):
    """q, k, v, dO (fp32 values that are exactly bf16) in token-major (B*L, H*64) layout.
    uniform:   q * 0.05 -> scaled scores of about +-0.1: a key let in or dropped by the tail mask changes every O row by about 1/Lk;
    saturated: scaled scores spanning about +-40 (most rows are one-hot);
    lastmax:   every query shares a direction with the last key: each row's maximum sits in the last key chunk, after the others (online rescale);
    equal:     q = 0, every score is exactly 0."""
    g = torch.Generator().manual_seed(seed)
    D = H * 64
    q = torch.randn(B * Lq, D, generator=g)
    k = torch.randn(B * Lk, D, generator=g)
    if regime == "uniform":
        q = q * 0.05
    elif regime == "saturated":
        q, k = q * 3.0, k * 3.0
    elif regime == "lastmax":
        d = torch.where(torch.rand(B, 1, D, generator=g) < 0.5, -0.5, 0.5)
        q = (q.view(B, Lq, D) + 2 * d).view(B * Lq, D)
        k.view(B, Lk, D)[:, -1:] = 3 * d
    elif regime == "equal":
        q = torch.zeros_like(q)
    v = torch.randn(B * Lk, D, generator=g)
    do = torch.randn(B * Lq, D, generator=g)
    return [x.bfloat16().float() for x in (q, k, v, do)]


def _placed(x, rows_pad, ld, col):
    """x (M, D) placed at column `col` of an (M + rows_pad, ld) bf16 buffer that is NaN everywhere else; returns (buffer, view)."""
    M, D = x.shape
    buf = _nan_like((M + rows_pad, ld), torch.bfloat16)
    buf[:M, col:col + D] = x.bfloat16().cuda()
    return buf, buf[:M, col:col + D]


def _heads(x, B, L, H):
    return x.double().reshape(B, L, H, 64).permute(0, 2, 1, 3)


def _unheads(x):
    B, H, L, _ = x.shape
    return x.permute(0, 2, 1, 3).reshape(B * L, H * 64)


def _untouched(buf, before, rows, c0, c1, what):
    """Everything of buf outside rows [0, rows) x columns [c0, c1) still equals `before` bit for bit."""
    mask = torch.ones(buf.shape, dtype=torch.bool)
    mask[:rows, c0:c1] = False
    assert bool((_bits(buf)[mask] == _bits(before)[mask]).all()), f"{what}: written outside its rows / head columns"


@pytest.mark.parametrize("B,H,Lq,Lk,regime", ATTN_CASES)
def test_attention_train_matches_fp64(TO, B, H, Lq, Lk, regime):
    scale = 0.125
    D = H * 64
    q, k, v, do = _attn_inputs(B, H, Lq, Lk, regime, seed=1000 * H + 10 * Lq + Lk)
    PAD = 64
    qbuf, qv = _placed(q, PAD, 3 * D + 16, 8)                  # q inside a wider QKV-like buffer at a column offset
    kvbuf, kv_k = _placed(k, PAD, 2 * D + 16, 8)
    kvbuf[:B * Lk, 8 + D:8 + 2 * D] = v.bfloat16().cuda()
    kv_v = kvbuf[:B * Lk, 8 + D:8 + 2 * D]
    dobuf, dov = _placed(do, PAD, D + 24, 16)
    obuf = _nan_like((B * Lq + PAD, D + 16), torch.bfloat16)
    lse_buf = _nan_like((B * H * Lq + PAD,), torch.float32)
    o_before, lse_before = obuf.cpu(), lse_buf.cpu()
    ov = obuf[:B * Lq, 8:8 + D]
    lse = lse_buf[:B * H * Lq].view(B * H, Lq)
    TO.attention_train_fwd(qv, kv_k, kv_v, ov, lse, B, H, Lq, Lk, scale)
    dqbuf = _nan_like((B * Lq + PAD, D + 16), torch.bfloat16)
    dkvbuf = _nan_like((B * Lk + PAD, 2 * D + 16), torch.bfloat16)
    delta_buf = _nan_like((B * H * Lq + PAD,), torch.float32)
    dq_before, dkv_before, delta_before = dqbuf.cpu(), dkvbuf.cpu(), delta_buf.cpu()
    delta = delta_buf[:B * H * Lq].view(B * H, Lq)
    TO.attention_train_bwd(qv, kv_k, kv_v, ov, dov, lse, delta, dqbuf[:B * Lq, 8:8 + D], dkvbuf[:B * Lk, 8:8 + D], dkvbuf[:B * Lk, 8 + D:8 + 2 * D],
                           B, H, Lq, Lk, scale)
    torch.cuda.synchronize()
    _untouched(obuf.cpu(), o_before, B * Lq, 8, 8 + D, "O")
    _untouched(dqbuf.cpu(), dq_before, B * Lq, 8, 8 + D, "dQ")
    _untouched(dkvbuf.cpu(), dkv_before, B * Lk, 8, 8 + 2 * D, "dK / dV")
    assert torch.equal(_bits(lse_buf.cpu()[B * H * Lq:]), _bits(lse_before[B * H * Lq:])), "LSE written past B*H*Lq"
    assert torch.equal(_bits(delta_buf.cpu()[B * H * Lq:]), _bits(delta_before[B * H * Lq:])), "Delta written past B*H*Lq"

    Q, K, V, dO = _heads(q, B, Lq, H), _heads(k, B, Lk, H), _heads(v, B, Lk, H), _heads(do, B, Lq, H)
    Sraw = Q @ K.transpose(-1, -2)                              # unscaled scores, exact in fp64 (products of bf16 values)
    S = scale * Sraw
    P = torch.softmax(S, -1)
    O64 = P @ V
    Ok = _heads(ov.float().cpu(), B, Lq, H)                      # the kernel's stored O (bf16)
    # score error, per row, in natural-log units: the fp32 tensor-core dot over 64 products loses at most 64 * 2^-23 of sum |q k| (truncating
    # adds assumed); scale * log2(e) is an fp32 constant (u), the fma with the row maximum rounds once (u of |s - m|) and ms = m * sl2 once (u |m|).
    A = (Q.abs() @ K.abs().transpose(-1, -2)).amax(-1, keepdim=True)
    Smax = Sraw.abs().amax(-1, keepdim=True)
    eps_s = scale * (64 * 2.0 ** -23 * A + 5 * U * Smax)
    # fp32 arithmetic besides the scores: P V accumulates Lk terms in fp32 (2^-23 per add, truncation assumed), l sums Lk terms and is rescaled once
    # per 64-key chunk, ex2.approx is within 2^-22 relative: 2^-23 (2 Lk + 8) in all.
    eps_f_k = 2.0 ** -23 * (2 * Lk + 8)
    eps_f_q = 2.0 ** -23 * (2 * Lq + 8)
    B8 = 2.0 ** -8                                             # one bf16 rounding (8 significant bits)

    # O: P is rounded to bf16 before P V (B8 of each P_k |V_k|), O is rounded on store (B8 |O|); a score error eps_s moves P_k by
    # P_k (eps_s + sum_j P_j eps_s), i.e. O by eps_s (P|V| + |O|); the fp32 terms scale the same way.
    PV = P @ V.abs()
    bound_o = SECOND_ORDER * ((B8 + eps_s + eps_f_k) * PV + (B8 + eps_s + eps_f_k) * O64.abs())
    _assert_within(_unheads(Ok), _unheads(O64), _unheads(bound_o), f"O {regime}")

    # LSE = m sl2 + log2(l), base 2: the score error (eps_s / ln 2) and l's fp32 relative error (eps_f / ln 2), log2f within 2^-22 of its
    # result (|log2 l| <= log2(Lk) + 1), one add (u |LSE|).
    lse64 = torch.logsumexp(S, -1) / math.log(2)
    bound_lse = SECOND_ORDER * ((eps_s.squeeze(-1) + eps_f_k) / math.log(2) + 2.0 ** -22 * (math.log2(Lk) + 1) + U * lse64.abs())
    _assert_within(lse.cpu().view(B, H, Lq), lse64, bound_lse, f"LSE {regime}")

    # Delta = sum_d dO O with the kernel's bf16 O: the 64 products are exact in fp32; each thread sums 16 of them, two shuffles add the rest.
    delta64 = (dO * Ok).sum(-1)
    bound_delta = gamma(18) * (dO * Ok).abs().sum(-1)
    _assert_within(delta.cpu().view(B, H, Lq), delta64, bound_delta, f"Delta {regime}")

    # backward reference: the formulas of the kernels in fp64 with the kernel's O in Delta (so that Delta is the one dS uses)
    dP = dO @ V.transpose(-1, -2)
    dS = scale * P * (dP - delta64.unsqueeze(-1))
    dQ64, dK64, dV64 = dS @ K, dS.transpose(-1, -2) @ Q, P.transpose(-1, -2) @ dO
    # P rebuilt as 2^(s sl2 - LSE): the score error, the stored LSE's error (its bound, in natural units) and ex2 (2^-22)
    eps_p = eps_s + bound_lse.unsqueeze(-1) * math.log(2) + 2.0 ** -22
    # dS = scale P (dP - Delta), rounded to bf16 for the dQ / dK products: P's error, B8 for the rounding, 3 fp32 roundings (u each);
    # dP is an fp32 tensor-core dot over 64 products (64 * 2^-23 of sum |dO V|), Delta carries its own summation bound.
    e_ds = (B8 + eps_p + 3 * U) * dS.abs() + scale * P * (64 * 2.0 ** -23 * (dO.abs() @ V.abs().transpose(-1, -2)) + bound_delta.unsqueeze(-1))
    bound_dq = SECOND_ORDER * (e_ds @ K.abs() + eps_f_k * (dS.abs() @ K.abs()) + B8 * dQ64.abs())
    bound_dk = SECOND_ORDER * (e_ds.transpose(-1, -2) @ Q.abs() + eps_f_q * (dS.abs().transpose(-1, -2) @ Q.abs()) + B8 * dK64.abs())
    # dV = P^T dO: P rounded to bf16 (B8) with its own error eps_p, fp32 accumulation over Lq, the store (B8 |dV|)
    bound_dv = SECOND_ORDER * (((B8 + eps_p) * P).transpose(-1, -2) @ dO.abs() + eps_f_q * (P.transpose(-1, -2) @ dO.abs()) + B8 * dV64.abs())
    dq_k = dqbuf[:B * Lq, 8:8 + D].float().cpu()
    dk_k = dkvbuf[:B * Lk, 8:8 + D].float().cpu()
    dv_k = dkvbuf[:B * Lk, 8 + D:8 + 2 * D].float().cpu()
    _assert_within(dq_k, _unheads(dQ64), _unheads(bound_dq), f"dQ {regime}")
    _assert_within(dk_k, _unheads(dK64), _unheads(bound_dk), f"dK {regime}")
    _assert_within(dv_k, _unheads(dV64), _unheads(bound_dv), f"dV {regime}")


# ================================================================================================ softmax rows (tf32 accuracy mode)
def _softmax_rows(n, ld, seed):
    """rows: N(0, 3) scores, rows offset by +1e3 and -1e3, one row with a single dominant entry; NaN beyond n."""
    g = torch.Generator().manual_seed(seed)
    rows = 48
    S = torch.randn(rows, n, generator=g) * 3
    S[8:16] += 1e3
    S[16:24] -= 1e3
    S[24] = -5.0
    S[24, n // 2] = 30.0
    Sb = torch.full((rows, ld), float("nan"))
    Sb[:, :n] = S
    return Sb


@pytest.mark.parametrize("dt", ACT, ids=DT_ID.get)
@pytest.mark.parametrize("n", [1, 31, 32, 33, 77, 265, 300])
def test_softmax_rows_match_fp64(G, TO, dt, n):
    ld = n + 8 - n % 8 + 8                                     # ld > n
    Sb = _softmax_rows(n, ld, seed=n)
    S = Sb.cuda()
    P = torch.full((Sb.shape[0], ld), -3.0, device="cuda").to(dt)   # sentinel beyond n
    TO.softmax_fwd(S, P, n)
    Pk = P.cpu()
    assert bool((Pk[:, n:].float() == -3.0).all()), "P written beyond n"
    Sd = Sb[:, :n].double()
    P64 = torch.softmax(Sd, -1)
    y = (Sd - Sd.amax(-1, keepdim=True)).abs()                 # |s - max|
    # per element, relative to P: s - max rounds once (u |y|), __expf(-y) is within (2 + 1.173 |y|) ulp (CUDA Programming Guide, ulp <= 2^-23
    # relative); the sum carries the P-weighted average of those errors plus its fp32 summation (ceil(n/32) per lane + 5 shuffles), then 1/sum
    # and the product round once each.  The store adds half an ulp of the stored value.
    e_k = U * y + 2.0 ** -23 * (2 + 1.173 * y)
    depth = -(-n // 32) + 5
    e_sum = gamma(depth) + (P64 * e_k).sum(-1, keepdim=True)
    bound = SECOND_ORDER * (e_k + e_sum + 2 * U) * P64 + _half_ulp(Pk[:, :n], dt)
    _assert_within(Pk[:, :n].float(), P64, bound, f"softmax_fwd n={n}")

    # backward: dS = alpha P (dP - sum_j P_j dP_j) on the kernel's stored P
    g = torch.Generator().manual_seed(n + 1)
    dPb = torch.full((Sb.shape[0], ld + 8), float("nan"))
    dPb[:, :n] = torch.randn(Sb.shape[0], n, generator=g)
    dS = torch.full((Sb.shape[0], ld), -3.0, device="cuda").to(dt)
    alpha = 0.125
    TO.softmax_bwd(P, dPb.cuda(), dS, n, alpha)
    dSk = dS.cpu()
    assert bool((dSk[:, n:].float() == -3.0).all()), "dS written beyond n"
    Pd, dPd = Pk[:, :n].double(), dPb[:, :n].double()
    dot = (Pd * dPd).sum(-1, keepdim=True)
    ref = alpha * Pd * (dPd - dot)
    # the dot: n products (u each) summed at depth ceil(n/32) + 5; the difference rounds once, alpha = 2^-3 is exact, the two products round
    # once each; the store adds half an ulp.
    e_dot = gamma(depth + 1) * (Pd * dPd).abs().sum(-1, keepdim=True)
    bound = SECOND_ORDER * (alpha * Pd.abs() * (e_dot + U * (dPd - dot).abs()) + 2 * U * ref.abs()) + _half_ulp(dSk[:, :n], dt)
    _assert_within(dSk[:, :n].float(), ref, bound, f"softmax_bwd n={n}")


# ================================================================================================ GELU2 and SiLU backward
def _ramp(n, seed):
    """n values over [-60, 60]: an even grid (exact zeros included) plus random points."""
    g = torch.Generator().manual_seed(seed)
    x = torch.cat([torch.linspace(-60, 60, 241), torch.zeros(7), (torch.rand(max(n - 248, 0), generator=g) * 120 - 60)])
    return x[torch.randperm(x.numel(), generator=g)[:n]]


def _sig_bound(s, v, eps_s, eps_v, dy):
    """Error of fp32 dy * (s + v s (1 - s)) given s with relative error eps_s and v with relative error eps_v: d/ds of the bracket is at most
    1 + |v|; v s and (1 - s) and the product round once each, the add and the multiply by dy once each."""
    gfun = s + v * s * (1 - s)
    return (dy.abs() * (eps_s * s * (1 + v.abs()) + v.abs() * s * (1 - s).abs() * (eps_v + 3 * U) + U * gfun.abs()) + U * (dy * gfun).abs(), gfun)


@pytest.mark.parametrize("dt", ACT, ids=DT_ID.get)
# The launch is capped at 16 CTAs/SM (2112 CTAs on 132 SMs) of 256 threads, each taking 8 values per pass: one pass covers 4,325,376 values.
# 2.4M runs one pass on 1172 CTAs; 5M runs the grid-stride loop twice (more often on fewer SMs).
@pytest.mark.parametrize("n", [8, 2_400_000, 5_000_000])
def test_gelu2_matches_fp64(G, TO, dt, n):
    x = _ramp(n, seed=n).to(dt)
    u = x.cuda()
    a = torch.full_like(u, 7.0)
    TO.gelu2_fwd(u, a)
    xd = x.double()
    av = 1.702 * xd
    sig = torch.sigmoid(av)
    ref = xd * sig
    # y = x / (1 + __expf(-1.702f x)): the argument carries 2u relative (the fp32 constant and the product); __expf is within (2 + 1.173 |a|)
    # ulp; the add and the divide round once each: 2^-23 (3 + 2.2 |a|) relative in all.  Where exp(|a|) leaves fp32's range (|a| > 88.7) the
    # kernel's 1 + exp overflows and the result is 0: the true value is below |x| 2^-126 there, which the last term covers.
    bound = SECOND_ORDER * 2.0 ** -23 * (3 + 2.2 * av.abs()) * ref.abs() + xd.abs() * 2.0 ** -126 + _half_ulp(a.cpu(), dt)
    _assert_within(a.cpu(), ref, bound, f"gelu2_fwd {DT_ID[dt]}")
    g = torch.Generator().manual_seed(n + 3)
    dav = torch.randn(n, generator=g).to(dt)
    du = torch.full_like(u, 7.0)
    TO.gelu2_bwd(u, dav.cuda(), du)
    # du = da * (sg + 1.702 x sg (1 - sg)), sg = 1 / (1 + __expf(-1.702f x)) carries 2^-23 (2 + 2.2 |a|) + 2u relative; v = 1.702f x carries 2u
    e_s = 2.0 ** -23 * (2 + 2.2 * av.abs()) + 2 * U
    b, dref = _sig_bound(sig, av, e_s, 2 * U, dav.double())
    bound = SECOND_ORDER * b + dav.double().abs() * (1 + av.abs()) * 2.0 ** -126 + _half_ulp(du.cpu(), dt)
    _assert_within(du.cpu(), dav.double() * dref, bound, f"gelu2_bwd {DT_ID[dt]}")


@pytest.mark.parametrize("n", [8, 1000, 600_000])   # 600k: more than 16 x 132 x 256 elements, the grid-stride loop runs twice
def test_silu_bwd_matches_fp64(TO, n):
    x = _ramp(n, seed=n + 5)
    g = torch.Generator().manual_seed(n)
    dy = torch.randn(n, generator=g)
    dx = torch.full((n,), 7.0, device="cuda")
    TO.silu_bwd(x.cuda(), dy.cuda(), dx)
    xd = x.double()
    s = torch.sigmoid(xd)
    # s = 1 / (1 + expf(-x)): expf within 2 ulp (4u), the add and the divide u each -> 6u; fp32 output (no storage rounding)
    b, dref = _sig_bound(s, xd, 6 * U, 0.0, dy.double())
    _assert_within(dx.cpu(), dy.double() * dref, SECOND_ORDER * b, "silu_bwd")


# ================================================================================================ LayerNorm / AdaLayerNorm backward
def _ln_x(B, L, D, seed):
    """N(0, 1) rows, with rows of variance 1e-4 (where eps = 1e-5 matters) and rows carrying a DC offset of 20 sigma."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, L, D, generator=g)
    x[:, 0::3] *= 1e-2
    x[:, 1::3] += 20.0
    x[:, 2::5] = x[:, 2::5] * 1e-2 + 0.2
    return x


def _ln_bwd_bounds(x, dy, g, eps, NV):
    """fp64 reference and per-element error bounds of the kernel's LayerNorm backward (first order; u = 2^-24).
    Row sums in the kernel run at depth n_D = NV + 7 (each lane adds NV groups of four as (a + b) + (c + d), five shuffles follow)."""
    D = x.shape[-1]
    nD = NV + 7
    mean = x.mean(-1, keepdim=True)
    xc = x - mean
    var = (xc * xc).mean(-1, keepdim=True)
    rstd = 1 / torch.sqrt(var + eps)
    xhat = xc * rstd
    dxh = dy * g
    m1 = dxh.mean(-1, keepdim=True)
    m2 = (dxh * xhat).mean(-1, keepdim=True)
    dx = rstd * (dxh - m1 - xhat * m2)
    sig = torch.sqrt(var)
    e_mean = gamma(nD) * x.abs().mean(-1, keepdim=True) + U * mean.abs()           # the sum, then / D
    # sum (x - mean)^2: the shifted values carry e_mean + u |xc|; by Cauchy-Schwarz sum |xc| / sum xc^2 <= 1 / sigma
    e_q = 2 * e_mean / sig.clamp_min(1e-300) + 2 * U + gamma(nD + 1)
    e_rstd = 0.5 * (e_q * var / (var + eps) + 3 * U) + 2 * 2.0 ** -23                   # / D, + eps; rsqrtf within 2 ulp
    e_xhat = rstd * (e_mean + U * xc.abs()) + xhat.abs() * (e_rstd + U)              # absolute
    e_dxh = 2 * U * dxh.abs()                                                       # g = 1 + table rounds once; the product once
    e_m1 = (gamma(nD) + 2 * U) * dxh.abs().mean(-1, keepdim=True) + U * m1.abs()
    e_m2 = ((dxh.abs() * e_xhat).mean(-1, keepdim=True) + (gamma(nD + 1) + 3 * U) * (dxh * xhat).abs().mean(-1, keepdim=True) + U * m2.abs())
    t = dxh - m1 - xhat * m2
    e_t = e_dxh + e_m1 + e_xhat * m2.abs() + xhat.abs() * e_m2 + 3 * U * (dxh.abs() + m1.abs() + (xhat * m2).abs())
    e_dx = rstd * e_t + dx.abs() * (e_rstd + 2 * U)
    return dict(dx=dx, e_dx=e_dx, xhat=xhat, e_xhat=e_xhat)


@pytest.mark.parametrize("dt", ACT, ids=DT_ID.get)
@pytest.mark.parametrize("L", [1, 33, 265])
@pytest.mark.parametrize("NV", [1, 2, 3, 4, 5, 6, 7, 8])
def test_layernorm_bwd_matches_fp64(G, TO, NV, L, dt):
    D, B, eps = 128 * NV, 2, 1e-5
    x = _ln_x(B, L, D, seed=NV * 100 + L)
    gen = torch.Generator().manual_seed(NV + L)
    dy = torch.randn(B, L, D, generator=gen)
    gamma_ = 1 + 0.3 * torch.randn(D, generator=gen)
    dx0 = torch.randn(B, L, D, generator=gen)                   # the residual branch's gradient, accumulated onto
    dg0, db0 = torch.randn(D, generator=gen), torch.randn(D, generator=gen)
    dx, dg, db = dx0.cuda(), dg0.cuda(), db0.cuda()
    dxa = torch.full((B, L, D), 7.0, device="cuda").to(dt)
    TO.layernorm_bwd(x.cuda(), dy.cuda(), dx, gamma_.cuda(), dg, db, eps=eps, dx_act=dxa)
    r = _ln_bwd_bounds(x.double(), dy.double(), gamma_.double(), eps, NV)
    ref = dx0.double() + r["dx"]
    _assert_within(dx.cpu(), ref, SECOND_ORDER * (r["e_dx"] + U * ref.abs()), f"layernorm_bwd dx D={D}")
    _assert_bitwise(dxa.cpu(), _store_ref(G, dx.cpu(), dt), "dx_act")
    # dgamma / dbeta: 4 rows per thread, 8 warps in shared memory, one atomic per 32-row CTA onto the pre-filled value
    depth = 4 + 8 + B * -(-L // 32) + 1
    dyd = dy.double()
    prod = (dyd * r["xhat"]).reshape(-1, D)
    ref_g = dg0.double() + prod.sum(0)
    b_g = gamma(depth) * (dg0.double().abs() + prod.abs().sum(0)) + (dyd.abs() * r["e_xhat"]).reshape(-1, D).sum(0) + U * prod.abs().sum(0)
    _assert_within(dg.cpu(), ref_g, SECOND_ORDER * b_g, "dgamma (accumulated)")
    ref_b = db0.double() + dyd.reshape(-1, D).sum(0)
    _assert_within(db.cpu(), ref_b, gamma(depth) * (db0.double().abs() + dyd.abs().reshape(-1, D).sum(0)), "dbeta (accumulated)")


@pytest.mark.parametrize("dt", ACT, ids=DT_ID.get)
@pytest.mark.parametrize("L", [1, 33, 265])
@pytest.mark.parametrize("NV", [1, 3, 5, 8])
def test_ada_layernorm_bwd_matches_fp64(G, TO, NV, L, dt):
    D, B, eps = 128 * NV, 3, 1e-5
    x = _ln_x(B, L, D, seed=NV * 10 + L + 7)
    gen = torch.Generator().manual_seed(NV * 3 + L)
    dy = torch.randn(B, L, D, generator=gen)
    table = 0.2 * torch.randn(4, 2 * D, generator=gen)
    idx = torch.tensor([2, 0, 2])                               # two batch elements share a table row
    dx0 = torch.randn(B, L, D, generator=gen)
    dt0 = torch.randn(4, 2 * D, generator=gen)                  # pre-filled: dtable is accumulated onto
    dx, dtab = dx0.cuda(), dt0.cuda()
    dxa = torch.full((B, L, D), 7.0, device="cuda").to(dt)
    TO.ada_layernorm_bwd(x.cuda(), dy.cuda(), dx, table.cuda(), idx.cuda(), dtab, eps=eps, dx_act=dxa)
    gsel = 1 + table.double()[idx][:, None, :D]
    r = _ln_bwd_bounds(x.double(), dy.double(), gsel, eps, NV)
    ref = dx0.double() + r["dx"]
    _assert_within(dx.cpu(), ref, SECOND_ORDER * (r["e_dx"] + U * ref.abs()), f"ada_layernorm_bwd dx D={D}")
    _assert_bitwise(dxa.cpu(), _store_ref(G, dx.cpu(), dt), "dx_act")
    dyd = dy.double()
    prod = dyd * r["xhat"]
    ref_t = dt0.double().clone()
    bnd = torch.zeros_like(ref_t)
    n_cta = -(-L // 32)
    for row in range(4):
        sel = (idx == row)
        nb = int(sel.sum())
        if nb == 0:
            continue
        depth = 4 + 8 + nb * n_cta + 1
        ps, ds = prod[sel].reshape(-1, D), dyd[sel].reshape(-1, D)
        ref_t[row, :D] += ps.sum(0)
        ref_t[row, D:] += ds.sum(0)
        bnd[row, :D] = (gamma(depth) * (dt0.double()[row, :D].abs() + ps.abs().sum(0)) + (dyd[sel].abs() * r["e_xhat"][sel]).reshape(-1, D).sum(0)
                        + U * ps.abs().sum(0))
        bnd[row, D:] = gamma(depth) * (dt0.double()[row, D:].abs() + ds.abs().sum(0))
    _assert_within(dtab.cpu(), ref_t, SECOND_ORDER * bnd, "dtable (accumulated; unselected rows unchanged)")


# ================================================================================================ colsum
@pytest.mark.parametrize("dt", ACT, ids=DT_ID.get)
@pytest.mark.parametrize("rows", [1, 63, 64, 65, 5300])
@pytest.mark.parametrize("N,path", [(1, "scalar"), (7, "scalar"), (8, "vector"), (8, "offset"), (1000, "vector"), (1000, "offset"), (3072, "vector"),
                                    (3072, "offset")])
def test_colsum_matches_fp64(TO, dt, rows, N, path):
    """vector: 16-byte loads (N % 8 == 0, 32-byte aligned base); offset: the same columns 2 elements into the row (scalar path); NaN beyond N."""
    off = 2 if path == "offset" else 0
    ld = N + off + 8
    g = torch.Generator().manual_seed(rows * 7 + N)
    x = (torch.randn(rows, N, generator=g) * torch.logspace(-2, 2, N)).to(dt)
    buf = torch.full((rows, ld), float("nan")).to(dt)
    buf[:, off:off + N] = x
    buf = buf.cuda()
    out = torch.full((N,), float("nan"), device="cuda")         # overwritten, not accumulated onto
    TO.colsum(buf[:, off:off + N], out)
    xd = x.double()
    # per column: each thread adds 8 rows of a 64-row slab, 8 warps are added in shared memory, one atomic per slab: depth 16 + ceil(rows / 64)
    depth = 16 + -(-rows // 64)
    _assert_within(out.cpu(), xd.sum(0), gamma(depth) * xd.abs().sum(0), f"colsum {path}")


# ================================================================================================ bit-exact data movement
@pytest.mark.parametrize("dt", ACT, ids=DT_ID.get)
@pytest.mark.parametrize("n,path,with_scale", [(8, "vector", False), (1027, "vector", True), (1027, "scalar", True), (1027, "scalar", False),
                                               (3_000_001, "vector", True), (3_000_001, "scalar", True)])
def test_cast_scale_bitwise(G, TO, dt, n, path, with_scale):
    """out = T(x * s): the vector path (16-byte aligned, n / 4 float4s plus a scalar tail of n % 4) and the scalar path (misaligned input).
    3M elements: the grid-stride loops run more than once."""
    g = torch.Generator().manual_seed(n)
    x = torch.randn(n + 1, generator=g) * 10
    xin = x.cuda()[1:] if path == "scalar" else x.cuda()[:n]
    out = torch.full((n + 4,), 7.0, device="cuda").to(dt)
    s = torch.tensor([0.7])
    TO.cast_scale(xin, out[:n], s.cuda() if with_scale else None)
    prod = xin.cpu() * (s if with_scale else 1.0)               # fp32 product, as the kernel forms it
    _assert_bitwise(out[:n].cpu(), _store_ref(G, prod, dt), "cast_scale")
    assert bool((out[n:].float() == 7.0).all())


def _rand_bits(shape, dt, seed):
    g = torch.Generator().manual_seed(seed)
    if dt == torch.float32:
        return torch.randint(-2 ** 31, 2 ** 31 - 1, shape, generator=g, dtype=torch.int64).to(torch.int32).view(torch.float32)
    return torch.randint(-2 ** 15, 2 ** 15 - 1, shape, generator=g, dtype=torch.int64).to(torch.int16).view(torch.bfloat16)


@pytest.mark.parametrize("dt,path", [(torch.float32, "scalar"), (torch.bfloat16, "vector"), (torch.bfloat16, "scalar")])
@pytest.mark.parametrize("rows,cols", [(1, 1), (63, 65), (64, 64), (795, 136)])
@pytest.mark.parametrize("batch", [1, 3])
def test_transpose_bitwise(TO, dt, path, rows, cols, batch):
    """Both kernels: the 64x64 16-byte one (2-byte elements, aligned, strides % 8 == 0) and the 32x32 element one (4-byte elements, or an odd
    leading dimension).  Random bit patterns (NaN payloads included) must arrive unchanged; output columns >= rows stay untouched."""
    ld_in = -(-cols // 8) * 8 + (8 if path == "vector" else 3)
    ld_out = -(-rows // 8) * 8 + (8 if path == "vector" else 5)
    src = _rand_bits((batch, rows + 1, ld_in), dt, seed=rows * cols + batch)
    x = src.cuda()[:, :rows, :cols]                              # batch stride (rows + 1) * ld_in
    out = _rand_bits((batch, cols + 2, ld_out), dt, seed=7).cuda()
    before = out.cpu()
    TO.transpose(x if batch > 1 else x[0], out[:, :cols] if batch > 1 else out[0, :cols])
    got, ref = out.cpu(), before.clone()
    ref[:, :cols, :rows] = src[:, :rows, :cols].transpose(1, 2)
    _assert_bitwise(got, ref, "transpose")


@pytest.mark.parametrize("dt", ACT, ids=DT_ID.get)
def test_heads_split_merge_bitwise(TO, dt):
    B, H, L = 3, 5, 77
    D = H * 64
    ld = 3 * D + 16                                              # ld > H * 64, the head block at a 16-byte aligned column offset
    tok = _rand_bits((B * L, ld), dt, seed=11)
    heads = torch.full((B * H, L, 64), 7.0, dtype=dt, device="cuda")
    TO.heads_split(tok.cuda()[:, 8 + D:8 + 2 * D], heads, B, H, L)
    ref = tok[:, 8 + D:8 + 2 * D].reshape(B, L, H, 64).permute(0, 2, 1, 3).reshape(B * H, L, 64)
    _assert_bitwise(heads.cpu(), ref, "heads_split")
    back = _rand_bits((B * L, ld), dt, seed=12).cuda()
    before = back.cpu()
    TO.heads_merge(heads, back[:, 8 + D:8 + 2 * D], B, H, L)
    exp = before.clone()
    exp[:, 8 + D:8 + 2 * D] = tok[:, 8 + D:8 + 2 * D]
    _assert_bitwise(back.cpu(), exp, "heads_merge (other columns untouched)")


@pytest.mark.parametrize("n,D", [(4, 128), (5300, 1024)])   # 5.4M elements: the grid-stride loops run more than once
def test_gather_scatter_rows(TO, n, D):
    g = torch.Generator().manual_seed(n)
    table = torch.randn(100, D, generator=g)
    idx = torch.randint(0, 100, (n,), generator=g)
    idx[:4] = torch.tensor([5, 99, 5, 0])                       # repeated indices
    out = torch.full((n, D), 7.0, device="cuda")
    TO.gather_rows(table.cuda(), idx.cuda(), out)
    _assert_bitwise(out.cpu(), table[idx], "gather_rows")
    src = torch.randn(n, D, generator=g)
    acc = table.cuda()                                          # accumulated onto
    TO.scatter_add_rows(acc, idx.cuda(), src.cuda())
    ref = table.double().index_add(0, idx, src.double())
    # each element: atomics in any order onto the pre-filled value, depth = (times its row is indexed) + 1
    depth = torch.bincount(idx, minlength=100).double()[:, None] + 1
    bound = gamma(depth) * table.double().abs().index_add(0, idx, src.double().abs())
    _assert_within(acc.cpu(), ref, bound, "scatter_add_rows")


# ================================================================================================ embedding backward
def test_embed_bwd_matches_fp64(TO):
    B, L, D, H, W, K = 3, 260, 256, 5, 53, 64                   # L = 260 < H * W = 265; ids include the [MASK] class K
    num_embed = K + 1
    g = torch.Generator().manual_seed(4)
    ids = torch.randint(0, num_embed, (B, L), generator=g)
    ids[0, :5] = K
    dx = torch.randn(B, L, D, generator=g)
    de0, dh0, dw0 = torch.randn(num_embed, D, generator=g), torch.randn(H, D, generator=g), torch.randn(W, D, generator=g)
    de, dh, dw = de0.cuda(), dh0.cuda(), dw0.cuda()
    TO.embed_bwd(ids.cuda(), dx.cuda(), de, dh, dw)
    dxd = dx.double().reshape(B * L, D)
    flat = ids.reshape(-1)
    ref_e = de0.double().index_add(0, flat, dxd)
    cnt = torch.bincount(flat, minlength=num_embed).double()[:, None] + 1
    abs_e = de0.double().abs().index_add(0, flat, dxd.abs())
    _assert_within(de.cpu(), ref_e, cnt * U / (1 - cnt * U) * abs_e, "demb (atomics onto the pre-filled table)")
    pos = torch.arange(L)
    hrow, wrow = pos // W, pos % W
    dxl = dx.double()                                           # (B, L, D)
    ref_h = dh0.double().index_add(0, hrow, dxl.sum(0))
    abs_h = dh0.double().abs().index_add(0, hrow, dxl.abs().sum(0))
    ref_w = dw0.double().index_add(0, wrow, dxl.sum(0))
    abs_w = dw0.double().abs().index_add(0, wrow, dxl.abs().sum(0))
    # fixed-order sums: a height row adds B * W values and the pre-filled one, a width row B * H values and the pre-filled one
    _assert_within(dh.cpu(), ref_h, gamma(B * W + 1) * abs_h, "dheight")
    _assert_within(dw.cpu(), ref_w, gamma(B * H + 1) * abs_w, "dwidth")


# ================================================================================================ a training step on NaN-filled workspaces
def _train_step(G, precision, fill, use_graph):
    """One forward + loss + backward of a D = 256, 2-layer denoiser whose engine allocates every buffer (packed weights, activations, scratch)
    filled with `fill`.  Returns {name: tensor} of the loss, log_model_prob, logits and every parameter gradient."""
    from oracle import diffsound_oracle as O
    from tests.helpers import build_dt, portable_uniform
    from diffsound_b200 import train_ops
    K, D, NL, NH, CD, B, L = 64, 256, 2, 4, 96, 3, 265
    sd = O.make_transformer_state_dict(K=K, D=D, n_layer=NL, n_head=NH, cond_dim=CD, seed=21)
    m = build_dt(K, D, NL, NH, CD, sd=sd)
    eng = m.transformer.train_engine
    eng.__init__(m.transformer, precision=precision)
    eng.use_cuda_graph = use_graph
    eng._act = lambda *shape: torch.full(shape, fill, dtype=eng.adt, device=eng.device)
    eng._f32 = lambda *shape: torch.full(shape, fill, dtype=torch.float32, device=eng.device)
    gen = torch.Generator().manual_seed(22)
    cond = torch.randn(B, 77, CD, generator=gen)
    x0 = torch.randint(0, K, (B, L), generator=gen).cuda()
    t, pt = torch.tensor([3, 0, 77]).cuda(), torch.tensor([0.01, 0.02, 0.005]).cuda()
    x_t = train_ops.q_sample(x0, t, portable_uniform(23, (B, K + 1, L)).cuda(), m._sched(), 100)
    loss, prob, grads = G.run_loss_and_grads(m, x0, x_t, cond.cuda(), t, pt)
    out = {"loss": loss.reshape(1), "log_model_prob": prob, "logits": eng.workspace(B, L, 77)["logits"]}
    out.update({"grad " + n: g for n, g in grads.items()})
    return {k: v.detach().float().cpu().clone() for k, v in out.items()}


@pytest.mark.parametrize("use_graph", [False, True], ids=["eager", "graph"])
@pytest.mark.parametrize("precision", ["tf32", "bf16"])
def test_training_step_on_nan_filled_buffers(G, precision, use_graph):
    """No kernel of the step may read a buffer element that nothing wrote (the padding columns of P, the transposed wgrad scratch, ...).
    A read of an unwritten element shows up as a NaN, so every output must be finite.  The run must also agree with zero-filled runs, which
    catches a NaN dropped by fmaxf into a different finite value.  If two zero-filled runs agree bit for bit, so must the NaN-filled one.  They
    do not: the LayerNorm-backward, colsum and scatter atomics add in a different order on every run, and that noise reaches every gradient
    downstream of them.  Two runs show only a sample of it: on an H100, four zero-filled runs agreed bit for bit on a tensor that the next run
    changed in one column (one dtable element one ulp off, flipping its TF32 rounding in the AdaLN Linear's weight-gradient GEMM).  So each
    tensor may differ from the clean run by twice the clean runs' difference or by 2^-12 of its largest magnitude, whichever is larger: above
    such a flip (measured up to 2.7e-6 of the tensor's maximum) and far below the O(1) change of a masked NaN, which the 3e38 run catches
    independently of this tolerance."""
    c1 = _train_step(G, precision, 0.0, use_graph)
    c2 = _train_step(G, precision, 0.0, use_graph)
    nr = _train_step(G, precision, float("nan"), use_graph)
    # fmaxf drops a NaN but not a huge value: a read through a max (the softmax row maximum) of a 3e38 fill overflows the exponentials or the
    # following sums, and an arithmetic read overflows too, so this run must also be finite
    big = _train_step(G, precision, 3.0e38, use_graph)
    assert c1.keys() == nr.keys() == big.keys()
    for name in c1:
        assert bool(torch.isfinite(nr[name]).all()), f"{name}: non-finite after a NaN-filled run"
        assert bool(torch.isfinite(big[name]).all()), f"{name}: non-finite after a run on buffers filled with 3e38"
    if all(torch.equal(_bits(c1[n]), _bits(c2[n])) for n in c1):
        for name in c1:
            assert torch.equal(_bits(nr[name]), _bits(c1[name])), f"{name}: clean runs agree bit for bit, the NaN-filled run does not"
        return
    for name in c1:
        spread = float((c1[name] - c2[name]).abs().max())
        diff = float((nr[name] - c1[name]).abs().max())
        tol = max(2 * spread, 2.0 ** -12 * float(c1[name].abs().max()))
        assert diff <= tol, f"{name}: NaN-filled run differs by {diff:.3e}, clean runs by {spread:.3e}, allowed {tol:.3e}"
