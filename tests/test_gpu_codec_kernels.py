"""The SpecVQGAN decoder's and the MelGAN vocoder's support kernels (csrc/decoder.cu, csrc/vocoder.cu) and the GEMM's calibration epilogue, each
against a plain torch restatement of the same operation on the H100.

Data-movement kernels (gather, upsample, padding, token scatter) are compared bit for bit.  Arithmetic kernels (GroupNorm, softmax) are compared
with fp64 at tolerances that a dropped lo half of an fp16 (hi | lo) pair (2^-12 relative, DESIGN section 3) would exceed.  The CPU stand-ins that
tests/test_cpu_codec_host.py runs in place of the split-fp16 kernels are checked here against the real kernels, bit for bit."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def G():
    from tests import gpu_common
    return gpu_common


def _bits(t):
    """Integer view of a float tensor on the CPU: equal bits, not merely equal values (-0.0 != +0.0, NaN payloads compare)."""
    t = t.contiguous().cpu()
    return t.view({torch.float32: torch.int32, torch.float16: torch.int16, torch.float64: torch.int64}[t.dtype])


def _assert_bitwise(got, ref):
    assert got.shape == ref.shape and got.dtype == ref.dtype, (got.shape, ref.shape, got.dtype, ref.dtype)
    bad = int((_bits(got) != _bits(ref)).sum())
    assert bad == 0, f"{bad} of {ref.numel()} elements differ"


def _pad_hw(x):
    """(B, H, W, C) -> (B, H+2, W+2, C) with an exactly zero border."""
    return F.pad(x, (0, 0, 1, 1, 1, 1))


def _tf32_pair(G, v, dim=-1):
    hi = G.tf32_round_ref(v)
    return torch.cat([hi, G.tf32_round_ref(v - hi)], dim)


def _f16_pair(v, dim=-1):
    hi = v.half()
    return torch.cat([hi, (v - hi.float()).half()], dim)  # v - hi in fp32, as the kernels compute it


def _is_tf32(t):
    return bool(((_bits(t.float()) & 0x1FFF) == 0).all())


def _f16_ulp(h):
    """ulp of each fp16 value, in fp64, from its exponent field: 2^(E - 25), and 2^-24 for zero and subnormals (E = 0)."""
    e = (_bits(h).int() >> 10) & 0x1F
    return torch.pow(2.0, (e.clamp(min=1) - 25).double())


def _assert_lo_within_half_ulp(hi, lo):
    hi, lo = hi.cpu(), lo.cpu()
    bad = lo.double().abs() > 0.5 * _f16_ulp(hi)
    if bool(bad.any()):
        i = bad.nonzero()[0].tolist()
        raise AssertionError(f"{int(bad.sum())} lo halves exceed half an ulp of hi, first at {i}: hi={float(hi[tuple(i)])!r} lo={float(lo[tuple(i)])!r}")


# ------------------------------------------------------------------------------------------------------------ codebook_gather_padded
@pytest.mark.parametrize("B,H,W,E,n_codes", [(2, 5, 53, 256, 256), (3, 7, 4, 260, 97)])  # E = 260: 65 float4 slots, more than a warp has lanes
def test_codebook_gather_padded_all_forms(G, B, H, W, E, n_codes):
    from oracle import diffsound_oracle as O
    ops = G.ops
    g = torch.Generator().manual_seed(E + H)
    cb = torch.randn(n_codes, E, generator=g) * torch.logspace(-3, 2, E)
    ids = torch.randint(0, n_codes, (B, H * W), generator=g)  # column-major token order, as the denoiser emits it
    ref = _pad_hw(cb[O.column_major_reverse(ids, H, W)].view(B, H, W, E))
    idc, cbc = ids.cuda(), cb.cuda()
    _assert_bitwise(ops.codebook_gather_padded(idc, cbc, H, W, round_out=False), ref)
    _assert_bitwise(ops.codebook_gather_padded(idc, cbc, H, W, round_out=True), G.tf32_round_ref(ref))
    _assert_bitwise(ops.codebook_gather_padded(idc, cbc, H, W, split=True), _tf32_pair(G, ref))
    _assert_bitwise(ops.codebook_gather_padded(idc, cbc, H, W, split_f16=True), _f16_pair(ref))


@pytest.mark.parametrize("split_f16", [False, True])
def test_codebook_gather_err_flag(G, split_f16):
    ops = G.ops
    B, H, W, E, n_codes = 2, 5, 53, 64, 50
    g = torch.Generator().manual_seed(7)
    cb = torch.randn(n_codes, E, generator=g).cuda()
    ids = torch.randint(0, n_codes, (B, H * W), generator=g)
    flag = torch.zeros(1, dtype=torch.int32, device="cuda")
    ops.codebook_gather_padded(ids.cuda(), cb, H, W, split_f16=split_f16, err_flag=flag)
    assert int(flag) == 0
    for bad in (-1, n_codes):
        b_ids = ids.clone()
        b_ids[1, 17] = bad
        flag.zero_()
        ops.codebook_gather_padded(b_ids.cuda(), cb, H, W, split_f16=split_f16, err_flag=flag)
        assert int(flag) == 1, bad


# ------------------------------------------------------------------------------------------------------------ GroupNorm
def _gn_input(B, H, W, C, groups, seed):
    """Interior (B, H, W, C): per-group scales from 1e-2 to 1e1 and offsets of up to one standard deviation.  The 1e-2 groups make eps visible:
    their variance is 1e-4, so eps 1e-5 instead of 1e-6 moves rstd by 4 %."""
    g = torch.Generator().manual_seed(seed)
    cg = C // groups
    scale = torch.logspace(-2, 1, groups).repeat_interleave(cg)
    off = (torch.rand(groups, generator=g) * 2 - 1).repeat_interleave(cg)
    return (torch.randn(B, H, W, C, generator=g) + off) * scale


def _gn_ref_stats(x_int, groups):
    B, H, W, C = x_int.shape
    xd = x_int.double().reshape(B, H * W, groups, C // groups)
    return torch.stack([xd.sum((1, 3)), (xd * xd).sum((1, 3))], -1)  # (B, groups, 2): sum, sumsq


@pytest.mark.parametrize("B,H,W,C", [(2, 5, 53, 128),    # C/groups = 4: staged per-thread partials; rows_per_block clamps at 16
                                     (2, 5, 53, 96),     # C/groups = 3: shared-memory atomics
                                     (2, 5, 53, 64),     # C/groups = 2: shared-memory atomics
                                     (2, 80, 848, 128)])  # the 80 x 848 level: rows_per_block clamps at 256
def test_groupnorm_stats_matches_fp64(G, B, H, W, C):
    groups = 32
    x = _gn_input(B, H, W, C, groups, seed=C + H)
    x[1, ..., :C // groups] += 20.0 * x[1, ..., :C // groups].std()  # a DC offset of 20 sigma: cancellation in E[x^2] - mean^2
    xc = _pad_hw(x).cuda()
    st = G.ops.groupnorm_stats(xc, groups=groups)
    xd = x.cuda().double().reshape(B, H * W, groups, C // groups)
    ref = torch.stack([xd.sum((1, 3)), (xd * xd).sum((1, 3))], -1)
    abs_sum = torch.stack([xd.abs().sum((1, 3)), (xd * xd).sum((1, 3))], -1)
    # each thread sums at most 128 rows of one channel in fp32 before the fp64 reduction: 128 * 2^-24 = 7.6e-6 of sum |x| (or of sum x^2)
    err = (st - ref).abs()
    assert bool((err <= 8e-6 * abs_sum).all()), float((err / abs_sum).max())
    cnt = H * W * (C // groups)
    mean, mean_ref = st[..., 0] / cnt, ref[..., 0] / cnt
    var, var_ref = st[..., 1] / cnt - mean * mean, ref[..., 1] / cnt - mean_ref * mean_ref
    # the same bound carried through var = E[x^2] - mean^2
    var_tol = 8e-6 * (abs_sum[..., 1] / cnt + 2 * mean_ref.abs() * abs_sum[..., 0] / cnt)
    assert bool(((var - var_ref).abs() <= var_tol).all())
    print(f"groupnorm_stats C={C} P={(H + 2) * (W + 2)}: max var rel err {float(((var - var_ref).abs() / var_ref).max()):.2e}")


_GN_CASES = {
    "rows128": (2, 5, 53, 128, 0),          # one CTA per padded row (256 % (C/4) == 0)
    "rows512": (2, 5, 53, 512, 0),
    "flat96": (2, 10, 13, 96, 0),           # flat-index kernel: 24 float4 slots do not divide 256
    "compact": (2, 5, 53, 512, 272),        # token rows (B, Lp, C) with Lp > H*W (the decoder's attention blocks)
    "uncached": (65, 5, 53, 128, 272),      # B * groups = 2080 > 2048: mean / rstd recomputed per element from fp64 stats
}


@pytest.mark.parametrize("case", list(_GN_CASES))
def test_groupnorm_apply_matches_fp64(G, case):
    ops = G.ops
    B, H, W, C, Lp = _GN_CASES[case]
    groups, eps = 32, 1e-6
    cg = C // groups
    x = _gn_input(B, H, W, C, groups, seed=C + B)
    x[:, :, :, 5 * cg:6 * cg] = 0.75  # one constant, exactly representable group: var = 0, output = beta
    g = torch.Generator().manual_seed(C)
    gamma, beta = torch.randn(C, generator=g) * 0.5 + 1.0, torch.randn(C, generator=g) * 0.5
    xc, gc, bc = _pad_hw(x).cuda(), gamma.cuda(), beta.cuda()
    stats = _gn_ref_stats(x.cuda(), groups)  # exact statistics: this test is about the apply kernel alone
    gn = F.group_norm(x.cuda().double().permute(0, 3, 1, 2), groups, gc.double(), bc.double(), eps=eps).permute(0, 2, 3, 1)  # (B, H, W, C)

    def layout(v, Co):  # interior values -> the kernel's output layout, zero outside
        if Lp:
            return F.pad(v.reshape(B, H * W, Co), (0, 0, 0, Lp - H * W))
        return _pad_hw(v)

    for swish in (False, True):
        ref_i = gn * torch.sigmoid(gn) if swish else gn
        ref = layout(ref_i, C)
        scale = float(ref.abs().max())
        tol = 3e-6 * scale  # fp32 normalise + affine (a few ulps), __expf / __fdividef in swish; a missing fp16 lo half is 2.4e-4 relative
        outside = layout(torch.ones_like(ref_i), C) == 0
        const = ref_i[..., 5 * cg:6 * cg]
        b_const = beta[5 * cg:6 * cg].cuda().expand_as(const)

        def run(**kw):
            Co = 2 * C if (kw.get("split") or kw.get("split_f16")) else C
            shape = (B, Lp, Co) if Lp else (B, H + 2, W + 2, Co)
            out = torch.full(shape, float("nan"), dtype=torch.float16 if kw.get("split_f16") else torch.float32, device="cuda")
            ops.groupnorm_apply(xc, stats, gc, bc, eps=eps, swish=swish, compact_len=Lp, out=out, groups=groups, **kw)
            return out

        # plain fp32
        o = run(round_out=False)
        assert torch.equal(_bits(o[outside[..., 0]]), torch.zeros_like(_bits(o[outside[..., 0]])))  # border / padding rows: exactly +0
        assert float((o.double() - ref).abs().max()) <= tol, (swish, float((o.double() - ref).abs().max()) / scale)
        oc = (o[:, 1:H + 1, 1:W + 1] if not Lp else o[:, :H * W].reshape(B, H, W, C))[..., 5 * cg:6 * cg]
        if swish:
            assert float((oc.double() - b_const.double() * torch.sigmoid(b_const.double())).abs().max()) <= tol
        else:
            assert torch.equal(oc, b_const)
        # TF32-rounded
        o = run(round_out=True)
        assert _is_tf32(o)
        assert bool(((o.double() - ref).abs() <= 2.0 ** -11 * ref.abs() + tol).all())
        # split-TF32 pair: both halves TF32-valued, hi + lo at fp32-class accuracy
        o = run(split=True)
        hi, lo = o[..., :C], o[..., C:]
        assert _is_tf32(hi) and _is_tf32(lo)
        assert float((hi.double() + lo.double() - ref).abs().max()) <= tol
        assert float(o[outside[..., 0]].abs().max()) == 0.0
        # split-fp16 pair: |lo| <= half an ulp of hi, hi + lo at fp32-class accuracy
        o = run(split_f16=True)
        hi, lo = o[..., :C], o[..., C:]
        err = float((hi.double() + lo.double() - ref).abs().max())
        print(f"groupnorm_apply {case} swish={swish}: f16 pair err {err / scale:.2e} of max|ref|")
        assert err <= tol
        _assert_lo_within_half_ulp(hi, lo)
        assert float(o[outside[..., 0]].abs().max()) == 0.0


# ------------------------------------------------------------------------------------------------------------ upsample, softmax, token add
@pytest.mark.parametrize("B,H,W,C", [(2, 5, 53, 512), (2, 5, 53, 4)])
def test_upsample2x_padded_bitwise(G, B, H, W, C):
    ops = G.ops
    g = torch.Generator().manual_seed(C)
    x = torch.randn(B, H, W, C, generator=g) * torch.logspace(-4, 3, C)
    xp = _pad_hw(x)
    xp[:, 0], xp[:, -1], xp[:, :, 0], xp[:, :, -1] = float("nan"), float("nan"), float("nan"), float("nan")  # the input border is never read
    ref = _pad_hw(x.repeat_interleave(2, 1).repeat_interleave(2, 2))
    xc = xp.cuda()
    _assert_bitwise(ops.upsample2x_padded(xc, round_out=False), ref)
    _assert_bitwise(ops.upsample2x_padded(xc, round_out=True), G.tf32_round_ref(ref))
    _assert_bitwise(ops.upsample2x_padded(xc, split=True), _tf32_pair(G, ref))
    _assert_bitwise(ops.upsample2x_padded(xc, split_f16=True), _f16_pair(ref))


@pytest.mark.parametrize("n_valid", [1, 31, 32, 33, 265])
def test_softmax_rows_matches_fp64(G, n_valid):
    ld, rows = 272, 300
    g = torch.Generator().manual_seed(n_valid)
    x = torch.randn(rows, ld, generator=g) * 3
    x[:100] += 1e3
    x[100:200] -= 1e3
    x[:, n_valid:] = 1e30  # columns beyond n_valid must not enter the max or the sum
    ref = torch.softmax(x[:, :n_valid].double(), -1)
    for round_out in (False, True):
        o = G.ops.softmax_rows_(x.clone().cuda(), n_valid, round_out=round_out).cpu()
        assert bool(torch.isfinite(o).all())
        assert torch.equal(_bits(o[:, n_valid:]), torch.zeros(rows, ld - n_valid, dtype=torch.int32))
        # expf (2 ulp), a 9-term fp32 sum per lane plus a 5-level tree, one division: 2e-6 relative per element
        tol = 2e-6 * ref + (2.0 ** -11 * ref if round_out else 0)
        assert bool(((o[:, :n_valid].double() - ref).abs() <= tol).all())
        if round_out:
            assert _is_tf32(o)


def test_tokens_add_to_padded_bitwise(G):
    B, H, W, C, Lp = 2, 5, 53, 512, 272
    g = torch.Generator().manual_seed(11)
    tok = torch.randn(B, Lp, C, generator=g)
    tok[:, H * W:] = float("nan")  # padding token rows are never read
    xp = torch.randn(B, H + 2, W + 2, C, generator=g)  # border filled too: it must come back unchanged
    ref = xp.clone()
    ref[:, 1:H + 1, 1:W + 1] += tok[:, :H * W].reshape(B, H, W, C)
    out = G.ops.tokens_add_to_padded_(tok.cuda(), xp.cuda())
    _assert_bitwise(out, ref)


# ------------------------------------------------------------------------------------------------------------ MelGAN: lrelu_pad
@pytest.mark.parametrize("channel_major", [False, True])
@pytest.mark.parametrize("B,T,C,pad", [(2, 300, 64, 3), (2, 40, 80, 39), (1, 5, 32, 4)])  # pad = T - 1: the largest reflection
def test_lrelu_pad_bitwise(G, B, T, C, pad, channel_major):
    ops = G.ops
    g = torch.Generator().manual_seed(T + C)
    x = torch.randn(B, T, C, generator=g) * torch.logspace(-3, 2, C)
    xin = x.transpose(1, 2).contiguous() if channel_major else x
    Cp = (C + 31) // 32 * 32
    for reflect in (True, False):
        ref = F.pad(F.leaky_relu(x, 0.2).transpose(1, 2), (pad, pad), mode="reflect" if reflect else "constant").transpose(1, 2).contiguous()
        xc = xin.cuda()
        kw = dict(reflect=reflect, channel_major=channel_major)
        _assert_bitwise(ops.lrelu_pad(xc, pad, round_out=False, **kw), ref)
        _assert_bitwise(ops.lrelu_pad(xc, pad, round_out=True, **kw), G.tf32_round_ref(ref))
        refp = F.pad(ref, (0, Cp - C))  # split rows [hi (Cp) | lo (Cp)], channel columns >= C exactly zero
        _assert_bitwise(ops.lrelu_pad(xc, pad, split=True, **kw), _tf32_pair(G, refp))


# ------------------------------------------------------------------------------------------------------------ split-fp16 stand-ins vs kernels
@pytest.mark.parametrize("T,pad", [(10, 9), (848, 9), (4, 3)])  # T = pad + 1: every padding row reflects from the far end
def test_mel_pack_f16_matches_cpu_stand_in(G, T, pad):
    from tests import cpu_state_gemm_emulation as E
    B, Cm, Kp = 2, 80, 96
    g = torch.Generator().manual_seed(T)
    mel = torch.randn(B, Cm, T, generator=g) * torch.logspace(-6, 2, Cm)[:, None]  # lo halves reach fp16 subnormals
    got = G.ops.mel_pack_f16(mel.cuda(), pad, Kp)
    _assert_bitwise(got, E.mel_pack_f16(mel, pad, Kp))
    E._LIVE.clear()


@pytest.mark.parametrize("d", [1, 3, 9])
@pytest.mark.parametrize("reflect", [True, False])
def test_edge_pad_f16_matches_cpu_stand_in(G, d, reflect):
    from tests import cpu_state_gemm_emulation as E
    B, T, P, ld, c0, ncols = 2, 50, 9, 128, 32, 64
    g = torch.Generator().manual_seed(d)
    s = torch.full((B, T + 2 * P, ld), -1234.0, dtype=torch.float16)  # sentinel everywhere outside the interior rows
    s[:, P:P + T] = torch.randn(B, T, ld, generator=g).half()
    got = s.cuda()
    G.ops.edge_pad_f16(got, T, P, d, c0, ncols, reflect=reflect)
    ref = s.clone()
    E.edge_pad_f16(ref, T, P, d, c0, ncols, reflect=reflect)
    _assert_bitwise(got, ref)
    changed = torch.zeros_like(s, dtype=torch.bool)
    changed[:, P - d:P, c0:c0 + ncols] = True
    changed[:, P + T:P + T + d, c0:c0 + ncols] = True
    assert torch.equal(_bits(got.cpu()[~changed]), _bits(s[~changed]))  # rows beyond d and columns outside [c0, c0 + ncols) untouched


@pytest.mark.parametrize("scale", [1.0, 2.0 ** 3, 2.0 ** -5])
def test_split_f16_matches_cpu_stand_in(G, scale):
    from tests import cpu_state_gemm_emulation as E
    g = torch.Generator().manual_seed(int(scale * 64))
    e = torch.rand(257, 96, generator=g) * 46 - 30  # |scale * x| from 2^-30 (fp16 subnormals and below) to 2^16
    x = torch.sign(torch.randn(257, 96, generator=g)) * torch.pow(2.0, e)
    x = x.clamp(-65504.0, 65504.0)
    x[0, :4] = torch.tensor([65504.0, -65504.0, 6.1e-5, 5.96e-8])
    x = x / scale
    got = G.ops.split_f16(x.cuda(), scale)
    _assert_bitwise(got, E.split_f16(x, scale))
    E._LIVE.clear()


# ------------------------------------------------------------------------------------------------------------ GEMM calibration epilogue
def _amax_problem(M, N, a_rows=None, seed=0):
    """fp16 A / W / fp32 bias on a 1/8 grid: every product and every 64-term sum is exact in fp32, so kernel and fp64 stand-in agree bit for bit."""
    g = torch.Generator().manual_seed(seed)
    K = 64
    a = (torch.randint(-8, 9, (a_rows or M, K), generator=g) / 4).half()
    w = (torch.randint(-8, 9, (N, K), generator=g) / 8).half()
    bias = torch.randint(-16, 17, (N,), generator=g) / 8
    return a, w, bias, K


def _run_amax(G, a, w, bias, M, N, K, ldo, *, flags=0, geo=None, amax0=0.0, out=None, split=False):
    ops = G.ops
    ac, wc, bc = a.cuda(), w.cuda(), bias.cuda()
    if out is None:
        out = torch.full((M, 2 * ldo if split else ldo), 7.0, dtype=torch.float16 if split else torch.float32, device="cuda")
    amax = torch.full((1,), amax0, dtype=torch.float32, device="cuda")
    ops.gemm_desc(A=ac.data_ptr(), W=wc.data_ptr(), out=out.data_ptr(), M=M, N=N, K=K, taps=[(0, 0, 0, 0)], a_rows=a.shape[0], a_cols=K, lda=K,
                  ldw=K, w_cols=K, ldo=2 * ldo if split else ldo, bias=bc, flags=flags | (ops.OUT_F16_SPLIT if split else 0), geo=geo, amax_out=amax,
                  split_off=ldo if split else 0)
    torch.cuda.synchronize()
    return out, amax


def _stand_in_amax(a, w, bias, M, N, K, ldo, *, flags=0, geo=None, amax0=0.0):
    from tests import cpu_state_gemm_emulation as E
    a, w = E.track(a.clone()), E.track(w.clone())
    out = E.track(torch.zeros(M, ldo, dtype=torch.float32))
    amax = torch.full((1,), amax0, dtype=torch.float32)
    E.gemm_desc(A=a.data_ptr(), W=w.data_ptr(), out=out.data_ptr(), M=M, N=N, K=K, taps=[(0, 0, 0, 0)], a_rows=a.shape[0], a_cols=K, lda=K, ldw=K,
                w_cols=K, ldo=ldo, bias=bias, flags=flags | E.NO_STORE, geo=geo, amax_out=amax)
    E._LIVE.clear()
    return amax


_AMAX_CASES = {  # name: (M, N, ldo, a_rows, geo)
    "vector": (300, 128, 128, None, None),                 # whole 32-column chunks, 16-byte aligned: the vectorised epilogue
    "n_tail": (300, 33, 33, None, None),                   # N tail: scalar epilogue
    "ldo_odd": (300, 128, 129, None, None),                # aligned N, unaligned ldo: scalar epilogue
    "geo": (2 * 70, 128, 128, None, (70, 10, 1, 6, 1, 9)),  # border rows of two 7 x 10 padded images are stored as zeros
    "a_rows": (200, 128, 128, 256, None),                  # rows >= M of the last tile are computed but neither stored nor counted
}


def _amax_inputs(case):
    M, N, ldo, a_rows, geo = _AMAX_CASES[case]
    a, w, bias, K = _amax_problem(M, N, a_rows, seed=M + N + ldo)
    if a_rows:
        a[M:] = 1000.0
    if geo:
        P, Wp, y0, y1, x0, x1 = geo
        p = torch.arange(M) % P
        border = ~((p // Wp >= y0) & (p // Wp < y1) & (p % Wp >= x0) & (p % Wp < x1))
        a[border] = 1000.0  # a masked row would dominate amax if it were counted
    return M, N, ldo, geo, a, w, bias, K


@pytest.mark.parametrize("case", list(_AMAX_CASES))
def test_gemm_amax_equals_max_of_stored_output(G, case):
    ops = G.ops
    M, N, ldo, geo, a, w, bias, K = _amax_inputs(case)
    out, amax = _run_amax(G, a, w, bias, M, N, K, ldo, geo=geo)
    stored = out[:, :N]
    _assert_bitwise(amax.cpu(), stored.abs().max().reshape(1).cpu())
    assert float(amax) < 1000.0 or not (geo or case == "a_rows")
    assert torch.equal(out[:, N:], torch.full_like(out[:, N:], 7.0))  # columns beyond N in a wider row untouched
    # the stand-in of tests/cpu_state_gemm_emulation.py agrees (exact arithmetic: bit for bit)
    _assert_bitwise(_stand_in_amax(a, w, bias, M, N, K, ldo, geo=geo), amax.cpu())
    # NO_STORE: same amax, output untouched -- fp32 and split-fp16 outputs
    out_ns, amax_ns = _run_amax(G, a, w, bias, M, N, K, ldo, geo=geo, flags=ops.NO_STORE)
    _assert_bitwise(amax_ns, amax)
    assert torch.equal(out_ns, torch.full_like(out_ns, 7.0))
    _, amax_sp = _run_amax(G, a, w, bias, M, N, K, ldo, geo=geo, split=True)
    out_sp, amax_sp_ns = _run_amax(G, a, w, bias, M, N, K, ldo, geo=geo, split=True, flags=ops.NO_STORE)
    _assert_bitwise(amax_sp, amax)
    _assert_bitwise(amax_sp_ns, amax)
    assert torch.equal(out_sp, torch.full_like(out_sp, 7.0))
    # amax accumulates across launches: a larger value already there stays
    hi = float(amax) * 2 + 1
    _, amax_keep = _run_amax(G, a, w, bias, M, N, K, ldo, geo=geo, amax0=hi)
    assert float(amax_keep) == hi
    assert float(_stand_in_amax(a, w, bias, M, N, K, ldo, geo=geo, amax0=hi)) == hi


@pytest.mark.parametrize("case", ["vector", "n_tail", "ldo_odd"])
@pytest.mark.parametrize("bad", [float("nan"), float("inf")])
def test_gemm_amax_keeps_nan_and_inf(G, case, bad):
    """The MelGAN calibration (vocoder_engine.py) rejects a launch site whose amax is not finite: a NaN or inf anywhere in the output must reach
    amax on the vectorised epilogue path as on the scalar one."""
    ops = G.ops
    M, N, ldo, geo, a, w, bias, K = _amax_inputs(case)
    bias[N // 2] = bad
    for flags in (0, ops.NO_STORE):
        _, amax = _run_amax(G, a, w, bias, M, N, K, ldo, flags=flags)
        v = float(amax)
        assert (v != v) if bad != bad else v == float("inf"), (case, bad, flags, v)
    s = float(_stand_in_amax(a, w, bias, M, N, K, ldo))
    assert (s != s) if bad != bad else s == float("inf")
