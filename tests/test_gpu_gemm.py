"""wgmma GEMM parity: TF32 / BF16 operands pre-rounded on the host so the only error left is fp32 accumulation order."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def G():
    from tests import gpu_common
    return gpu_common


def _ref(a, w, bias=None, res=None, gelu=False, taps=None, out_rows=None):
    a, w = a.double(), w.double()
    if taps is None:
        y = a @ w.T
    else:
        K = a.shape[1]
        M = out_rows or a.shape[0]
        y = torch.zeros(M, w.shape[0], dtype=torch.float64)
        for i, s in enumerate(taps):
            idx = torch.arange(M) + s
            ok = (idx >= 0) & (idx < a.shape[0])
            sh = torch.zeros(M, K, dtype=torch.float64)
            sh[ok] = a[idx[ok]]
            y += sh @ w[:, i * K:(i + 1) * K].T
    if bias is not None:
        y = y + bias.double()
    if gelu:
        y = y * torch.sigmoid(1.702 * y)
    if res is not None:
        y = y + res.double()
    return y


@pytest.mark.parametrize("M,N,K,bn", [(128, 128, 32, 128), (128, 256, 128, 256), (530, 256, 1024, 0), (4240, 1024, 1024, 0), (1000, 3072, 1024, 256),
                                      (265, 4096, 1024, 128), (300, 1024, 4096, 0), (77 * 3, 2048, 512, 0), (200, 33, 64, 0), (130, 260, 100, 0)])
def test_gemm_tf32(G, M, N, K, bn):
    g = torch.Generator().manual_seed(M + N + K)
    a = G.tf32_round_ref(torch.randn(M, K, generator=g))
    w = G.tf32_round_ref(torch.randn(N, K, generator=g) * 0.05)
    bias = torch.randn(N, generator=g)
    out = G.ops.gemm(a.cuda(), w.cuda(), bias.cuda(), block_n=bn, cta_pair=-1)  # explicit tile width, no split-fp16 fusion
    torch.cuda.synchronize()
    assert G.relerr(out, _ref(a, w, bias)) < 2e-5


@pytest.mark.parametrize("M,N,K", [(256, 256, 64), (512, 256, 1024), (530, 256, 1024), (4240, 1024, 1024), (1000, 3072, 1024), (300, 1024, 4096),
                                   (77 * 3, 2048, 512), (200, 33, 64), (130, 260, 100), (129, 512, 96)])
@pytest.mark.parametrize("dtype", ["tf32", "f16"])
def test_gemm_cta_pair(G, M, N, K, dtype):
    """256-wide tiles forced through the cta_pair hint: same answers as the fp64 reference, incl. M / N / K tails."""
    g = torch.Generator().manual_seed(M * 7 + N + K)
    a, w = torch.randn(M, K, generator=g), torch.randn(N, K, generator=g) * 0.05
    bias, res = torch.randn(N, generator=g), torch.randn(M, N, generator=g)
    if dtype == "tf32":
        a, w = G.tf32_round_ref(a), G.tf32_round_ref(w)
        if (K * 4) % 16:
            pytest.skip("leading dimension must be a multiple of 16 bytes")
        out = G.ops.gemm(a.cuda(), w.cuda(), bias.cuda(), res.cuda(), cta_pair=1)
    else:
        a, w = a.half(), w.half()
        if (K * 2) % 16:
            pytest.skip("leading dimension must be a multiple of 16 bytes")
        out = G.ops.gemm(a.cuda(), w.cuda(), bias.cuda(), res.cuda(), dtype=G.ops.F16, cta_pair=1)
    torch.cuda.synchronize()
    assert G.relerr(out, _ref(a.float(), w.float(), bias, res)) < 2e-5


def test_gemm_cta_pair_persistent_and_taps(G):
    g = torch.Generator().manual_seed(11)
    M, N, K = 3000, 1024, 512
    a = torch.randn(M, K, generator=g).half()
    w = (torch.randn(N, K, generator=g) * 0.05).half()
    bias = torch.randn(N, generator=g)
    ref = _ref(a.float(), w.float(), bias, gelu=True)
    out = G.ops.gemm(a.cuda(), w.cuda(), bias.cuda(), dtype=G.ops.F16, gelu=True, cta_pair=1, max_ctas=6)  # 3 pairs, many tiles each
    assert G.relerr(out, ref) < 2e-5
    rows, C, Nn = 7 * 60, 64, 96
    a = G.tf32_round_ref(torch.randn(rows, C, generator=g))
    w = G.tf32_round_ref(torch.randn(Nn, 3 * C, generator=g) * 0.1)
    out = G.ops.gemm(a.cuda(), w.cuda(), taps=[-7, 0, 7], cta_pair=1)
    assert G.relerr(out, _ref(a, w, taps=[-7, 0, 7])) < 2e-5
    Bt = 3
    a = G.tf32_round_ref(torch.randn(Bt, 265, 512, generator=g)); w = G.tf32_round_ref(torch.randn(Bt, 265, 512, generator=g))
    out = G.ops.gemm(a.cuda(), w.cuda(), alpha=0.5, cta_pair=1)
    assert G.relerr(out, 0.5 * torch.einsum("bmk,bnk->bmn", a.double(), w.double())) < 2e-5


def test_gemm_epilogues_and_persistence(G):
    g = torch.Generator().manual_seed(1)
    M, N, K = 2000, 1024, 512
    a = G.tf32_round_ref(torch.randn(M, K, generator=g))
    w = G.tf32_round_ref(torch.randn(N, K, generator=g) * 0.05)
    bias, res = torch.randn(N, generator=g), torch.randn(M, N, generator=g)
    ref = _ref(a, w, bias, res, gelu=True)
    # max_ctas=5 forces many tiles per CTA: exercises the smem ring wrap across tiles
    out = G.ops.gemm(a.cuda(), w.cuda(), bias.cuda(), res.cuda(), gelu=True, max_ctas=5)
    assert G.relerr(out, ref) < 2e-5
    # in-place residual (x += proj(y)) and tf32-rounded output
    x = res.cuda().clone()
    G.ops.gemm(a.cuda(), w.cuda(), bias.cuda(), x, out=x)
    assert G.relerr(x, _ref(a, w, bias, res)) < 2e-5
    out = G.ops.gemm(a.cuda(), w.cuda(), bias.cuda(), round_out=True)
    assert torch.equal(out.cpu(), G.tf32_round_ref(G.ops.gemm(a.cuda(), w.cuda(), bias.cuda()).cpu()))


def _out_view(M, N, pad, dtype):
    """A sentinel-filled (M, N + pad) buffer and its (M, N) view: the GEMM writes the view with ldo = N + pad."""
    buf = torch.full((M, N + pad), 7.0, dtype=dtype, device="cuda")
    return buf, buf[:, :N]


def _residual_view(M, N, pad, g):
    """None, or an (M, N) residual view of an (M, N + pad) buffer: ld_res = N + pad."""
    return None if pad is None else torch.randn(M, N + pad, generator=g).cuda()[:, :N]


def _assert_rounded(out, ref, u):
    """Every element within the output type's rounding (u: half an ulp, relative) of the fp64 value, on top of the fp32 result's own 2e-5."""
    ref = ref.double().cpu()
    err = (out.double().cpu() - ref).abs()
    assert bool((err <= u * ref.abs() + 2e-5 * float(ref.abs().max())).all())


def _check_2byte_gemm(G, dt, M, N, K, ldo_pad=0, res_pad=None):
    """A bf16 GEMM (no bias) or an f16 GEMM (bias + GELU2) with fp32 and 2-byte outputs, vs fp64: the fp32 output within 2e-5, the 2-byte output
    within its type's rounding of the fp64 value, and columns beyond N of a wider output row untouched."""
    f16 = dt == "f16"
    g = torch.Generator().manual_seed(3 if f16 else 2)
    a = torch.randn(M, K, generator=g).to(torch.float16 if f16 else torch.bfloat16)
    w = (torch.randn(N, K, generator=g) * 0.05).to(a.dtype)
    bias = torch.randn(N, generator=g) if f16 else None
    res = _residual_view(M, N, res_pad, g)
    ref = _ref(a.float(), w.float(), bias, None if res is None else res.cpu(), gelu=f16)
    kw = dict(dtype=G.ops.F16 if f16 else G.ops.BF16, gelu=f16)
    bc = None if bias is None else bias.cuda()
    buf, out = _out_view(M, N, ldo_pad, torch.float32)
    G.ops.gemm(a.cuda(), w.cuda(), bc, res, out=out, **kw)
    assert G.relerr(out, ref) < 2e-5
    bufh, outh = _out_view(M, N, ldo_pad, a.dtype)
    G.ops.gemm(a.cuda(), w.cuda(), bc, res, out=outh, **kw)
    assert outh.dtype == a.dtype and G.relerr(outh.float(), ref) < (1e-3 if f16 else 5e-3)
    _assert_rounded(outh, ref, 2.0 ** (-11 if f16 else -8))
    for b in (buf, bufh):
        assert torch.equal(b[:, N:], torch.full_like(b[:, N:], 7.0))


def test_gemm_bf16(G):
    _check_2byte_gemm(G, "bf16", 777, 512, 1024)


def test_gemm_f16(G):
    _check_2byte_gemm(G, "f16", 4240, 1024, 1024)


# the layouts that take the scalar epilogue: an N tail (33, 100), an output view with ldo = N + 2, a residual view with ld_res = N + 1
@pytest.mark.parametrize("M,N,K,ldo_pad,res_pad", [(300, 33, 128, 0, None), (300, 100, 256, 0, None), (300, 128, 128, 2, None), (300, 128, 128, 0, 1)])
@pytest.mark.parametrize("dt", ["bf16", "f16"])
def test_gemm_2byte_scalar_epilogue(G, dt, M, N, K, ldo_pad, res_pad):
    _check_2byte_gemm(G, dt, M, N, K, ldo_pad, res_pad)


def test_gemm_activation_flags(G):
    g = torch.Generator().manual_seed(6)
    M, N, K = 300, 64, 96
    a = G.tf32_round_ref(torch.randn(M, K, generator=g))
    w = G.tf32_round_ref(torch.randn(N, K, generator=g) * 0.2)
    bias, res = torch.randn(N, generator=g), torch.randn(M, N, generator=g)
    y = a.double() @ w.double().T + bias.double()
    out = G.ops.gemm(a.cuda(), w.cuda(), bias.cuda(), res.cuda(), lrelu=True)
    assert G.relerr(out, torch.nn.functional.leaky_relu(y, 0.2) + res.double()) < 2e-5
    out = G.ops.gemm(a.cuda(), w.cuda(), bias.cuda(), res.cuda(), lrelu=True, res_before_act=True)
    assert G.relerr(out, torch.nn.functional.leaky_relu(y + res.double(), 0.2)) < 2e-5
    out = G.ops.gemm(a.cuda(), w.cuda(), bias.cuda(), tanh=True)
    assert G.relerr(out, torch.tanh(y)) < 2e-5


def test_gemm_taps_and_row_mask(G):
    """3 taps with row shifts (-7, 0, +7) and a zero-border mask: the implicit-GEMM form used by the conv layers."""
    g = torch.Generator().manual_seed(4)
    rows, C, N = 7 * 30, 64, 96
    a = G.tf32_round_ref(torch.randn(rows, C, generator=g))
    w = G.tf32_round_ref(torch.randn(N, 3 * C, generator=g) * 0.1)
    taps = [-7, 0, 7]
    ref = _ref(a, w, taps=taps)
    out = G.ops.gemm(a.cuda(), w.cuda(), taps=taps)
    assert G.relerr(out, ref) < 2e-5
    geo = (7 * 10, 7, 1, 9, 1, 6)  # images of 10x7 rows, interior y in [1,9), x in [1,6)
    out = G.ops.gemm(a.cuda(), w.cuda(), taps=taps, geo=geo).cpu()
    r = torch.arange(rows)
    y, x = (r % 70) // 7, r % 7
    inside = (y >= 1) & (y < 9) & (x >= 1) & (x < 6)
    assert float(out[~inside].abs().max()) == 0.0
    assert G.relerr(out[inside], ref[inside]) < 2e-5


def test_gemm_batched(G):
    g = torch.Generator().manual_seed(5)
    Bt, M, N, K = 3, 265, 265, 512
    a = G.tf32_round_ref(torch.randn(Bt, M, K, generator=g))
    w = G.tf32_round_ref(torch.randn(Bt, N, K, generator=g))
    out = G.ops.gemm(a.cuda(), w.cuda(), alpha=0.5)
    ref = 0.5 * torch.einsum("bmk,bnk->bmn", a.double(), w.double())
    assert G.relerr(out, ref) < 2e-5


def test_gemm_split_tf32_recovers_fp32_accuracy(G):
    """3-pass split-TF32 (hi*Whi + lo*Whi + hi*Wlo) with taps: error ~1e-6 where single-pass TF32 gives ~5e-4."""
    g = torch.Generator().manual_seed(8)
    rows, C, N = 7 * 30, 80, 96          # C = 80 exercises the padding to Cp = 96
    a = torch.randn(rows, C, generator=g) * torch.logspace(-2, 2, C)   # wide dynamic range
    w = torch.randn(N, 3 * C, generator=g) * 0.1
    taps = [-7, 0, 7]
    ref = _ref(a, w, taps=taps)
    asp = G.ops.split_tf32(a.cuda())
    wsp = G.ops.pack_split_weight(w.cuda(), 3)
    out = G.ops.gemm_split(asp, wsp, taps=taps)
    e3 = G.relerr(out, ref)
    e1 = G.relerr(G.ops.gemm(G.ops.round_tf32(a.cuda()), G.ops.round_tf32(w.cuda()), taps=taps), ref)
    print("split-tf32 err", e3, "single tf32 err", e1)
    assert e3 < 5e-6 and e1 > 10 * e3
    # weight-format split of an activation (attention K / V^T operands), batched
    q = torch.randn(2, 40, 64, generator=g); k = torch.randn(2, 48, 64, generator=g)
    s = G.ops.gemm_split(G.ops.split_tf32(q.cuda()), G.ops.split_tf32(k.cuda(), w_format=True), alpha=0.125)
    assert G.relerr(s, 0.125 * torch.einsum("bmk,bnk->bmn", q.double(), k.double())) < 5e-6


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("M,N,K", [(128, 128, 64), (256, 512, 200), (1024, 1024, 5300), (4096, 1024, 795), (77, 64, 265), (265, 64, 77), (96, 200, 130)])
def test_gemm_mn_major_operands(G, dt, M, N, K):
    """Operands as they lie in memory with the reduction dimension as ROWS (weight-gradient / P^T dO shapes): out = a^T w, a^T w_k, a w."""
    g = torch.Generator().manual_seed(M * 7 + N * 3 + K)
    code = G.ops.BF16 if dt == torch.bfloat16 else G.ops.F16
    ld_a, ld_w = (M + 7) // 8 * 8 + 8, (N + 7) // 8 * 8 + 16  # padded leading dimensions: garbage beyond the extents must never be read
    a_store = torch.full((K, ld_a), float("nan")).to(dt)
    w_store = torch.full((K, ld_w), float("nan")).to(dt)
    a_store[:, :M] = torch.randn(K, M, generator=g).to(dt)
    w_store[:, :N] = (torch.randn(K, N, generator=g) * 0.1).to(dt)
    a_km, w_km = a_store.cuda()[:, :M], w_store.cuda()[:, :N]            # (K, M), (K, N) row-strided views of the padded buffers
    ref = a_store[:, :M].double().T @ w_store[:, :N].double()
    out = G.ops.gemm(a_km, w_km, dtype=code, a_mn=True, w_mn=True)
    assert out.shape == (M, N) and G.relerr(out, ref) < 2e-5
    # mixed: A K-major (M, K) with W MN-major (K, N), and A MN-major with W K-major (N, K)
    a_rm = a_store[:, :M].T.contiguous().cuda()
    w_rm = w_store[:, :N].T.contiguous().cuda()
    if K % 8 == 0:
        assert G.relerr(G.ops.gemm(a_rm, w_km, dtype=code, w_mn=True), ref) < 2e-5
        assert G.relerr(G.ops.gemm(a_km, w_rm, dtype=code, a_mn=True), ref) < 2e-5
    bias = torch.randn(N, generator=g)
    outb = G.ops.gemm(a_km, w_km, bias.cuda(), dtype=code, a_mn=True, w_mn=True, alpha=0.5, block_n=128)
    assert G.relerr(outb, 0.5 * ref + bias.double()) < 2e-5


def test_gemm_mn_major_batched(G):
    g = torch.Generator().manual_seed(11)
    Bt, Lq, Lk = 5, 265, 77
    P = torch.rand(Bt, Lq, 80, generator=g).bfloat16()       # (Lq rows = reduction, Lk columns) inside an 80-wide buffer
    dO = torch.randn(Bt, Lq, 64, generator=g).bfloat16()
    Pc = P.cuda()[:, :, :Lk]
    out = G.ops.gemm(Pc, dO.cuda(), dtype=G.ops.BF16, a_mn=True, w_mn=True)   # dV = P^T dO
    ref = torch.einsum("bqk,bqd->bkd", P[:, :, :Lk].double(), dO.double())
    assert out.shape == (Bt, Lk, 64) and G.relerr(out, ref) < 2e-5
    V = torch.randn(Bt, Lk, 64, generator=g).bfloat16()
    out2 = G.ops.gemm(Pc, V.cuda(), dtype=G.ops.BF16, w_mn=True)             # O = P V with V as stored
    assert G.relerr(out2, torch.einsum("bqk,bkd->bqd", P[:, :, :Lk].double(), V.double())) < 2e-5
