"""Ordered stream-K in the wgmma GEMM keeps every output bit: each case runs once with the automatic schedule (stream-K wherever the tiles leave a
partial last wave) and once forced data-parallel (schedule=1), and the two outputs must be identical as integers.  Every case here has a partial last
wave; all but qkv and mlp1 (three waves or more, which stay data-parallel) run under three waves, so the automatic schedule does split tiles
between neighbouring CTAs."""
import pytest
import torch

pytestmark = pytest.mark.gpu

M_DENOISER = 16 * 265  # the denoiser's token rows at batch 16: tiles_m = 34


@pytest.fixture(scope="module")
def ops():
    from tests import gpu_common
    return gpu_common.ops


def _same_bits(x, y):
    itype = {4: torch.int32, 2: torch.int16}[x.element_size()]
    assert x.shape == y.shape
    xi, yi = x.contiguous().view(itype), y.contiguous().view(itype)
    n_diff = int((xi != yi).sum())
    assert n_diff == 0, f"{n_diff} of {x.numel()} elements differ between the stream-K and data-parallel schedules"


def _both(run):
    """run(schedule) -> output tensor (a fresh one per call); returns (auto, data-parallel)."""
    a = run(0).clone()
    d = run(1).clone()
    torch.cuda.synchronize()
    return a, d


def _pair(ops, rows, cols, g, std=1.0):
    return ops.split_f16((torch.randn(rows, cols, generator=g) * std).cuda())


# (name, N, K, split_out, gelu, in-place residual): the six split-fp16 GEMMs of a denoiser layer
DENOISER = [("qkv", 3072, 1024, True, False, False), ("proj1", 1024, 1024, False, False, True), ("q2", 1024, 1024, True, False, False),
            ("proj2", 1024, 1024, False, False, True), ("mlp1", 4096, 1024, True, True, False), ("mlp2", 1024, 4096, False, False, True)]


@pytest.mark.parametrize("name,N,K,split_out,gelu,residual", DENOISER, ids=[d[0] for d in DENOISER])
def test_denoiser_f16x3_shapes(ops, name, N, K, split_out, gelu, residual):
    g = torch.Generator().manual_seed(N + K)
    a = _pair(ops, M_DENOISER, K, g, 0.5)
    w = _pair(ops, N, K, g, K ** -0.5)
    bias = (torch.randn(N, generator=g) * 0.1).cuda()
    x0 = torch.randn(M_DENOISER, N, generator=g).cuda()

    def run(schedule):
        if residual:  # proj / mlp2: out = x + (a W^T + b), in place on the fp32 stream
            x = x0.clone()
            return ops.gemm_f16x3(a, w, bias, residual=x, out=x, schedule=schedule)
        return ops.gemm_f16x3(a, w, bias, gelu=gelu, split_out=split_out, schedule=schedule)

    auto, dp = _both(run)
    _same_bits(auto, dp)
    assert torch.isfinite(auto.float()).all() and auto.float().abs().max() > 0


def test_decoder_9tap_f16x3_conv(ops):
    # a SpecVQGAN 3x3 conv as implicit GEMM over a zero-bordered channels-last image: 9 spatial taps x (lo*hi, hi*lo, hi*hi), border rows masked
    B, H, W_, C, N = 2, 62, 82, 128, 256
    Hp, Wp = H + 2, W_ + 2
    M = B * Hp * Wp  # 10752 rows: 84 x 2 = 168 tiles
    g = torch.Generator().manual_seed(9)
    img = torch.zeros(B, Hp, Wp, C)
    img[:, 1:H + 1, 1:W_ + 1] = torch.randn(B, H, W_, C, generator=g)
    a = ops.split_f16(img.view(M, C).cuda())
    # W row n = [tap 0 hi | tap 0 lo | tap 1 hi | tap 1 lo | ...]
    w = ops.split_f16((torch.randn(N * 9, C, generator=g) * (9 * C) ** -0.5).cuda()).view(N, 18 * C)
    shifts, acol, wcol = [], [], []
    for j, (dy, dx) in enumerate((dy, dx) for dy in (-1, 0, 1) for dx in (-1, 0, 1)):
        s = dy * Wp + dx
        shifts += [s, s, s]
        acol += [C, 0, 0]
        wcol += [2 * C * j, 2 * C * j + C, 2 * C * j]
    bias = (torch.randn(N, generator=g) * 0.1).cuda()
    geo = (Hp * Wp, Wp, 1, H + 1, 1, W_ + 1)

    def run(schedule):
        out = torch.empty(M, 2 * N, dtype=torch.float16, device="cuda")
        return ops.gemm(a, w, bias, out=out, dtype=ops.F16, taps=shifts, tap_acol=acol, tap_wcol=wcol, k_per_tap=C, geo=geo, split_out=True, schedule=schedule)

    auto, dp = _both(run)
    _same_bits(auto, dp)


def test_vocoder_resident_w_conv(ops):
    # MelGAN's narrow-channel conv form: seven 64-deep fp16 taps, N <= 128 (one 128-wide tile column, tiles_m > SM count)
    T, C, N, KT = 40000, 64, 64, 7
    g = torch.Generator().manual_seed(7)
    a = torch.randn(T, C, generator=g).half().cuda()
    w = (torch.randn(N, KT * C, generator=g) * (KT * C) ** -0.5).half().cuda()
    bias = (torch.randn(N, generator=g) * 0.1).cuda()
    taps = [(j - KT // 2, 0, j * C, 0) for j in range(KT)]

    def run(schedule):
        out = torch.empty(T, N, device="cuda")
        ops.gemm_desc(A=a.data_ptr(), W=w.data_ptr(), out=out.data_ptr(), M=T, N=N, K=C, taps=taps, lda=C, ldw=KT * C, ldo=N, a_rows=T, a_cols=C,
                      w_cols=KT * C, bias=bias, flags=ops.LRELU, resident_w=1, schedule=schedule)
        return out

    auto, dp = _both(run)
    _same_bits(auto, dp)


@pytest.mark.parametrize("dt,M,N,K,bn", [("bf16", M_DENOISER, 1024, 1024, 0), ("tf32", M_DENOISER, 1024, 1024, 0), ("bf16", M_DENOISER, 2048, 512, 256),
                                         ("tf32", M_DENOISER, 1536, 768, 256), ("f16", 3000, 700, 200, 128)])
def test_single_pass_dtypes(ops, dt, M, N, K, bn):
    g = torch.Generator().manual_seed(M + N + K)
    tdt = {"bf16": torch.bfloat16, "f16": torch.float16, "tf32": torch.float32}[dt]
    kind = {"bf16": ops.BF16, "f16": ops.F16, "tf32": ops.TF32}[dt]
    a = torch.randn(M, K, generator=g).to(tdt).cuda()
    w = (torch.randn(N, K, generator=g) * K ** -0.5).to(tdt).cuda()
    bias = torch.randn(N, generator=g).cuda()
    res = torch.randn(M, N, generator=g).cuda()
    auto, dp = _both(lambda s: ops.gemm(a, w, bias, res, dtype=kind, block_n=bn, schedule=s))
    _same_bits(auto, dp)


@pytest.mark.parametrize("a_mn,w_mn", [(False, True), (True, True)], ids=["dgrad", "wgrad"])
def test_mn_major_operands(ops, a_mn, w_mn):
    # training: dX = dY W with W (out, in) as stored (W MN-major); dW = dY^T X with both operands token-major
    g = torch.Generator().manual_seed(5)
    if a_mn:
        Kr, M, N = 4240, 2048, 2048
        a = torch.randn(Kr, M, generator=g).bfloat16().cuda()
    else:
        Kr, M, N = 1024, M_DENOISER, 1024
        a = torch.randn(M, Kr, generator=g).bfloat16().cuda()
    w = (torch.randn(Kr, N, generator=g) * Kr ** -0.5).bfloat16().cuda()
    auto, dp = _both(lambda s: ops.gemm(a, w, dtype=ops.BF16, a_mn=a_mn, w_mn=True, out_bf16=True, block_n=128, schedule=s))
    _same_bits(auto, dp)


def test_batched(ops):
    g = torch.Generator().manual_seed(3)
    a = torch.randn(3, 1000, 512, generator=g).bfloat16().cuda()  # 8 x 8 x 3 = 192 tiles
    w = (torch.randn(1024, 512, generator=g) * 512 ** -0.5).bfloat16().cuda()
    auto, dp = _both(lambda s: ops.gemm(a, w, dtype=ops.BF16, gelu=True, block_n=128, schedule=s))
    _same_bits(auto, dp)


def test_amax_out(ops):
    g = torch.Generator().manual_seed(11)
    M, N, K = M_DENOISER, 512, 1024
    a = torch.randn(M, K, generator=g).half().cuda()
    w = (torch.randn(N, K, generator=g) * K ** -0.5).half().cuda()
    res = {}
    for s in (0, 1):
        out = torch.empty(M, N, device="cuda")
        amax = torch.zeros(1, device="cuda")
        ops.gemm_desc(A=a.data_ptr(), W=w.data_ptr(), out=out.data_ptr(), M=M, N=N, K=K, taps=[(0, 0, 0, 0)], lda=K, ldw=K, ldo=N, a_rows=M, a_cols=K,
                      w_cols=K, flags=ops.TANH, amax_out=amax, block_n=128, schedule=s)
        res[s] = (out, amax)
    torch.cuda.synchronize()
    _same_bits(res[0][0], res[1][0])
    _same_bits(res[0][1], res[1][1])
    assert float(res[0][1]) == float(res[0][0].abs().max())


@pytest.mark.parametrize("M,N,K,max_ctas", [(M_DENOISER, 512, 1024, 0), (M_DENOISER, 512, 1024, 131), (M_DENOISER, 512, 4096, 120),
                                             (133 * 128, 128, 1024, 0), (133 * 128, 128, 4096, 0), (133 * 128, 128, 128, 0)])
def test_tiny_heads_and_tails(ops, M, N, K, max_ctas):
    # a grid just below the tile count (136 or 133 tiles): each CTA owns barely more than one tile's k-blocks, so heads and tails of a single
    # k-block occur, and with K = 128 every split tile is cut after its first of two k-blocks
    g = torch.Generator().manual_seed(M + K + max_ctas)
    a = _pair(ops, M, K, g, 0.5)
    w = _pair(ops, N, K, g, K ** -0.5)
    x0 = torch.randn(M, N, generator=g).cuda()

    def run(schedule):
        x = x0.clone()
        return ops.gemm_f16x3(a, w, None, residual=x, out=x, max_ctas=max_ctas, schedule=schedule)

    auto, dp = _both(run)
    _same_bits(auto, dp)


def test_graph_replays_reset_the_workspace(ops):
    # two stream-K launches and their data-parallel twins captured into one CUDA graph, replayed twice: every replay must find the flags clear
    g = torch.Generator().manual_seed(2)
    N, K = 1024, 1024
    a = _pair(ops, M_DENOISER, K, g, 0.5)
    w = _pair(ops, N, K, g, K ** -0.5)
    w2 = _pair(ops, 3 * N, K, g, K ** -0.5)
    bias = (torch.randn(N, generator=g) * 0.1).cuda()
    outs = [torch.empty(M_DENOISER, N, device="cuda") for _ in range(2)] + [torch.empty(M_DENOISER, 6 * N, dtype=torch.float16, device="cuda") for _ in range(2)]

    def seq():
        for s in (0, 1):
            ops.gemm_f16x3(a, w, bias, out=outs[s], schedule=s)
            ops.gemm_f16x3(a, w2, None, split_out=True, out=outs[2 + s], schedule=s)

    seq()  # eager first: lazy set-up (kernel attributes, the stream-K workspace) stays out of the capture
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        seq()
    for _ in range(2):
        for o in outs:
            o.fill_(float("nan"))
        graph.replay()
        torch.cuda.synchronize()
        _same_bits(outs[0], outs[1])
        _same_bits(outs[2], outs[3])
        assert torch.isfinite(outs[0]).all() and torch.isfinite(outs[2]).all()
