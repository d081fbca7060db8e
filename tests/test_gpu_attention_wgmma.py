"""The wgmma split-fp16 attention (csrc/attention_tc_split.cu) against fp64: the edges of its 64-row query tiles and 64-key chunks, more
(batch, head, tile pair) units than CTAs, the engine's packed buffers, large scores, the rows it must not write, and run-to-run bits."""
import itertools

import pytest
import torch

pytestmark = pytest.mark.gpu

LQ = [1, 9, 63, 64, 65, 128, 265]
LK = [1, 8, 9, 16, 63, 64, 65, 77, 265, 288]


@pytest.fixture(scope="module")
def ops():
    from tests import gpu_common
    return gpu_common.ops


def _pair(p, C):
    return p[:, :C].double() + p[:, C:2 * C].double()


def _heads(x, B, L, H):
    return x.view(B, L, H, 64).permute(0, 2, 1, 3)


def _ref(q, k, v, B, H, Lq, Lk):
    """fp64 softmax(Q K^T / 8) V of fp64 (B*L, H*64) matrices."""
    s = _heads(q, B, Lq, H) @ _heads(k, B, Lk, H).transpose(-1, -2) * 0.125
    return (torch.softmax(s, -1) @ _heads(v, B, Lk, H)).permute(0, 2, 1, 3).reshape(B * Lq, H * 64)


def _run(ops, B, H, Lq, Lk, qs=1.5, ks=1.5, g=None):
    D = H * 64
    q = torch.randn(B * Lq, D, device="cuda", generator=g) * qs
    k = torch.randn(B * Lk, D, device="cuda", generator=g) * ks
    v = torch.randn(B * Lk, D, device="cuda", generator=g)
    qp, kp, vp = ops.split_f16(q), ops.split_f16(k), ops.split_f16(v)
    out = torch.full((B * Lq, 2 * D), float("nan"), dtype=torch.float16, device="cuda")
    ops.attention_tc_split(qp[:, :D], kp[:, :D], vp[:, :D], out[:, :D], q_lo=D, k_lo=D, v_lo=D, o_lo=D, B=B, H=H, Lq=Lq, Lk=Lk, scale=0.125)
    return out, _ref(_pair(qp, D), _pair(kp, D), _pair(vp, D), B, H, Lq, Lk)


def _check(out, ref, D, tol=3e-6):
    got = _pair(out, D)
    assert torch.isfinite(got).all()
    err = float((got - ref).abs().max() / ref.abs().max())
    assert err < tol, err


@pytest.mark.parametrize("Lq,Lk", list(itertools.product(LQ, LK)))
def test_tile_and_chunk_edges(ops, Lq, Lk):
    """Every query-tile edge (one row, a partial tile, 64 / 65 rows, an odd last tile) against every key-chunk edge (one key, partial and
    exact chunks, the bench's 77 and 265, 288)."""
    g = torch.Generator(device="cuda").manual_seed(Lq * 1000 + Lk)
    out, ref = _run(ops, 2, 2, Lq, Lk, g=g)
    _check(out, ref, 128)


def test_long_key_sequence(ops):
    """Keys stream through the ring chunk by chunk: no limit on Lk from shared memory."""
    out, ref = _run(ops, 2, 3, 130, 700, g=torch.Generator(device="cuda").manual_seed(7))
    _check(out, ref, 192)


@pytest.mark.parametrize("B,H,Lq,Lk", [(37, 5, 265, 265), (64, 16, 265, 77)])
def test_more_units_than_ctas(ops, B, H, Lq, Lk):
    out, ref = _run(ops, B, H, Lq, Lk, g=torch.Generator(device="cuda").manual_seed(B))
    _check(out, ref, H * 64)


def test_engine_packed_views(ops):
    """The engine's calls: self-attention off qkv = [Qh Kh Vh | Ql Kl Vl] (lo at 3D) and cross-attention of q2 = [Qh | Ql] against the
    last layer's K / V columns of kv_all = [every layer's Kh Vh | every layer's Kl Vl] (lo at n_layer * 2D)."""
    B, H, L, Lc, NL = 3, 16, 265, 77, 19
    D = H * 64
    g = torch.Generator(device="cuda").manual_seed(11)
    qkv = ops.split_f16(torch.randn(B * L, 3 * D, device="cuda", generator=g))
    att = torch.full((B * L, 2 * D), float("nan"), dtype=torch.float16, device="cuda")
    ops.attention_tc_split(qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:3 * D], att[:, :D], q_lo=3 * D, k_lo=3 * D, v_lo=3 * D, o_lo=D, B=B, H=H, Lq=L, Lk=L,
                           scale=0.125)
    full = _pair(qkv, 3 * D)
    _check(att, _ref(full[:, :D], full[:, D:2 * D], full[:, 2 * D:], B, H, L, L), D)

    q2 = ops.split_f16(torch.randn(B * L, D, device="cuda", generator=g))
    kv_all = ops.split_f16(torch.randn(B * Lc, NL * 2 * D, device="cuda", generator=g))
    li = NL - 1
    kv = kv_all[:, li * 2 * D:]
    ops.attention_tc_split(q2[:, :D], kv[:, :D], kv[:, D:2 * D], att[:, :D], q_lo=D, k_lo=NL * 2 * D, v_lo=NL * 2 * D, o_lo=D, B=B, H=H, Lq=L, Lk=Lc,
                           scale=0.125)
    kvd = _pair(kv_all, NL * 2 * D)[:, li * 2 * D:(li + 1) * 2 * D]
    _check(att, _ref(_pair(q2, D), kvd[:, :D], kvd[:, D:], B, H, L, Lc), D)


def test_scores_of_forty(ops):
    """Scaled scores of +40 and -40: every query row is +-5 times one key row of +-1 entries, so Q K^T is exact in fp32 and the check
    is on the softmax and P V alone."""
    B, H, Lq, Lk = 2, 4, 265, 265
    D = H * 64
    g = torch.Generator(device="cuda").manual_seed(40)
    k = torch.randint(0, 2, (B * Lk, D), device="cuda", generator=g).float() * 2 - 1
    pick = torch.randint(0, Lk, (B, Lq), device="cuda", generator=g) + torch.arange(B, device="cuda")[:, None] * Lk
    sign = torch.randint(0, 2, (B * Lq, 1), device="cuda", generator=g).float() * 2 - 1
    q = 5.0 * sign * k[pick.reshape(-1)]
    v = torch.randn(B * Lk, D, device="cuda", generator=g)
    qp, kp, vp = ops.split_f16(q), ops.split_f16(k), ops.split_f16(v)
    out = torch.full((B * Lq, 2 * D), float("nan"), dtype=torch.float16, device="cuda")
    ops.attention_tc_split(qp[:, :D], kp[:, :D], vp[:, :D], out[:, :D], q_lo=D, k_lo=D, v_lo=D, o_lo=D, B=B, H=H, Lq=Lq, Lk=Lk, scale=0.125)
    qd, kd = _pair(qp, D), _pair(kp, D)
    s = _heads(qd, B, Lq, H) @ _heads(kd, B, Lk, H).transpose(-1, -2) * 0.125
    assert float(s.max()) == 40.0 and float(s.min()) == -40.0
    _check(out, _ref(qd, kd, _pair(vp, D), B, H, Lq, Lk), D)


def test_leaves_other_rows_and_columns_alone(ops):
    """The output view is rows [0, B*Lq) and head columns of a wider NaN-filled buffer: nothing outside it changes, though the last query
    tile of every head runs 64 rows."""
    B, H, Lq, Lk = 3, 2, 65, 77
    D = H * 64
    g = torch.Generator(device="cuda").manual_seed(3)
    q = ops.split_f16(torch.randn(B * Lq, D, device="cuda", generator=g))
    k = ops.split_f16(torch.randn(B * Lk, D, device="cuda", generator=g))
    v = ops.split_f16(torch.randn(B * Lk, D, device="cuda", generator=g))
    buf = torch.full((B * Lq + 70, 2 * D + 64), float("nan"), dtype=torch.float16, device="cuda")
    ops.attention_tc_split(q[:, :D], k[:, :D], v[:, :D], buf[:, :D], q_lo=D, k_lo=D, v_lo=D, o_lo=D + 32, B=B, H=H, Lq=Lq, Lk=Lk, scale=0.125)
    assert torch.isnan(buf[B * Lq:]).all()
    assert torch.isnan(buf[:B * Lq, D:D + 32]).all() and torch.isnan(buf[:B * Lq, 2 * D + 32:]).all()
    got = buf[:B * Lq, :D].double() + buf[:B * Lq, D + 32:2 * D + 32].double()
    ref = _ref(_pair(q, D), _pair(k, D), _pair(v, D), B, H, Lq, Lk)
    assert float((got - ref).abs().max() / ref.abs().max()) < 3e-6


def test_same_bits_every_launch_and_in_a_graph(ops):
    B, H, L = 4, 16, 265
    D = H * 64
    g = torch.Generator(device="cuda").manual_seed(5)
    qkv = ops.split_f16(torch.randn(B * L, 3 * D, device="cuda", generator=g))
    outs = [torch.zeros(B * L, 2 * D, dtype=torch.float16, device="cuda") for _ in range(3)]

    def run(o):
        ops.attention_tc_split(qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:3 * D], o[:, :D], q_lo=3 * D, k_lo=3 * D, v_lo=3 * D, o_lo=D, B=B, H=H, Lq=L,
                               Lk=L, scale=0.125)

    run(outs[0])
    run(outs[1])
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        run(outs[2])
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])
