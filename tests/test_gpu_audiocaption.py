"""ACT audio captioning on the GPU: the new kernels per element against fp64, the encoder memory against the fp64 oracle, greedy and beam ids
against the reference's fixtures, graph replay, batch invariance and untouched sentinels."""
import math
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests.test_cpu_audiocaption import CASES, EOS, SOS, V, config, fixture_mels  # noqa: E402
import _pkg  # noqa: E402

_pkg.load()
from diffsound_b200 import ops  # noqa: E402
from diffsound_b200.evaluation.audiocaption import ACT, beam_decode, greedy_decode  # noqa: E402
from oracle import act_oracle as O  # noqa: E402

pytestmark = pytest.mark.gpu
dev = "cuda"
EPS32 = 2.0 ** -24
SENT = -7777.0


def unpair(p, D):
    return p[:, :D].double() + p[:, D:2 * D].double()


def attend64(q, K, Vv, scale):
    s = (K @ q) * scale
    p = torch.softmax(s, 0)
    return p @ Vv, p


def attn_bound(q, K, Vv, n):
    """fp32 steps: dot products over 64 terms, exp / sum over n, P.V over n terms, then the fp16 pair (2^-22 relative)."""
    vmax = float(Vv.abs().max()) if Vv.numel() else 0.0
    smax = float(q.abs().sum() * K.abs().max()) * 0.125
    return vmax * (6 * 64 * EPS32 * smax + (n + 8) * 4 * EPS32) + vmax * 2.0 ** -21


@pytest.mark.parametrize("Lm", [1, 64, 213, 216])
def test_cross_attention_vs_fp64(Lm):
    B, H, D, R = 5, 8, 512, 3
    kv = torch.randn(B * Lm, 2 * D, device=dev)
    q = torch.randn(R, D, device=dev)
    clips = torch.tensor([4, 0, 2], dtype=torch.int32, device=dev)  # a subset of the clips, out of order
    out = torch.full((R + 1, 2 * D), SENT, dtype=torch.float16, device=dev)
    ops.caption_cross_attention(q, kv, clips, out, R=R, H=H, Lm=Lm, v_off=D, scale=0.125)
    o = unpair(out[:R], D).cpu()
    for r in range(R):
        c = int(clips[r])
        for h in range(H):
            sl = slice(64 * h, 64 * h + 64)
            K = kv[c * Lm:(c + 1) * Lm, sl].double().cpu()
            Vv = kv[c * Lm:(c + 1) * Lm, D + 64 * h:D + 64 * h + 64].double().cpu()
            want, _ = attend64(q[r, sl].double().cpu(), K, Vv, 0.125)
            assert float((o[r, sl] - want).abs().max()) <= attn_bound(q[r, sl].double().cpu(), K, Vv, Lm)
    assert bool((out[R] == SENT).all())


def test_tree_attention_vs_fp64():
    """Rows with paths of 1 ... 2001 slots; rows 2 and 3 share a prefix; slots scattered over the pool."""
    H, D = 8, 512
    lens = [1, 2, 63, 64, 65, 513, 2001]
    n_slots = 6000
    g = torch.Generator().manual_seed(1)
    perm = torch.randperm(n_slots, generator=g)
    paths, used = [], 0
    for i, n in enumerate(lens):
        if i == 3:  # share the first 60 slots of row 2's path
            p = torch.cat([paths[2][:60], perm[used:used + n - 60]])
            used += n - 60
        else:
            p = perm[used:used + n]
            used += n
        paths.append(p)
    kp = torch.randn(n_slots, D, device=dev)
    vp = torch.randn(n_slots, D, device=dev)
    R = len(lens)
    qkv = torch.randn(R, 3 * D, device=dev)
    kp0, vp0 = kp.clone(), vp.clone()
    flat = torch.cat(paths).to(torch.int32).to(dev)
    start = torch.tensor(np.concatenate([[0], np.cumsum(lens)[:-1]]), dtype=torch.int64, device=dev)
    pos = torch.tensor([n - 1 for n in lens], dtype=torch.int32, device=dev)
    out = torch.full((R, 2 * D), SENT, dtype=torch.float16, device=dev)
    ops.caption_tree_attention(qkv, kp, vp, flat, start, pos, out, R=R, H=H, scale=0.125, max_len=max(lens))
    own = torch.stack([p[-1] for p in paths]).to(dev)
    assert torch.equal(kp[own], qkv[:, D:2 * D]) and torch.equal(vp[own], qkv[:, 2 * D:])
    other = torch.ones(n_slots, dtype=torch.bool, device=dev)
    other[own] = False
    assert torch.equal(kp[other], kp0[other]) and torch.equal(vp[other], vp0[other])  # only the rows' own slots are written
    o = unpair(out, D).cpu()
    K_all, V_all = kp.double().cpu(), vp.double().cpu()
    for r, p in enumerate(paths):
        for h in range(H):
            sl = slice(64 * h, 64 * h + 64)
            qh = qkv[r, sl].double().cpu()
            want, _ = attend64(qh, K_all[p][:, sl], V_all[p][:, sl], 0.125)
            assert float((o[r, sl] - want).abs().max()) <= attn_bound(qh, K_all[p][:, sl], V_all[p][:, sl], len(p))


def test_attention_refuses_paths_and_clips_out_of_range():
    """A row whose path is longer than max_len, leaves the path list or names a slot outside the pool, and a row whose clip is outside the
    batch, set the error flag and write nothing; the valid row beside them is unaffected."""
    H, D = 8, 512
    kp, vp = torch.randn(100, D, device=dev), torch.randn(100, D, device=dev)
    kp0, vp0 = kp.clone(), vp.clone()
    qkv = torch.randn(4, 3 * D, device=dev)
    path = torch.tensor([0, 1, 2, 3, 4, 5, 6, 7, 8, 100], dtype=torch.int32, device=dev)
    start = torch.tensor([0, 0, 6, 5], dtype=torch.int64, device=dev)
    pos = torch.tensor([1, 7, 5, 4], dtype=torch.int32, device=dev)  # row 1 longer than max_len, row 2 leaves the list, row 3 reaches slot 100
    out = torch.full((4, 2 * D), SENT, dtype=torch.float16, device=dev)
    err = torch.zeros(1, dtype=torch.int32, device=dev)
    ops.caption_tree_attention(qkv, kp, vp, path, start, pos, out, R=4, H=H, scale=0.125, max_len=5, err_flag=err)
    assert int(err) == 1 and bool((out[1:] == SENT).all()) and not bool((out[0] == SENT).any())
    assert torch.equal(kp[2:], kp0[2:]) and torch.equal(vp[2:], vp0[2:])
    kv = torch.randn(3 * 4, 2 * D, device=dev)
    clips = torch.tensor([2, 3, -1], dtype=torch.int32, device=dev)
    out = torch.full((3, 2 * D), SENT, dtype=torch.float16, device=dev)
    err.zero_()
    ops.caption_cross_attention(qkv[:3, :D].contiguous(), kv, clips, out, R=3, H=H, Lm=4, v_off=D, scale=0.125, err_flag=err)
    assert int(err) == 1 and bool((out[1:] == SENT).all()) and not bool((out[0] == SENT).any())


@pytest.mark.parametrize("Vn", [1, 31, 4097, 16384])
def test_select_vs_fp64(Vn):
    R = 4
    x = torch.randn(R, Vn, device=dev) * 3
    if Vn > 1:
        x[0, :] = torch.round(x[0, :])  # exact ties
        x[1, Vn // 2] = x[1, 0] = x[1].max() + 1  # tied maximum: the lower index wins
    k = min(3, Vn)
    vals = torch.empty(R, k, device=dev)
    idx = torch.empty(R, k, dtype=torch.int64, device=dev)
    err = torch.zeros(1, dtype=torch.int32, device=dev)
    ops.caption_select_topk(x, k, vals, idx, err_flag=err)
    assert int(err) == 0
    xd = x.double().cpu()
    ls = torch.log_softmax(xd, 1)
    for r in range(R):
        order = sorted(range(Vn), key=lambda j: (-float(x[r, j]), j))[:k]
        assert idx[r].tolist() == order
        bound = 4 * EPS32 * (float(xd[r].abs().max()) + math.log(Vn) + 1) + Vn * EPS32
        assert float((vals[r].double().cpu() - ls[r, order]).abs().max()) <= bound
    ys = torch.full((R, 3), -5, dtype=torch.int64, device=dev)
    tok = torch.zeros(R, dtype=torch.int64, device=dev)
    pos = torch.ones(R, dtype=torch.int32, device=dev)
    ops.caption_select_greedy(x, ys, tok, pos, err_flag=err)
    want = [sorted(range(Vn), key=lambda j: (-float(x[r, j]), j))[0] for r in range(R)]
    assert ys[:, 2].tolist() == want and tok.tolist() == want and pos.tolist() == [2] * R and ys[:, :2].eq(-5).all()
    x[2, 0] = float("nan")
    ops.caption_select_greedy(x, ys, tok, pos, err_flag=err)
    assert int(err) == 1


def _model(name):
    c = CASES[name]
    m = ACT(config(c), V)
    m.load_state_dict(O.seeded_state_dict(m.state_dict(), c["seed"], EOS, c["eos_bias"]))
    return m.to(dev).eval(), c


@pytest.fixture(scope="module")
def ref():
    return dict(np.load(os.path.join(ROOT, "tests", "golden", "act_ref.npz")))


@pytest.mark.parametrize("B,T", [(1, 848), (3, 848), (3, 860), (64, 848)])
def test_encoder_memory_vs_oracle(B, T):
    m, _ = _model("cap")
    mels = O.seeded_mels(7, B, T)
    got = m.encode(mels.to(dev)).transpose(0, 1).double().cpu()
    rows = range(B) if B <= 3 else (0, 31, 63)
    sd = {k: v.cpu() for k, v in m.state_dict().items()}
    want = O.encode(sd, mels[list(rows)])
    err = float((got[list(rows)] - want).abs().max() / want.abs().max())
    assert err < 3e-5, err


def test_greedy_forward_and_beams_match_reference(ref):
    m, c = _model("full")
    mels = fixture_mels().to(dev)
    mem = m.encode(mels)
    assert float((mem.transpose(0, 1).cpu() - torch.from_numpy(ref["full_memory"])).abs().max()) < 3e-5 * float(np.abs(ref["full_memory"]).max())
    logits = m.decode(mem, torch.from_numpy(ref["tgt"]).to(dev)).transpose(0, 1).cpu()
    assert float((logits - torch.from_numpy(ref["full_forward"])).abs().max()) < 3e-5 * float(np.abs(ref["full_forward"]).max())
    ys = greedy_decode(m, mels, SOS, EOS, 30).cpu().numpy()
    want = ref["full_greedy"]
    if not np.array_equal(ys, want):  # a differing id must sit on a top-two gap within the logits' error bound
        sd = {k: v.cpu() for k, v in m.state_dict().items()}
        memo = O.encode(sd, mels.cpu())
        for b, t in zip(*np.nonzero(ys != want)):
            lg = O.decode(sd, memo[b:b + 1], torch.from_numpy(want[b:b + 1, :t]), c["nhead"])[0, -1]
            top = torch.topk(lg, 2).values
            assert float(top[0] - top[1]) < 3e-5 * float(lg.abs().max())
            break
    for bw in (2, 3):
        assert np.array_equal(beam_decode(mels, m, SOS, EOS, beam_width=bw).cpu().numpy(), ref[f"full_beam{bw}"])


@pytest.mark.parametrize("bw", [2, 3])
def test_beam_at_the_queue_cap_matches_reference(ref, bw):
    m, _ = _model("cap")
    got = beam_decode(fixture_mels().to(dev), m, SOS, EOS, beam_width=bw).cpu().numpy()
    assert np.array_equal(got, ref[f"cap_beam{bw}"])


def test_graph_replay_and_batch_invariance():
    m, _ = _model("cap")
    mels = O.seeded_mels(9, 6).to(dev)
    eng = m.engine
    ys_graph = greedy_decode(m, mels, SOS, EOS, 30)
    ys_graph2 = greedy_decode(m, mels, SOS, EOS, 30)
    eng.use_cuda_graph = False
    mem_eager = eng.encode(mels)
    ys_eager = greedy_decode(m, mels, SOS, EOS, 30)
    eng.use_cuda_graph = True
    assert torch.equal(ys_graph, ys_eager) and torch.equal(ys_graph, ys_graph2)
    assert torch.equal(eng.encode(mels), mem_eager)
    alone = torch.cat([greedy_decode(m, mels[i:i + 1], SOS, EOS, 30) for i in range(6)])
    assert torch.equal(alone, ys_graph)
    b_all = beam_decode(mels[:3], m, SOS, EOS, beam_width=2)
    for i in range(3):
        one = beam_decode(mels[i:i + 1], m, SOS, EOS, beam_width=2)[0]
        row = b_all[i]
        assert torch.equal(row[:one.numel()], one) and bool((row[one.numel():] == EOS).all())
