"""Melception on the H100: each new kernel against a torch restatement, DSB_GEMM_RELU on both epilogue paths, the full forward against the fp64
oracle over clip lengths, batch sizes and both weight regimes, the drop-in against the reference golden, and the metrics from GPU features."""
import os
import tempfile

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from oracle import melception_oracle as MO  # noqa: E402
from tests.helpers import GOLD  # noqa: E402

DEV = "cuda"
TOL = 4e-5  # full forward, per feature: max |gpu - fp64 oracle| / max |oracle|; 4x the largest measured (9.3e-6, H100 80GB HBM3 at 700 W)


@pytest.fixture(scope="module")
def G():
    from tests import gpu_common
    return gpu_common


def mel_input(seed, B, T):
    rng = np.random.Generator(np.random.Philox(seed))
    return torch.from_numpy(rng.random(size=(B, 80, T), dtype=np.float32)) * 4 - 2


def build(sd, features=MO.FEATURES, aux_logits=True):
    from diffsound_b200.evaluation.feature_extractors.melception import Melception
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "w.pt")
        torch.save({"model": sd}, path)
        return Melception(309, list(features), path, aux_logits=aux_logits).to(DEV).eval()


def pair_of(v):
    hi = v.half()
    return torch.cat([hi, (v - hi.float()).half()], -1)


def value_of(p):
    C = p.shape[-1] // 2
    return p[..., :C].double() + p[..., C:].double()


def pair_grid(B, Hp, Wp, C, win, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    v = torch.zeros(B, Hp, Wp, C)
    y0, x0, H, W = win
    v[:, y0:y0 + H, x0:x0 + W] = (torch.rand(B, H, W, C, generator=g) * 2 - 1) * scale
    return pair_of(v).to(DEV)


# ---------------------------------------------------------------------------------------------------------------- kernels
@pytest.mark.parametrize("H,W,C", [(35, 43, 288), (17, 20, 96), (17, 21, 192), (4, 5, 8)])
def test_space_to_depth_is_a_bit_exact_copy(G, H, W, C):
    from diffsound_b200 import ops
    B, Hpi, Wpi, win = 2, H + 6, W + 6, (3, 3, H, W)
    x = pair_grid(B, Hpi, Wpi, C, win, 1)
    Hpo, Wpo, o = (H + 1) // 2 + 4, (W + 1) // 2 + 5, (2, 3)
    out = torch.full((B, Hpo, Wpo, 8 * C), float("nan"), dtype=torch.float16, device=DEV)
    ops.pair_space_to_depth(x, win, out, o)
    ref = torch.zeros_like(out)
    xw = x[:, 3:3 + H, 3:3 + W]
    for ph in range(4):
        s = xw[:, ph >> 1::2, ph & 1::2]
        ref[:, o[0]:o[0] + s.shape[1], o[1]:o[1] + s.shape[2], ph * C:(ph + 1) * C] = s[..., :C]
        ref[:, o[0]:o[0] + s.shape[1], o[1]:o[1] + s.shape[2], 4 * C + ph * C:4 * C + (ph + 1) * C] = s[..., C:]
    assert torch.equal(out.view(torch.int16), ref.view(torch.int16))


@pytest.mark.parametrize("scale", [1.0, 0.25, 8.0])
def test_maxpool_copies_the_winning_pair(G, scale):
    from diffsound_b200 import ops
    B, C, H, W = 2, 96, 17, 23
    win = (3, 3, H, W)
    x = pair_grid(B, H + 6, W + 6, C, win, 2)
    x[0, 5, 5:8] = x[0, 5, 6]  # exact ties: the first pixel in (dy, dx) order wins (all three are equal pairs, so any winner copies the same bits)
    Ho, Wo = (H - 3) // 2 + 1, (W - 3) // 2 + 1
    Ctot, off = 160, 48
    out = torch.full((B, Ho + 2, Wo + 2, 2 * Ctot), float("nan"), dtype=torch.float16, device=DEV)
    ops.pair_maxpool3s2(x, win, out, (1, 1), out_ptr=out.data_ptr() + 2 * off, ldo=2 * Ctot, lo_off=Ctot, scale=scale)
    xw = x[:, 3:3 + H, 3:3 + W]
    cand = torch.stack([xw[:, dy:dy + 2 * Ho - 1:2, dx:dx + 2 * Wo - 1:2] for dy in range(3) for dx in range(3)], 0)  # (9, B, Ho, Wo, 2C)
    idx = value_of(cand).argmax(0, keepdim=True)
    win_hi = torch.gather(cand[..., :C], 0, idx).squeeze(0)
    win_lo = torch.gather(cand[..., C:], 0, idx).squeeze(0)
    hi = (win_hi.float() * scale).half()
    lo = (win_lo.float() * scale).half()
    got = out[:, 1:1 + Ho, 1:1 + Wo]
    assert torch.equal(got[..., off:off + C].view(torch.int16), hi.view(torch.int16))
    assert torch.equal(got[..., Ctot + off:Ctot + off + C].view(torch.int16), lo.view(torch.int16))
    ring = out.clone()
    ring[:, 1:1 + Ho, 1:1 + Wo] = 0
    assert torch.equal(ring[..., off:off + C], torch.zeros_like(ring[..., off:off + C]))
    assert torch.isnan(out[..., :off]).all()  # other channel slices untouched


def test_avgpool_against_fp64(G):
    from diffsound_b200 import ops
    B, C, Hp, Wp, win = 2, 64, 12, 30, (2, 3, 8, 25)
    x = pair_grid(B, Hp, Wp, C, win, 3, scale=300.0)
    out = ops.pair_avgpool3(x, win)
    v = value_of(x).permute(0, 3, 1, 2)
    ref = F.avg_pool2d(v, 3, 1, 1, count_include_pad=True).permute(0, 2, 3, 1)
    mask = torch.zeros(1, Hp, Wp, 1, dtype=torch.bool, device=DEV)
    mask[:, 2:10, 3:28] = True
    ref = torch.where(mask, ref, torch.zeros_like(ref))
    err = (value_of(out) - ref).abs()
    # nine fp32 additions, one fp32 division, one re-split: a few fp32 ulps of the largest partial sum
    assert float(err.max()) <= 8 * 2.0 ** -24 * 9 * float(v.abs().max()), float(err.max())
    assert torch.equal(value_of(out)[~mask.expand_as(ref)], torch.zeros_like(ref[~mask.expand_as(ref)]))


def test_channel_mean_against_fp64(G):
    from diffsound_b200 import ops
    B, C, Hp, Wp, win = 3, 200, 19, 44, (1, 2, 17, 41)
    x = pair_grid(B, Hp, Wp, C, win, 4, scale=512.0)
    got = ops.pair_channel_mean(x, win, inv_scale=2.0 ** -9)
    ref = value_of(x)[:, 1:18, 2:43].mean((1, 2)) * 2.0 ** -9
    assert float((got.double() - ref).abs().max()) <= 2.0 ** -24 * float(ref.abs().max()) * 2
    assert torch.equal(got, ops.pair_channel_mean(x, win, inv_scale=2.0 ** -9))  # fixed summation order


@pytest.mark.parametrize("norm", [False, True])
def test_stem_against_fp64(G, norm):
    from diffsound_b200 import ops
    g = torch.Generator().manual_seed(5)
    B, T = 2, 101
    x = (torch.rand(B, 80, T, generator=g) * 6 - 1).to(DEV)
    w = (torch.rand(32, 9, generator=g) - 0.5).to(DEV)
    b = (torch.rand(32, generator=g) - 0.5).to(DEV)
    mean = (torch.rand(80, generator=g) * 2).to(DEV) if norm else None
    std = (torch.rand(80, generator=g) + 0.5).to(DEV) if norm else None
    Ho, Wo = 39, (T - 3) // 2 + 1
    out = torch.full((B, Ho + 2, Wo + 4, 64), float("nan"), dtype=torch.float16, device=DEV)
    ops.mel_stem(x, w, b, out, Hp=Ho + 2, Wp=Wo + 4, y0=1, x0=2, scale=4.0, mean=mean, std=std)
    xn = x.double()
    if norm:
        xn = (xn - mean.double()[:, None]) / std.double()[:, None]
    ref = torch.relu(F.conv2d(xn.unsqueeze(1), w.double().view(32, 1, 3, 3), b.double(), stride=2)).permute(0, 2, 3, 1) * 4.0
    got = value_of(out)
    assert float((got[:, 1:1 + Ho, 2:2 + Wo] - ref).abs().max()) <= 1e-6 * float(ref.abs().max())
    inner = torch.zeros_like(got, dtype=torch.bool)
    inner[:, 1:1 + Ho, 2:2 + Wo] = True
    assert torch.equal(got[~inner], torch.zeros_like(got[~inner]))


@pytest.mark.parametrize("N", [96, 40])  # 40: the last 32-column chunk is partial, so it runs the scalar epilogue
def test_gemm_relu_flag(G, N):
    from diffsound_b200 import ops
    g = torch.Generator().manual_seed(6)
    M, K = 300, 128
    a = (torch.rand(M, K, generator=g) * 2 - 1).to(DEV)
    w = (torch.rand(N, K, generator=g) * 2 - 1).to(DEV)
    bias = (torch.rand(N, generator=g) - 0.5).to(DEV)
    ap, wp = ops.split_f16(a), ops.split_f16(w)
    off = ops.gemm_f16x3(ap, wp, bias)
    on = ops.gemm_f16x3(ap, wp, bias, relu=True)
    assert torch.equal(on, torch.where(off < 0, torch.zeros_like(off), off))  # the flag adds exactly the ReLU
    ref = torch.relu(a.double() @ w.double().T + bias.double())
    assert float((on.double() - ref).abs().max()) <= 1e-5 * float(ref.abs().max())
    # pair output
    poff = ops.gemm_f16x3(ap, wp, bias, split_out=True)
    pon = ops.gemm_f16x3(ap, wp, bias, split_out=True, relu=True)
    neg = (value_of(poff) < 0).repeat(1, 2)
    assert torch.equal(pon.view(torch.int16)[~neg], poff.view(torch.int16)[~neg])
    assert (pon[neg] == 0).all()
    # residual before the activation (the last launch of a chained 5x5)
    res = (torch.rand(M, N, generator=g) - 0.5).to(DEV)
    rr = ops.gemm_f16x3(ap, wp, bias, residual=res, relu=True, res_before_act=True)
    assert float((rr.double() - torch.relu(a.double() @ w.double().T + bias.double() + res.double())).abs().max()) <= 1e-5 * float(ref.abs().max())


# ---------------------------------------------------------------------------------------------------------------- full forward
_SD = {}


def sd_for(init):
    if init not in _SD:
        _SD[init] = MO.make_melception_state_dict({"he": 21, "wide": 22}[init], init)
    return _SD[init]


@pytest.fixture(scope="module")
def models():
    ms = {}
    yield lambda init: ms.setdefault(init, build(sd_for(init)))
    ms.clear()
    torch.cuda.empty_cache()


@pytest.mark.parametrize("init", ["he", "wide"])
@pytest.mark.parametrize("T", [96, 848, 860])
@pytest.mark.parametrize("B", [1, 3, 65])
def test_forward_against_fp64_oracle(G, models, init, T, B):
    m = models(init)
    assert m.engine.max_batch == 64  # B = 65 is one clip past a full pass: two CUDA graphs
    x = mel_input(1000 + T + B, B, T).to(DEV)
    got = m(x)
    ref = MO.melception_forward(sd_for(init), x, MO.FEATURES, torch.float64)
    errs = {}
    for name, gf, rf in zip(MO.FEATURES, got, ref):
        assert gf.shape == rf.shape and gf.dtype == torch.float32, (name, gf.shape, rf.shape)
        errs[name] = float((gf.double() - rf).abs().max() / rf.abs().max())
    print(f"melception {init} T={T} B={B}: " + " ".join(f"{k}={v:.2e}" for k, v in errs.items()))
    assert max(errs.values()) < TOL, errs


@pytest.mark.parametrize("tag", ["he", "wide"])
def test_dropin_matches_reference_golden(G, tag):
    ref = np.load(os.path.join(GOLD, "melception_ref.npz"))
    seed, B, T, xseed = ref[f"{tag}.cfg"].tolist()
    m = build(MO.make_melception_state_dict(seed, tag))
    got = m(mel_input(xseed, B, T).to(DEV))
    for name, g_ in zip(MO.FEATURES, got):
        r = torch.from_numpy(ref[f"{tag}.{name}"]).double()
        err = float((g_.double().cpu() - r).abs().max() / r.abs().max())
        print(f"golden {tag} {name}: {err:.2e}")
        assert err < TOL, (tag, name, err)


def test_features_list_orders_and_early_exit(G):
    sd = sd_for("he")
    x = mel_input(7, 2, 96).to(DEV)
    full = dict(zip(MO.FEATURES, build(sd)(x)))
    for fl in (["64"], ["192", "64"], ["768"], ["2048"], ["logits"], ["logits_unbiased"], ["logits", "logits_unbiased", "2048"],
               ["2048", "768", "192", "64", "logits", "logits_unbiased"]):
        m = build(sd, features=fl)
        got = m(x)
        assert isinstance(got, tuple) and len(got) == len(fl)
        for name, g_ in zip(fl, got):
            assert torch.equal(g_, full[name]), (fl, name)
        assert list(m.convert_features_tuple_to_dict(got)) == fl
    assert full["64"].shape == (2, 64, 1, 1) and full["192"].shape == (2, 192, 1, 1) and full["768"].shape == (2, 768, 1, 1)
    assert full["2048"].shape == (2, 2048) and full["logits"].shape == (2, 309)


def test_cuda_graph_replay_equals_eager(G):
    m = build(sd_for("he"))
    x = mel_input(8, 3, 96).to(DEV)
    a = m(x)
    b = m(x)  # second call replays the captured graph
    m.engine.use_cuda_graph = False
    c = m(x)
    for u, v, w_ in zip(a, b, c):
        assert torch.equal(u, v) and torch.equal(u, w_)


def test_repack_after_to_load_and_inplace_change(G, tmp_path):
    from diffsound_b200.evaluation.feature_extractors.melception import Melception
    sd1, sd2 = sd_for("he"), MO.make_melception_state_dict(23, "he")
    path = str(tmp_path / "w.pt")
    torch.save({"model": sd1}, path)
    m = Melception(309, ["2048", "logits"], path).eval()  # built on the CPU, moved after
    with pytest.raises(RuntimeError, match="CUDA"):
        m(mel_input(9, 1, 96))
    m = m.to(DEV)
    x = mel_input(9, 2, 96).to(DEV)
    r1 = MO.melception_forward(sd1, x, ["2048", "logits"])
    g1 = m(x)
    assert float((g1[1].double() - r1[1]).abs().max() / r1[1].abs().max()) < TOL
    m.load_state_dict(sd2)
    r2 = MO.melception_forward(sd2, x, ["2048", "logits"])
    g2 = m(x)
    assert float((g2[0].double() - r2[0]).abs().max() / r2[0].abs().max()) < TOL
    with torch.no_grad():
        m.fc.bias.add_(1.0)  # in place: no load_state_dict, no .to()
    g3 = m(x)
    assert float((g3[1].double() - (r2[1] + 1.0)).abs().max() / r2[1].abs().max()) < TOL


def test_errors(G):
    m = build(sd_for("he"), features=["2048"])
    x = mel_input(10, 1, 96)
    with pytest.raises(RuntimeError):
        m(x)  # CPU tensor: no fallback
    with pytest.raises(RuntimeError, match="eval mode"):
        m.train()(x.to(DEV))
    m.eval()
    with pytest.raises(RuntimeError, match="non-finite"):
        m(x.to(DEV) * 1e7)  # activations beyond fp16 even at the calibrated scales
    bad = dict(sd_for("he"))
    bad["Mixed_6b.branch7x7_2.bn.running_var"] = torch.full_like(bad["Mixed_6b.branch7x7_2.bn.running_var"], float("nan"))
    with pytest.raises(RuntimeError):
        build(bad, features=["2048"])(x.to(DEV))


def test_metrics_from_gpu_features_match_oracle_features(G):
    from diffsound_b200.evaluation.metrics import fid, isc, kid, kl
    sd = sd_for("he")
    fl = ["logits_unbiased", "2048", "logits"]
    m = build(sd, features=fl)
    xf, xr = mel_input(11, 64, 96).to(DEV), mel_input(12, 32, 96).to(DEV)
    keys = [f"Y{k:04d}" for k in range(32)]
    names_f = [f"/f/cls_0/{k}_sample_{n}.npy" for k in keys for n in range(2)]
    names_r = [f"/r/val/{k}_mel.npy" for k in keys]

    def feats(x, names, gpu):
        v = m(x) if gpu else MO.melception_forward(sd, x, fl, torch.float64)
        d = {k: t.float().cpu() for k, t in zip(fl, v)}
        d["2048_head"] = d["2048"][:, :24].contiguous()  # full-rank slice: FID's sqrtm is well conditioned on it (N = 64 > 24)
        d["file_path_"] = names
        return d

    g1, g2, o1, o2 = feats(xf, names_f, True), feats(xr, names_r, True), feats(xf, names_f, False), feats(xr, names_r, False)
    rel = lambda a, b: abs(a - b) / abs(b)
    k_g, k_o = kl.calculate_kl(g1, g2, "logits", "caps"), kl.calculate_kl(o1, o2, "logits", "caps")
    i_g, i_o = isc.calculate_isc(g1, "logits_unbiased", 2020, True, 10), isc.calculate_isc(o1, "logits_unbiased", 2020, True, 10)
    f_g, f_o = fid.calculate_fid(g1, g2, "2048_head"), fid.calculate_fid(o1, o2, "2048_head")
    d_g, d_o = kid.calculate_kid(g1, g2, 100, 1000, 3, None, 1, 2020, "2048"), kid.calculate_kid(o1, o2, 100, 1000, 3, None, 1, 2020, "2048")
    print("metrics gpu", k_g, i_g, f_g, d_g, "\nmetrics oracle", k_o, i_o, f_o, d_o)
    assert rel(k_g["kullback_leibler_divergence"], k_o["kullback_leibler_divergence"]) < 1e-4
    assert rel(i_g["inception_score_mean"], i_o["inception_score_mean"]) < 1e-4
    assert rel(f_g["frechet_inception_distance"], f_o["frechet_inception_distance"]) < 1e-4
    f = o1["2048"].double().numpy()
    mean_kernel = float(np.mean((f @ f.T / f.shape[1] + 1) ** 3))
    assert abs(d_g["kernel_inception_distance_mean"] - d_o["kernel_inception_distance_mean"]) < 1e-4 * mean_kernel
    assert np.isfinite(fid.calculate_fid(g1, g2, "2048")["frechet_inception_distance"])
