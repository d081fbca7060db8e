"""The SpecVQGAN mel front end on the H100: the pack kernel bit for bit, dsb_mel_log per element against fp64, the full path against the fp64
oracle within the bound derived in tests/mel_reference.py, determinism and batch invariance, the encoder / DALLE.reconstruct on a GPU mel, and
the drop-ins."""
import os
import subprocess
import sys

import numpy as np
import pytest
import scipy.io.wavfile
import torch

pytestmark = pytest.mark.gpu

from oracle import mel_oracle as O  # noqa: E402
from tests import mel_reference as R  # noqa: E402
from tests.helpers import GOLD, ROOT  # noqa: E402

SENT = -12345.0


@pytest.fixture(scope="module")
def G():
    from tests import gpu_common
    return gpu_common


@pytest.fixture(scope="module")
def eng(G):
    from diffsound_b200 import mel_engine as ME
    return ME.MelEngine("cuda")


def clips():
    z = np.load(os.path.join(GOLD, "audio_clips.npz"))
    return {k: z[k].astype(np.float32) / 32768.0 for k in z.files}


@pytest.mark.parametrize("length", [513, 1000, 1024, 1025, 22050, 220160, 220500])
@pytest.mark.parametrize("B", [1, 3, 64])
def test_pack_is_bit_identical_to_restatement(G, length, B):
    g = torch.Generator().manual_seed(length + B)
    wav = (torch.rand(B, length, generator=g) * 2 - 1) * 0.9
    wav[0, 0], wav[-1, -1] = 3.99, -3.99                     # the borders land in the reflected rows
    rows = length // 256 + 4
    extra = 4096
    buf = torch.full((B * rows * 512 + extra,), SENT, dtype=torch.float16, device="cuda")
    out = buf[:B * rows * 512].view(B, rows, 512)
    err = torch.zeros(1, dtype=torch.int32, device="cuda")
    G.ops.wav_frames_f16(wav.cuda(), out, rows=rows, err_flag=err)
    ref = R.frames_f16(wav, rows)
    assert torch.equal(out.cpu(), ref) and int(err.item()) == 0
    assert bool((buf[B * rows * 512:] == SENT).all())
    # reflect borders: padded sample 512 - j is x[j], and 512 + length - 1 + j is x[length - 1 - j]
    full = (out[..., :256].float() + out[..., 256:].float()).cpu().reshape(B, -1) / 8192
    assert torch.allclose(full[:, 512 - torch.arange(1, 513)], wav[:, 1:513], atol=2.0 ** -36, rtol=2.0 ** -21)   # lo halves of tiny samples are fp16 subnormals
    n_tail = rows * 256 - (length + 1024)
    if n_tail > 0:
        assert not full[:, length + 1024:].any()


def test_pack_sets_err_flag(G):
    for bad in (float("nan"), float("inf"), 4.0, -4.0, 17.0):
        wav = torch.zeros(2, 2000)
        wav[1, 1234] = bad
        err = torch.zeros(1, dtype=torch.int32, device="cuda")
        G.ops.wav_frames_f16(wav.cuda(), err_flag=err)
        assert int(err.item()) == 1, bad
    err = torch.zeros(1, dtype=torch.int32, device="cuda")
    G.ops.wav_frames_f16(torch.full((2, 2000), 3.999).cuda(), err_flag=err)
    assert int(err.item()) == 0
    with pytest.raises(RuntimeError):
        G.ops.wav_frames_f16(torch.zeros(1, 512).cuda())


def _mel_kernel(G, eng, spec, T_out, extra=1000):
    B = spec.shape[0]
    buf = torch.full((B * 80 * T_out + extra,), SENT, device="cuda")
    out = buf[:B * 80 * T_out].view(B, 80, T_out)
    G.ops.mel_log(spec.cuda(), eng.n_bins, eng.fb_start, eng.fb_len, eng.fb_w, T_out, out=out)
    assert bool((buf[B * 80 * T_out:] == SENT).all())
    return out.cpu()


@pytest.mark.parametrize("T,T_out", [(1, 1), (37, 37), (862, 860), (900, 860)])
def test_mel_log_kernel_against_fp64(G, eng, T, T_out):
    g = torch.Generator().manual_seed(T)
    B = 3
    scale = 10.0 ** (torch.rand(B, T, 1, generator=g) * 10 - 7)          # mels from far below 1e-5 to far above 10
    spec = torch.randn(B, T, eng.n_cols, generator=g) * scale
    spec[:, :, 2 * eng.n_bins:] = float("nan")                           # padding columns are never read
    got = _mel_kernel(G, eng, spec, T_out)
    want, mel, dense = R.mel_log(spec, eng.n_bins, eng.fb_start.cpu(), eng.fb_len.cpu(), eng.fb_w.cpu(), T_out)
    # fp32 steps: magnitude within 2 ulp, the filter sum within (n_m + 1) ulp of the mel, then the log steps
    width = (dense != 0).sum(1).double()
    dmel = (width[None, :, None] + 3) * 2.0 ** -24 * mel
    bound = R.bound_from_mel(mel, dmel)
    err = (got.double() - want).abs()
    print(f"mel_log T={T}: max err {float(err.max()):.3g}, max err / bound {float((err / bound).max()):.3g}")
    assert got.shape == (B, 80, T_out) and bool((err <= bound).all())


def test_mel_log_exact_ends(G, eng):
    T = 40
    spec = torch.zeros(1, T, eng.n_cols)
    got = _mel_kernel(G, eng, spec, T)
    assert bool((got == 0.0).all())
    # a flat magnitude c in every bin gives mel = c * sum(f_m); choose c so that every mel is at least 10
    fsum = eng.fb_w.double().sum(1).min().item()
    for c in (1.01 * 10.0 / fsum, 1e3):
        spec = torch.zeros(1, T, eng.n_cols)
        spec[:, :, 0:2 * eng.n_bins:2] = c
        got = _mel_kernel(G, eng, spec, T)
        assert bool((got == 1.0).all()), c


def _cases():
    c = clips()
    n = 220500
    t = np.arange(n) / 22050.0
    g = np.random.default_rng(7)
    out = {name: O.pad_or_trim(c[name], n).astype(np.float32) for name in c}
    out["silence"] = np.zeros(n, np.float32)
    imp = np.zeros(n, np.float32)
    imp[0] = imp[-1] = 1.0
    out["impulses"] = imp
    out["dc"] = np.full(n, 0.5, np.float32)
    for k in (6, 100, 352, 100.5, 6.25):
        out[f"sine_bin{k}"] = np.sin(2 * np.pi * (k * 22050 / 1024) * t).astype(np.float32)
    out["noise_0dB"] = np.clip(g.standard_normal(n) * 0.5, -1, 1).astype(np.float32)
    out["noise_-60dB"] = (g.standard_normal(n) * 0.5e-3).astype(np.float32)
    return out


def test_full_path_within_derived_bound(G, eng):
    cases = _cases()
    names = list(cases)
    wav = torch.from_numpy(np.stack([cases[k] for k in names])).cuda()
    got = eng(wav).cpu().double().numpy()
    basis = O.mel_basis()
    worst, worst_ratio = 0.0, 0.0
    for i, k in enumerate(names):
        y = cases[k].astype(np.float64)
        mel = O.mel_power(y, basis)[:, :860]
        want = O.log_steps(mel)
        bound = R.full_path_bound(y, basis, mel).numpy()
        err = np.abs(got[i] - want)
        print(f"{k:14s} max err {err.max():.3g}  max err / bound {(err / bound).max():.3g}")
        assert got[i].shape == (80, 860) and np.all(err <= bound), k
        worst, worst_ratio = max(worst, err.max()), max(worst_ratio, (err / bound).max())
        if k == "silence":
            assert not got[i].any()
    print(f"full path: largest error {worst:.3g}, largest error / bound {worst_ratio:.3g}")


def test_determinism_graph_and_batch_invariance(G, eng):
    c = clips()
    g = np.random.default_rng(3)
    wav = np.stack([np.roll(c["original_0"], int(s)) * float(a) for s, a in zip(g.integers(0, 220500, 64), g.uniform(0.1, 1.0, 64))])
    x = torch.from_numpy(wav.astype(np.float32)).cuda()
    a = eng(x)
    b = eng(x)
    e = eng(x, use_graph=False)
    assert torch.equal(a, b) and torch.equal(a, e)
    for j in (0, 17, 63):
        assert torch.equal(eng(x[j:j + 1]), a[j:j + 1])


def test_encoder_tokens_and_reconstruct_on_gpu_mel(G, eng):
    from tests.test_gpu_decoder import build_vq
    y = O.pad_or_trim(clips()["original_0"], 220500).astype(np.float32)
    mel_gpu = eng(torch.from_numpy(y)[None].cuda())[:, None, :, :848]
    mel_ref = torch.from_numpy(O.log_mel(y.astype(np.float64))[:, :848]).float()[None, None].cuda()
    torch.manual_seed(5)
    m = build_vq(256, 256, 128, (1, 1, 2, 2, 4))
    m.encode(mel_ref)
    zf = m.last_latent.permute(0, 2, 3, 1).reshape(-1, 256).cpu()
    g = torch.Generator().manual_seed(6)
    cb = zf.mean(0, keepdim=True) + torch.randn(256, 256, generator=g) * zf.std(0, keepdim=True)
    m.quantize.embedding.weight.data.copy_(cb.cuda())
    m.enc_engine.repack()
    _, _, info_ref = m.encode(mel_ref)
    z_ref = m.last_latent.permute(0, 2, 3, 1).reshape(-1, 256).double().cpu()
    _, _, info = m.encode(mel_gpu)
    ids, ids_ref = info[2].view(-1).cpu(), info_ref[2].view(-1).cpu()
    agree = float((ids == ids_ref).float().mean())
    d = ((z_ref[:, None, :] - cb.double()[None]) ** 2).sum(-1)              # distances of the oracle-mel latents to every code
    bad = (ids != ids_ref).nonzero().view(-1)
    gaps = (d[bad, ids[bad]] - d[bad, ids_ref[bad]]) / d[bad, ids_ref[bad]]
    print("GPU mel -> encoder: token agreement", agree, "relative distance gaps of mismatches", gaps.tolist())
    assert agree >= 0.99 and bool((gaps < 1e-3).all())
    from diffsound_b200.utils import builders
    dalle = builders.build_dalle(K=64, D=128, NL=2, NH=2, CD=64, seed=0)
    rec = dalle.reconstruct(mel_gpu)
    assert rec.shape == (1, 1, 80, 848) and bool(torch.isfinite(rec).all())


def test_dropins_match_batched_path(G, eng, tmp_path):
    from diffsound_b200.feature_extraction import extract_mel_spectrogram as X
    c = clips()
    src = tmp_path / "wavs"
    src.mkdir()
    for name, x in c.items():
        scipy.io.wavfile.write(str(src / f"{name}.wav"), 22050, np.round(x * 32768).astype(np.int16))
    ys = {name: X.pad_or_trim(X.read_wav(str(src / f"{name}.wav")), 220500) for name in c}
    batched = X.mel_spectrogram(torch.from_numpy(np.stack([ys[k] for k in c]).astype(np.float32)).cuda()).cpu().numpy()
    for i, name in enumerate(c):
        assert np.array_equal(X.TRANSFORMS(ys[name]), batched[i]), name
        y, mel = X.get_spectrogram(str(src / f"{name}.wav"), None, 220500, save_results=False)
        assert np.array_equal(y, ys[name]) and np.array_equal(mel, batched[i])
    out = tmp_path / "mels"
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "extract_mel.py"), "-i", str(src), "-o", str(out), "--batch", "2"],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    for i, name in enumerate(c):
        saved = np.load(str(out / f"{name}_mel.npy"))
        assert saved.dtype == np.float32 and np.array_equal(saved, batched[i]), name
