"""The SpecVQGAN mel front end without a GPU: the fp64 oracle pinned to torch.stft and torchaudio's Slaney filterbank, the packed DFT weights,
MelEngine's host orchestration on plain-torch stand-ins of its three kernels, WAV reading, the CLI's dry run, and what ptxas made of mel.cu."""
import json
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest
import scipy.io.wavfile
import torch

from oracle import mel_oracle as O
from tests import cpu_state_gemm_emulation as E
from tests import mel_reference as R
from tests.helpers import GOLD, ROOT

import _pkg  # noqa: E402

_pkg.load()
from diffsound_b200 import mel_engine as ME  # noqa: E402
from diffsound_b200 import ops, packing  # noqa: E402
from diffsound_b200.feature_extraction import extract_mel_spectrogram as X  # noqa: E402


def clips():
    z = np.load(os.path.join(GOLD, "audio_clips.npz"))
    return {k: z[k].astype(np.float32) / 32768.0 for k in z.files}


def torch_log_mel(y):
    """The librosa-compatible path of two independent installed implementations: torch.stft (reflect, periodic Hann, fp64) and torchaudio's
    Slaney filterbank (computed in fp64, stored as float32 as librosa stores it)."""
    import torchaudio
    spec = torch.stft(torch.from_numpy(np.asarray(y, dtype=np.float64)), 1024, 256, window=torch.hann_window(1024, periodic=True, dtype=torch.float64),
                      center=True, pad_mode="reflect", return_complex=True).abs()
    dt = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    try:
        fb = torchaudio.functional.melscale_fbanks(513, 125.0, 7600.0, 80, 22050, norm="slaney", mel_scale="slaney").T.float().double()
    finally:
        torch.set_default_dtype(dt)
    return R.log_steps(fb @ spec)[:, :860].numpy()


def test_basis_matches_torchaudio_and_covers_bins_6_to_352():
    import torchaudio
    b = O.mel_basis()
    dt = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)   # torchaudio's arithmetic in fp64; librosa rounds twice to float32 (triangle, then normalised)
    try:
        ta = torchaudio.functional.melscale_fbanks(513, 125.0, 7600.0, 80, 22050, norm="slaney", mel_scale="slaney").T.numpy()
    finally:
        torch.set_default_dtype(dt)
    assert np.array_equal(ta != 0, b != 0)
    assert np.all(np.abs(ta - b) <= 2 * 2.0 ** -24 * np.abs(ta))
    nz = np.nonzero(b.any(axis=0))[0]
    assert (nz[0], nz[-1], len(nz)) == (6, 352, 347)
    assert b.dtype == np.float32 and np.array_equal(ME.mel_basis(), b)   # the package's own basis, bit for bit
    k0, nb, starts, lens, w = ME.filter_table(b)
    assert (k0, nb) == (6, 347) and lens.min() >= 3 and lens.max() <= 24
    for m in range(80):
        dense = np.zeros(nb, np.float32)
        dense[starts[m]:starts[m] + lens[m]] = w[m, :lens[m]]
        assert np.array_equal(dense, b[m, 6:353])


def test_magnitude_matches_torch_stft_fp64():
    y = clips()["original_0"][:30000].astype(np.float64)
    ref = torch.stft(torch.from_numpy(y), 1024, 256, window=torch.hann_window(1024, periodic=True, dtype=torch.float64), center=True,
                     pad_mode="reflect", return_complex=True).abs().numpy()
    mag = O.stft_mag(y)
    assert mag.shape == ref.shape == (513, 1 + 30000 // 256)
    assert np.abs(mag - ref).max() <= 1e-12 * max(1.0, np.abs(ref).max())


@pytest.mark.parametrize("name", ["original_0", "generated_0"])
def test_oracle_log_mel_matches_torch_path_on_fixture_clips(name):
    y = O.pad_or_trim(clips()[name], 220500)
    mel = O.log_mel(y)
    assert mel.shape == (80, 860) and 1 + 220500 // 256 == 862
    assert np.abs(mel - torch_log_mel(y)).max() < 2e-6
    assert 0.0 <= mel.min() and mel.max() <= 1.0 and mel.std() > 0.05


def test_pad_or_trim_follows_get_spectrogram():
    c = clips()
    short = c["generated_0"]                              # 88200 samples: zero-padded to 220500
    n = len(short)
    assert n == 88200 and len(c["original_0"]) == 220500
    y = O.pad_or_trim(short, 220500)
    assert len(y) == 220500 and np.array_equal(y[:n], short.astype(np.float64)) and not y[n:].any()
    assert np.array_equal(X.pad_or_trim(short, 220500), y)
    long_ = np.concatenate([c["original_0"], c["generated_0"]])
    assert np.array_equal(X.pad_or_trim(long_, 220500), long_[:220500].astype(np.float64))
    for n in (513, 1000, 22050):
        m = O.log_mel(O.pad_or_trim(c["original_0"], n))
        assert m.shape == (80, 1 + n // 256) and np.abs(m - torch_log_mel(O.pad_or_trim(c["original_0"], n))).max() < 2e-6
    with pytest.raises(ValueError):
        X.pad_or_trim(short, 512)


def test_packed_dft_pairs_reproduce_the_fp64_basis(monkeypatch):
    monkeypatch.setattr(ops, "split_f16", E.split_f16)
    k0, nb = 6, 347
    n_cols = (2 * nb + 7) // 8 * 8
    w = torch.from_numpy(ME.dft_weights(k0, nb, n_cols))
    assert n_cols == 696 and not w[694:].any()
    # exact argument reduction: bin k, sample n uses the angle of (k n) mod 1024
    n = np.arange(1024)
    win = 0.5 - 0.5 * np.cos(2 * np.pi * n / 1024)
    assert np.allclose(w[2 * 94].numpy(), win * np.cos(2 * np.pi * 100 * n / 1024), atol=1e-13, rtol=0)
    pc = packing.PackedConv([w[:, j * 256:(j + 1) * 256] for j in range(4)], torch.zeros(n_cols))
    pair = pc.w.view(n_cols, 4, 2, 256).double()
    rec = ((pair[:, :, 0] + pair[:, :, 1]) * pc.alpha).reshape(n_cols, 1024)
    # 22 bits per weight; weights so small that the lo half is an fp16 subnormal keep 2^-25 of absolute precision before alpha
    assert torch.all((rec - w).abs() <= 2.0 ** -22 * w.abs() + 2.0 ** -25 * pc.alpha)
    assert float((rec - w).abs().max()) <= 2.0 ** -22 * float(w.abs().max())


def _frames_standin(wav, out, *, rows, err_flag=None):
    out.copy_(R.frames_f16(wav, rows))
    bad = ~(wav.abs() < R.LIMIT)
    if err_flag is not None and bool(bad.any()):
        err_flag.fill_(1)
    return out


def _mel_log_standin(spec, n_bins, fb_start, fb_len, fb_w, T_out, out=None):
    y, _, _ = R.mel_log(spec, n_bins, fb_start, fb_len, fb_w, T_out)
    return y.float()


def test_engine_orchestration_on_cpu_standins(monkeypatch):
    """MelEngine's buffers, tap list, strides and alpha with plain-torch stand-ins of the pack kernel, dsb_gemm_ex and the mel kernel."""
    monkeypatch.setattr(ops, "split_f16", E.split_f16)
    monkeypatch.setattr(ops, "gemm_desc", E.gemm_desc)
    monkeypatch.setattr(ops, "wav_frames_f16", _frames_standin)
    monkeypatch.setattr(ops, "mel_log", _mel_log_standin)
    eng = ME.MelEngine("cpu")
    E.track(eng.dft.w)
    alloc = eng._alloc
    monkeypatch.setattr(eng, "_alloc", lambda B, n: tuple(E.track(t) for t in alloc(B, n)))
    c = clips()
    for length in (1000, 5000):
        wav = np.stack([c["original_0"][:length], c["generated_0"][7000:7000 + length]])
        out = eng(torch.from_numpy(wav), use_graph=False)
        assert out.shape == (2, 80, 1 + length // 256)
        for b in range(2):
            ref = O.log_mel(wav[b].astype(np.float64))
            assert np.abs(out[b].numpy() - ref).max() < 1e-5, (length, b)
    bad = torch.from_numpy(np.stack([c["original_0"][:1000]])).clone()
    bad[0, 10] = float("nan")
    with pytest.raises(RuntimeError, match="finite"):
        eng(bad, use_graph=False)
    with pytest.raises(ValueError):
        eng(torch.zeros(1, 512), use_graph=False)


@pytest.mark.parametrize("kind", ["int16", "int32", "float32", "uint8"])
def test_read_wav_scales_like_librosa(tmp_path, kind):
    g = np.random.default_rng(0)
    x = (g.random((3000, 2)) * 2 - 1) * 0.9
    if kind == "float32":
        data = x.astype(np.float32)
        want = data.mean(axis=1)
    elif kind == "uint8":
        data = np.round(x * 127 + 128).astype(np.uint8)
        want = ((data.astype(np.float32) - 128) / 128).mean(axis=1)
    else:
        bits = 16 if kind == "int16" else 32
        data = np.round(x * (2 ** (bits - 1) - 1)).astype(kind)
        want = (data.astype(np.float32) / 2.0 ** (bits - 1)).mean(axis=1)
    p = str(tmp_path / "a.wav")
    scipy.io.wavfile.write(p, 22050, data)
    got = X.read_wav(p)
    assert got.dtype == np.float32 and got.shape == (3000,) and np.allclose(got, want, rtol=0, atol=1e-7)
    scipy.io.wavfile.write(p, 22050, data[:, 0])
    assert np.allclose(X.read_wav(p), want * 0 + (data[:, 0].astype(np.float64) - (128 if kind == "uint8" else 0)) /
                       (1.0 if kind == "float32" else (128 if kind == "uint8" else 2.0 ** (8 * data.dtype.itemsize - 1))), atol=1e-7)
    scipy.io.wavfile.write(p, 16000, data)
    with pytest.raises(ValueError, match="22050"):
        X.read_wav(p)


def test_reference_constants_only():
    X.MelSpectrogram(sr=22050, nfft=1024, fmin=125, fmax=7600, nmels=80, hoplen=256, spec_power=1)
    for bad in (dict(sr=16000), dict(nfft=2048), dict(nmels=128), dict(hoplen=512), dict(spec_power=2), dict(fmax=8000)):
        kw = dict(sr=22050, nfft=1024, fmin=125, fmax=7600, nmels=80, hoplen=256, spec_power=1)
        kw.update(bad)
        with pytest.raises(ValueError):
            X.MelSpectrogram(**kw)
    with pytest.raises(ValueError):
        X.MelSpectrogram(22050, 1024, 125, 7600, 80, 256, 1, inverse=True)
    with pytest.raises(NotImplementedError):
        X.get_spectrogram("x.wav", "out", 220500, folder_name="melspec_other")


def test_extract_mel_dry_run_lists_files(tmp_path):
    src = tmp_path / "in"
    (src / "sub").mkdir(parents=True)
    for p in ("b.wav", "a.wav", "sub/c.v1.wav", "notes.txt"):
        (src / p).write_bytes(b"")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "extract_mel.py"), "-i", str(src), "-o", str(tmp_path / "out"), "--dry-run"],
                       capture_output=True, text=True, check=True)
    d = json.loads(r.stdout.strip().splitlines()[-1])
    assert d["n_files"] == 3 and d["length"] == 220500
    assert [os.path.relpath(f["mel"], str(tmp_path / "out")) for f in d["files"]] == ["a_mel.npy", "b_mel.npy", os.path.join("sub", "c_mel.npy")]


def test_entry_points_declared_and_bound():
    hdr = open(os.path.join(ROOT, "include", "diffsound_b200.h")).read()
    from diffsound_b200 import _lib
    for name in ("dsb_wav_frames_f16", "dsb_mel_log"):
        assert re.search(r"\bint " + name + r"\(", hdr) and name in _lib.SIGNATURES
    assert "#define DSB_WAV_SCALE 8192.0f" in hdr and "#define DSB_WAV_LIMIT 4.0f" in hdr
    assert (ops.WAV_SCALE, ops.WAV_LIMIT) == (8192.0, 4.0)


def _tool(name):
    cand = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", name)
    return cand if os.access(cand, os.X_OK) else shutil.which(name)


def test_mel_kernels_sass_has_no_spills_or_local_memory(tmp_path):
    nvcc, cuobjdump = _tool("nvcc"), _tool("cuobjdump")
    if not nvcc or not cuobjdump:
        pytest.skip("nvcc / cuobjdump not installed")
    csrc = os.path.join(ROOT, "text-to-sound-synthesis_b200", "csrc")
    out = str(tmp_path / "mel.cubin")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo", "--expt-relaxed-constexpr", "-I",
                        os.path.join(ROOT, "include"), "-I", csrc, "-Xptxas", "-v", "-cubin", os.path.join(csrc, "mel.cu"), "-o", out],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    props = re.findall(r"Function properties for (\S+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert {p[0] for p in props} >= {"_ZN3dsb21wav_frames_f16_kernelEPKfxiiP6__halfiPi", "_ZN3dsb14mel_log_kernelEPKfxxiiPKiS3_S1_iiPf"}
    assert all(p[1:] == ("0", "0", "0") for p in props), props
    sass = subprocess.run([cuobjdump, "-sass", out], capture_output=True, text=True, check=True).stdout
    assert not re.search(r"\b(LDL|STL)\b", sass)
