"""SpecVQGAN's log-mel spectrogram on sm_90a (reference Codebook/feature_extraction/extract_mel_spectrogram.py, TRANSFORMS :141-151, with
librosa 0.8.0's stft and filters.mel): 22050 Hz audio -> (80, <= 860) mels in [0, 1].

Three launches per batch, captured once per (B, length) as a CUDA graph:
  * dsb_wav_frames_f16: the reflect-padded clip as rows of 256 samples, split-fp16 pairs of 2^13 x;
  * dsb_gemm_ex: the periodic-Hann windowed DFT as a 4-tap conv over those rows (frame t = rows t ... t+3), split-fp16 3-pass form, fp32 out.
    Only the 347 bins 6 ... 352 that some mel filter covers are computed: N = 694 columns (re, im interleaved), padded to 696;
  * dsb_mel_log: |X|, the sparse filterbank, max(., 1e-5), log10, *20, -20, +100, /100, clip(0, 1), mel-major.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from . import ops
from .graphs import GraphCache
from .packing import PackedConv

SR, N_FFT, HOP, FMIN, FMAX, N_MELS, MAX_FRAMES = 22050, 1024, 256, 125.0, 7600.0, 80, 860
N_TAPS = N_FFT // HOP


def _hz_to_mel(f):
    """librosa.hz_to_mel(htk=False): the Slaney scale, linear below 1 kHz, logarithmic above."""
    f = np.asarray(f, dtype=np.float64)
    f_sp, min_log_hz = 200.0 / 3, 1000.0
    min_log_mel, logstep = min_log_hz / f_sp, math.log(6.4) / 27.0
    return np.where(f >= min_log_hz, min_log_mel + np.log(np.maximum(f, 1e-300) / min_log_hz) / logstep, f / f_sp)


def _mel_to_hz(m):
    m = np.asarray(m, dtype=np.float64)
    f_sp, min_log_hz = 200.0 / 3, 1000.0
    min_log_mel, logstep = min_log_hz / f_sp, math.log(6.4) / 27.0
    return np.where(m >= min_log_mel, min_log_hz * np.exp(logstep * (m - min_log_mel)), f_sp * m)


def mel_basis() -> np.ndarray:
    """librosa.filters.mel(sr=22050, n_fft=1024, fmin=125, fmax=7600, n_mels=80) as librosa 0.8.0 stores it: triangles in fp64 rounded to
    float32, then times the Slaney area normalisation 2 / (f[m+2] - f[m]) and rounded to float32 again."""
    fftfreqs = np.linspace(0, SR / 2, 1 + N_FFT // 2)
    mel_f = _mel_to_hz(np.linspace(_hz_to_mel(FMIN), _hz_to_mel(FMAX), N_MELS + 2))
    fdiff = np.diff(mel_f)
    ramps = np.subtract.outer(mel_f, fftfreqs)
    w = np.zeros((N_MELS, 1 + N_FFT // 2), dtype=np.float32)
    for i in range(N_MELS):
        w[i] = np.maximum(0, np.minimum(-ramps[i] / fdiff[i], ramps[i + 2] / fdiff[i + 1]))
    w *= (2.0 / (mel_f[2:N_MELS + 2] - mel_f[:N_MELS]))[:, None]
    return w


def filter_table(basis: np.ndarray):
    """The filterbank's support (first bin, number of bins) and its compact form: per filter the first bin (relative to the support's first),
    the number of bins and the float32 weights, zero-padded to the widest filter."""
    nz = np.nonzero(basis.any(axis=0))[0]
    k0, nb = int(nz[0]), int(nz[-1]) - int(nz[0]) + 1
    starts, lens, rows = [], [], []
    for m in range(basis.shape[0]):
        idx = np.nonzero(basis[m])[0]
        starts.append(int(idx[0]) - k0)
        lens.append(int(idx[-1]) - int(idx[0]) + 1)
        rows.append(basis[m, idx[0]:idx[-1] + 1])
    w = np.zeros((basis.shape[0], max(lens)), dtype=np.float32)
    for m, r in enumerate(rows):
        w[m, :len(r)] = r
    return k0, nb, np.array(starts, dtype=np.int32), np.array(lens, dtype=np.int32), w


def dft_weights(k0: int, nb: int, n_cols: int) -> np.ndarray:
    """(n_cols, 1024) fp64: row 2i = w[n] cos(2 pi k n / 1024), row 2i + 1 = -w[n] sin(2 pi k n / 1024) for bin k = k0 + i, w the periodic Hann
    window; the argument is reduced exactly as (k n) mod 1024.  Rows past 2 nb are zero."""
    n = np.arange(N_FFT)
    win = 0.5 - 0.5 * np.cos(2 * np.pi * n / N_FFT)
    k = np.arange(k0, k0 + nb)
    ang = 2 * np.pi * ((k[:, None] * n[None, :]) % N_FFT) / N_FFT
    out = np.zeros((n_cols, N_FFT))
    out[0:2 * nb:2] = win * np.cos(ang)
    out[1:2 * nb:2] = -win * np.sin(ang)
    return out


def frames_out(length: int) -> int:
    """Frames librosa.stft(center=True) gives, 1 + length // 256, and how many TrimSpec(860) keeps."""
    return min(1 + length // HOP, MAX_FRAMES)


class MelEngine:
    """TRANSFORMS of the reference on a batch of clips: __call__(wav (B, length) fp32 CUDA) -> (B, 80, min(1 + length // 256, 860)) fp32."""

    def __init__(self, device="cuda"):
        self.device = torch.device(device)
        if self.device.type == "cuda" and self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        basis = mel_basis()
        self.k0, self.n_bins, starts, lens, w = filter_table(basis)
        self.n_cols = (2 * self.n_bins + 7) // 8 * 8  # fp32 output rows 16-byte aligned for the GEMM's stores
        dft = torch.from_numpy(dft_weights(self.k0, self.n_bins, self.n_cols)).to(self.device)
        self.dft = PackedConv([dft[:, j * HOP:(j + 1) * HOP] for j in range(N_TAPS)], torch.zeros(self.n_cols, device=self.device))
        self.fb_start = torch.from_numpy(starts).to(self.device)
        self.fb_len = torch.from_numpy(lens).to(self.device)
        self.fb_w = torch.from_numpy(w).to(self.device)
        self._ws = {}
        self._graphs = GraphCache()

    def _alloc(self, B, length):
        T = 1 + length // HOP
        frames = torch.empty(B, ops.wav_frame_rows(length), 2 * HOP, dtype=torch.float16, device=self.device)
        spec = torch.empty(B, T, self.n_cols, dtype=torch.float32, device=self.device)
        err = torch.zeros(1, dtype=torch.int32, device=self.device)
        return frames, spec, err

    def _run(self, wav):
        B, length = wav.shape
        ws = self._ws.get((B, length))
        if ws is None:
            ws = self._ws[(B, length)] = self._alloc(B, length)
        frames, spec, err = ws
        R, T = frames.shape[1], spec.shape[1]
        err.zero_()
        ops.wav_frames_f16(wav, frames, rows=R, err_flag=err)
        self.dft.launch(spatial=[(j, 0, HOP, 0) for j in range(N_TAPS)], A=frames.data_ptr(), out=spec.data_ptr(), M=T, lda=2 * HOP, ldo=self.n_cols,
                        batch=B, a_rows=R, a_cols=2 * HOP, a_batch_stride=R * 2 * HOP, out_batch_stride=T * self.n_cols, dtype=ops.F16,
                        alpha=1.0 / ops.WAV_SCALE)
        out = ops.mel_log(spec, self.n_bins, self.fb_start, self.fb_len, self.fb_w, frames_out(length))
        return out, err

    @torch.no_grad()
    def __call__(self, wav: torch.Tensor, *, use_graph: bool = True) -> torch.Tensor:
        if wav.dim() != 2:
            raise ValueError(f"MelEngine takes (B, length) audio, got shape {tuple(wav.shape)}")
        B, length = wav.shape
        if length <= N_FFT // 2:
            raise ValueError(f"clips must be longer than {N_FFT // 2} samples (librosa's reflect padding), got {length}")
        if wav.device != self.device:
            raise RuntimeError(f"MelEngine on {self.device} got audio on {wav.device} (no CPU fallback)")
        wav = wav.float().contiguous()
        if use_graph:
            out, err = self._graphs.run((B, length), self._run, wav)
        else:
            out, err = self._run(wav)
        if int(err.item()):
            raise RuntimeError(f"audio samples must be finite with |x| < {ops.WAV_LIMIT:g}")
        return out
