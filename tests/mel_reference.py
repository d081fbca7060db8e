"""Plain-torch restatements of the two mel kernels' contracts (include/diffsound_b200.h: dsb_wav_frames_f16, dsb_mel_log) and the error bound
of the GPU log-mel against the fp64 oracle.  TEST INFRASTRUCTURE -- never imported by the product package."""
import math

import numpy as np
import torch

SCALE, LIMIT, HOP, PAD = 8192.0, 4.0, 256, 512


def frames_f16(wav, rows=None):
    """dsb_wav_frames_f16: (B, length) fp32 -> (B, rows, 512) fp16 [hi | lo] of 2^13 * the reflect-padded clip, zeros past its end."""
    wav = wav.float().cpu()
    B, length = wav.shape
    rows = length // HOP + 4 if rows is None else rows
    p = torch.nn.functional.pad(wav[:, None], (PAD, PAD), mode="reflect")[:, 0]
    full = torch.zeros(B, rows * HOP)
    n = min(p.shape[1], rows * HOP)                                              # the last frame ends at 256 (length // 256) + 1024
    full[:, :n] = p[:, :n]
    s = full * SCALE
    h = s.to(torch.float16)
    lo = (s - h.float()).to(torch.float16)
    return torch.cat([h.view(B, rows, HOP), lo.view(B, rows, HOP)], dim=2)


def mel_log(spec, n_bins, fb_start, fb_len, fb_w, T_out):
    """dsb_mel_log's arithmetic in fp64 on the given fp32 spectra (the exact value its fp32 steps approximate)."""
    s = spec.double().cpu()[:, :T_out, :2 * n_bins].reshape(spec.shape[0], T_out, n_bins, 2)
    mag = (s[..., 0] ** 2 + s[..., 1] ** 2).sqrt()                             # (B, T, n_bins)
    n_mels = fb_w.shape[0]
    dense = torch.zeros(n_mels, n_bins, dtype=torch.float64)
    for m in range(n_mels):
        a, n = int(fb_start[m]), int(fb_len[m])
        dense[m, a:a + n] = fb_w[m, :n].double().cpu()
    mel = torch.einsum("mk,btk->bmt", dense, mag)
    return log_steps(mel), mel, dense


def log_steps(mel):
    y = (20.0 * torch.log10(mel.clamp_min(1e-5)) - 20.0 + 100.0) / 100.0
    return y.clamp(0.0, 1.0)


# fp32 rounding of the kernel's own steps after the mel sum (log10f within 2 ulp, then *20, -20, +100, /100 each rounded): below 1e-6 in y
STEP_ERR = 1e-6


def bound_from_mel(mel, dmel):
    """Per-element bound on |y(mel') - y(mel)| for |mel' - mel| <= dmel, y = the clipped log steps (monotone), plus STEP_ERR."""
    y = log_steps(mel)
    return torch.maximum(log_steps(mel + dmel) - y, y - log_steps((mel - dmel).clamp_min(0.0))) + STEP_ERR


# The split-fp16 DFT: each operand is a (hi | lo) pair carrying 22 bits (|x - hi - lo| <= 2^-22 |x|, the dropped lo*lo term <= 2^-22 |x w|),
# so the products are within 3 * 2^-22 of x*w; the fp32 accumulation runs 16 k-blocks of 3 x 64 products inside wgmma, each promoted into the
# fp32 accumulator with an FADD: at most 208 roundings in sequence, each within 2^-23 (allowing truncation inside the MMA).
EPS_DFT = 3 * 2.0 ** -22 + 208 * 2.0 ** -23


def full_path_bound(y, basis_f32, mel_true):
    """Bound on |GPU log-mel - oracle log-mel| per (mel, frame) of clip y (fp64, after pad / trim), mel_true (80, T_out) the oracle's mel.

    Each DFT output (re or im) of frame t is within EPS_DFT * A_t of its exact value, A_t = sum_n |x_n| w_n over the frame; so |X_k| is within
    sqrt(2) EPS_DFT A_t (+ 2 ulp for the fp32 magnitude), and the filter sum within sum_k f_mk of that, plus (n_m + 1) 2^-24 of the mel for its
    n_m fp32 FMAs.  That bound on the mel is carried through the monotone log steps (bound_from_mel)."""
    T = mel_true.shape[1]
    p = np.pad(np.asarray(y, dtype=np.float64), PAD, mode="reflect")
    idx = np.arange(T)[:, None] * HOP + np.arange(1024)[None, :]
    win = 0.5 - 0.5 * np.cos(2 * np.pi * np.arange(1024) / 1024)
    A = torch.from_numpy(np.abs(p[idx]) @ win)                                   # (T,)
    bas = torch.from_numpy(basis_f32.astype(np.float64))
    width = (bas != 0).sum(1).double()
    mel = torch.as_tensor(mel_true, dtype=torch.float64)
    dmel = bas.sum(1)[:, None] * math.sqrt(2) * EPS_DFT * A[None, :] + (width[:, None] + 3) * 2.0 ** -24 * mel
    return bound_from_mel(mel, dmel)
