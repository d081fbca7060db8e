"""fp64 numpy restatement of SpecVQGAN's mel front end (reference Codebook/feature_extraction/extract_mel_spectrogram.py: get_spectrogram
:166-187, TRANSFORMS :141-151) as librosa 0.8.0 computes it, with only the mel basis rounded to float32 as librosa stores it:
  1. y = the clip zero-padded or cut to `length`;
  2. |stft(y, n_fft=1024, hop_length=256)|: center=True reflect padding of 512, periodic Hann window, 1 + length // 256 frames;
  3. mel_basis @ spec, mel_basis = filters.mel(sr=22050, n_fft=1024, fmin=125, fmax=7600, n_mels=80) (Slaney scale and area norm);
  4. max(1e-5, .), log10, *20, -20, +100, /100, clip(0, 1), the first 860 frames.
Written independently of the package (the tests pin it to torch.stft and torchaudio's Slaney filterbank)."""
import numpy as np

SR, N_FFT, HOP, FMIN, FMAX, N_MELS, MAX_FRAMES = 22050, 1024, 256, 125.0, 7600.0, 80, 860


def hz_to_mel(f):
    f = np.atleast_1d(np.asarray(f, dtype=np.float64))
    out = f / (200.0 / 3)
    hi = f >= 1000.0
    out[hi] = 15.0 + np.log(f[hi] / 1000.0) / (np.log(6.4) / 27.0)
    return out


def mel_to_hz(m):
    m = np.atleast_1d(np.asarray(m, dtype=np.float64))
    out = m * (200.0 / 3)
    hi = m >= 15.0
    out[hi] = 1000.0 * np.exp((np.log(6.4) / 27.0) * (m[hi] - 15.0))
    return out


def mel_basis():
    """(80, 513) float32, librosa.filters.mel's arithmetic: float32 triangles, then the fp64 Slaney norm, rounded to float32 again."""
    freqs = np.arange(N_FFT // 2 + 1) * (SR / N_FFT)
    edges = mel_to_hz(np.linspace(hz_to_mel(FMIN)[0], hz_to_mel(FMAX)[0], N_MELS + 2))
    out = np.zeros((N_MELS, N_FFT // 2 + 1), dtype=np.float32)
    for m in range(N_MELS):
        lo, c, hi = edges[m], edges[m + 1], edges[m + 2]
        up = (freqs - lo) / (c - lo)
        down = (hi - freqs) / (hi - c)
        tri = np.clip(np.minimum(up, down), 0.0, None).astype(np.float32)
        out[m] = (tri.astype(np.float64) * (2.0 / (hi - lo))).astype(np.float32)
    return out


def pad_or_trim(wav, length):
    """get_spectrogram's rule: zeros after a short clip, the first `length` samples of a long one (fp64)."""
    wav = np.asarray(wav, dtype=np.float64)
    y = np.zeros(length)
    n = min(len(wav), length)
    y[:n] = wav[:n]
    return y


def stft_mag(y):
    """(513, 1 + len(y) // 256) fp64 |STFT| with librosa.stft's framing."""
    y = np.asarray(y, dtype=np.float64)
    p = np.pad(y, N_FFT // 2, mode="reflect")
    T = 1 + len(y) // HOP
    win = 0.5 - 0.5 * np.cos(2 * np.pi * np.arange(N_FFT) / N_FFT)
    idx = np.arange(T)[:, None] * HOP + np.arange(N_FFT)[None, :]
    return np.abs(np.fft.rfft(p[idx] * win, axis=1)).T


def mel_power(y, basis=None):
    """(80, T) fp64 mel_basis @ |STFT| before the log steps."""
    basis = mel_basis() if basis is None else basis
    return basis.astype(np.float64) @ stft_mag(y)


def log_steps(mel):
    """Steps 4 of the transform on a mel (fp64), trimmed to 860 frames."""
    y = (20.0 * np.log10(np.maximum(1e-5, mel)) - 20.0 + 100.0) / 100.0
    return np.clip(y, 0.0, 1.0)[:, :MAX_FRAMES]


def log_mel(y):
    """TRANSFORMS(y): (80, min(1 + len(y) // 256, 860)) fp64."""
    return log_steps(mel_power(y))
