"""Drop-in for the reference's Codebook/feature_extraction/extract_mel_spectrogram.py (and Diffsound/vocoder/mel2wav/extract_mel_spectrogram.py):
the SpecVQGAN transform from 22050 Hz audio to (80, <= 860) log-mel spectrograms in [0, 1], computed on the GPU by MelEngine.

  TRANSFORMS(y)                      numpy 1-D clip -> numpy (80, min(1 + len(y) // 256, 860)) float32
  get_spectrogram(path, save_dir, length, folder_name='melspec_10s_22050hz', save_results=True)
                                     the reference's signature and pad / trim rule; writes <name>_mel.npy (save_results) or returns (y, mel)
  mel_spectrogram(wav)               batched: CUDA (B, length) -> (B, 80, min(1 + length // 256, 860)) fp32
  read_wav(path)                     what librosa.load(path, sr=22050) returns for a 22050 Hz WAV (no resampling)

Only the reference's constants are supported (sr 22050, n_fft 1024, hop 256, 80 mels over 125 ... 7600 Hz, magnitude spectrum); inverse
transforms and resampling are not provided.
"""
from __future__ import annotations

import os

import numpy as np
import scipy.io.wavfile
import torch

from .. import mel_engine as _me

_ENGINES = {}


def _engine(device) -> _me.MelEngine:
    if device not in _ENGINES:
        _ENGINES[device] = _me.MelEngine(device)
    return _ENGINES[device]


class MelSpectrogram:
    """The reference's MelSpectrogram(sr, nfft, fmin, fmax, nmels, hoplen, spec_power) restricted to the one configuration TRANSFORMS uses;
    other values (and inverse=True) are refused."""
    CONFIG = dict(sr=_me.SR, nfft=_me.N_FFT, fmin=_me.FMIN, fmax=_me.FMAX, nmels=_me.N_MELS, hoplen=_me.HOP, spec_power=1)

    def __init__(self, sr, nfft, fmin, fmax, nmels, hoplen, spec_power, inverse=False):
        given = dict(sr=sr, nfft=nfft, fmin=fmin, fmax=fmax, nmels=nmels, hoplen=hoplen, spec_power=spec_power)
        bad = {k: v for k, v in given.items() if float(v) != float(self.CONFIG[k])}
        if bad or inverse:
            raise ValueError(f"only the SpecVQGAN transform {self.CONFIG} is supported (forward only), got {bad or 'inverse=True'}")


class _Transforms:
    """TRANSFORMS: MelSpectrogram -> LowerThresh(1e-5) -> Log10 -> *20 -> -20 -> +100 -> /100 -> Clip(0, 1) -> TrimSpec(860)."""

    def __call__(self, y):
        y = np.asarray(y)
        if y.ndim != 1:
            raise ValueError(f"TRANSFORMS takes a 1-D clip, got shape {y.shape}")
        wav = torch.from_numpy(np.ascontiguousarray(y, dtype=np.float32)).to(_default_device())[None]
        return mel_spectrogram(wav)[0].cpu().numpy()


TRANSFORMS = _Transforms()


def _default_device():
    if not torch.cuda.is_available():
        raise RuntimeError("the mel spectrogram runs on a CUDA device (no CPU fallback)")
    return torch.device("cuda", torch.cuda.current_device())


def mel_spectrogram(wav: torch.Tensor) -> torch.Tensor:
    """(B, length) or (length,) audio on a CUDA device -> (B, 80, min(1 + length // 256, 860)) fp32 log-mel (the batch dimension is kept only if
    given).  length must exceed 512 (librosa's reflect padding needs it)."""
    if not wav.is_cuda:
        raise RuntimeError("mel_spectrogram needs a CUDA tensor (no CPU fallback)")
    one = wav.dim() == 1
    out = _engine(wav.device)(wav[None] if one else wav)
    return out[0] if one else out


def read_wav(path) -> np.ndarray:
    """float32 mono samples of a 22050 Hz WAV as librosa.load(path, sr=22050) gives them: integer PCM divided by full scale (2^(bits-1); 8-bit
    unsigned centred at 128), channels averaged.  Any other rate raises ValueError (resampling is out of scope)."""
    sr, data = scipy.io.wavfile.read(path)
    if sr != _me.SR:
        raise ValueError(f"{path}: sample rate {sr} Hz, expected {_me.SR} Hz (resample it first)")
    if data.dtype == np.uint8:
        x = (data.astype(np.float32) - 128.0) / 128.0
    elif np.issubdtype(data.dtype, np.integer):
        x = data.astype(np.float32) / float(2 ** (8 * data.dtype.itemsize - 1))
    elif np.issubdtype(data.dtype, np.floating):
        x = data.astype(np.float32)
    else:
        raise ValueError(f"{path}: unsupported sample type {data.dtype}")
    if x.ndim == 2:
        x = x.mean(axis=1, dtype=np.float32)
    return x


def pad_or_trim(wav, length: int) -> np.ndarray:
    """get_spectrogram's rule: zeros after a short clip, the first `length` samples of a long one (float64, as the reference's np.zeros)."""
    length = int(length)
    if length <= _me.N_FFT // 2:
        raise ValueError(f"length must exceed {_me.N_FFT // 2} samples (reflect padding), got {length}")
    y = np.zeros(length)
    n = min(len(wav), length)
    y[:n] = wav[:n]
    return y


def mel_file_name(audio_path) -> str:
    """<name>_mel.npy, name = the file name up to its first '.' (the reference's audio_name)."""
    return os.path.basename(str(audio_path)).split(".")[0] + "_mel.npy"


def get_spectrogram(audio_path, save_dir, length, folder_name="melspec_10s_22050hz", save_results=True):
    if folder_name != "melspec_10s_22050hz":
        raise NotImplementedError(folder_name)
    y = pad_or_trim(read_wav(audio_path), length)
    mel_spec = TRANSFORMS(y)
    if save_results:
        os.makedirs(save_dir, exist_ok=True)
        np.save(os.path.join(save_dir, mel_file_name(audio_path)), mel_spec)
    else:
        return y, mel_spec
