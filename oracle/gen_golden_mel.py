"""Writes tests/golden/audio_clips.npz: two real 22050 Hz int16 clips shipped with the reference (Codebook/vocoder_audioset/logs/audioset),
kept under half a megabyte: the whole of original_0 (220500 samples, get_spectrogram's default length) and the first 4 s of the MelGAN output
generated_0 (88200 samples, so that padding it to 220500 takes get_spectrogram's zero-pad branch).  Data only: the mel tests compute everything
else from these samples.

    python oracle/gen_golden_mel.py [reference checkout]     # default: oracle.ref_harness.REF_ROOT"""
import os
import sys

import numpy as np
import scipy.io.wavfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle.ref_harness import REF_ROOT  # noqa: E402

CLIPS = {"original_0": None, "generated_0": 4 * 22050}  # name -> samples kept (None: all)


def main(ref):
    src = os.path.join(ref, "Codebook", "vocoder_audioset", "logs", "audioset")
    out = {}
    for name, keep in CLIPS.items():
        sr, data = scipy.io.wavfile.read(os.path.join(src, name + ".wav"))
        assert sr == 22050 and data.dtype == np.int16 and data.ndim == 1, (name, sr, data.dtype, data.shape)
        out[name] = data[:keep]
    dst = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "audio_clips.npz")
    np.savez_compressed(dst, **out)
    print("wrote", dst, {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else REF_ROOT)
