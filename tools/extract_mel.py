"""WAV clips -> SpecVQGAN log-mel spectrograms on the GPU (the reference's Codebook/feature_extraction/extract_mel_spectrogram.py CLI).

    python tools/extract_mel.py -i clips/ -o data/features/val/melspec_10s_22050hz [-l 220500] [--batch 64] [--workers 8]
    python tools/extract_mel.py -i clips/ -o out/ --dry-run        # list input -> output files; no GPU

Every *.wav under the input directory (searched recursively, sorted) becomes <output>/<same subdirectory>/<name>_mel.npy, an (80, <= 860)
float32 array: the layout tools/evaluate_samples.py --reals reads.  Files are read on a thread pool, padded or cut to --length samples as
get_spectrogram does, and run through the GPU in batches.  Clips must be 22050 Hz (no resampling).  Prints one JSON summary line.
"""
import argparse
import json
import os
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def plan(input_dir, output_dir):
    """[(wav path, mel path)] in sorted order."""
    found = []
    for d, _, files in os.walk(input_dir):
        found += [os.path.join(d, f) for f in files if f.lower().endswith(".wav")]
    found.sort()
    out = []
    for p in found:
        rel = os.path.relpath(os.path.dirname(p), input_dir)
        out.append((p, os.path.normpath(os.path.join(output_dir, rel, os.path.basename(p).split(".")[0] + "_mel.npy"))))
    return out


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("-i", "--input_dir", required=True)
    ap.add_argument("-o", "--output_dir", required=True)
    ap.add_argument("-l", "--length", type=int, default=220500)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--workers", type=int, default=8, help="threads reading WAV files")
    ap.add_argument("--dry-run", action="store_true")
    a = ap.parse_args(argv)
    if a.length <= 512:
        ap.error("--length must exceed 512 samples (reflect padding)")
    jobs = plan(a.input_dir, a.output_dir)
    if a.dry_run:
        print(json.dumps({"n_files": len(jobs), "length": a.length, "files": [{"wav": w, "mel": m} for w, m in jobs]}))
        return 0
    import torch
    import _pkg
    _pkg.load()
    from diffsound_b200.feature_extraction import extract_mel_spectrogram as X
    dev = torch.device("cuda", torch.cuda.current_device())
    load = lambda p: X.pad_or_trim(X.read_wav(p), a.length).astype(np.float32)
    t0 = time.perf_counter()
    with ThreadPoolExecutor(a.workers) as pool:
        for s in range(0, len(jobs), a.batch):
            chunk = jobs[s:s + a.batch]
            wav = torch.from_numpy(np.stack(list(pool.map(load, [w for w, _ in chunk])))).to(dev)
            mels = X.mel_spectrogram(wav).cpu().numpy()
            for (_, m), mel in zip(chunk, mels):
                os.makedirs(os.path.dirname(m), exist_ok=True)
                np.save(m, mel)
    dt = time.perf_counter() - t0
    print(json.dumps({"n_files": len(jobs), "length": a.length, "seconds": round(dt, 3), "clips_per_s": round(len(jobs) / dt, 2) if dt else None}))
    return 0


if __name__ == "__main__":
    sys.exit(main())
