"""Validation loss and perplexity of the autoregressive SpecVQGAN transformer (Codebook/configs/caps_transformer*.yaml) on the H100 kernels: the
`val/loss` Net2NetTransformer.validation_step logs (cond_transformer.py:353-370), over caption / mel pairs.

    python tools/ar_val_loss.py --config caps_transformer.yaml --ckpt last.ckpt --clip-ckpt ViT-B-32.pt --captions val.csv \\
        --mels data/features/val/melspec_10s_22050hz [--batch-size 64] [--bpe vocab.txt.gz] [--codec-ckpt codebook.ckpt]

Every caption of the CSV (`file_name,caption`) is scored against the mel `<file name without extension>_mel.npy` found anywhere under --mels
(tools/extract_mel.py mirrors its input's subdirectories; a needed name found twice is refused).  The mel is prepared as the configs' validation data
prepares it (Codebook/specvqgan/data/caps.py VASSpecs): center-cropped to 80 x 848 (CropImage, random_crop: False), then mapped from the
log-mel's [0, 1] to the codec's [-1, 1] as `image = 2 * input - 1`.  The condition is the caption's CLIP ViT-B/32 pooled text feature
(tools/generate_samples_ar.py's caption_features).  Each batch runs validation_step in one causal pass; the result is the token-weighted mean
loss over all 265 tokens of every pair and its perplexity exp(loss).

The reference's validation set pairs each mel with one caption, its first (caps.py VASFeats loads `<vid>1`'s feature).  This tool scores every
caption in the CSV, so its number equals the reference's `val/loss` when the CSV lists only the first caption of each clip; with all captions it
is the mean over every (caption, mel) pair.

--dry-run builds the model on the CPU, reads the captions, pairs each with its mel (shapes checked) and stops before the first kernel."""
import argparse
import math
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import _pkg  # noqa: E402

_pkg.load()
from tools import generate_samples_ar as G  # noqa: E402
from tools.generate_samples import read_captions  # noqa: E402

MEL_SHAPE = (80, 848)  # spec_crop_len 848 of the caps_transformer configs' data block
TOKENS = G.GRID[0] * G.GRID[1]


def pair_mels(caps, mel_dir):
    """[(mel path, caption)] for every caption in file order, the mel found by name anywhere under mel_dir.  A missing mel raises
    FileNotFoundError and a name present in two subdirectories ValueError, each naming the file."""
    found = {}
    for d, _, files in os.walk(mel_dir):
        for f in files:
            if f.endswith("_mel.npy"):
                found.setdefault(f, []).append(os.path.join(d, f))
    jobs = []
    for name, texts in caps.items():
        key = os.path.basename(name).split(".")[0] + "_mel.npy"
        paths = sorted(found.get(key, []))
        if not paths:
            raise FileNotFoundError(f"no mel for {name}: no {key} under {mel_dir} (make it with tools/extract_mel.py)")
        if len(paths) > 1:
            raise ValueError(f"{key} is under --mels more than once: {', '.join(paths)}")
        jobs += [(paths[0], t) for t in texts]
    return jobs


def load_mel(path):
    """(80, W >= 848) log-mel in [0, 1] -> the codec's input: its center 80 x 848 crop (albumentations CenterCrop: offset (W - 848) // 2) as
    2 * crop - 1, fp32 (caps.py VASSpecs.__getitem__)."""
    m = np.load(path)
    h, w = m.shape
    if h < MEL_SHAPE[0] or w < MEL_SHAPE[1]:
        raise ValueError(f"{path}: mel {m.shape} is smaller than {MEL_SHAPE}")
    y, x = (h - MEL_SHAPE[0]) // 2, (w - MEL_SHAPE[1]) // 2
    crop = torch.from_numpy(np.ascontiguousarray(m[y:y + MEL_SHAPE[0], x:x + MEL_SHAPE[1]], dtype=np.float32))
    return 2 * crop - 1


@torch.no_grad()
def score(model, text, tokenizer, jobs, batch_size):
    """Token-weighted mean of validation_step's loss over the (mel path, caption) jobs, batch_size pairs per call; model and text on the GPU."""
    total, count = 0.0, 0
    for i in range(0, len(jobs), batch_size):
        chunk = jobs[i:i + batch_size]
        feats = G.caption_features(text, tokenizer, [t for _, t in chunk])  # (B, 512, 1)
        batch = {"image": torch.stack([load_mel(p) for p, _ in chunk]).cuda(), "feature": feats.permute(0, 2, 1)}
        loss = float(model.validation_step(batch, i // batch_size))
        total += loss * len(chunk) * TOKENS  # every token counts (no ignored targets)
        count += len(chunk) * TOKENS
    return total / count, count


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--config", required=True, help="Codebook/configs/caps_transformer*.yaml")
    ap.add_argument("--ckpt", default=None, help="Lightning checkpoint of the transformer ({'state_dict': ...})")
    ap.add_argument("--codec-ckpt", default=None, help="SpecVQGAN Lightning checkpoint (only needed if --ckpt does not hold first_stage_model.*)")
    ap.add_argument("--clip-ckpt", default=None, help="OpenAI CLIP ViT-B/32 weights (state_dict or TorchScript archive)")
    ap.add_argument("--bpe", default=None, help="bpe_simple_vocab_16e6.txt.gz (default: $DIFFSOUND_BPE_VOCAB or the reference checkout)")
    ap.add_argument("--captions", required=True, help="CSV with file_name,caption columns")
    ap.add_argument("--mels", required=True, help="directory searched recursively for <name>_mel.npy files (tools/extract_mel.py's output)")
    ap.add_argument("--batch-size", type=int, default=64)
    ap.add_argument("--dry-run", action="store_true")
    a = ap.parse_args(argv)
    a.vocoder_ckpt = None
    model, text, tokenizer, _ = G.build(a)
    jobs = pair_mels(read_captions(a.captions), a.mels)
    print(f"{len(jobs)} caption / mel pairs, batch {a.batch_size}")
    if a.dry_run:
        for path, _ in jobs:
            load_mel(path)
        return model, text, tokenizer, jobs
    model, text = model.cuda().eval(), text.cuda()
    mean, count = score(model, text, tokenizer, jobs, a.batch_size)
    print(f"val/loss {mean:.6f}  perplexity {math.exp(mean):.4f}  ({count} tokens)")
    return mean


if __name__ == "__main__":
    main()
