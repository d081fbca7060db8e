"""Caption generated clips with ACT (Codebook/AudiocaptionLoss/eval.py:277-279): greedy and beam sizes 2 and 3, on the H100.

    python tools/caption_samples.py --fakes samples/ --captions val.csv --ckpt ACTm.pth --vocab words_list.p --out DIR [--dry-run]

Pairs every `<stem>_mel_sample_<j>.npy` (pipeline.save_clip's names, 80 x 848) with the five reference captions of `<stem>.wav` in the CSV,
reads each mel transposed to (848, 80) as the reference's TTS_eval loader does, and writes per mode `DIR/<mode>_predictions.csv`
(file_name, caption_predicted) and `DIR/<mode>_references.csv` (file_name, caption_1 ... caption_5): the two tables the reference's
evaluate_metrics reads.  Prints one JSON line with clips/s per mode, the GPU name and its power limit.  --dry-run only pairs the files.
The ACT config is the released settings.yaml decoder (nhid 512, 4 layers, 8 heads, feed-forward 2048, GELU)."""
import argparse
import csv
import json
import os
import re
import subprocess
import sys
import time
from types import SimpleNamespace as NS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools.generate_samples import read_captions  # noqa: E402

MODES = (("greedy", 0), ("beam2", 2), ("beam3", 3))


def pair_files(fakes, captions):
    caps = read_captions(captions)
    pairs = []
    for name in sorted(os.listdir(fakes)):
        m = re.fullmatch(r"(.+)_mel_sample_(\d+)\.npy", name)
        if not m:
            continue
        refs = caps.get(m.group(1) + ".wav")
        if refs is None:
            raise SystemExit(f"{name}: no captions for {m.group(1)}.wav in {captions}")
        if len(refs) != 5:
            raise SystemExit(f"{m.group(1)}.wav has {len(refs)} captions in {captions}, the caption metrics need 5")
        pairs.append((os.path.join(fakes, name), m.group(1) + ".wav", refs))
    if not pairs:
        raise SystemExit(f"no <stem>_mel_sample_<j>.npy files in {fakes}")
    return pairs


def words_of(ids, words_list, eos_ind):
    """eval.py's post-processing of one decoded row (eval_greedy / eval_beam, then decode_output): drop <sos>; a row with no <eos> gets
    eos_ind written over its last word; the caption is the words before the first '<eos>'."""
    row = list(ids[1:])
    if row and eos_ind not in row:
        row[-1] = eos_ind
    out = [words_list[i] for i in row]
    if "<eos>" in out:
        out = out[:out.index("<eos>")]
    return " ".join(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--fakes", required=True)
    ap.add_argument("--captions", required=True)
    ap.add_argument("--ckpt", required=True)
    ap.add_argument("--vocab", required=True)
    ap.add_argument("--out", required=True)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--dry-run", action="store_true")
    a = ap.parse_args()
    pairs = pair_files(a.fakes, a.captions)
    if a.dry_run:
        print(json.dumps(dict(clips=len(pairs), captions_per_clip=5, modes=[m for m, _ in MODES])))
        return
    import pickle

    import numpy as np
    import torch
    import _pkg
    _pkg.load()
    from diffsound_b200.evaluation.audiocaption import ACT, beam_decode, greedy_decode
    with open(a.vocab, "rb") as f:
        words_list = pickle.load(f)
    sos, eos = words_list.index("<sos>"), words_list.index("<eos>")
    cfg = NS(encoder=NS(model="audioset", freeze=False, pretrained=False),
             decoder=NS(nhead=8, nhid=512, nlayers=4, dropout=0.2, dim_feedforward=2048, activation="gelu"),
             word_embedding=NS(pretrained=False, freeze=False), path=NS())
    model = ACT(cfg, len(words_list))
    model.load_state_dict(torch.load(a.ckpt, map_location="cpu")["model"])
    model = model.cuda().eval()
    os.makedirs(a.out, exist_ok=True)
    rates = {}
    for mode, bw in MODES:
        preds = []
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for i in range(0, len(pairs), a.batch):
            chunk = pairs[i:i + a.batch]
            x = torch.from_numpy(np.stack([np.load(p).T for p, _, _ in chunk]).astype(np.float32)).cuda()
            ids = greedy_decode(model, x, sos, eos, 30) if bw == 0 else beam_decode(x, model, sos, eos, beam_width=bw)
            preds += [words_of(r, words_list, eos) for r in ids.tolist()]
        torch.cuda.synchronize()
        rates[mode] = len(pairs) / (time.perf_counter() - t0)
        with open(os.path.join(a.out, f"{mode}_predictions.csv"), "w", newline="") as f:
            w = csv.writer(f)
            w.writerow(["file_name", "caption_predicted"])
            w.writerows([(wav, p) for (_, wav, _), p in zip(pairs, preds)])
        with open(os.path.join(a.out, f"{mode}_references.csv"), "w", newline="") as f:
            w = csv.writer(f)
            w.writerow(["file_name"] + [f"caption_{k}" for k in range(1, 6)])
            w.writerows([[wav] + refs for _, wav, refs in pairs])
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps(dict(clips=len(pairs), clips_per_s={k: round(v, 2) for k, v in rates.items()}, gpu=smi)))


if __name__ == "__main__":
    main()
