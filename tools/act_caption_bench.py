"""ACT captioning throughput: the caption engine against the reference's algorithm (oracle/act_oracle.py: the whole prefix re-run for every
position or expanded node, fp32 torch on the same GPU), alternated in one process.

Workloads, B = 64 clips of 80 x 848 with seeded weights (nhid 512, 4 layers, V = 5000, the fixture's weight seed): 'cap' (random weights: the
beam searches run into the qsize > 2000 cut-off) and 'eos' (the <eos> logit biased by --eos-bias so that the beam searches end on <eos> after
some words, as a trained model's do; the default was chosen with the fp32 oracle on the CPU, and mean_words reports what the run produced).
Modes: greedy (30 words, no early stop) and beams 2 and 3.  The reference's greedy_decode is batched, so it runs on all B clips, as the
engine does; its beam search goes one clip at a time and is timed on the first --ref-clips clips, reported per clip.  Prints one JSON line."""
import argparse
import json
import os
import subprocess
import sys
import time
from types import SimpleNamespace as NS

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import _pkg  # noqa: E402

_pkg.load()
from diffsound_b200.evaluation.audiocaption import ACT, beam_decode, greedy_decode  # noqa: E402
from oracle import act_oracle as O  # noqa: E402

V, SOS, EOS, NHEAD = 5000, 0, 9, 8
WEIGHT_SEED, EOS_BIAS = 11, 2.3


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=64)
    ap.add_argument("--ref-clips", type=int, default=2)
    ap.add_argument("--eos-bias", type=float, default=EOS_BIAS)
    ap.add_argument("--reps", type=int, default=2)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "act_caption_bench measures on the GPU"
    cfg = NS(encoder=NS(model="audioset", freeze=False, pretrained=False),
             decoder=NS(nhead=NHEAD, nhid=512, nlayers=4, dropout=0.2, dim_feedforward=2048, activation="gelu"),
             word_embedding=NS(pretrained=False, freeze=False), path=NS())
    mels = O.seeded_mels(21, a.B).cuda()
    res = {}
    for wl, bias in (("cap", 0.0), ("eos", a.eos_bias)):
        m = ACT(cfg, V)
        m.load_state_dict(O.seeded_state_dict(m.state_dict(), WEIGHT_SEED, EOS, bias))
        m = m.cuda().eval()
        sd = {k: v.cuda() for k, v in m.state_dict().items()}
        greedy_decode(m, mels, SOS, EOS, 30)  # warm-up: packing, graphs
        for mode, bw in (("greedy", 0), ("beam2", 2), ("beam3", 3)):
            eng_t, ref_t, lens = [], [], []
            for _ in range(a.reps):
                t, ids = timed(lambda: greedy_decode(m, mels, SOS, EOS, 30) if bw == 0 else beam_decode(mels, m, SOS, EOS, beam_width=bw))
                eng_t.append(t)
                lens.append(float((ids[:, 1:] != EOS).sum(1).float().mean()))  # words after <sos>, <eos> and padding excluded

                def reference():
                    with torch.no_grad():
                        if bw == 0:
                            return O.greedy_decode(sd, O.encode(sd, mels, torch.float32), NHEAD, SOS, 30, torch.float32)
                        mem = O.encode(sd, mels[:a.ref_clips], torch.float32)
                        return [O.beam_decode_one(lambda w, c=c: O.next_logprobs(sd, mem[c], w, NHEAD, torch.float32), SOS, EOS, bw, 1)
                                for c in range(a.ref_clips)]
                ref_t.append(timed(reference)[0])
            res[f"{wl}_{mode}"] = dict(engine_clips_per_s=round(a.B / min(eng_t), 2), reference_clips_per_s=round((a.B if bw == 0 else a.ref_clips) / min(ref_t), 3),
                                       mean_words=round(lens[0], 1))
            print(wl, mode, res[f"{wl}_{mode}"], file=sys.stderr, flush=True)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps(dict(B=a.B, ref_clips=a.ref_clips, eos_bias=a.eos_bias, gpu=smi, results=res)))


if __name__ == "__main__":
    main()
