"""Melception feature extraction throughput: the sm_90a kernels (CUDA graph replay) against the same network on cuDNN through stock PyTorch
(the fp32 oracle, with torch's default TF32 convolutions -- what the reference's evaluate.py runs -- and with TF32 off), timed alternately in one
process with CUDA events.  Seeded bounded ('he') weights; B clips of 80 x T.  Prints one JSON line.

    python tools/melception_bench.py [--batch 64] [--T 848] [--iters 10]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

GFLOP_PER_CLIP = 112.9  # 2 * MACs of the 94 convolutions + fc at 80 x 848 (scaled by T / 848 for other lengths)
FEATS = ["logits_unbiased", "2048", "logits"]


def timed(fn, iters):
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b) / 1e3)
    return sorted(ts)[len(ts) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--T", type=int, default=848)
    ap.add_argument("--iters", type=int, default=10)
    a = ap.parse_args()
    import _pkg
    _pkg.load()
    import tempfile
    from diffsound_b200.evaluation.feature_extractors.melception import Melception
    from oracle import melception_oracle as MO
    sd = MO.make_melception_state_dict(21, "he")
    with tempfile.TemporaryDirectory() as d:
        torch.save({"model": sd}, os.path.join(d, "w.pt"))
        m = Melception(309, FEATS, os.path.join(d, "w.pt")).cuda().eval()
    g = torch.Generator().manual_seed(0)
    x = (torch.rand(a.batch, 80, a.T, generator=g) * 4 - 2).cuda()
    sd_dev = {k: v.cuda() for k, v in sd.items()}
    ours = lambda: m(x)
    cudnn = lambda: MO.melception_forward(sd_dev, x, FEATS, torch.float32)

    def with_tf32(flag, fn):
        def run():
            old = torch.backends.cudnn.allow_tf32
            torch.backends.cudnn.allow_tf32 = flag
            try:
                return fn()
            finally:
                torch.backends.cudnn.allow_tf32 = old
        return run
    legs = {"kernels": ours, "cudnn_tf32": with_tf32(True, cudnn), "cudnn_fp32": with_tf32(False, cudnn)}
    outs = {k: f() for k, f in legs.items()}  # warm-up: packing, calibration, graph capture, cuDNN algorithm choice
    for f in legs.values():
        f()
    times = {k: [] for k in legs}
    for _ in range(3):  # alternate the legs so that clock and neighbour noise hit all of them
        for k, f in legs.items():
            times[k].append(timed(f, a.iters))
    gflop = GFLOP_PER_CLIP * a.T / 848
    res = {"batch": a.batch, "T": a.T}
    for k, ts in times.items():
        t = sorted(ts)[1]
        res[k] = {"s_per_batch": round(t, 5), "clips_per_s": round(a.batch / t, 1), "tflops": round(a.batch * gflop / t / 1e3, 1)}
    ref = outs["cudnn_fp32"]
    res["agreement_vs_cudnn_fp32"] = {k: {n: float((o.double() - r.double()).abs().max() / r.double().abs().max()) for n, o, r in zip(FEATS, outs[k], ref)}
                                      for k in ("kernels", "cudnn_tf32")}
    res["gpu"] = torch.cuda.get_device_name()
    try:
        res["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                                            capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        res["power_limit"] = "unknown"
    print(json.dumps(res))


if __name__ == "__main__":
    main()
