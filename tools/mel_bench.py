"""Log-mel extraction throughput at B ten-second clips (220500 samples, 860 frames): this library's path (pack -> split-fp16 DFT GEMM -> mel / log
kernel, CUDA graph replay) against torch.stft (cuFFT, fp32) + a matmul with the same float32 basis + the same normalisation, alternated in one
process with CUDA events.  A separate torch.profiler run gives each kernel's share of one call and the DFT GEMM's achieved TFLOP/s, counted from
shapes (frames x 694 columns x 1024 x 2 x 3 passes; 3.7 GFLOP per clip).  Writes one JSON line (stdout and --out).

    python tools/mel_bench.py [--batch 64] [--iters 20] [--out results/mel_bench.json]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

LENGTH = 220500


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


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # the measurement still stands; say why the card could not be read
        return f"unavailable ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import _pkg
    _pkg.load()
    from diffsound_b200 import mel_engine as ME
    B = a.batch
    g = torch.Generator(device="cuda").manual_seed(0)
    wav = (torch.rand(B, LENGTH, device="cuda", generator=g) * 2 - 1) * 0.5
    eng = ME.MelEngine("cuda")
    basis = torch.from_numpy(ME.mel_basis()).cuda()
    win = torch.hann_window(1024, periodic=True, device="cuda")

    def ours():
        return eng(wav)

    def cufft():
        spec = torch.stft(wav, 1024, 256, window=win, center=True, pad_mode="reflect", return_complex=True).abs()
        mel = torch.matmul(basis, spec)
        return ((torch.log10(mel.clamp_min(1e-5)) * 20 - 20 + 100) / 100).clamp(0, 1)[:, :, :ME.MAX_FRAMES]

    for _ in range(3):  # warm every shape: graph capture, cuFFT plan, cuBLAS heuristics
        x, y = ours(), cufft()
    torch.cuda.synchronize()
    agree = float((x - y).abs().max())
    t_ours, t_fft = [], []
    for _ in range(5):
        t_ours.append(timed(ours, a.iters))
        t_fft.append(timed(cufft, a.iters))
    so, sf = float(np.median(t_ours)), float(np.median(t_fft))

    T = 1 + LENGTH // ME.HOP
    gflop_clip = T * 2 * eng.n_bins * ME.N_FFT * 2 * 3 / 1e9
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(10):
            eng(wav)
        torch.cuda.synchronize()
    per = {}
    for ev in prof.key_averages():
        if ev.device_type.name == "CUDA" and ev.count:
            per[ev.key] = per.get(ev.key, 0.0) + ev.device_time_total / 10 / 1e6   # seconds per call
    total = sum(per.values())
    kern = {k[:60]: {"us_per_call": round(v * 1e6, 1), "share": round(v / total, 3)} for k, v in sorted(per.items(), key=lambda kv: -kv[1])}
    gemm_s = sum(v for k, v in per.items() if "gemm" in k.lower())
    res = {"card": card(), "batch": B, "length": LENGTH, "frames": T,
           "ours": {"s_per_batch": round(so, 5), "clips_per_s": round(B / so, 1)},
           "torch_stft_cufft_fp32": {"s_per_batch": round(sf, 5), "clips_per_s": round(B / sf, 1)},
           "ours_over_cufft_time": round(so / sf, 3), "max_abs_diff_vs_cufft": agree,
           "gemm_gflop_per_clip": round(gflop_clip, 3), "gemm_tflops": round(gflop_clip * B / gemm_s / 1e3, 1) if gemm_s else None,
           "kernels": kern}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
