"""Where one p_sample step's time goes: B = 16, f16x3, the full-size denoiser, under torch.profiler with CUDA activities.

Runs warm-up steps, then profiles --steps steps (replays of the captured step graph, as bench.py runs them; --eager launches each kernel
from Python instead).  Every kernel of a step is assigned to its launch position in the denoiser's fixed sequence (embed, then per layer
AdaLN1, qkv, self-attention, proj1, AdaLN2, q2, cross-attention, proj2, LN, mlp1, mlp2, then the final LN and the logits GEMM); whatever
else the step launches is "sampler".  Prints us per step for each position (per-layer positions summed over the layers, and their per-layer
mean), its share of the step, and the gap: step span minus the time at least one kernel runs.  Kernels launched with programmatic
dependent launch start before their predecessor ends, so the positions add up to more than the step; the overlap line says by how much.
A profile in its own process: do not time anything else in the same run.

    python tools/step_breakdown.py [--steps 5] [--warmup 3] [--eager] [--trace step.pt.trace.json]
"""
import argparse
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench import synthetic_cond  # noqa: E402
import _pkg  # noqa: E402
_pkg.load()
from diffsound_b200.utils.builders import build_diffusion_transformer  # noqa: E402

LAYER_POS = ["ada_ln1", "gemm_qkv", "attn_self", "gemm_proj1", "ada_ln2", "gemm_q2", "attn_cross", "gemm_proj2", "ln", "gemm_mlp1", "gemm_mlp2"]


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[torch.cuda.current_device()]
    except Exception as e:  # the numbers below still stand; say that the card could not be read
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--layers", type=int, default=19)
    ap.add_argument("--eager", action="store_true", help="launch every kernel from Python instead of replaying the step graph")
    ap.add_argument("--trace", default=None, help="also export the chrome trace here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("step_breakdown needs a GPU")

    torch.manual_seed(0)
    m = build_diffusion_transformer(256, 1024, args.layers, 16, 512, precision="f16x3")
    m.truncation = "top0.85r"
    m.use_cuda_graph = not args.eager
    cond = synthetic_cond(args.batch, 1).cuda()
    torch.manual_seed(1234)
    warm = list(range(99, 99 - args.warmup, -1))
    m._run_steps(cond, args.batch, warm, warm)
    torch.cuda.synchronize()
    steps = list(range(99, 99 - args.steps - 1, -1))  # one extra step: the last one is only the end marker of the one before
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        m._run_steps(cond, args.batch, steps, steps)
        torch.cuda.synchronize()
    if args.trace:
        os.makedirs(os.path.dirname(os.path.abspath(args.trace)), exist_ok=True)
        prof.export_chrome_trace(args.trace)

    kern = sorted(((e.time_range.start, e.time_range.end, e.name) for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
                   and "memcpy" not in e.name.lower() and "memset" not in e.name.lower()), key=lambda k: k[0])
    starts = [i for i, k in enumerate(kern) if "embed_tokens_kernel" in k[2]]
    if len(starts) < args.steps + 1:
        sys.exit(f"found {len(starts)} denoiser passes in the trace, expected {args.steps + 1}: the profiler did not record the step's kernels")
    n_fwd = 1 + 11 * args.layers + 2
    tot = {}
    span = busy = 0.0
    for s in range(args.steps):
        ks = kern[starts[s]:starts[s + 1]]
        if len(ks) < n_fwd:
            sys.exit(f"step {s}: {len(ks)} kernels, fewer than the {n_fwd} the denoiser launches")
        span += kern[starts[s + 1]][0] - ks[0][0]
        end = ks[0][0]
        for t0, t1, _ in ks:  # union of the kernel intervals: with programmatic dependent launch a kernel starts before its predecessor ends
            busy += max(0.0, t1 - max(t0, end))
            end = max(end, t1)
        for i, (t0, t1, name) in enumerate(ks):
            if i == 0:
                pos = "embed"
            elif i < 1 + 11 * args.layers:
                pos = LAYER_POS[(i - 1) % 11]
            elif i == 1 + 11 * args.layers:
                pos = "final_ln"
            elif i == 2 + 11 * args.layers:
                pos = "gemm_logits"
            else:
                pos = "sampler"
            tot[pos] = tot.get(pos, 0.0) + (t1 - t0)
    n = args.steps
    step_us = span / n
    busy /= n
    print(f"GPU: {gpu_info()}")
    print(f"B={args.batch} f16x3, {args.layers} layers, {n} profiled steps, {'eager' if args.eager else 'graph replay'}: {step_us:8.1f} us per step")
    print(f"{'position':<12} {'us/step':>9} {'us/layer':>9} {'share':>7}")
    order = ["embed"] + LAYER_POS + ["final_ln", "gemm_logits", "sampler"]
    for pos in order:
        us = tot.get(pos, 0.0) / n
        per_layer = f"{us / args.layers:9.1f}" if pos in LAYER_POS else " " * 9
        print(f"{pos:<12} {us:9.1f} {per_layer} {100 * us / step_us:6.1f}%")
    attn = (tot.get("attn_self", 0.0) + tot.get("attn_cross", 0.0)) / n
    print(f"{'gap':<12} {step_us - busy:9.1f} {'':9} {100 * (step_us - busy) / step_us:6.1f}%  (no kernel running)")
    print(f"{'overlap':<12} {sum(tot.values()) / n - busy:9.1f} {'':9} {'':7}  (summed kernel time past the union: a kernel's early start,"
          " waiting for its predecessor, is counted in its own time)")
    print(f"{'attention':<12} {attn:9.1f} {attn / args.layers:9.1f} {100 * attn / step_us:6.1f}%  (both launches)")


if __name__ == "__main__":
    main()
