"""Per-shape time of the split-fp16 (f16x3) wgmma GEMM under its two tile schedules: auto (ordered stream-K where the tiles leave a partial last
wave) and forced data-parallel (schedule=1).

The six GEMMs of a denoiser layer plus the logits GEMM, at the denoiser's token count for --batch clips (M = batch x 265).  Each timed launch
sequence is one CUDA graph of --layers launches over distinct weight sets (as bench.py's gemm_roofline does: no launch finds its weights warm in
L2), replayed --reps times between CUDA events.  The two schedules alternate --rounds times; each reports the median and the range of its rounds.
`bit_equal` compares one launch of each schedule on the same inputs, as integers.  One JSON line on stdout.

    python tools/gemm_f16x3_shapes.py [--batch 16] [--layers 19] [--rounds 3] [--reps 10]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

L_TOK = 265
D = 1024
# name, N, K, epilogue: 'split' = fp16 (hi | lo) output, 'gelu' = GELU2 + split output, 'res' = in-place fp32 residual, 'f32' = plain fp32
SHAPES = [("qkv", 3 * D, D, "split"), ("proj1", D, D, "res"), ("q2", D, D, "split"), ("proj2", D, D, "res"), ("mlp1", 4 * D, D, "gelu"),
          ("mlp2", D, 4 * D, "res"), ("logits", 256, D, "f32")]


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        name, power = [v.strip() for v in r.stdout.splitlines()[0].split(",")]
        return {"gpu": name, "power_limit": power}
    except Exception as e:  # the timing does not depend on it; report what is missing
        return {"gpu": torch.cuda.get_device_name(), "power_limit": f"unavailable ({type(e).__name__})"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--layers", type=int, default=19)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gemm_f16x3_shapes.py needs a CUDA device")
    import _pkg
    _pkg.load()
    from diffsound_b200 import ops

    M = args.batch * L_TOK
    g = torch.Generator(device="cuda").manual_seed(0)
    res = {}
    for name, N, K, epi in SHAPES:
        a = ops.split_f16(torch.randn(M, K, device="cuda", generator=g) * 0.5)
        ws = [ops.split_f16(torch.randn(N, K, device="cuda", generator=g) * K ** -0.5) for _ in range(args.layers)]
        bias = torch.randn(N, device="cuda", generator=g) * 0.1
        x0 = torch.randn(M, N, device="cuda", generator=g)
        out = torch.empty(M, 2 * N, dtype=torch.float16, device="cuda") if epi in ("split", "gelu") else x0.clone()

        def launch(w, schedule):
            if epi == "res":
                ops.gemm_f16x3(a, w, bias, residual=out, out=out, schedule=schedule)
            else:
                ops.gemm_f16x3(a, w, bias, gelu=epi == "gelu", split_out=epi != "f32", out=out, schedule=schedule)

        # bit equality: one launch per schedule from the same inputs
        outs = []
        for s in (0, 1):
            out.copy_(x0) if epi in ("res", "f32") else out.zero_()
            launch(ws[0], s)
            outs.append(out.clone())
        torch.cuda.synchronize()
        itype = torch.int32 if outs[0].element_size() == 4 else torch.int16
        bit_equal = bool(torch.equal(outs[0].view(itype), outs[1].view(itype)))

        graphs = {}
        for s in (0, 1):
            for w in ws:  # warm-up outside the capture (kernel attributes, the stream-K workspace)
                launch(w, s)
            torch.cuda.synchronize()
            gr = torch.cuda.CUDAGraph()
            with torch.cuda.graph(gr):
                for w in ws:
                    launch(w, s)
            gr.replay()
            graphs[s] = gr
        torch.cuda.synchronize()
        times = {0: [], 1: []}
        for _ in range(args.rounds):
            for s in (0, 1):
                st, en = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                st.record()
                for _ in range(args.reps):
                    graphs[s].replay()
                en.record()
                en.synchronize()
                times[s].append(st.elapsed_time(en) * 1e3 / (args.reps * args.layers))
        tiles = -(-M // 128) * -(-N // 128)

        def summary(v):
            v = sorted(v)
            return {"us": round(v[len(v) // 2], 2), "min": round(v[0], 2), "max": round(v[-1], 2)}

        res[name] = {"M": M, "N": N, "K": K, "tiles": tiles, "auto": summary(times[0]), "data_parallel": summary(times[1]),
                     "speedup": round(sorted(times[1])[len(times[1]) // 2] / sorted(times[0])[len(times[0]) // 2], 3), "bit_equal": bit_equal}
        del graphs, ws, a, out, outs
        torch.cuda.empty_cache()
    line = {"tool": "gemm_f16x3_shapes", **gpu_info(), "batch": args.batch, "layers": args.layers, "rounds": args.rounds, "reps": args.reps,
            "bit_equal": all(r["bit_equal"] for r in res.values()), "shapes": res}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
