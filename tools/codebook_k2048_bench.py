"""Cost of the 2048-code AudioSet codebook (caps_2048.yaml) against the 256-code one on one GPU, as one JSON line.

    python tools/codebook_k2048_bench.py [--batch 16] [--rounds 2] [--replays 50]

Full-size denoiser (19 layers, D = 1024, random init), B = 16, K = 256 and K = 2048 alternated in one process (rounds x both).  Per K:
  sampler_us   one launch of the fused sampling-loop kernel (warp kernel at K = 256, CTA-per-column kernel at K = 2048), CUDA events over
               replays of a CUDA graph that holds `replays` launches
  step_ms      one diffusion step: denoiser forward + sampling-loop launch, CUDA events over replays of a graph of both
  sample_ms    DiffusionTransformer.sample(): 100 steps from all-[MASK], top0.85r, the CUDA-graph loop
  clips_per_s  text -> wav: pipeline.synthesize (sample, SpecVQGAN decode, MelGAN vocode) on resident caption embeddings
Each number is the median over rounds.  The GPU's name and power limit are read in the same run."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def events_ms(fn, iters):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e) / iters


def graph_of(fn, n):
    """A CUDA graph holding n calls of fn (warmed up once on a side stream first)."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(n):
            fn()
    return g


def measure(K, B, replays, voc):
    from diffsound_b200 import ops, pipeline
    from diffsound_b200.utils import builders
    dalle = builders.build_dalle(K=K, NL=19, precision="f16x3", seed=0)
    tr = dalle.transformer
    L = tr.shape
    g = torch.Generator().manual_seed(1)
    cond = torch.randn(B, 77, 512, generator=g)
    cond = (cond / cond.norm(dim=-1, keepdim=True)).cuda()
    eng = tr.transformer.engine
    kv = eng.encode_condition(cond)
    loop = tr._sampler_ops()[1]
    x = torch.full((B, L), K, dtype=torch.long, device="cuda")
    t = torch.full((B,), 99, dtype=torch.long, device="cuda")
    tp = t.clone()
    nthreads, inc = ops.aten_rand_geometry(B * (K + 1) * L)
    n_sched = 100
    t_s = torch.arange(99, -1, -1, device="cuda")
    ctrl = torch.tensor([1234, 0, inc, nthreads, 0, n_sched, 0, 0], dtype=torch.int64, device="cuda")
    logits = eng.forward(x, kv, t, 77).clone()

    def sampler():
        loop(logits, x, t, tp, tr._sched(), ctrl, t_s, t_s, T=100, trunc_mode=1, trunc_r=0.85, trunc_k=0)

    gs = graph_of(sampler, replays)
    sampler_us = 1e3 * events_ms(gs.replay, 5) / replays

    def step():
        lg = eng.forward(x, kv, t, 77)
        loop(lg, x, t, tp, tr._sched(), ctrl, t_s, t_s, T=100, trunc_mode=1, trunc_r=0.85, trunc_k=0)

    gstep = graph_of(step, 10)
    step_ms = events_ms(gstep.replay, 3) / 10

    tr.truncation = "top0.85r"

    def sample():
        torch.manual_seed(7)
        return tr.sample(None, None, cond, filter_ratio=0, batch_size=B)["content_token"]

    sample()
    sample_ms = events_ms(sample, 3)
    tok = sample()
    assert int(tok.min()) >= 0 and int(tok.max()) < K

    def synth():
        torch.manual_seed(7)
        pipeline.synthesize(dalle, voc, cond, sample_type="top0.85r", codec_batch=32)

    synth()
    clips_per_s = B / (1e-3 * events_ms(synth, 3))
    del dalle, tr, eng, gs, gstep
    torch.cuda.empty_cache()
    return dict(sampler_us=sampler_us, step_ms=step_ms, sample_ms=sample_ms, clips_per_s=clips_per_s)


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--replays", type=int, default=50)
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("codebook_k2048_bench.py needs a GPU")
    import _pkg
    _pkg.load()
    from diffsound_b200.utils import builders
    voc = builders.build_vocoder(os.path.join(ROOT, "oracle", "_ref", "best_netG.pt"))
    runs = {256: [], 2048: []}
    for _ in range(args.rounds):
        for K in (256, 2048):
            runs[K].append(measure(K, args.batch, args.replays, voc))
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    out = {"gpu": torch.cuda.get_device_name(), "nvidia_smi": q, "batch": args.batch, "layers": 19, "D": 1024, "rounds": args.rounds}
    for K, rs in runs.items():
        out[f"K{K}"] = {k: round(statistics.median(r[k] for r in rs), 3) for k in rs[0]}
        out[f"K{K}"]["all"] = rs
    out["clips_per_s_ratio_2048_over_256"] = round(out["K2048"]["clips_per_s"] / out["K256"]["clips_per_s"], 4)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
