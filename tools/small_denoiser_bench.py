"""Cost of Diffsound's small denoiser (caps_small_transformer.yaml: 18 layers, D = 512, 16 heads of 32) against caps.yaml's (19 layers, D = 1024,
16 heads of 64) on one GPU; writes small_denoiser_bench.json to --out and prints it as one JSON line.

    python tools/small_denoiser_bench.py --out DIR [--batch 16] [--rounds 2] [--iters 200]

  attention_us   one launch of the split-fp16 attention core at head_dim 32 and 64, B = 16, self (265 x 265) and cross (265 x 77), CUDA events
                 around replays of a CUDA graph of `iters` launches (best of 5)
Per model (f16x3, random init, B = 16, the two models alternated in one process, rounds x both):
  step_ms        one diffusion step: denoiser forward + sampling-loop launch, CUDA events over replays of a graph of both
  sample_ms      DiffusionTransformer.sample(): 100 steps from all-[MASK], top0.85r, the CUDA-graph loop
  clips_per_s    text -> wav: pipeline.synthesize (sample, SpecVQGAN decode, MelGAN vocode) on resident caption embeddings
  attention_share   the attention kernels' share of the device time of one denoiser forward, from torch.profiler in a separate pass
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
from tools.codebook_k2048_bench import events_ms, graph_of  # noqa: E402

MODELS = ("caps_small_transformer", "caps")


def attention_us(B, iters):
    from diffsound_b200 import ops
    L, H, out = 265, 16, {}
    g = torch.Generator(device="cuda").manual_seed(0)
    for hd in (32, 64):
        C = H * hd
        for name, Lk in (("self", L), ("cross", 77)):
            q = ops.split_f16(torch.randn(B * L, C, device="cuda", generator=g))
            k = ops.split_f16(torch.randn(B * Lk, C, device="cuda", generator=g))
            v = ops.split_f16(torch.randn(B * Lk, C, device="cuda", generator=g))
            o = torch.empty(B * L, 2 * C, dtype=torch.float16, device="cuda")

            def run():
                ops.attention_tc_split(q[:, :C], k[:, :C], v[:, :C], o[:, :C], q_lo=C, k_lo=C, v_lo=C, o_lo=C, B=B, H=H, Lq=L, Lk=Lk,
                                       scale=hd ** -0.5, head_dim=hd)

            graph = graph_of(run, iters)  # replayed: back-to-back launches with no host enqueue cost between them
            graph.replay()
            out[f"hd{hd}_{name}"] = round(1e3 * min(events_ms(graph.replay, 1) for _ in range(5)) / iters, 2)
    return out


def attention_share(eng, x, kv, t):
    """Device time of the attention kernels over all device time of one denoiser forward (torch.profiler, CUDA activity)."""
    from torch.profiler import ProfilerActivity, profile
    eng.forward(x, kv, t, 77)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        eng.forward(x, kv, t, 77)
        torch.cuda.synchronize()
    total = attn = 0.0
    for e in prof.key_averages():
        us = e.self_device_time_total
        total += us
        if "attention" in e.key:
            attn += us
    return round(attn / total, 4), round(total / 1e3, 3)


def measure(name, B, voc, with_profile):
    from diffsound_b200 import ops, pipeline
    from diffsound_b200.utils import builders
    dalle = builders.build_dalle(**builders.DALLE_CONFIGS[name], precision="f16x3", seed=0)
    tr = dalle.transformer
    L, K = tr.shape, tr.num_classes - 1
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
    t_s = torch.arange(99, -1, -1, device="cuda")
    ctrl = torch.tensor([1234, 0, inc, nthreads, 0, 100, 0, 0], dtype=torch.int64, device="cuda")

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
    r = dict(step_ms=step_ms, sample_ms=sample_ms, clips_per_s=clips_per_s)
    if with_profile:
        r["attention_share"], r["profiled_forward_ms"] = attention_share(eng, x, kv, t)
    del dalle, tr, eng, gstep
    torch.cuda.empty_cache()
    return r


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--out", required=True, help="directory for small_denoiser_bench.json")
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--iters", type=int, default=200)
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("small_denoiser_bench.py needs a GPU")
    import _pkg
    _pkg.load()
    from diffsound_b200.utils import builders
    voc = builders.build_vocoder(os.path.join(ROOT, "oracle", "_ref", "best_netG.pt"))
    out = {"gpu": torch.cuda.get_device_name(),
           "nvidia_smi": subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                                        text=True).stdout.strip(),
           "batch": args.batch, "rounds": args.rounds, "attention_us": attention_us(args.batch, args.iters)}
    runs = {m: [] for m in MODELS}
    for i in range(args.rounds):
        for m in MODELS:
            runs[m].append(measure(m, args.batch, voc, with_profile=(i == args.rounds - 1)))
    for m, rs in runs.items():
        out[m] = {k: round(statistics.median(r[k] for r in rs if k in r), 4) for k in rs[-1]}
        out[m]["all"] = rs
    out["step_ratio_small_over_caps"] = round(out["caps_small_transformer"]["step_ms"] / out["caps"]["step_ms"], 4)
    out["clips_per_s_ratio_small_over_caps"] = round(out["caps_small_transformer"]["clips_per_s"] / out["caps"]["clips_per_s"], 4)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "small_denoiser_bench.json"), "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
