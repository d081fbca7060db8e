"""Autoregressive SpecVQGAN transformer (caps_transformer.yaml) against Diffsound on one GPU, as one JSON line.

    python tools/ar_bench.py [--batches 16 96] [--rounds 3] [--profile-tokens 24]

Full-size models with random init: the AR model (19 layers, D = 1024, V = 256) and Diffsound's DALLE (19 layers, D = 1024, K = 256).  Per batch:
  ar_sample_ms    Net2NetTransformer.sample(): 265 tokens from no prefix, top_k 100, sampled (the KV-cached decode, one CUDA graph per position)
  diff_sample_ms  DiffusionTransformer.sample(): 100 steps from all-[MASK], top0.85r
The two are alternated in one process, one warm-up call each, then `rounds` calls each; numbers are medians over rounds.
A separate run under torch.profiler (eager launches, so every kernel is its own event) attributes one decode step to its launch roles (each GEMM,
decode attention, LayerNorm, GELU, sampler) over `profile-tokens` tokens at B = 16.  bytes_per_step is the split-fp16 weights plus the fp32 KV
cache read at the mean position, from shapes; bound_ms = bytes / 3.35 TB/s (the H100 SXM data-sheet HBM3 bandwidth).  The GPU's name and power
limit are read in the same run."""
import argparse
import collections
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12


def events_ms(fn, iters=1):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e) / iters


NAMED = {"ar_embed_kernel": "embed", "layernorm_kernel": "layernorm", "ar_attention_kernel": "attention", "ar_gelu_split_kernel": "gelu_split",
         "ar_sample_kernel": "sampler"}
# a GEMM call (one or more kernels) is named by the launches around it: AREngine._step runs
#   embed, n_layer x [layernorm, QKV, attention, proj, layernorm, MLP1, gelu_split, MLP2], layernorm, head, sampler
GEMM_ROLE = {("layernorm", "attention"): "gemm_qkv", ("attention", "layernorm"): "gemm_proj", ("layernorm", "gelu_split"): "gemm_mlp1",
             ("gelu_split", "layernorm"): "gemm_mlp2", ("layernorm", "sampler"): "gemm_head"}


def role_of(name):
    for k, v in NAMED.items():
        if k in name:
            return v
    return None


def weight_bytes(eng):
    n = sum(w.pair.numel() * 2 for lay in eng.layers for w in (lay["wqkv"], lay["wo"], lay["w1"], lay["w2"])) + eng.whead.pair.numel() * 2
    n += sum(lay[k].numel() * 4 for lay in eng.layers for k in ("bqkv", "bo", "bm1", "bm2", "g1", "b1", "g2", "b2"))
    return n


def profile_step(ar, B, tokens):
    from torch.profiler import ProfilerActivity, profile
    tr = ar.transformer
    feats = torch.randn(B, 512, 1, device="cuda")
    x0 = torch.zeros(B, 0, dtype=torch.long, device="cuda")
    tr.engine.use_cuda_graph = False
    ar.sample(x0, feats, tokens, sample=True, top_k=100)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        ar.sample(x0, feats, tokens, sample=True, top_k=100)
        torch.cuda.synchronize()
    tr.engine.use_cuda_graph = True
    kern = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "Memcpy" not in e.name and "Memset" not in e.name),
                  key=lambda e: e.time_range.start)
    names = [role_of(e.name) for e in kern]
    first = names.index("embed")  # the condition embedding GEMM runs once before the first position
    kern, names = kern[first:], names[first:]
    tot = collections.defaultdict(float)
    for i, e in enumerate(kern):
        r = names[i]
        if r is None:
            prev = next((n for n in reversed(names[:i]) if n is not None), None)
            nxt = next((n for n in names[i + 1:] if n is not None), None)
            r = GEMM_ROLE.get((prev, nxt), "other")
        tot[r] += e.time_range.elapsed_us()
    if names.count("embed") != tokens:
        return {"error": f"{names.count('embed')} positions in the trace, expected {tokens}"}
    step_us = sum(tot.values()) / tokens
    return {"step_us_kernels": round(step_us, 1),
            "per_role_us": {k: round(v / tokens, 1) for k, v in sorted(tot.items(), key=lambda kv: -kv[1])},
            "share": {k: round(v / tokens / step_us, 4) for k, v in sorted(tot.items(), key=lambda kv: -kv[1])}}


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--batches", type=int, nargs="+", default=[16, 96])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--profile-tokens", type=int, default=24)
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("ar_bench.py needs a GPU")
    import _pkg
    _pkg.load()
    from diffsound_b200.utils import builders
    ar = builders.build_ar_transformer(builders.ar_transformer_config(**builders.AR_CONFIGS["caps_transformer"]), seed=0)
    dalle = builders.build_dalle(K=256, NL=19, precision="f16x3", seed=0)
    dt = dalle.transformer
    dt.truncation = "top0.85r"
    out = {"gpu": torch.cuda.get_device_name(),
           "nvidia_smi": subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                                        text=True).stdout.strip(), "rounds": args.rounds}
    for B in args.batches:
        g = torch.Generator().manual_seed(B)
        feats = torch.randn(B, 512, 1, generator=g)
        feats = (feats / feats.norm(dim=1, keepdim=True)).cuda()
        cond = torch.randn(B, 77, 512, generator=g)
        cond = (cond / cond.norm(dim=-1, keepdim=True)).cuda()
        x0 = torch.zeros(B, 0, dtype=torch.long, device="cuda")

        def ar_sample():
            return ar.sample(x0, feats, 265, temperature=1.0, sample=True, top_k=100)[0]

        def diff_sample():
            return dt.sample(None, None, cond, filter_ratio=0, batch_size=B)["content_token"]

        ar_sample(), diff_sample()
        runs = {"ar_sample_ms": [], "diff_sample_ms": []}
        for _ in range(args.rounds):
            runs["ar_sample_ms"].append(round(events_ms(ar_sample), 2))
            runs["diff_sample_ms"].append(round(events_ms(diff_sample), 2))
        ids = ar_sample()
        assert ids.shape == (B, 265) and int(ids.min()) >= 0 and int(ids.max()) < 256
        eng = ar.transformer.engine
        wb = weight_bytes(eng)
        kv_mean = 19 * 2 * 1024 * 4 * B * (265 / 2)  # fp32 K and V of every layer at the mean position
        r = {k: statistics.median(v) for k, v in runs.items()}
        r.update(runs=runs, ar_step_ms=round(r["ar_sample_ms"] / 265, 4), ar_over_diff=round(r["ar_sample_ms"] / r["diff_sample_ms"], 3),
                 weight_bytes=wb, kv_bytes_mean=int(kv_mean), bytes_per_step=int(wb + kv_mean),
                 bound_ms_per_step=round((wb + kv_mean) / HBM_BYTES_PER_S * 1e3, 4), launches_per_step=eng.launches_per_step)
        out[f"B{B}"] = r
    out["profile_B16"] = profile_step(ar, 16, args.profile_tokens)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
