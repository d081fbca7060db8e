"""Scoring the autoregressive SpecVQGAN transformer: the full-sequence causal pass (AREngine.prefill) against the KV-cached teacher-forced forward,
as one JSON line.

    python tools/ar_loss_bench.py [--configs caps_transformer caps_transformer_small] [--batches 16 64] [--rounds 5]
    python tools/ar_loss_bench.py --profile OUT_DIR [--batches 16]      # kernel time breakdown of one prefill (a separate run)

Full-size models with random init.  Per config and batch, the scoring of one shared_step batch (265 tokens after a 1-row condition, T = 265):
  kv_forward_ms   GPTFeats.forward(z[:, :-1], feats): the KV-cached decode, one CUDA graph replayed per position
  prefill_loss_ms GPTFeats.forward_loss(z[:, :-1], feats, z, 0): one causal pass with M = B * T GEMMs, the logits and the cross-entropy
The two alternate in one process after one warm-up call each; numbers are medians over rounds.  loss_gap is |prefill loss - F.cross_entropy of
the KV-cached logits| of the last round.  attention_us: one launch of the causal and the non-causal split attention at L = 266, B = 16, 16 heads,
per head_dim (CUDA events over 200 launches, median of 5).  --profile runs one prefill at the first batch size under torch.profiler with eager
launches and prints each kernel's share of the device time.  The GPU's name and power limit are read in the same run."""
import argparse
import collections
import json
import math
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import _pkg  # noqa: E402

_pkg.load()
from diffsound_b200 import ops  # noqa: E402
from diffsound_b200.utils.builders import AR_CONFIGS, ar_transformer_config, build_ar_transformer  # noqa: E402

N_TOK = 265


def events_ms(fn, iters=1):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e) / iters


def inputs(V, B, seed=0):
    g = torch.Generator().manual_seed(seed)
    z = torch.randint(0, V, (B, N_TOK), generator=g).cuda()
    f = torch.randn(B, 512, 1, generator=g)
    return z, (f / f.norm(dim=1, keepdim=True)).cuda()


def scoring(name, batches, rounds):
    m = build_ar_transformer(ar_transformer_config(**AR_CONFIGS[name]), seed=0)
    tr, V = m.transformer, AR_CONFIGS[name]["V"]
    out = {}
    for B in batches:
        z, feats = inputs(V, B)
        kv = lambda: tr(z[:, :-1], feats)
        pf = lambda: tr.forward_loss(z[:, :-1], feats, z, 0)
        kv(), pf()
        t_kv, t_pf = [], []
        for _ in range(rounds):
            t_kv.append(events_ms(kv))
            t_pf.append(events_ms(pf))
        logits, _, _ = kv()
        _, loss, _ = pf()
        gap = abs(float(loss) - float(F.cross_entropy(logits.reshape(-1, V), z.reshape(-1))))
        out[f"B{B}"] = {"kv_forward_ms": round(statistics.median(t_kv), 3), "prefill_loss_ms": round(statistics.median(t_pf), 3),
                        "speedup": round(statistics.median(t_kv) / statistics.median(t_pf), 2), "loss": round(float(loss), 6), "loss_gap": gap}
    del m, tr
    torch.cuda.empty_cache()
    return out


def attention_us(hd, B=16, H=16, L=266):
    D = H * hd
    qkv = ops.split_f16(torch.randn(B * L, 3 * D, device="cuda"))
    o = torch.empty(B * L, 2 * D, dtype=torch.float16, device="cuda")
    a = dict(q_lo=3 * D, k_lo=3 * D, v_lo=3 * D, o_lo=D, B=B, H=H, scale=1.0 / math.sqrt(hd))
    calls = {"causal": lambda: ops.attention_tc_split_causal(qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:3 * D], o[:, :D], L=L, head_dim=hd, **a),
             "non_causal": lambda: ops.attention_tc_split(qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:3 * D], o[:, :D], Lq=L, Lk=L, head_dim=hd, **a)}
    res = {k: [] for k in calls}
    for fn in calls.values():
        events_ms(fn, 20)
    for _ in range(5):
        for k, fn in calls.items():
            res[k].append(events_ms(fn, 200) * 1e3)
    return {k: round(statistics.median(v), 2) for k, v in res.items()}


def profile(B, out_dir):
    from torch.profiler import ProfilerActivity, profile as tprofile
    m = build_ar_transformer(ar_transformer_config(**AR_CONFIGS["caps_transformer"]), seed=0)
    tr = m.transformer
    tr.engine.use_cuda_graph = False  # eager launches: every kernel is its own event
    z, feats = inputs(256, B)
    for _ in range(2):
        tr.forward_loss(z[:, :-1], feats, z, 0)
    torch.cuda.synchronize()
    with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
        tr.forward_loss(z[:, :-1], feats, z, 0)
        torch.cuda.synchronize()
    per = collections.Counter()
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            per[ev.name] += ev.device_time
    total = sum(per.values())
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        prof.export_chrome_trace(os.path.join(out_dir, f"prefill_B{B}.pt.trace.json"))
    return {"B": B, "device_us": round(total, 1),
            "kernels": [{"name": n[:90], "us": round(t, 1), "share": round(t / total, 4)} for n, t in per.most_common(12)]}


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--configs", nargs="+", default=["caps_transformer", "caps_transformer_small"])
    ap.add_argument("--batches", nargs="+", type=int, default=[16, 64])
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--profile", default=None, help="directory for the profiler trace; runs the kernel breakdown only")
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("ar_loss_bench needs a CUDA GPU")
    out = {"gpu": torch.cuda.get_device_name(),
           "nvidia_smi": subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                                        text=True).stdout.strip()}
    if a.profile is not None:
        out["profile"] = profile(a.batches[0], a.profile)
    else:
        out["attention_us_L266"] = {f"hd{hd}": attention_us(hd) for hd in (64, 32)}
        for name in a.configs:
            out[name] = scoring(name, a.batches, a.rounds)
    print(json.dumps(out))
    return out


if __name__ == "__main__":
    main()
