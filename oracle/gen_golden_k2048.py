"""Generate the K = 2048 (caps_2048.yaml, AudioSet codebook) fixtures of tests/golden/ by running the UNMODIFIED reference on CPU.

    python oracle/gen_golden_k2048.py      # needs the reference tree; writes tests/golden/

  schedule_k2048.npz          the eight schedule buffers at N = 2049 classes (alpha_schedule depends on N)
  sampler_cases_k2048.npz     predict_start (+ truncation) -> q_posterior -> Gumbel-argmax through the reference's own methods at K = 2048, for
                              no truncation, top0.85r and top20p; inputs are regenerated from portable_uniform seeds (gen_golden.sampler_case_inputs),
                              outputs stored as next ids (int16), 6-column heads of log_pred and of the posterior, and top-2 margins
  caps_2048_state_dict.json   key -> shape of the reference DALLE built with caps_2048.yaml's content codec and diffusion model
"""
from __future__ import annotations

import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_harness as rh  # noqa: E402
from oracle.gen_golden import GOLD, sampler_case_inputs  # noqa: E402

K = 2048
CASES = (0, 1, 2)
TRUNCS = {"top0.85r": "nuc", None: "raw", "top20p": "topk"}


def gen_schedule_k2048(model):
    tr = model.transformer
    names = ["log_at", "log_bt", "log_ct", "log_cumprod_at", "log_cumprod_bt", "log_cumprod_ct", "log_1_min_ct", "log_1_min_cumprod_ct"]
    np.savez_compressed(os.path.join(GOLD, "schedule_k2048.npz"), **{n: getattr(tr, n).numpy() for n in names})


def gen_sampler_cases_k2048(model):
    """The reference's predict_start tail, truncation wrapper, q_posterior and Gumbel-argmax at K = 2048 (the style of gen_golden.gen_sampler_cases)."""
    tr = model.transformer
    res = {}
    for case in CASES:
        logits, x_t, t, u = sampler_case_inputs(case, K=K)
        tr.transformer.forward = lambda *_a, _l=logits, **_k: _l
        model.this_save_path = None
        for trunc, name in TRUNCS.items():
            ps = type(tr).predict_start.__get__(tr)
            if trunc:
                ps = model.predict_start_with_truncation(ps, trunc)
            if case == 0:
                log_x = torch.log(torch.nn.functional.one_hot(x_t, K + 1).permute(0, 2, 1).float())
            else:
                log_x = torch.log(torch.nn.functional.one_hot(x_t, K + 1).permute(0, 2, 1).float().clamp(min=1e-30))
            lp = ps(log_x, None, t)
            post = tr.q_posterior(lp, log_x, t)
            g = -torch.log(-torch.log(u + 1e-30) + 1e-30)
            tag = f"c{case}_{name}"
            res[tag + "_next"] = (g + post).argmax(1).numpy().astype(np.int16)
            res[tag + "_post_head"] = post[:, :, :6].numpy()
            res[tag + "_lp_head"] = lp[:, :, :6].numpy()
            top2 = (g + post).topk(2, dim=1).values
            res[tag + "_margin"] = (top2[:, 0] - top2[:, 1]).numpy()
    np.savez_compressed(os.path.join(GOLD, "sampler_cases_k2048.npz"), **res)


def gen_state_dict_shapes_k2048():
    """caps_2048.yaml's model at full size: the content codec (n_embed 2048) and the diffusion model (num_embed 2048).  The CLIP condition
    embedding is left out (it loads a checkpoint); its keys are those of caps.yaml, which the existing drop-in tests pin."""
    model, _ = rh.build_dalle(K=K, seed=0)
    shapes = {k: list(v.shape) for k, v in model.state_dict().items()}
    with open(os.path.join(GOLD, "caps_2048_state_dict.json"), "w") as f:
        json.dump(shapes, f, indent=0, sort_keys=True)


if __name__ == "__main__":
    assert rh.available(), "reference tree not found"
    torch.set_grad_enabled(False)
    small, _ = rh.build_dalle(K=K, overrides=dict(n_layer=1, n_embd=64, n_head=1, dec_ch=32, dec_ch_mult=[1, 1, 1, 1, 2]), seed=0)
    gen_schedule_k2048(small)
    gen_sampler_cases_k2048(small)
    gen_state_dict_shapes_k2048()
    for f in ("schedule_k2048.npz", "sampler_cases_k2048.npz", "caps_2048_state_dict.json"):
        print(f, os.path.getsize(os.path.join(GOLD, f)) // 1024, "KB")
