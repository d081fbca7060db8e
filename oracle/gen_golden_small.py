"""Generate the head_dim-32 (caps_small_transformer.yaml) fixtures of tests/golden/ by running the UNMODIFIED reference on CPU.

    python oracle/gen_golden_small.py      # needs the reference tree; writes tests/golden/

  xf_small_tiny.npz                   a tiny head_dim-32 denoiser (K = 32, D = 64, 2 layers, 2 heads, B = 3, L = 265), in the layout of
                                      gen_golden.gen_xf_tiny's xf_tiny.npz: inputs, the transformer's logits, the truncating predict_start and
                                      q_posterior, and a free-running 100-step sample().  Its parameters are loaded into the reference from
                                      portable_params (numpy Philox), so the fixture stores only their shapes and the schedule buffers
  caps_small_transformer_state_dict.json   key -> shape of the reference DALLE built with caps_small_transformer.yaml's content codec and
                                      diffusion model (n_layer 18, n_embd 512, position embed_dim 512: the three values that differ from caps.yaml)
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
from oracle.gen_golden import GOLD, portable_uniform, sd_np  # noqa: E402


def portable_params(shapes: dict) -> dict:
    """Parameters of the given shapes from numpy Philox, bit-identical on every platform (tests/test_cpu_small_denoiser.py regenerates them):
    biases 0 +- 0.05, 1-D weights (the LayerNorm affines) 1 +- 0.05, every other weight +- 0.035 (standard deviation 0.02, the reference's
    init scale).  Nonzero biases and non-unit affines pin those paths too."""
    out = {}
    for i, (name, shape) in enumerate(sorted(shapes.items())):
        u = portable_uniform(7000 + i, shape) - 0.5
        if name.endswith("bias"):
            out[name] = u * 0.1
        elif len(shape) == 1:
            out[name] = 1.0 + u * 0.1
        else:
            out[name] = u * 0.07
    return out


def gen_xf_small_tiny():
    K, D, NL, NH, CD = 32, 64, 2, 2, 64
    model, _ = rh.build_dalle(K=K, overrides=dict(n_layer=NL, n_embd=D, n_head=NH, condition_dim=CD, dec_ch=32,
                                                  dec_ch_mult=[1, 1, 1, 1, 2], dec_z_channels=64, embed_dim=64), seed=0)
    tr = model.transformer  # DiffusionTransformer
    shapes = {n: list(p.shape) for n, p in tr.named_parameters()}
    params = portable_params(shapes)
    for n, p in tr.named_parameters():
        p.copy_(params[n])
    g = torch.Generator().manual_seed(11)
    B, L = 3, 265
    cond = torch.randn(B, 77, CD, generator=g)
    cond = cond / cond.norm(dim=-1, keepdim=True)
    x_t = torch.randint(0, K + 1, (B, L), generator=g)
    t = torch.tensor([99, 41, 0])
    logits = tr.transformer(x_t.clone(), cond, t)
    log_x = torch.log(torch.nn.functional.one_hot(x_t, K + 1).permute(0, 2, 1).float().clamp(min=1e-30))
    wrapped = model.predict_start_with_truncation(tr.predict_start, "top0.85r")
    lp = wrapped(log_x, cond, t)
    post = tr.q_posterior(lp, log_x, t)
    # free-running reference sample(): global CPU generator, exactly as generate_content would
    model.truncation_forward = True
    tr.predict_start = wrapped
    buffers = {k: v for k, v in sd_np(tr.state_dict()).items() if k not in shapes}  # the schedule; the parameters are regenerated
    torch.manual_seed(4321)
    tok = tr.sample(condition_token=None, condition_mask=None, condition_embed=cond, filter_ratio=0, batch_size=B)["content_token"]
    np.savez_compressed(os.path.join(GOLD, "xf_small_tiny.npz"), __cfg=np.array([K, D, NL, NH, CD, B, L]), __seed=np.array([4321]),
                        __param_shapes=np.array(json.dumps(shapes, sort_keys=True)),
                        in_cond=cond.numpy(), in_x_t=x_t.numpy().astype(np.int16), in_t=t.numpy(),
                        out_logits=logits.numpy(), out_lp=lp.numpy(), out_post=post.numpy(),
                        out_sample_tokens=tok.numpy().astype(np.int16), **{"sd." + k: v for k, v in buffers.items()})
    print("xf_small_tiny: logits", tuple(logits.shape), "tokens", tok[0, :8].tolist())


def gen_state_dict_shapes_small():
    """caps_small_transformer.yaml's model at full size.  The CLIP condition embedding is left out (it loads a checkpoint); its keys are those
    of caps.yaml, which the existing drop-in tests pin."""
    model, _ = rh.build_dalle(overrides=dict(n_layer=18, n_embd=512), seed=0)
    shapes = {k: list(v.shape) for k, v in model.state_dict().items()}
    with open(os.path.join(GOLD, "caps_small_transformer_state_dict.json"), "w") as f:
        json.dump(shapes, f, indent=0, sort_keys=True)


if __name__ == "__main__":
    assert rh.available(), "reference tree not found"
    torch.set_grad_enabled(False)
    gen_xf_small_tiny()
    gen_state_dict_shapes_small()
    for f in ("xf_small_tiny.npz", "caps_small_transformer_state_dict.json"):
        print(f, os.path.getsize(os.path.join(GOLD, f)) // 1024, "KB")
