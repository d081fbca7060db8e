"""Helpers for the -m gpu tests: load the product package, move oracle state dicts to the device."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
import _pkg  # noqa: E402

_pkg.load()
from diffsound_b200 import ops  # noqa: E402,F401

DEV = "cuda"


def tf32_round_ref(x: torch.Tensor) -> torch.Tensor:
    """cvt.rna.tf32.f32 emulation (round to nearest, ties away from zero) on any device."""
    xi = x.contiguous().view(torch.int32)
    r = ((xi + 0x1000) & ~0x1FFF)
    return torch.where(torch.isfinite(x), r.view(torch.float32), x)


def run_loss_and_grads(m, x0, x_t, cond, t, pt):
    """One training forward + fused loss + backward of the drop-in DiffusionTransformer m: (loss, exp(log_model_prob), {name: gradient})."""
    from diffsound_b200.modeling.transformers.diffusion_transformer import denoiser_loss
    for p in m.parameters():
        p.requires_grad_(True)
        p.grad = None
    names, params = zip(*m.transformer.named_parameters())
    loss, prob, vb, hits = denoiser_loss(m, x0, x_t, cond, t, pt, True, True)
    loss.backward()
    return loss.detach(), prob, {n: p.grad for n, p in zip(names, params)}


def relerr(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))
