"""Shared helpers for the parity tests (CPU side)."""
import os

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")


def load_golden(name):
    z = np.load(os.path.join(GOLD, name))
    sd = {k[3:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("sd.")}
    rest = {k: z[k] for k in z.files if not k.startswith("sd.")}
    return sd, rest


def portable_uniform(seed, shape):
    rng = np.random.Generator(np.random.Philox(seed))
    return torch.from_numpy(rng.random(size=tuple(shape), dtype=np.float32))


def sampler_case_inputs(case, B=2, K=256, L=265):
    """Must stay identical to oracle/gen_golden.py:sampler_case_inputs (inputs are regenerated, not stored)."""
    scale = [1.0, 6.0, 40.0, 2.0, 12.0][case % 5]
    logits = (portable_uniform(100 + case, (B, K, L)) - 0.5) * scale
    u = portable_uniform(200 + case, (B, K + 1, L))
    t_pair = [(99, 99), (57, 12), (1, 1), (0, 0), (98, 33)][case % 5]
    t = torch.tensor([t_pair[i % 2] for i in range(B)], dtype=torch.long)
    ids = (portable_uniform(300 + case, (B, L)) * K).long().clamp(max=K - 1)
    masked = portable_uniform(400 + case, (B, L)) < ([1.1, 0.35, 0.05, 0.02, 0.9][case % 5])
    x_t = torch.where(masked, torch.full_like(ids, K), ids)
    return logits, x_t, t, u


def build_dt(K, D, NL, NH, CD, sd=None, spatial=(5, 53), T=100, precision="f16"):
    """The drop-in DiffusionTransformer (the package must already be loaded)."""
    from diffsound_b200.utils.builders import build_diffusion_transformer
    return build_diffusion_transformer(K, D, NL, NH, CD, sd, spatial=spatial, T=T, precision=precision)


def rel_err(a, b):
    """max |a-b| / max|b|  -- the 'relative' of north_star's 1e-3 (relative to the tensor's scale)."""
    return float((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30))


def bpe_vocab_file(dirpath):
    """The CLIP BPE merge table (stored as two parts below 1 MB) reassembled into `dirpath`; returns its path."""
    out = os.path.join(str(dirpath), "bpe_simple_vocab_16e6.txt.gz")
    with open(out, "wb") as f:
        for i in range(2):
            with open(os.path.join(GOLD, f"bpe_simple_vocab_16e6.txt.gz.part{i}"), "rb") as part:
                f.write(part.read())
    return out
