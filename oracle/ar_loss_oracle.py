"""CPU fp32 restatement of the autoregressive SpecVQGAN transformer's loss -- test infrastructure: GPT.forward's
F.cross_entropy(logits, targets) (Codebook/specvqgan/modules/transformer/mingpt.py:183-185) and Net2NetTransformer.shared_step's, which slices
the logits at cond_size - 1 first (Codebook/specvqgan/models/cond_transformer.py:106, :358-359), over oracle.ar_oracle.forward's logits."""
from __future__ import annotations

import torch
import torch.nn.functional as F

from oracle import ar_oracle as A


def loss(sd: dict, idx: torch.Tensor, feats: torch.Tensor, targets: torch.Tensor, *, first_row: int = 0, n_layer: int, n_head: int,
         prefix: str = "") -> torch.Tensor:
    """F.cross_entropy (ignore_index -100) of A.forward's logits rows first_row ... against targets (B, T - first_row): GPT.forward's loss at
    first_row 0, shared_step's at first_row = cond_size - 1."""
    logits = A.forward(sd, idx, feats, n_layer=n_layer, n_head=n_head, prefix=prefix)[:, first_row:]
    return F.cross_entropy(logits.reshape(-1, logits.size(-1)), targets.reshape(-1))
