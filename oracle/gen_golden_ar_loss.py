"""Generate tests/golden/ar_loss.npz from the UNMODIFIED reference autoregressive transformer (Codebook/specvqgan/modules/transformer/mingpt.py
GPT.forward with targets, Codebook/specvqgan/models/cond_transformer.py shared_step's slicing + F.cross_entropy) on CPU.

Run from the repository root where the reference checkout is readable:  python oracle/gen_golden_ar_loss.py
Same import stubs and the same seeded weights as oracle/gen_golden_ar.py (the reference's own init under torch.manual_seed(seed), then
oracle.ar_oracle.perturb_); the tests rebuild the weights from the seed and restate the loss with oracle.ar_loss_oracle.
Per case (B = 2 for the tiny configs, B = 1 at caps_transformer width):
  <case>/z, <case>/feats       the token sequence z (B, 265 or fewer) and the (B, Cf, Tc) features
  <case>/gpt_targets           targets (B, Tc + n) of GPT.forward(z[:, :-1], embeddings, targets), a few set to -100
  <case>/gpt_loss              that loss (mingpt.py:183-185)
  <case>/step_loss             shared_step's loss: F.cross_entropy(logits[:, Tc - 1:], z) of GPTFeats.forward(z[:, :-1], feats)
  <case>/meta                  [V, Tc, seed, n_embd, n_layer, n_head, Cf]
  full/logits                  GPTFeats.forward's logits of the width case
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ar_oracle as A  # noqa: E402
from oracle.gen_golden_ar import OUT, install_stubs, ref_gpt  # noqa: E402

# name, V, Tc, n tokens, seed, B, width (n_embd, n_layer, n_head, Cf)
CASES = [("v32_tc1", 32, 1, 265, 41, 2, None), ("v32_tc3", 32, 3, 263, 42, 2, None), ("v2048_tc1", 2048, 1, 40, 43, 2, None),
         ("v2048_tc3", 2048, 3, 40, 44, 2, None), ("full", 256, 1, 265, 45, 1, (1024, 19, 16, 512))]


@torch.no_grad()
def main():
    install_stubs()
    from specvqgan.modules.transformer.mingpt import GPT
    out = {}
    for name, V, Tc, n, seed, B, width in CASES:
        D, NL, NH, Cf = width or (A.TINY["n_embd"], A.TINY["n_layer"], A.TINY["n_head"], A.TINY["Cf"])
        g = ref_gpt(V, D, NL, NH, Cf, seed)
        gen = torch.Generator().manual_seed(seed)
        z = torch.randint(0, V, (B, n), generator=gen)
        feats = torch.randn(B, Cf, Tc, generator=gen)
        feats = feats / feats.norm(dim=1, keepdim=True)
        idx = z[:, :-1]
        tg = torch.randint(0, V, (B, Tc + n - 1), generator=gen)
        tg[0, :2] = -100  # the condition rows' first targets and a few scattered ones are ignored
        tg[B - 1, torch.randperm(Tc + n - 1, generator=gen)[:5]] = -100
        emb = g.embedder(feats).permute(0, 2, 1)  # GPTFeats.forward's Conv1d branch
        _, gpt_loss, _ = GPT.forward(g, idx, embeddings=emb, targets=tg)
        logits, _, _ = g(idx, feats)
        step_loss = F.cross_entropy(logits[:, Tc - 1:].reshape(-1, logits.size(-1)), z.reshape(-1))
        out.update({f"{name}/z": z.numpy(), f"{name}/feats": feats.numpy(), f"{name}/gpt_targets": tg.numpy(),
                    f"{name}/gpt_loss": np.float32(gpt_loss.item()), f"{name}/step_loss": np.float32(step_loss.item()),
                    f"{name}/meta": np.array([V, Tc, seed, D, NL, NH, Cf])})
        if width is not None:
            out[f"{name}/logits"] = logits.numpy()
        print(name, float(gpt_loss), float(step_loss))
    np.savez_compressed(os.path.join(OUT, "ar_loss.npz"), **out)
    print("wrote", os.path.join(OUT, "ar_loss.npz"))


if __name__ == "__main__":
    main()
