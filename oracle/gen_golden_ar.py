"""Generate tests/golden/ar_*.npz / ar_state_dict_keys.json from the UNMODIFIED reference autoregressive transformer
(Codebook/specvqgan/modules/transformer/mingpt.py GPTFeats, Codebook/specvqgan/models/cond_transformer.py Net2NetTransformer) on CPU.

Run from the repository root where the reference checkout is readable:  python oracle/gen_golden_ar.py
The reference imports pytorch_lightning, omegaconf.listconfig and train.instantiate_from_config; the three small import stubs below stand in
for them.  Weights are the reference's own seeded init (torch.manual_seed(seed) before construction) followed by oracle.ar_oracle.perturb_
(pos_emb is zero at init); the tests rebuild the same weights from the same seed with this package's drop-in, whose init order is the
reference's.  Fixtures:
  ar_forward.npz      teacher-forced logits of GPTFeats.forward, B = 1: tiny configs (D = 128, 2 layers, V = 32 / 2048, Tc = 1 / 3) and one
                      caps_transformer-width forward
  ar_sample.npz       Net2NetTransformer.sample ids, greedy and torch.multinomial (CPU generator seeded per case), nopix and half, top_k
                      None / 1 / 5 / V, temperature 1 / 0.7
  ar_state_dict_keys.json  key -> shape of the full Net2NetTransformer for caps_transformer, caps_transformer_2048, caps_transformer_small
"""
from __future__ import annotations

import importlib
import json
import os
import sys
import types

import numpy as np
import torch
import torch.nn as nn
import yaml

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ar_oracle as A  # noqa: E402

REF_CODEBOOK = os.path.join(os.environ.get("DIFFSOUND_REFERENCE", "/root/reference"), "Codebook")
OUT = os.path.join(ROOT, "tests", "golden")
CONFIGS = ("caps_transformer", "caps_transformer_2048", "caps_transformer_small")


class AttrDict(dict):
    """The attribute access OmegaConf gives the reference's configs."""
    __getattr__ = dict.__getitem__


def attr(o):
    if isinstance(o, dict):
        return AttrDict({k: attr(v) for k, v in o.items()})
    if isinstance(o, list):
        return [attr(v) for v in o]
    return o


def instantiate(config):
    if config is None:
        return None
    mod, cls = config["target"].rsplit(".", 1)
    return getattr(importlib.import_module(mod), cls)(**config.get("params", dict()))


def install_stubs():
    train = types.ModuleType("train")
    train.instantiate_from_config = instantiate
    sys.modules["train"] = train
    pl = types.ModuleType("pytorch_lightning")
    pl.LightningModule = nn.Module
    sys.modules.setdefault("pytorch_lightning", pl)
    om, oml = types.ModuleType("omegaconf"), types.ModuleType("omegaconf.listconfig")
    oml.ListConfig = list
    om.listconfig = oml
    sys.modules["omegaconf"] = om
    sys.modules["omegaconf.listconfig"] = oml
    sys.path.insert(0, REF_CODEBOOK)


def ref_gpt(V, n_embd, n_layer, n_head, Cf, seed):
    from specvqgan.modules.transformer.mingpt import GPTFeats
    fe, gc = A.gpt_config(V, n_embd, n_layer, n_head, Cf)
    torch.manual_seed(seed)
    g = GPTFeats(attr(fe), gc).eval()
    A.perturb_(g.state_dict(), seed)
    return g


@torch.no_grad()
def main():
    install_stubs()
    from specvqgan.models.cond_transformer import Net2NetTransformer
    fwd = {}
    cases = [("v32_tc1", 32, 266, 1, 11), ("v32_tc3", 32, 266, 3, 12), ("v2048_tc1", 2048, 40, 1, 13), ("v2048_tc3", 2048, 40, 3, 14)]
    for name, V, T, Tc, seed in cases:
        g = ref_gpt(V, A.TINY["n_embd"], A.TINY["n_layer"], A.TINY["n_head"], A.TINY["Cf"], seed)
        gen = torch.Generator().manual_seed(seed)
        idx = torch.randint(0, V, (1, T - Tc), generator=gen)
        feats = torch.randn(1, A.TINY["Cf"], Tc, generator=gen)
        logits, _, _ = g(idx, feats)
        fwd.update({f"{name}/idx": idx.numpy(), f"{name}/feats": feats.numpy(), f"{name}/logits": logits.numpy(),
                    f"{name}/meta": np.array([V, Tc, seed])})
    g = ref_gpt(256, 1024, 19, 16, 512, 21)  # caps_transformer width
    gen = torch.Generator().manual_seed(21)
    idx = torch.randint(0, 256, (1, 265), generator=gen)
    feats = torch.randn(1, 512, 1, generator=gen)
    feats = feats / feats.norm(dim=1, keepdim=True)  # a pooled CLIP feature is L2-normalised
    logits, _, _ = g(idx, feats)
    fwd.update({"full/idx": idx.numpy(), "full/feats": feats.numpy(), "full/logits": logits.numpy(), "full/meta": np.array([256, 1, 21])})
    np.savez_compressed(os.path.join(OUT, "ar_forward.npz"), **fwd)

    smp = {}
    V, seed, steps = 32, 31, 16
    g = ref_gpt(V, A.TINY["n_embd"], A.TINY["n_layer"], A.TINY["n_head"], A.TINY["Cf"], seed)
    stub = types.SimpleNamespace(transformer=g, pkeep=1.0, top_k_logits=lambda lg, k: Net2NetTransformer.top_k_logits(None, lg, k))
    gen = torch.Generator().manual_seed(seed)
    feats = torch.randn(2, A.TINY["Cf"], 1, generator=gen)
    gt = torch.randint(0, V, (2, steps), generator=gen)
    smp.update(feats=feats.numpy(), gt=gt.numpy(), meta=np.array([V, seed, steps]))
    i = 0
    for mode in ("nopix", "half"):
        x0 = gt[:, :0] if mode == "nopix" else gt[:, :steps // 2]
        for top_k in (None, 1, 5, V):
            for temperature in (1.0, 0.7):
                for do_sample in (False, True):
                    torch.manual_seed(1000 + i)
                    out, _ = Net2NetTransformer.sample(stub, x0, feats, steps - x0.shape[1], temperature=temperature, sample=do_sample, top_k=top_k)
                    key = f"c{i}"
                    smp[key + "/ids"] = out.numpy()
                    smp[key + "/args"] = np.array([0 if mode == "nopix" else 1, -1 if top_k is None else top_k, temperature, int(do_sample), 1000 + i],
                                                  dtype=np.float64)
                    i += 1
    np.savez_compressed(os.path.join(OUT, "ar_sample.npz"), **smp)

    keys = {}
    for name in CONFIGS:
        with open(os.path.join(REF_CODEBOOK, "configs", name + ".yaml")) as f:
            cfg = yaml.safe_load(f)["model"]
        cfg["params"]["first_stage_config"]["params"]["ckpt_path"] = None
        m = instantiate(attr(cfg))
        keys[name] = {k: list(v.shape) for k, v in m.state_dict().items()}
        del m
    with open(os.path.join(OUT, "ar_state_dict_keys.json"), "w") as f:
        json.dump(keys, f, indent=0, sort_keys=True)
    print("wrote", [n for n in os.listdir(OUT) if n.startswith("ar_")])


if __name__ == "__main__":
    main()
