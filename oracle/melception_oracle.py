"""CPU/GPU oracle for the Melception feature extractor -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

A functional restatement, in plain torch at a chosen dtype (fp32 or fp64), of the reference's Melception forward
(Codebook/evaluation/feature_extractors/melception.py:23-113) over torchvision's Inception3 (models/inception.py: BasicConv2d = bias-free conv,
BatchNorm2d(eps=0.001), ReLU; InceptionA-E).  It takes a state dict with the reference's own key names.  ``make_melception_state_dict`` draws
seeded weights from a portable numpy Philox stream (no checkpoint ships with the reference).  Pinned against the reference itself by
tests/golden/melception_ref.npz (oracle/gen_golden_melception.py).
"""
from __future__ import annotations

from typing import Dict, Sequence

import numpy as np
import torch
import torch.nn.functional as F

FEATURES = ("64", "192", "768", "2048", "logits_unbiased", "logits")


def _blocks():
    """Inception3's registration order: (module name, [(conv name, cin, cout, (kh, kw))])."""
    A = lambda cin, pf: [("branch1x1", cin, 64, (1, 1)), ("branch5x5_1", cin, 48, (1, 1)), ("branch5x5_2", 48, 64, (5, 5)),
                         ("branch3x3dbl_1", cin, 64, (1, 1)), ("branch3x3dbl_2", 64, 96, (3, 3)), ("branch3x3dbl_3", 96, 96, (3, 3)),
                         ("branch_pool", cin, pf, (1, 1))]
    B = lambda cin: [("branch3x3", cin, 384, (3, 3)), ("branch3x3dbl_1", cin, 64, (1, 1)), ("branch3x3dbl_2", 64, 96, (3, 3)),
                     ("branch3x3dbl_3", 96, 96, (3, 3))]
    C = lambda cin, c7: [("branch1x1", cin, 192, (1, 1)), ("branch7x7_1", cin, c7, (1, 1)), ("branch7x7_2", c7, c7, (1, 7)),
                         ("branch7x7_3", c7, 192, (7, 1)), ("branch7x7dbl_1", cin, c7, (1, 1)), ("branch7x7dbl_2", c7, c7, (7, 1)),
                         ("branch7x7dbl_3", c7, c7, (1, 7)), ("branch7x7dbl_4", c7, c7, (7, 1)), ("branch7x7dbl_5", c7, 192, (1, 7)),
                         ("branch_pool", cin, 192, (1, 1))]
    D = lambda cin: [("branch3x3_1", cin, 192, (1, 1)), ("branch3x3_2", 192, 320, (3, 3)), ("branch7x7x3_1", cin, 192, (1, 1)),
                     ("branch7x7x3_2", 192, 192, (1, 7)), ("branch7x7x3_3", 192, 192, (7, 1)), ("branch7x7x3_4", 192, 192, (3, 3))]
    E = lambda cin: [("branch1x1", cin, 320, (1, 1)), ("branch3x3_1", cin, 384, (1, 1)), ("branch3x3_2a", 384, 384, (1, 3)),
                     ("branch3x3_2b", 384, 384, (3, 1)), ("branch3x3dbl_1", cin, 448, (1, 1)), ("branch3x3dbl_2", 448, 384, (3, 3)),
                     ("branch3x3dbl_3a", 384, 384, (1, 3)), ("branch3x3dbl_3b", 384, 384, (3, 1)), ("branch_pool", cin, 192, (1, 1))]
    return [("Conv2d_1a_3x3", [("", 1, 32, (3, 3))]), ("Conv2d_2a_3x3", [("", 32, 32, (3, 3))]), ("Conv2d_2b_3x3", [("", 32, 64, (3, 3))]),
            ("Conv2d_3b_1x1", [("", 64, 80, (1, 1))]), ("Conv2d_4a_3x3", [("", 80, 192, (3, 3))]),
            ("Mixed_5b", A(192, 32)), ("Mixed_5c", A(256, 64)), ("Mixed_5d", A(288, 64)), ("Mixed_6a", B(288)),
            ("Mixed_6b", C(768, 128)), ("Mixed_6c", C(768, 160)), ("Mixed_6d", C(768, 160)), ("Mixed_6e", C(768, 192)),
            ("AuxLogits", [("conv0", 768, 128, (1, 1)), ("conv1", 128, 768, (5, 5))]),
            ("Mixed_7a", D(768)), ("Mixed_7b", E(1280)), ("Mixed_7c", E(2048))]


def state_dict_shapes(num_classes: int = 309, aux_logits: bool = True):
    """[(key, shape)] of the reference Melception's state dict, in its order."""
    out = []
    for blk, convs in _blocks():
        if blk == "AuxLogits" and not aux_logits:
            continue
        for name, cin, cout, (kh, kw) in convs:
            p = f"{blk}.{name}." if name else f"{blk}."
            out += [(p + "conv.weight", (cout, cin, kh, kw))]
            out += [(p + "bn." + k, (cout,)) for k in ("weight", "bias", "running_mean", "running_var")] + [(p + "bn.num_batches_tracked", ())]
        if blk == "AuxLogits":
            out += [("AuxLogits.fc.weight", (num_classes, 768)), ("AuxLogits.fc.bias", (num_classes,))]
    return out + [("fc.weight", (num_classes, 2048)), ("fc.bias", (num_classes,))]


def make_melception_state_dict(seed: int, init: str = "he", num_classes: int = 309, aux_logits: bool = True) -> Dict[str, torch.Tensor]:
    """Seeded Melception weights from numpy Philox uniforms (exact arithmetic only: the same bits on every platform).
    'he':   conv weights U(-a, a) with std sqrt(2 / fan_in); BN gamma in [0.5, 1.5], beta and running mean in [-0.2, 0.2], running var in [0.5, 2]:
            activations stay O(10) through the network, like a trained checkpoint's.
    'wide': the reference's own init (torchvision Inception3 init_weights: trunc-normal std 0.1 convs and fc, identity BN; here a zero-mean
            bounded Irwin-Hall(3) stand-in with std 0.1), whose activations grow to ~1e12 by Mixed_7c."""
    if init not in ("he", "wide"):
        raise ValueError("init must be 'he' or 'wide'")
    rng = np.random.Generator(np.random.Philox(seed))
    u = lambda shape, lo, hi: (lo + (hi - lo) * rng.random(size=shape, dtype=np.float64)).astype(np.float32)
    sd = {}
    for key, shape in state_dict_shapes(num_classes, aux_logits):
        if key.endswith("num_batches_tracked"):
            sd[key] = torch.tensor(0, dtype=torch.long)
            continue
        if init == "wide":
            if key.endswith("weight") and len(shape) > 1:
                v = ((rng.random(size=shape) + rng.random(size=shape) + rng.random(size=shape) - 1.5) * 0.2).astype(np.float32)
            elif key.endswith("bn.weight") or key.endswith("running_var"):
                v = np.ones(shape, np.float32)
            else:
                v = np.zeros(shape, np.float32)
        elif key.endswith("conv.weight"):
            fan_in = shape[1] * shape[2] * shape[3]
            a = float(np.sqrt(3.0) * np.sqrt(2.0 / fan_in))
            v = u(shape, -a, a)
        elif key.endswith("fc.weight"):
            a = float(np.sqrt(3.0 / shape[1]))
            v = u(shape, -a, a)
        elif key.endswith("bn.weight"):
            v = u(shape, 0.5, 1.5)
        elif key.endswith("running_var"):
            v = u(shape, 0.5, 2.0)
        else:  # bn.bias, running_mean, fc.bias
            v = u(shape, -0.2, 0.2)
        sd[key] = torch.from_numpy(v)
    return sd


def state_dict_checksum(sd: Dict[str, torch.Tensor]) -> np.ndarray:
    """Per tensor (fp64 sum, fp64 sum of squares), in key order."""
    return np.array([[float(v.double().sum()), float((v.double() ** 2).sum())] for v in sd.values()], dtype=np.float64)


def melception_forward(sd: Dict[str, torch.Tensor], x: torch.Tensor, features_list: Sequence[str], dtype=torch.float64):
    """The reference Melception.forward (melception.py:23-113) in eval mode: x (B, 80, T) -> tuple of features in features_list order; the
    forward stops after the last requested feature, as the reference's does.  Runs on x's device."""
    dev = x.device
    p = {k: v.to(dev, dtype) for k, v in sd.items() if not k.endswith("num_batches_tracked")}
    rem = list(features_list)
    feats = {}

    def conv(x, name, stride=1, padding=(0, 0)):
        x = F.conv2d(x, p[name + ".conv.weight"], stride=stride, padding=padding)
        x = F.batch_norm(x, p[name + ".bn.running_mean"], p[name + ".bn.running_var"], p[name + ".bn.weight"], p[name + ".bn.bias"], False, 0.0, 0.001)
        return F.relu(x)

    def take(name, v):
        feats[name] = v
        rem.remove(name)
        return not rem

    def out():
        return tuple(feats[a] for a in features_list)

    def block_a(x, n):
        b1 = conv(x, n + ".branch1x1")
        b5 = conv(conv(x, n + ".branch5x5_1"), n + ".branch5x5_2", padding=(2, 2))
        b3 = conv(conv(conv(x, n + ".branch3x3dbl_1"), n + ".branch3x3dbl_2", padding=(1, 1)), n + ".branch3x3dbl_3", padding=(1, 1))
        bp = conv(F.avg_pool2d(x, 3, 1, 1), n + ".branch_pool")
        return torch.cat([b1, b5, b3, bp], 1)

    def block_b(x, n):
        b3 = conv(x, n + ".branch3x3", stride=2)
        bd = conv(conv(conv(x, n + ".branch3x3dbl_1"), n + ".branch3x3dbl_2", padding=(1, 1)), n + ".branch3x3dbl_3", stride=2)
        return torch.cat([b3, bd, F.max_pool2d(x, 3, 2)], 1)

    def block_c(x, n):
        r, c = (0, 3), (3, 0)
        b1 = conv(x, n + ".branch1x1")
        b7 = conv(conv(conv(x, n + ".branch7x7_1"), n + ".branch7x7_2", padding=r), n + ".branch7x7_3", padding=c)
        bd = conv(x, n + ".branch7x7dbl_1")
        for i, pad in ((2, c), (3, r), (4, c), (5, r)):
            bd = conv(bd, n + f".branch7x7dbl_{i}", padding=pad)
        bp = conv(F.avg_pool2d(x, 3, 1, 1), n + ".branch_pool")
        return torch.cat([b1, b7, bd, bp], 1)

    def block_d(x, n):
        b3 = conv(conv(x, n + ".branch3x3_1"), n + ".branch3x3_2", stride=2)
        b7 = conv(conv(conv(x, n + ".branch7x7x3_1"), n + ".branch7x7x3_2", padding=(0, 3)), n + ".branch7x7x3_3", padding=(3, 0))
        b7 = conv(b7, n + ".branch7x7x3_4", stride=2)
        return torch.cat([b3, b7, F.max_pool2d(x, 3, 2)], 1)

    def block_e(x, n):
        b1 = conv(x, n + ".branch1x1")
        b3 = conv(x, n + ".branch3x3_1")
        b3 = torch.cat([conv(b3, n + ".branch3x3_2a", padding=(0, 1)), conv(b3, n + ".branch3x3_2b", padding=(1, 0))], 1)
        bd = conv(conv(x, n + ".branch3x3dbl_1"), n + ".branch3x3dbl_2", padding=(1, 1))
        bd = torch.cat([conv(bd, n + ".branch3x3dbl_3a", padding=(0, 1)), conv(bd, n + ".branch3x3dbl_3b", padding=(1, 0))], 1)
        bp = conv(F.avg_pool2d(x, 3, 1, 1), n + ".branch_pool")
        return torch.cat([b1, b3, bd, bp], 1)

    h = x.to(dtype).unsqueeze(1)
    h = conv(h, "Conv2d_1a_3x3", stride=2)
    h = conv(h, "Conv2d_2a_3x3")
    h = conv(h, "Conv2d_2b_3x3", padding=(1, 1))
    if "64" in rem and take("64", F.adaptive_avg_pool2d(h, (1, 1))):
        return out()
    h = conv(conv(h, "Conv2d_3b_1x1"), "Conv2d_4a_3x3")
    if "192" in rem and take("192", F.adaptive_avg_pool2d(h, (1, 1))):
        return out()
    for n in ("Mixed_5b", "Mixed_5c", "Mixed_5d"):
        h = block_a(h, n)
    h = block_b(h, "Mixed_6a")
    for n in ("Mixed_6b", "Mixed_6c", "Mixed_6d", "Mixed_6e"):
        h = block_c(h, n)
    if "768" in rem and take("768", F.adaptive_avg_pool2d(h, (1, 1))):
        return out()
    h = block_e(block_e(block_d(h, "Mixed_7a"), "Mixed_7b"), "Mixed_7c")
    h = torch.flatten(F.adaptive_avg_pool2d(h, (1, 1)), 1)
    if "2048" in rem and take("2048", h):
        return out()
    if "logits_unbiased" in rem:
        h = h.mm(p["fc.weight"].T)
        if take("logits_unbiased", h):
            return out()
        h = h + p["fc.bias"].unsqueeze(0)
    else:
        h = F.linear(h, p["fc.weight"], p["fc.bias"])
    feats["logits"] = h
    return out()
