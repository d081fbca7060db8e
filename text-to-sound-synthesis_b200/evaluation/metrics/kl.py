"""Paired KL divergence KL(real_i || fake_i): same signature, return dict and torch arithmetic as the reference's calculate_kl
(Codebook/evaluation/metrics/kl.py:4-78).  Every fake is paired with the real that shares its key: the file stem without '_mel' and without
everything from '_sample_' on.  The Diffsound evaluation's dataset ('caps') is supported; 'vas' / 'vggsound' keys are not."""
from pathlib import Path

import torch


def path_to_sharedkey(path, dataset_name, classes=None):
    if dataset_name.lower() != "caps":
        raise NotImplementedError(f"KL pairing is implemented for dataset_name='caps', not {dataset_name!r}")
    return Path(path).stem.replace("_mel", "").split("_sample_")[0]


def calculate_kl(featuresdict_1, featuresdict_2, feat_layer_name, dataset_name, classes=None):
    if feat_layer_name != "logits":
        raise ValueError("the KL metric is defined on 'logits'")
    if "file_path_" not in featuresdict_1 or "file_path_" not in featuresdict_2:
        raise ValueError("KL needs the file paths of both feature sets ('file_path_')")
    key = lambda p: path_to_sharedkey(p, dataset_name, classes)
    fakes = {}
    for p, f in {p: f for p, f in zip(featuresdict_1["file_path_"], featuresdict_1[feat_layer_name])}.items():
        fakes.setdefault(key(p), []).append(f)
    reals = {key(p): f for p, f in zip(featuresdict_2["file_path_"], featuresdict_2[feat_layer_name])}
    pred, target = [], []
    for k, real in reals.items():  # in the order of the reals; a real without fakes contributes nothing
        group = fakes.get(k, [])
        pred += group
        target += [real] * len(group)
    p1 = torch.stack(pred, 0).softmax(dim=1)
    p2 = torch.stack(target, 0).softmax(dim=1)
    kl = torch.nn.functional.kl_div((p1 + 1e-6).log(), p2, reduction="sum") / len(p1)
    return {"kullback_leibler_divergence": float(kl)}
