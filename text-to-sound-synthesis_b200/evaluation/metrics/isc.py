"""Inception Score: same signature, return dict, RandomState shuffle and fp64 arithmetic as the reference's calculate_isc
(Codebook/evaluation/metrics/isc.py:5-32)."""
import numpy as np
import torch


def calculate_isc(featuresdict, feat_layer_name, rng_seed, samples_shuffle, splits):
    logits = featuresdict[feat_layer_name]
    if not (torch.is_tensor(logits) and logits.dim() == 2):
        raise ValueError("ISc needs a 2-D logit tensor")
    n = logits.shape[0]
    if samples_shuffle:
        logits = logits[np.random.RandomState(rng_seed).permutation(n), :]
    logits = logits.double()
    prob, logp = logits.softmax(dim=1), logits.log_softmax(dim=1)
    scores = []
    for k in range(splits):
        lo, hi = k * n // splits, (k + 1) * n // splits
        p, lp = prob[lo:hi], logp[lo:hi]
        marginal = p.mean(dim=0, keepdim=True)
        scores.append((p * (lp - marginal.log())).sum(dim=1).mean().exp().item())
    return {"inception_score_mean": float(np.mean(scores)), "inception_score_std": float(np.std(scores))}
