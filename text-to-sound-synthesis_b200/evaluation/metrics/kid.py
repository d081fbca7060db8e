"""Kernel Inception Distance: same signature, return dict, RandomState draws and host arithmetic (numpy on the features' own dtype) as the
reference's calculate_kid (Codebook/evaluation/metrics/kid.py:6-72): unbiased polynomial-kernel MMD^2 over random subsets."""
import numpy as np
import torch


def _poly(X, Y, degree, gamma, coef0):
    g = 1.0 / X.shape[1] if gamma in (None, "none", "null", "None") else gamma
    return (np.matmul(X, Y.T) * g + coef0) ** degree


def polynomial_mmd(features_1, features_2, degree, gamma, coef0):
    kxx = _poly(features_1, features_1, degree, gamma, coef0)
    kyy = _poly(features_2, features_2, degree, gamma, coef0)
    kxy = _poly(features_1, features_2, degree, gamma, coef0)
    m = kxx.shape[0]
    off_x = (kxx.sum(axis=1) - np.diagonal(kxx)).sum()  # row sums without the diagonal, then their total
    off_y = (kyy.sum(axis=1) - np.diagonal(kyy)).sum()
    cross = kxy.sum(axis=0).sum()
    return (off_x + off_y) / (m * (m - 1)) - 2 * cross / (m * m)


def calculate_kid(featuresdict_1, featuresdict_2, subsets, subset_size, degree, gamma, coef0, rng_seed, feat_layer_name):
    f1, f2 = featuresdict_1[feat_layer_name], featuresdict_2[feat_layer_name]
    if not (torch.is_tensor(f1) and f1.dim() == 2 and torch.is_tensor(f2) and f2.dim() == 2 and f1.shape[1] == f2.shape[1]):
        raise ValueError("KID needs two 2-D feature tensors of the same width")
    m = min(subset_size, len(f2), len(f1))
    f1, f2 = f1.cpu().numpy(), f2.cpu().numpy()
    rng = np.random.RandomState(rng_seed)
    mmds = np.zeros(subsets)
    for i in range(subsets):
        a = f1[rng.choice(len(f1), m, replace=False)]
        b = f2[rng.choice(len(f2), m, replace=False)]
        mmds[i] = polynomial_mmd(a, b, degree, gamma, coef0)
    return {"kernel_inception_distance_mean": float(np.mean(mmds)), "kernel_inception_distance_std": float(np.std(mmds))}
