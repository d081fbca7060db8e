"""Frechet Inception Distance: same signature, return dict and fp64 host arithmetic as the reference's calculate_fid
(Codebook/evaluation/metrics/fid.py:5-63): numpy mean / covariance of the (N, D) features, scipy.linalg.sqrtm of the covariance product."""
import numpy as np
import scipy.linalg
import torch


def _stats(features):
    if not (torch.is_tensor(features) and features.dim() == 2):
        raise ValueError("FID needs a 2-D feature tensor")
    a = features.numpy()
    return np.atleast_1d(np.mean(a, axis=0)), np.atleast_2d(np.cov(a, rowvar=False))


def calculate_fid(featuresdict_1, featuresdict_2, feat_layer_name):
    mu1, s1 = _stats(featuresdict_1[feat_layer_name])
    mu2, s2 = _stats(featuresdict_2[feat_layer_name])
    if mu1.shape != mu2.shape or s1.shape != s2.shape:
        raise ValueError("FID: the two feature sets have different dimensions")
    root = scipy.linalg.sqrtm(s1.dot(s2))
    if not np.isfinite(root).all():  # nearly singular product: regularise both covariances, as the reference does
        eye = np.eye(s1.shape[0]) * 1e-6
        root = scipy.linalg.sqrtm((s1 + eye).dot(s2 + eye))
    if np.iscomplexobj(root):
        if not np.allclose(np.diagonal(root).imag, 0, atol=1e-3):
            raise ValueError(f"FID: imaginary component {np.max(np.abs(root.imag))}")
        root = root.real
    d = mu1 - mu2
    return {"frechet_inception_distance": float(d.dot(d) + np.trace(s1) + np.trace(s2) - 2 * np.trace(root))}
