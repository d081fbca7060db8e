"""Restatements of the reference Codebook/evaluation/metrics/: same signatures, return dicts and random draws."""
