"""Feature extractors (reference Codebook/evaluation/feature_extractors/)."""
