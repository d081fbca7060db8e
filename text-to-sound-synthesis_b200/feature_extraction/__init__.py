"""Feature extraction (reference Codebook/feature_extraction/)."""
