"""Drop-ins for the reference Codebook/evaluation package: the Melception feature extractor and the KL / ISc / FID / KID metrics."""
