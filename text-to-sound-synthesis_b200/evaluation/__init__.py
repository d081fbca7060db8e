"""Drop-ins for the reference Codebook/evaluation package (the Melception feature extractor and the KL / ISc / FID / KID metrics) and for
Codebook/AudiocaptionLoss (the ACT captioning transformer, in audiocaption/)."""
