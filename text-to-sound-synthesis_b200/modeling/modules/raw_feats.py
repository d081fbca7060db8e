"""Drop-in for Codebook/specvqgan/modules/misc/raw_feats.py::RawFeatsStage: the condition stage of the caps_transformer configs passes the
(B, Cf, Tc) features through unchanged (a fake VQ-model interface, no parameters)."""
import torch


class RawFeatsStage(object):
    def __init__(self):
        pass

    def eval(self):
        return self

    def encode(self, c):
        return c, None, (None, None, c)

    def decode(self, c):
        return c

    def get_input(self, batch, k):
        x = batch[k]
        x = x.permute(0, 2, 1).to(memory_format=torch.contiguous_format)
        return x.float()
