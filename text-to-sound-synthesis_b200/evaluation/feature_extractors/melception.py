"""Drop-in for Codebook/evaluation/feature_extractors/melception.py::Melception (the Diffsound evaluation's feature extractor).

Same constructor, the same state_dict keys and shapes as torchvision's Inception3 with the 1-channel Conv2d_1a_3x3 (580 entries with the default
aux_logits=True), the same forward contract (features_list order, early exit after the last requested feature, '64' / '192' / '768' as
(B, C, 1, 1)) and convert_features_tuple_to_dict, so a YAML `target:` swap in evaluate.py's config is the whole integration.  The modules only hold
parameters under torchvision's names (torchvision is not imported); compute is MelceptionEngine (CUDA kernels, no CPU path).  Eval mode only:
BatchNorm batch statistics are not implemented.
"""
import torch
from torch import nn

from ...engine_base import EngineModule
from ...melception_engine import FEATURES, MelceptionEngine


class BasicConv2d(nn.Module):
    """torchvision's BasicConv2d parameter layout: bias-free conv + BatchNorm2d(eps=0.001) (ReLU follows in the engine)."""

    def __init__(self, cin, cout, kernel_size, **kw):
        super().__init__()
        self.conv = nn.Conv2d(cin, cout, kernel_size, bias=False, **kw)
        self.bn = nn.BatchNorm2d(cout, eps=0.001)


class _Block(nn.Module):
    def __init__(self, convs):
        super().__init__()
        for name, cin, cout, k in convs:
            setattr(self, name, BasicConv2d(cin, cout, k))


def _inception_a(cin, pf):
    return _Block([("branch1x1", cin, 64, 1), ("branch5x5_1", cin, 48, 1), ("branch5x5_2", 48, 64, 5), ("branch3x3dbl_1", cin, 64, 1),
                   ("branch3x3dbl_2", 64, 96, 3), ("branch3x3dbl_3", 96, 96, 3), ("branch_pool", cin, pf, 1)])


def _inception_b(cin):
    return _Block([("branch3x3", cin, 384, 3), ("branch3x3dbl_1", cin, 64, 1), ("branch3x3dbl_2", 64, 96, 3), ("branch3x3dbl_3", 96, 96, 3)])


def _inception_c(cin, c7):
    return _Block([("branch1x1", cin, 192, 1), ("branch7x7_1", cin, c7, 1), ("branch7x7_2", c7, c7, (1, 7)), ("branch7x7_3", c7, 192, (7, 1)),
                   ("branch7x7dbl_1", cin, c7, 1), ("branch7x7dbl_2", c7, c7, (7, 1)), ("branch7x7dbl_3", c7, c7, (1, 7)),
                   ("branch7x7dbl_4", c7, c7, (7, 1)), ("branch7x7dbl_5", c7, 192, (1, 7)), ("branch_pool", cin, 192, 1)])


def _inception_d(cin):
    return _Block([("branch3x3_1", cin, 192, 1), ("branch3x3_2", 192, 320, 3), ("branch7x7x3_1", cin, 192, 1), ("branch7x7x3_2", 192, 192, (1, 7)),
                   ("branch7x7x3_3", 192, 192, (7, 1)), ("branch7x7x3_4", 192, 192, 3)])


def _inception_e(cin):
    return _Block([("branch1x1", cin, 320, 1), ("branch3x3_1", cin, 384, 1), ("branch3x3_2a", 384, 384, (1, 3)), ("branch3x3_2b", 384, 384, (3, 1)),
                   ("branch3x3dbl_1", cin, 448, 1), ("branch3x3dbl_2", 448, 384, 3), ("branch3x3dbl_3a", 384, 384, (1, 3)),
                   ("branch3x3dbl_3b", 384, 384, (3, 1)), ("branch_pool", cin, 192, 1)])


class _InceptionAux(nn.Module):
    """Parameters of torchvision's InceptionAux (present in the checkpoints, never run by Melception.forward)."""

    def __init__(self, cin, num_classes):
        super().__init__()
        self.conv0 = BasicConv2d(cin, 128, 1)
        self.conv1 = BasicConv2d(128, 768, 5)
        self.fc = nn.Linear(768, num_classes)


class Melception(EngineModule):
    def __init__(self, num_classes, features_list, feature_extractor_weights_path, aux_logits=True, transform_input=False, dropout=0.5, **kwargs):
        """As the reference: Inception3(num_classes, aux_logits, ...) with a 1-channel Conv2d_1a_3x3, no max pools in the stem, weights loaded
        strictly from torch.load(path)['model'] and frozen.  transform_input and dropout have no effect on the reference's forward either."""
        super().__init__()
        if kwargs:
            raise TypeError(f"Melception: unsupported arguments {sorted(kwargs)}")
        unknown = [f for f in features_list if f not in FEATURES]
        if unknown:
            raise ValueError(f"unknown features {unknown}; choose from {FEATURES}")
        self.features_list = list(features_list)
        self.aux_logits, self.transform_input = aux_logits, transform_input
        self.Conv2d_1a_3x3 = BasicConv2d(1, 32, 3)
        self.Conv2d_2a_3x3 = BasicConv2d(32, 32, 3)
        self.Conv2d_2b_3x3 = BasicConv2d(32, 64, 3)
        self.Conv2d_3b_1x1 = BasicConv2d(64, 80, 1)
        self.Conv2d_4a_3x3 = BasicConv2d(80, 192, 3)
        self.Mixed_5b = _inception_a(192, 32)
        self.Mixed_5c = _inception_a(256, 64)
        self.Mixed_5d = _inception_a(288, 64)
        self.Mixed_6a = _inception_b(288)
        self.Mixed_6b = _inception_c(768, 128)
        self.Mixed_6c = _inception_c(768, 160)
        self.Mixed_6d = _inception_c(768, 160)
        self.Mixed_6e = _inception_c(768, 192)
        self.AuxLogits = _InceptionAux(768, num_classes) if aux_logits else None
        self.Mixed_7a = _inception_d(768)
        self.Mixed_7b = _inception_e(1280)
        self.Mixed_7c = _inception_e(2048)
        self.fc = nn.Linear(2048, num_classes)
        self.engine = MelceptionEngine(self)
        state_dict = torch.load(feature_extractor_weights_path, map_location="cpu")
        self.load_state_dict(state_dict["model"])
        for p in self.parameters():
            p.requires_grad_(False)

    @torch.no_grad()
    def forward(self, x):
        """x (B, 80, T) fp32 CUDA (normalised mels) -> tuple of the features in features_list order."""
        if self.training:
            raise RuntimeError("Melception runs in eval mode only (BatchNorm batch statistics are not implemented): call .eval() first, as "
                               "evaluate.py does")
        feats = self.engine.forward(x, self.features_list)
        return tuple(feats[a] for a in self.features_list)

    def convert_features_tuple_to_dict(self, features):
        """Recover the {name: feature} mapping from forward()'s tuple."""
        message = "Features must be the output of forward function"
        assert type(features) is tuple and len(features) == len(self.features_list), message
        return dict(zip(self.features_list, features))
