"""Drop-in for Diffsound/vocoder/modules.py::Generator (MelGAN, inference side).  Same constructor, same state_dict keys
(`model.{i}.{bias,weight_g,weight_v}`, `model.{i}.block.{2,4}.*`, `model.{i}.shortcut.*`), so the shipped checkpoint
`vocoder/logs/vggsound/best_netG.pt` loads unchanged.  Modules only hold parameters; compute is `VocoderEngine`.
"""
import numpy as np
import torch
from torch import nn

from ..engine_base import EngineModule
from ..vocoder_engine import VocoderEngine


def _wn(m):
    return torch.nn.utils.weight_norm(m)  # parameter names weight_g / weight_v, as in the reference checkpoints


class _Holder(nn.Module):
    def forward(self, *a, **k):
        raise RuntimeError(f"{type(self).__name__} only stores parameters; compute runs in VocoderEngine (CUDA kernels)")


class ResnetBlock(_Holder):
    def __init__(self, dim, dilation=1):
        super().__init__()
        self.dilation = dilation
        self.block = nn.Sequential(nn.LeakyReLU(0.2), nn.ReflectionPad1d(dilation), _wn(nn.Conv1d(dim, dim, kernel_size=3, dilation=dilation)),
                                   nn.LeakyReLU(0.2), _wn(nn.Conv1d(dim, dim, kernel_size=1)))
        self.shortcut = _wn(nn.Conv1d(dim, dim, kernel_size=1))


class Generator(EngineModule):
    def __init__(self, input_size, ngf, n_residual_layers, precision="f16x3"):
        super().__init__()
        ratios = [8, 8, 2, 2]
        self.ratios = ratios
        self.hop_length = int(np.prod(ratios))
        self.n_residual_layers = n_residual_layers
        mult = int(2 ** len(ratios))
        model = [nn.ReflectionPad1d(3), _wn(nn.Conv1d(input_size, mult * ngf, kernel_size=7, padding=0))]
        for r in ratios:
            model += [nn.LeakyReLU(0.2), _wn(nn.ConvTranspose1d(mult * ngf, mult * ngf // 2, kernel_size=r * 2, stride=r, padding=r // 2 + r % 2,
                                                                output_padding=r % 2))]
            for j in range(n_residual_layers):
                model += [ResnetBlock(mult * ngf // 2, dilation=3 ** j)]
            mult //= 2
        model += [nn.LeakyReLU(0.2), nn.ReflectionPad1d(3), _wn(nn.Conv1d(ngf, 1, kernel_size=7, padding=0)), nn.Tanh()]
        self.model = nn.Sequential(*model)
        for m in self.modules():  # weights_init of the reference (modules.py:9-15)
            if isinstance(m, (nn.Conv1d, nn.ConvTranspose1d)):
                m.weight_v.data.normal_(0.0, 0.02)
        self.engine = VocoderEngine(self, precision=precision)

    @torch.no_grad()
    def forward(self, x):
        """mel in [0,1] (B, 80, T) -> waveform (B, 1, 256*T)   (modules.py:129-130); batched, unlike the reference script's B=1 loop."""
        return self.engine.forward(x)
