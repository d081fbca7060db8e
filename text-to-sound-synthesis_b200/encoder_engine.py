"""SpecVQGAN encoder + nearest-codebook quantiser on sm_90a: the training-time tokeniser behind DALLE.get_tokens (SURVEY.md section 8f N4).

Same machinery as the decoder (decoder_engine.py): zero-bordered channels-last images, every Conv2d a wgmma implicit GEMM with taps in
split-TF32 (the nearest-code argmin needs fp32-class latents), GroupNorm / AttnBlock kernels shared with the decoder.  New here:
  * Downsample (zero pad (0,1,0,1) + 3x3 stride-2 conv, model.py:55-75): the image is rearranged into its four stride-2 phases on the
    half-resolution padded grid (dsb_space_to_depth_padded); the strided conv is then a 9-tap GEMM with constant row shifts and per-tap A column
    offsets -- no im2col buffer;
  * VectorQuantizer.forward's argmin (quantize.py:56-63): |e|^2 - 2 z.e from one GEMM (alpha = -2, bias = |e|^2) + a row-argmin kernel.
Reference: specvqgan/modules/diffusionmodules/model.py:410-500 (Encoder), sound_synthesis/modeling/codecs/spec_codec/vqgan.py:48-54 (encode),
sound_synthesis/modeling/models/dalle_spec.py:71-78 (get_tokens).
"""
from __future__ import annotations

import torch

from . import ops
from .decoder_engine import DecoderEngine


class EncoderEngine(DecoderEngine):
    def __init__(self, vq):
        super().__init__(vq, precision="tf32x3")
        self.options = {}  # EncoderEngine(vq) takes no arguments of its own

    def _pack(self):
        vq, e = self.m, self.m.encoder
        if vq.quant_conv.weight.device.type != "cuda":
            raise RuntimeError("EncoderEngine needs the module on a CUDA device (no CPU fallback)")
        f = lambda p: p.detach().float().contiguous()
        self.w = {}

        def conv(name, m):
            self.w[name] = (self._pack_conv(m), f(m.bias), m.kernel_size[0])

        def gn(name, m):
            self.w[name] = (f(m.weight), f(m.bias), m.eps)

        def res(name, m):
            gn(name + ".norm1", m.norm1); conv(name + ".conv1", m.conv1); gn(name + ".norm2", m.norm2); conv(name + ".conv2", m.conv2)
            if hasattr(m, "nin_shortcut"):
                conv(name + ".nin", m.nin_shortcut)

        def attn(name, m):
            gn(name + ".norm", m.norm)
            for n in ("q", "k", "v", "proj_out"):
                conv(name + "." + n, getattr(m, n))

        conv("conv_in", e.conv_in)
        for lvl, down in enumerate(e.down):
            for j, blk in enumerate(down.block):
                res(f"down.{lvl}.block.{j}", blk)
            for j, a in enumerate(down.attn):
                attn(f"down.{lvl}.attn.{j}", a)
            if hasattr(down, "downsample"):
                conv(f"down.{lvl}.downsample", down.downsample.conv)
        res("mid.block_1", e.mid.block_1); attn("mid.attn_1", e.mid.attn_1); res("mid.block_2", e.mid.block_2)
        gn("norm_out", e.norm_out)
        conv("conv_out", e.conv_out)
        conv("quant_conv", vq.quant_conv)
        cb = f(vq.quantize.embedding.weight)
        self.codebook = cb
        self.cb_split = ops.pack_split_weight(cb, 1)          # (K, 3*Ep) W operand of the distance GEMM
        self.cb_sq = (cb.double() ** 2).sum(1).float()         # |e_k|^2, set-up time only
        self._graphs.clear()

    def _downsample(self, x, name):
        """x: padded (B, H+2, W+2, C) fp32 -> padded (B, H/2+2, W/2+2, C)."""
        w, b, _ = self.w[name]
        B, Hp, Wp, C = x.shape
        a = ops.space_to_depth_padded(x, split=True)            # (B, Ho, Wo, 8C) = [hi (4 phases x C) | lo]
        Ho, Wo = a.shape[1], a.shape[2]
        R = B * Ho * Wo
        taps, acol = [], []
        for dy in range(3):
            for dx in range(3):
                ph = 2 * (dy % 2) + (dx % 2)
                shift = (dy // 2) * Wo + (dx // 2)
                taps += [shift, shift, shift]                   # hi*Whi, lo*Whi, hi*Wlo (the weight is packed [Whi | Whi | Wlo] per tap)
                acol += [ph * C, 4 * C + ph * C, ph * C]
        out = torch.empty(B, Ho, Wo, w.shape[0], dtype=torch.float32, device=x.device)
        ops.gemm(a.view(R, 8 * C), w, b, None, out.view(R, -1), dtype=ops.TF32, taps=taps, tap_acol=acol, k_per_tap=C, geo=(Ho * Wo, Wo, 1, Ho - 1, 1, Wo - 1))
        self.launches += 2
        return out

    @torch.no_grad()
    def _encode_padded(self, x):
        e = self.m.encoder
        h = self._conv(x, "conv_in")
        for lvl in range(e.num_resolutions):
            for j in range(e.num_res_blocks):
                h = self._res(h, f"down.{lvl}.block.{j}")
                if len(e.down[lvl].attn) > 0:
                    h = self._attn(h, f"down.{lvl}.attn.{j}")
            if lvl != e.num_resolutions - 1:
                h = self._downsample(h, f"down.{lvl}.downsample")
        h = self._res(h, "mid.block_1")
        h = self._attn(h, "mid.attn_1")
        h = self._res(h, "mid.block_2")
        h = self._conv(self._gn(h, "norm_out"), "conv_out", presplit=True)
        return self._conv(h, "quant_conv")                       # (B, Hq+2, Wq+2, E), zero border

    @torch.no_grad()
    def encode(self, mel):
        """mel (B, 1, H, W) fp32 NCHW -> (z (B, E, H/16, W/16) after quant_conv, nearest-code ids (B, H/16 * W/16) row-major)."""
        self.ensure_current()
        B, Cin, H, W = mel.shape
        down = 2 ** (self.m.encoder.num_resolutions - 1)
        if H % down or W % down:
            raise RuntimeError(f"encoder input {H}x{W} must be divisible by {down}")
        self.launches = 0
        x = torch.nn.functional.pad(mel.detach().float().permute(0, 2, 3, 1), (0, 0, 1, 1, 1, 1)).contiguous()   # layout only
        zp = self._encode_padded(x)
        z = zp[:, 1:-1, 1:-1, :].contiguous()                    # (B, Hq, Wq, E)
        Hq, Wq, E = z.shape[1], z.shape[2], z.shape[3]
        d = ops.gemm_split(ops.split_tf32(z.view(-1, E)), self.cb_split, self.cb_sq, alpha=-2.0)   # |e|^2 - 2 z.e   (|z|^2 is constant per row)
        ids = ops.row_argmin(d, self.codebook.shape[0]).view(B, Hq * Wq)
        self.launches += 3
        return z.permute(0, 3, 1, 2).contiguous(), ids
