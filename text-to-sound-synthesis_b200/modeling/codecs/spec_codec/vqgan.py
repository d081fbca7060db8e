"""Drop-in for the decode side of sound_synthesis/modeling/codecs/spec_codec/vqgan.py::VQModel, plus the pieces it pulls from
specvqgan (Decoder: modules/diffusionmodules/model.py:570-671; VectorQuantizer.get_codebook_entry: modules/vqvae/quantize.py:88-103;
ColumnMajor: modules/transformer/permuter.py:21-55).  Same state_dict keys for quantize / post_quant_conv / decoder, so a
SpecVQGAN checkpoint's ["state_dict"] loads with strict=False exactly as the reference does (vqgan.py:44-52).

The modules only hold parameters; compute is `DecoderEngine` (wgmma implicit-GEMM convs on zero-padded channels-last
buffers + HBM-bound GroupNorm / upsample kernels).  The encoder / GAN losses (stage-1 training) are out of scope (SURVEY 8).
"""
import numpy as np
import torch
from torch import nn

from ....decoder_engine import DecoderEngine
from ....encoder_engine import EncoderEngine
from ....engine_base import EngineModule


class ColumnMajor(nn.Module):
    """Index permutation only (no arithmetic): same buffers and forward(x, reverse) as permuter.py:21-55."""

    def __init__(self, H, W):
        super().__init__()
        self.H, self.W = H, W
        idx = torch.tensor(np.arange(H * W).reshape(H, W).T.ravel())
        self.register_buffer("forward_shuffle_idx", idx)
        self.register_buffer("backward_shuffle_idx", torch.argsort(idx))

    def forward(self, x, reverse=False):
        return x[:, self.backward_shuffle_idx] if reverse else x[:, self.forward_shuffle_idx]


class Identity(nn.Module):
    """permuter.py Identity: token order unchanged, no buffers."""

    def forward(self, x, reverse=False):
        return x


class _Holder(nn.Module):
    def forward(self, *a, **k):
        raise RuntimeError(f"{type(self).__name__} only stores parameters; compute runs in DecoderEngine (CUDA kernels)")


def Normalize(c):
    return nn.GroupNorm(num_groups=32, num_channels=c, eps=1e-6, affine=True)


class ResnetBlock(_Holder):
    def __init__(self, cin, cout):
        super().__init__()
        self.in_channels, self.out_channels = cin, cout
        self.norm1 = Normalize(cin)
        self.conv1 = nn.Conv2d(cin, cout, 3, 1, 1)
        self.norm2 = Normalize(cout)
        self.conv2 = nn.Conv2d(cout, cout, 3, 1, 1)
        if cin != cout:
            self.nin_shortcut = nn.Conv2d(cin, cout, 1, 1, 0)


class AttnBlock(_Holder):
    def __init__(self, c):
        super().__init__()
        self.in_channels = c
        self.norm = Normalize(c)
        self.q = nn.Conv2d(c, c, 1)
        self.k = nn.Conv2d(c, c, 1)
        self.v = nn.Conv2d(c, c, 1)
        self.proj_out = nn.Conv2d(c, c, 1)


class Upsample(_Holder):
    def __init__(self, c, with_conv):
        super().__init__()
        self.with_conv = with_conv
        if with_conv:
            self.conv = nn.Conv2d(c, c, 3, 1, 1)


class Downsample(_Holder):
    def __init__(self, c, with_conv):
        super().__init__()
        assert with_conv
        self.with_conv = with_conv
        self.conv = nn.Conv2d(c, c, 3, 2, 0)  # applied after a (0,1,0,1) zero pad (model.py:55-75)


class Encoder(nn.Module):
    """Parameter holder with the reference's names (specvqgan/modules/diffusionmodules/model.py:410-475); compute runs in EncoderEngine."""

    def __init__(self, *, ch, out_ch, ch_mult=(1, 2, 4, 8), num_res_blocks, attn_resolutions, dropout=0.0, resamp_with_conv=True, in_channels,
                 resolution, z_channels, double_z=True, **ignore_kwargs):
        super().__init__()
        assert dropout == 0.0 and resamp_with_conv
        self.ch, self.num_resolutions, self.num_res_blocks = ch, len(ch_mult), num_res_blocks
        self.conv_in = nn.Conv2d(in_channels, ch, 3, 1, 1)
        curr_res = resolution
        in_ch_mult = (1,) + tuple(ch_mult)
        self.down = nn.ModuleList()
        block_in = ch
        for i_level in range(self.num_resolutions):
            block, attn = nn.ModuleList(), nn.ModuleList()
            block_in, block_out = ch * in_ch_mult[i_level], ch * ch_mult[i_level]
            for _ in range(num_res_blocks):
                block.append(ResnetBlock(block_in, block_out))
                block_in = block_out
                if curr_res in attn_resolutions:
                    attn.append(AttnBlock(block_in))
            down = nn.Module()
            down.block, down.attn = block, attn
            if i_level != self.num_resolutions - 1:
                down.downsample = Downsample(block_in, True)
                curr_res = curr_res // 2
            self.down.append(down)
        self.mid = nn.Module()
        self.mid.block_1 = ResnetBlock(block_in, block_in)
        self.mid.attn_1 = AttnBlock(block_in)
        self.mid.block_2 = ResnetBlock(block_in, block_in)
        self.norm_out = Normalize(block_in)
        self.conv_out = nn.Conv2d(block_in, 2 * z_channels if double_z else z_channels, 3, 1, 1)

    def forward(self, x):
        raise RuntimeError("call VQModel.encode (EncoderEngine); Encoder only stores parameters")


class Decoder(nn.Module):
    def __init__(self, *, ch, out_ch, ch_mult=(1, 2, 4, 8), num_res_blocks, attn_resolutions, dropout=0.0, resamp_with_conv=True, in_channels,
                 resolution, z_channels, give_pre_end=False, **ignorekwargs):
        super().__init__()
        assert dropout == 0.0 and resamp_with_conv and not give_pre_end
        self.ch, self.num_resolutions, self.num_res_blocks = ch, len(ch_mult), num_res_blocks
        block_in = ch * ch_mult[-1]
        curr_res = resolution // 2 ** (self.num_resolutions - 1)
        self.conv_in = nn.Conv2d(z_channels, block_in, 3, 1, 1)
        self.mid = nn.Module()
        self.mid.block_1 = ResnetBlock(block_in, block_in)
        self.mid.attn_1 = AttnBlock(block_in)
        self.mid.block_2 = ResnetBlock(block_in, block_in)
        self.up = nn.ModuleList()
        for i_level in reversed(range(self.num_resolutions)):
            block, attn = nn.ModuleList(), nn.ModuleList()
            block_out = ch * ch_mult[i_level]
            for _ in range(num_res_blocks + 1):
                block.append(ResnetBlock(block_in, block_out))
                block_in = block_out
                if curr_res in attn_resolutions:
                    attn.append(AttnBlock(block_in))
            up = nn.Module()
            up.block, up.attn = block, attn
            if i_level != 0:
                up.upsample = Upsample(block_in, True)
                curr_res = curr_res * 2
            self.up.insert(0, up)
        self.norm_out = Normalize(block_in)
        self.conv_out = nn.Conv2d(block_in, out_ch, 3, 1, 1)

    def forward(self, z):
        raise RuntimeError("call VQModel.decode / decode_tokens (DecoderEngine); Decoder only stores parameters")


class VectorQuantizer(nn.Module):
    def __init__(self, n_e, e_dim, beta=0.25):
        super().__init__()
        self.n_e, self.e_dim, self.beta = n_e, e_dim, beta
        self.embedding = nn.Embedding(n_e, e_dim)
        self.embedding.weight.data.uniform_(-1.0 / n_e, 1.0 / n_e)

    @torch.no_grad()
    def get_codebook_entry(self, indices, shape):
        """indices (N,) in row-major (b,h,w) order, shape (B,H,W,C) -> z_q (B,C,H,W)  (quantize.py:88-103); a pure gather."""
        z = self.embedding.weight.detach()[indices]
        if shape is not None:
            z = z.view(shape).permute(0, 3, 1, 2).contiguous()
        return z


class VQModel(EngineModule):
    def __init__(self, ddconfig, lossconfig=None, n_embed=256, embed_dim=256, ckpt_path=None, ignore_keys=[], image_key="image",
                 colorize_nlabels=None, monitor=None, precision="f16x3"):
        super().__init__()
        self.image_key = image_key
        self.ddconfig = dict(ddconfig)
        self.encoder = Encoder(**ddconfig)
        self.decoder = Decoder(**ddconfig)
        self.quantize = VectorQuantizer(n_embed, embed_dim, beta=0.25)
        self.quant_conv = nn.Conv2d(ddconfig["z_channels"], embed_dim, 1)
        self.post_quant_conv = nn.Conv2d(embed_dim, ddconfig["z_channels"], 1)
        self.engine = DecoderEngine(self, precision=precision)
        self.enc_engine = EncoderEngine(self)
        if ckpt_path is not None:
            self.init_from_ckpt(ckpt_path, ignore_keys=ignore_keys)

    def init_from_ckpt(self, path, ignore_keys=list()):
        sd = torch.load(path, map_location="cpu")["state_dict"]
        for k in list(sd.keys()):
            if any(k.startswith(ik) for ik in ignore_keys):
                del sd[k]
        self.load_state_dict(sd, strict=False)  # encoder / loss keys are ignored, as with the reference's strict=False
        print(f"Restored from {path}")

    @torch.no_grad()
    def encode(self, x):
        """mel (B, 1, H, W) -> (quant (B, E, H/16, W/16), None, (None, None, indices (B*H/16*W/16, 1)))  (vqgan.py:48-54).  The tokeniser is
        inference-only here (the frozen stage-1 codec of Diffsound training): no commitment loss / perplexity / one-hot encodings."""
        z, ids = self.enc_engine.encode(x)
        B, E, Hq, Wq = z.shape
        quant = self.quantize.get_codebook_entry(ids.reshape(-1), (B, Hq, Wq, E))
        self.last_latent = z  # pre-quantisation latent, kept for parity checks
        return quant, None, (None, None, ids.reshape(-1, 1))

    @torch.no_grad()
    def decode(self, quant):
        """quant (B, embed_dim, H, W) NCHW -> mel (B, out_ch, 16H, 16W)   (vqgan.py:62-65)."""
        return self.engine.decode_latents(quant)

    @torch.no_grad()
    def decode_tokens(self, ids, grid):
        """Fast path of DALLE.decode_to_img: column-major token ids (B, H*W) -> mel; un-permute + gather run in one kernel."""
        return self.engine.decode_tokens(ids, grid)
