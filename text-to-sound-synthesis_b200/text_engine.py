"""CLIP text tower on sm_90a (SURVEY.md section 8f N2): captions' token ids -> the (B, 77, 512) per-token embeddings the denoiser cross-attends to.

Same building blocks as the denoiser engine: fp16 wgmma GEMMs with fused bias / QuickGELU (= GELU2, x * sigmoid(1.702 x)) / residual epilogues,
one-warp-per-row LayerNorm, the mma.sync fp16 attention kernel with its causal flag (8 heads x 64, 77 positions), fp32 residual stream.
Reference: sound_synthesis/modeling/embeddings/clip_text_embedding.py:46-88, sound_synthesis/modeling/modules/clip/model.py:166-199 (blocks),
:323-329 (causal mask).  Runs once per caption batch (12 layers x 77 tokens: ~0.1 % of a 100-step sample()).
"""
from __future__ import annotations

import math

import torch

from . import ops
from .engine_base import PackedEngine


class TextTowerEngine(PackedEngine):
    def __init__(self, module):
        super().__init__(module)
        self.launches = 0

    def _pack(self):
        m = self.m
        dev = m.token_embedding.weight.device
        if dev.type != "cuda":
            raise RuntimeError("TextTowerEngine needs the module on a CUDA device (no CPU fallback)")
        f = lambda p: p.detach().float().contiguous()
        h = lambda p: ops.to_f16(p.detach().float().contiguous())
        self.D = m.token_embedding.weight.shape[1]
        self.H = m.transformer.resblocks[0].attn.num_heads
        if self.D // self.H != 64:
            raise RuntimeError("the attention kernel is specialised for head_dim 64")
        self.tok, self.pos = f(m.token_embedding.weight), f(m.positional_embedding)
        self.zero_w = torch.zeros(1, self.D, dtype=torch.float32, device=dev)
        self.layers = []
        for blk in m.transformer.resblocks:
            self.layers.append(dict(
                g1=f(blk.ln_1.weight), b1=f(blk.ln_1.bias), e1=blk.ln_1.eps, wqkv=h(blk.attn.in_proj_weight), bqkv=f(blk.attn.in_proj_bias),
                wo=h(blk.attn.out_proj.weight), bo=f(blk.attn.out_proj.bias), g2=f(blk.ln_2.weight), b2=f(blk.ln_2.bias), e2=blk.ln_2.eps,
                wfc=h(blk.mlp.c_fc.weight), bfc=f(blk.mlp.c_fc.bias), wpr=h(blk.mlp.c_proj.weight), bpr=f(blk.mlp.c_proj.bias)))
        self.gf, self.bf, self.ef = f(m.ln_final.weight), f(m.ln_final.bias), m.ln_final.eps

    @torch.no_grad()
    def forward(self, tokens: torch.Tensor, normalize: bool = True) -> torch.Tensor:
        """tokens (B, L) int64 (negative = padding, read as id 0 like the reference's in-place clamp) -> (B, L, D) fp32."""
        self.ensure_current()
        B, L = tokens.shape
        D, H = self.D, self.H
        if L > self.pos.shape[0]:
            raise RuntimeError(f"context length {L} exceeds the positional table ({self.pos.shape[0]})")
        M = B * L
        dev = tokens.device
        x = torch.empty(B, L, D, dtype=torch.float32, device=dev)
        err = torch.zeros(1, dtype=torch.int32, device=dev)
        # token + positional embedding through the grid-embedding kernel: "height" row l = position l, one all-zero "width" row
        ops.embed_tokens(tokens.contiguous(), self.tok, self.pos[:L].contiguous(), self.zero_w, out=x, err_flag=err)
        hbuf = torch.empty(M, D, dtype=torch.float16, device=dev)
        qkv = torch.empty(M, 3 * D, dtype=torch.float16, device=dev)
        att = torch.empty(M, D, dtype=torch.float16, device=dev)
        hid = torch.empty(M, self.layers[0]["wfc"].shape[0], dtype=torch.float16, device=dev)
        x2 = x.view(M, D)
        for lay in self.layers:
            ops.layernorm(x, lay["g1"], lay["b1"], out=hbuf.view(B, L, D), eps=lay["e1"])
            ops.gemm(hbuf, lay["wqkv"], lay["bqkv"], None, qkv, dtype=ops.F16)
            ops.attention(qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:], att, B=B, H=H, Lq=L, Lk=L, scale=1.0 / math.sqrt(64), causal=True)
            ops.gemm(att, lay["wo"], lay["bo"], x2, x2, dtype=ops.F16)
            ops.layernorm(x, lay["g2"], lay["b2"], out=hbuf.view(B, L, D), eps=lay["e2"])
            ops.gemm(hbuf, lay["wfc"], lay["bfc"], None, hid, dtype=ops.F16, gelu=True)
            ops.gemm(hid, lay["wpr"], lay["bpr"], x2, x2, dtype=ops.F16)
        out = ops.layernorm(x, self.gf, self.bf, eps=self.ef)
        if normalize:
            ops.l2_normalize_rows_(out)
        self.launches = 2 + 7 * len(self.layers) + (1 if normalize else 0)
        if int(err.item()):
            raise RuntimeError("token id out of range of the CLIP vocabulary")
        return out
