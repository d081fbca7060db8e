"""Denoiser execution engine: packs a Text2ImageTransformer's parameters for the sm_90a kernels and runs one
forward pass as a fixed sequence of C-ABI launches (12 per layer), CUDA-graph capturable.

What is hoisted relative to the reference (all algebraically identical):
  * the AdaLayerNorm timestep MLP  Linear(SiLU(emb[t]))  depends only on t -> a (T, 2D) table per norm, built once
    (reference recomputes it for every token batch: transformer_utils.py:145-147);
  * cross-attention K/V projections of cond_emb depend only on the caption -> one GEMM for all layers, once per
    sample() (reference recomputes them every step in every layer: transformer_utils.py:95,97);
  * query/key/value of self-attention run as one (3D x D) GEMM (reference: three Linears, :45-47).
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import torch

from . import ops
from .engine_base import PackedEngine
from .packing import SplitWeight


class DenoiserEngine(PackedEngine):
    def __init__(self, transformer, precision: str = "f16x3"):
        """precision: 'f16x3' -- the parity-grade tensor-core mode (default): every GEMM / attention operand is an fp16 (hi | lo) pair
                                (22 significand bits), products run as three fp16 wgmma passes (lo*hi + hi*lo + hi*hi) into one
                                fp32 register accumulator; fp32 residual stream / LayerNorm / softmax / logits.  fp32-class logits (the
                                reference computes its nn.Linear layers in fp32): free-running token ids reproduce the fp32 oracle;
                      'f16'   -- single-pass fp16 operands (11-bit significand = TF32's, at twice the TF32 rate): 3x fewer MMAs, logits
                                within ~1e-3 of fp32, token agreement ~99.6 % -- the throughput mode;
                      'tf32'  -- fp32 containers rounded to TF32, TF32 wgmma;
                      'fp32'  -- exact FFMA GEMMs (slow; the fp32-exact mode of SURVEY.md section 7.2)."""
        if precision not in ("f16x3", "f16", "tf32", "fp32"):
            raise ValueError("precision must be 'f16x3', 'f16', 'tf32' or 'fp32'")
        super().__init__(transformer, precision=precision)
        self.precision = precision
        self._ws: Dict[int, dict] = {}
        self.launches_per_forward = 0

    # ------------------------------------------------------------------ weights
    @property
    def device(self):
        return self.m.to_logits[1].weight.device

    def _prep(self, w: torch.Tensor):
        w = w.detach().float().contiguous()
        if self.precision == "f16x3":
            return SplitWeight(w)
        if self.precision == "f16":
            return ops.to_f16(w)
        return ops.round_tf32(w) if self.precision == "tf32" else w.clone()

    def _pack(self) -> None:
        m = self.m
        if self.device.type != "cuda":
            raise RuntimeError("DenoiserEngine needs the module on a CUDA device (no CPU fallback)")
        self.D = m.n_embd
        self.H = m.n_head
        self.n_layer = len(m.blocks)
        self.T = m.diffusion_step
        self.mlp_times = m.blocks[0].mlp[0].weight.shape[0] // m.n_embd
        D = self.D
        if D % 64 or D % self.H or D // self.H not in (64, 32):
            raise RuntimeError(f"kernels are specialised for head_dim 64 and 32 (n_embd={D}, n_head={self.H})")
        self.head_dim = D // self.H
        if self.head_dim == 32 and self.precision == "f16":
            raise RuntimeError(f"precision 'f16' has no head_dim-32 attention (n_embd={D}, n_head={self.H}); use 'f16x3', 'tf32' or 'fp32'")
        f = lambda p: p.detach().float().contiguous()
        self.layers = []
        kv_w, kv_b = [], []
        for blk in m.blocks:
            a1, a2 = blk.attn1, blk.attn2
            lay = dict(
                tab1=self._adaln_table(blk.ln1), tab2=self._adaln_table(blk.ln1_1),
                wqkv=self._prep(torch.cat([a1.query.weight, a1.key.weight, a1.value.weight], 0)),
                bqkv=f(torch.cat([a1.query.bias, a1.key.bias, a1.value.bias], 0)),
                wo1=self._prep(a1.proj.weight), bo1=f(a1.proj.bias),
                wq2=self._prep(a2.query.weight), bq2=f(a2.query.bias),
                wo2=self._prep(a2.proj.weight), bo2=f(a2.proj.bias),
                g2=f(blk.ln2.weight), b2=f(blk.ln2.bias), eps2=blk.ln2.eps,
                w1=self._prep(blk.mlp[0].weight), b1=f(blk.mlp[0].bias),
                w2=self._prep(blk.mlp[2].weight), bm2=f(blk.mlp[2].bias),
            )
            kv_w += [a2.key.weight, a2.value.weight]
            kv_b += [a2.key.bias, a2.value.bias]
            self.layers.append(lay)
        self.wkv_all = self._prep(torch.cat(kv_w, 0))          # (n_layer*2D, cond_dim)
        self.bkv_all = f(torch.cat(kv_b, 0))
        self.gf, self.bf, self.epsf = f(m.to_logits[0].weight), f(m.to_logits[0].bias), m.to_logits[0].eps
        self.wlog, self.blog = self._prep(m.to_logits[1].weight), f(m.to_logits[1].bias)
        ce = m.content_emb
        self.emb, self.hemb, self.wemb = f(ce.emb.weight), f(ce.height_emb.weight), f(ce.width_emb.weight)
        self.K = m.to_logits[1].weight.shape[0]
        self._ws.clear()

    def _adaln_table(self, ln) -> torch.Tensor:
        """(T, 2D) table of Linear(SiLU(emb[t])) in exact fp32 (transformer_utils.py:145-147)."""
        e = ln.emb.weight.detach().float().contiguous()
        return ops.gemm_f32(ops.silu(e), ln.linear.weight.detach().float().contiguous(), ln.linear.bias.detach().float().contiguous())

    # ------------------------------------------------------------------ workspaces
    def workspace(self, B: int, L: int) -> dict:
        key = (B, L)
        ws = self._ws.get(key)
        if ws is None:
            dev, M, D = self.device, B * L, self.D
            e = lambda *s: torch.empty(*s, dtype=torch.float32, device=dev)
            if self.precision == "f16x3":  # every GEMM A operand is an fp16 (hi | lo) pair: twice the columns
                a = lambda *s: torch.zeros(*s[:-1], 2 * s[-1], dtype=torch.float16, device=dev)
            else:
                a = (lambda *s: torch.empty(*s, dtype=torch.float16, device=dev)) if self.precision == "f16" else e  # GEMM A operands
            ws = dict(x=e(B, L, D), h=a(B, L, D), qkv=a(M, 3 * D), att=a(M, D), q2=a(M, D), hid=a(M, self.mlp_times * D),
                      logits=e(B, L, self.K), err=torch.zeros(1, dtype=torch.int32, device=dev))
            self._ws[key] = ws
        return ws

    def check_token_range(self, B: int, L: int) -> None:
        """Raise the reference's embedding error (dalle_mask_image_embedding.py:40-44 -> torch's index error) if a forward pass since the last check
        saw a token id >= num_embed; one 4-byte D2H read, call it once per sample() / training forward, outside any graph capture."""
        ws = self._ws.get((B, L))
        if ws is not None and int(ws["err"].item()) != 0:
            ws["err"].zero_()
            raise IndexError(f"index out of range in self: a content token id >= num_embed ({self.emb.shape[0]}) reached DalleMaskImageEmbedding")

    # ------------------------------------------------------------------ compute
    def _linear(self, a, w, bias, residual=None, out=None, gelu=False, round_out=False, split_out=False):
        if self.precision == "f16x3":
            return ops.gemm_f16x3(a, w.pair, bias, residual, out, alpha=w.alpha, gelu=gelu, split_out=split_out)
        if self.precision == "f16":
            return ops.gemm(a, w, bias, residual, out, dtype=ops.F16, gelu=gelu)
        if self.precision == "tf32":
            return ops.gemm(a, w, bias, residual, out, dtype=ops.TF32, gelu=gelu, round_out=round_out)
        return ops.gemm_f32(a, w, bias, residual, out, gelu=gelu)

    @torch.no_grad()
    def encode_condition(self, cond_emb: torch.Tensor) -> torch.Tensor:
        """cond_emb (B, Lc, cond_dim) -> K/V of every layer's cross-attention, (B*Lc, n_layer*2D)."""
        self.ensure_current()
        B, Lc, Cd = cond_emb.shape
        c = cond_emb.detach().float().reshape(B * Lc, Cd).contiguous()
        if self.precision == "f16x3":
            out = torch.empty(B * Lc, 2 * self.n_layer * 2 * self.D, dtype=torch.float16, device=c.device)  # (hi | lo) pair of every layer's K|V
            return self._linear(ops.split_f16(c), self.wkv_all, self.bkv_all, out=out, split_out=True)
        if self.precision == "tf32":
            c = ops.round_tf32(c)
        elif self.precision == "f16":
            c = ops.to_f16(c)
        out = torch.empty(B * Lc, self.n_layer * 2 * self.D, dtype=torch.float16 if self.precision == "f16" else torch.float32, device=c.device)
        return self._linear(c, self.wkv_all, self.bkv_all, out=out)

    @torch.no_grad()
    def forward(self, ids: torch.Tensor, kv_all: torch.Tensor, t: torch.Tensor, Lc: int, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """ids (B,L) int64, kv_all from encode_condition, t (B,) int64 -> logits (B, L, K) fp32 (the reference returns its
        'b l c -> b c l' view, transformer_utils.py:442; callers permute)."""
        if not self.packed:
            self.repack()
        B, L = ids.shape
        D, H = self.D, self.H
        ws = self.workspace(B, L)
        x, h, qkv, att, q2, hid = ws["x"], ws["h"], ws["qkv"], ws["att"], ws["q2"], ws["hid"]
        rnd = self.precision == "tf32"
        if self.precision == "f16x3":
            return self._forward_split(ids, kv_all, t, Lc, out)
        x2 = x.view(B * L, D)
        h2 = h.view(B * L, D)
        scale = 1.0 / math.sqrt(self.head_dim)
        hd_arg = {} if self.head_dim == 64 else dict(head_dim=self.head_dim)  # the head_dim-64 calls keep their exact arguments
        n = 0
        ops.embed_tokens(ids, self.emb, self.hemb, self.wemb, out=x, err_flag=ws["err"]); n += 1
        for li, lay in enumerate(self.layers):
            ops.ada_layernorm(x, lay["tab1"], t, out=h, round_out=rnd)
            self._linear(h2, lay["wqkv"], lay["bqkv"], out=qkv)
            if self.precision == "f16" and L <= 272:
                # K / V staged once per head by TMA, fp16 mma.sync over 16-row slabs
                ops.attention_tc(qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:], att, B=B, H=H, Lq=L, Lk=L, scale=scale)
            else:
                ops.attention(qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:], att, B=B, H=H, Lq=L, Lk=L, scale=scale, round_out=rnd, **hd_arg)
            self._linear(att, lay["wo1"], lay["bo1"], residual=x2, out=x2)
            ops.ada_layernorm(x, lay["tab2"], t, out=h, round_out=rnd)
            self._linear(h2, lay["wq2"], lay["bq2"], out=q2)
            kv = kv_all[:, li * 2 * D:(li + 1) * 2 * D]
            if self.precision == "f16" and Lc <= 272:
                ops.attention_tc(q2, kv[:, :D], kv[:, D:], att, B=B, H=H, Lq=L, Lk=Lc, scale=scale)
            else:
                ops.attention(q2, kv[:, :D], kv[:, D:], att, B=B, H=H, Lq=L, Lk=Lc, scale=scale, round_out=rnd, **hd_arg)
            self._linear(att, lay["wo2"], lay["bo2"], residual=x2, out=x2)
            ops.layernorm(x, lay["g2"], lay["b2"], out=h, eps=lay["eps2"], round_out=rnd)
            self._linear(h2, lay["w1"], lay["b1"], out=hid, gelu=True, round_out=rnd)
            self._linear(hid, lay["w2"], lay["bm2"], residual=x2, out=x2)
            n += 11
        ops.layernorm(x, self.gf, self.bf, out=h, eps=self.epsf, round_out=rnd)
        logits = ws["logits"] if out is None else out
        self._linear(h2, self.wlog, self.blog, out=logits.view(B * L, self.K))
        self.launches_per_forward = n + 2
        return logits

    @torch.no_grad()
    def _forward_split(self, ids, kv_all, t, Lc, out=None):
        """The 'f16x3' pass: same launch sequence as forward(), every tensor-core operand an fp16 (hi | lo) pair.
        qkv (M, 6D) = [Qh Kh Vh | Ql Kl Vl]; kv_all (B*Lc, 2 * n_layer*2D) = [hi of every layer's K|V | lo ...]."""
        B, L = ids.shape
        D, H = self.D, self.H
        ws = self.workspace(B, L)
        x, h, qkv, att, q2, hid = ws["x"], ws["h"], ws["qkv"], ws["att"], ws["q2"], ws["hid"]
        M = B * L
        x2, h2 = x.view(M, D), h.view(M, 2 * D)
        scale = 1.0 / math.sqrt(self.head_dim)
        hd_arg = {} if self.head_dim == 64 else dict(head_dim=self.head_dim)
        kv_lo = self.n_layer * 2 * D
        n = 0
        ops.embed_tokens(ids, self.emb, self.hemb, self.wemb, out=x, err_flag=ws["err"]); n += 1
        for li, lay in enumerate(self.layers):
            ops.ada_layernorm(x, lay["tab1"], t, out=h, split=True)
            self._linear(h2, lay["wqkv"], lay["bqkv"], out=qkv, split_out=True)
            ops.attention_tc_split(qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:3 * D], att[:, :D], q_lo=3 * D, k_lo=3 * D, v_lo=3 * D, o_lo=D,
                                   B=B, H=H, Lq=L, Lk=L, scale=scale, **hd_arg)
            self._linear(att, lay["wo1"], lay["bo1"], residual=x2, out=x2)
            ops.ada_layernorm(x, lay["tab2"], t, out=h, split=True)
            self._linear(h2, lay["wq2"], lay["bq2"], out=q2, split_out=True)
            kv = kv_all[:, li * 2 * D:]
            ops.attention_tc_split(q2[:, :D], kv[:, :D], kv[:, D:2 * D], att[:, :D], q_lo=D, k_lo=kv_lo, v_lo=kv_lo, o_lo=D,
                                   B=B, H=H, Lq=L, Lk=Lc, scale=scale, **hd_arg)
            self._linear(att, lay["wo2"], lay["bo2"], residual=x2, out=x2)
            ops.layernorm(x, lay["g2"], lay["b2"], out=h, eps=lay["eps2"], split=True)
            self._linear(h2, lay["w1"], lay["b1"], out=hid, gelu=True, split_out=True)
            self._linear(hid, lay["w2"], lay["bm2"], residual=x2, out=x2)
            n += 11
        ops.layernorm(x, self.gf, self.bf, out=h, eps=self.epsf, split=True)
        logits = ws["logits"] if out is None else out
        self._linear(h2, self.wlog, self.blog, out=logits.view(M, self.K))
        self.launches_per_forward = n + 2
        return logits

