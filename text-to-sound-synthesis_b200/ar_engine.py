"""Decode engine of the autoregressive SpecVQGAN transformer (Codebook/specvqgan/modules/transformer/mingpt.py GPTFeats / GPT): packs a
drop-in GPT's parameters for the sm_90a kernels and runs the model one position at a time with a per-layer fp32 KV cache.

The reference's Net2NetTransformer.sample (cond_transformer.py:124-194) re-runs the whole prefix for every token; because of the causal mask
the last row of that forward only needs the keys and values of the earlier positions, so caching them computes the same logits in exact
arithmetic.  One position of B rows is a fixed launch sequence (dsb_ar_* in include/diffsound_b200.h, GEMMs through ops.gemm_f16x3 with M = B):

    embed, n_layer x [LayerNorm, QKV, decode attention, proj + residual, LayerNorm, MLP1, GELU(erf) + split, MLP2 + residual], ln_f, head, sampler

The current position and the RNG state live in a device loop-control block that the sampler's last CTA advances, so the step is captured once as
a CUDA graph and replayed for every position.  Teacher-forced forward() runs the same steps and records every position's logits.  One precision:
every GEMM operand is an fp16 (hi | lo) pair ('f16x3', fp32-class results); the attention, softmax and sampler arithmetic is fp32.

Scoring (GPT.forward with targets, Net2NetTransformer.shared_step) knows the whole sequence up front, so prefill() runs every position in one pass
with M = B * T GEMMs on the same packed weights and one CUDA graph, for the latest (B, T):

    embed all, n_layer x [LayerNorm, QKV (split pair out), causal split attention, proj + residual, LayerNorm, MLP1, GELU(erf) + split,
    MLP2 + residual], ln_f, head, cross-entropy
"""
from __future__ import annotations

import math
from typing import Callable, Dict, Optional

import numpy as np
import torch

from . import ops
from .engine_base import PackedEngine
from .graphs import capture
from .packing import SplitWeight


class AREngine(PackedEngine):
    settings = ("use_cuda_graph",)

    def __init__(self, gpt, use_cuda_graph: bool = True):
        super().__init__(gpt, use_cuda_graph=use_cuda_graph)
        self.use_cuda_graph = use_cuda_graph
        self._ws: Dict[int, dict] = {}
        self._pf: Dict[tuple, dict] = {}  # the prefill workspace of the latest (B, T)
        self.launches_per_step = 0

    @property
    def device(self):
        return self.m.head.weight.device

    def _pack(self) -> None:
        m = self.m
        check_ar_shapes(m.config.vocab_size, m.config.n_embd, m.config.n_head, m.block_size)
        if self.device.type != "cuda":
            raise RuntimeError("AREngine needs the module on a CUDA device (no CPU fallback)")
        f = lambda p: p.detach().float().contiguous()
        self.D, self.H, self.V, self.P = m.config.n_embd, m.config.n_head, m.config.vocab_size, m.block_size
        self.layers = []
        for blk in m.blocks:
            a = blk.attn
            self.layers.append(dict(
                g1=f(blk.ln1.weight), b1=f(blk.ln1.bias), eps1=blk.ln1.eps,
                wqkv=SplitWeight(torch.cat([a.query.weight, a.key.weight, a.value.weight], 0)),
                bqkv=f(torch.cat([a.query.bias, a.key.bias, a.value.bias], 0)),
                wo=SplitWeight(a.proj.weight), bo=f(a.proj.bias),
                g2=f(blk.ln2.weight), b2=f(blk.ln2.bias), eps2=blk.ln2.eps,
                w1=SplitWeight(blk.mlp[0].weight), bm1=f(blk.mlp[0].bias),
                w2=SplitWeight(blk.mlp[2].weight), bm2=f(blk.mlp[2].bias)))
        self.gf, self.bf, self.epsf = f(m.ln_f.weight), f(m.ln_f.bias), m.ln_f.eps
        self.whead = SplitWeight(m.head.weight)
        self.tok_emb = f(m.tok_emb.weight)
        self.pos_emb = f(m.pos_emb.reshape(m.pos_emb.shape[-2], m.pos_emb.shape[-1]))
        emb = getattr(m, "embedder", None)
        if emb is not None:
            self.wc = f(emb.weight.reshape(emb.weight.shape[0], -1))
            self.bc = f(emb.bias) if emb.bias is not None else None
        self._ws.clear()
        self._pf.clear()

    # ------------------------------------------------------------------ workspaces
    def workspace(self, B: int) -> dict:
        """Per-B buffers, sized for block_size positions: activations of one position, the per-layer fp32 K / V caches, the token ids, the
        logits history, the loop-control block and the captured step graphs."""
        ws = self._ws.get(B)
        if ws is None:
            dev, D, P, V = self.device, self.D, self.P, self.V
            e = lambda *s: torch.empty(*s, dtype=torch.float32, device=dev)
            pair = lambda r, c: torch.zeros(r, 2 * c, dtype=torch.float16, device=dev)
            ws = dict(x=e(B, D), h=pair(B, D), qkv=e(B, 3 * D), att=pair(B, D), hid=e(B, 4 * D), hid2=pair(B, 4 * D), logits=e(B, V),
                      kc=[torch.zeros(B, P, D, dtype=torch.float32, device=dev) for _ in self.layers],
                      vc=[torch.zeros(B, P, D, dtype=torch.float32, device=dev) for _ in self.layers],
                      cond=e(B * P * D), ids=torch.zeros(B, P + 1, dtype=torch.int64, device=dev), hist=None,
                      ctrl=torch.zeros(ops.AR_CTRL_WORDS, dtype=torch.int64, device=dev),
                      host=torch.zeros(ops.AR_CTRL_WORDS, dtype=torch.int64).pin_memory(),
                      err=torch.zeros(2, dtype=torch.int32, device=dev), graphs={})
            self._ws[B] = ws
        return ws

    # ------------------------------------------------------------------ compute
    @torch.no_grad()
    def embed_condition(self, feats: torch.Tensor) -> torch.Tensor:
        """GPTFeats' Conv1d(Cf, D, 1) embedder (mingpt.py:286-289), once per call, in exact fp32: feats (B, Cf, Tc) -> (B, Tc, D)."""
        self.ensure_current()
        B, Cf, Tc = feats.shape
        a = feats.detach().float().permute(0, 2, 1).reshape(B * Tc, Cf).contiguous()
        return ops.gemm_f32(a, self.wc, self.bc).view(B, Tc, self.D)

    def _step(self, ws, Tc: int, temperature: float, top_k: Optional[int], sample: bool, hist) -> None:
        """One position: the fixed launch sequence (no host reads, capturable)."""
        D, H = self.D, self.H
        x, h, qkv, att, hid, hid2, ctrl = ws["x"], ws["h"], ws["qkv"], ws["att"], ws["hid"], ws["hid2"], ws["ctrl"]
        B = x.shape[0]
        cond = ws["cond"][:B * max(Tc, 1) * D].view(B, max(Tc, 1), D)[:, :Tc]
        scale = 1.0 / math.sqrt(D // H)
        ops.ar_embed(cond, self.tok_emb, self.pos_emb, ws["ids"], x, ctrl, err_flag=ws["err"][0:1])
        for li, lay in enumerate(self.layers):
            ops.layernorm(x, lay["g1"], lay["b1"], out=h, eps=lay["eps1"], split=True)
            ops.gemm_f16x3(h, lay["wqkv"].pair, lay["bqkv"], out=qkv, alpha=lay["wqkv"].alpha)
            ops.ar_attention(qkv, ws["kc"][li], ws["vc"][li], att, ctrl, H=H, scale=scale)
            ops.gemm_f16x3(att, lay["wo"].pair, lay["bo"], residual=x, out=x, alpha=lay["wo"].alpha)
            ops.layernorm(x, lay["g2"], lay["b2"], out=h, eps=lay["eps2"], split=True)
            ops.gemm_f16x3(h, lay["w1"].pair, lay["bm1"], out=hid, alpha=lay["w1"].alpha)
            ops.gelu_erf_split(hid, out=hid2)
            ops.gemm_f16x3(hid2, lay["w2"].pair, lay["bm2"], residual=x, out=x, alpha=lay["w2"].alpha)
        ops.layernorm(x, self.gf, self.bf, out=h, eps=self.epsf, split=True)
        ops.gemm_f16x3(h, self.whead.pair, None, out=ws["logits"], alpha=self.whead.alpha)
        ops.ar_sample(ws["logits"], ws["ids"], ctrl, Tc=Tc, temperature=temperature, top_k=top_k, sample=sample, logits_hist=hist,
                      err_flag=ws["err"][1:2])
        self.launches_per_step = 4 + 8 * len(self.layers)

    def _arm(self, ws, seed, offset, counter_offset, nthreads, n_pos, first) -> None:
        """(Re)load the device loop state: RNG (seed, offset), position 0, the number of positions and the first sampled one."""
        c = ws["host"]
        c[0] = np.array([seed & (2 ** 64 - 1)], dtype=np.uint64).view(np.int64)[0].item()
        c[1], c[2], c[3], c[4], c[5], c[6], c[7] = offset, counter_offset, nthreads, 0, n_pos, first, 0
        ws["ctrl"].copy_(c)  # blocking: the pinned staging buffer is rewritten by the next call

    @torch.no_grad()
    def run(self, cond: torch.Tensor, ids: torch.Tensor, n_pos: int, first: int, *, temperature: float = 1.0, top_k: Optional[int] = None,
            sample: bool = False, record_logits: bool = False, callback: Optional[Callable[[int], None]] = None):
        """Runs positions 0 ... n_pos - 1.  cond (B, Tc, D) fp32 (the embedded condition), ids (B, n) the given tokens; positions p >= first
        write the token of position p + 1 (ids[b, p - Tc + 1]).  Returns (ids (B, n_pos - Tc + 1) when first < n_pos else None, logits history
        (B, n_pos, V) when record_logits else None).  callback(k) runs on the host before the k-th sampled position."""
        self.ensure_current()
        B, Tc, _ = cond.shape
        n_given = ids.shape[1]
        dev = self.device
        ws = self.workspace(B)
        if Tc > 0:
            ws["cond"][:B * Tc * self.D].view(B, Tc, self.D).copy_(cond)
        hist = None
        if record_logits:
            if ws["hist"] is None:
                ws["hist"] = torch.zeros(B, self.P, self.V, dtype=torch.float32, device=dev)
            hist = ws["hist"]
        gen = torch.cuda.default_generators[dev.index if dev.index is not None else torch.cuda.current_device()]
        seed, offset = gen.initial_seed(), gen.get_offset()
        nthreads, counter_offset = ops.aten_rand_geometry(B * self.V, dev)
        if n_given:  # before the capture warm-up below, which already embeds position 0 (a token when Tc = 0)
            ws["ids"][:, :n_given].copy_(ids)
        key = (Tc, float(temperature), top_k, bool(sample), record_logits)
        g = ws["graphs"].get(key) if self.use_cuda_graph else None
        if self.use_cuda_graph and g is None:  # the warm-up runs one step: the loop state is re-armed afterwards
            self._arm(ws, seed, offset, counter_offset, nthreads, n_pos, first)
            g = ws["graphs"][key] = capture(lambda: self._step(ws, Tc, temperature, top_k, sample, hist), dev)
        self._arm(ws, seed, offset, counter_offset, nthreads, n_pos, first)
        if n_given:  # the warm-up step may have written a sampled token over the given ones
            ws["ids"][:, :n_given].copy_(ids)
        for p in range(n_pos):
            if callback is not None and p >= first:
                callback(p - first)
            if g is not None:
                g.replay()
            else:
                self._step(ws, Tc, temperature, top_k, sample, hist)
        n_sampled = max(0, n_pos - first)
        if sample:
            gen.set_offset(offset + n_sampled * counter_offset)
        err = ws["err"].tolist()  # one 8-byte read per call
        if any(err):
            ws["err"].zero_()
            if err[0]:
                raise IndexError(f"index out of range in self: a token id >= vocab_size ({self.V}) reached GPT.tok_emb")
            raise RuntimeError("probability tensor contains either `inf`, `nan` or element < 0")
        out_ids = ws["ids"][:, :n_pos - Tc + 1].clone() if first < n_pos else None
        out_hist = hist[:, :n_pos].clone() if record_logits else None
        return out_ids, out_hist

    # ------------------------------------------------------------------ full-sequence forward (scoring)
    def prefill_workspace(self, B: int, T: int) -> dict:
        """Buffers of prefill() for one (B, T): the (B * T)-row activations, logits, the static inputs of the captured graph and its graphs.  About
        B * T * (60 D + 4 V) bytes (1.06 GB at caps_transformer width, B = 64, T = 265), so only the latest shape is kept: a new (B, T) frees the old
        workspace and its graphs first."""
        ws = self._pf.get((B, T))
        if ws is None:
            self._pf.clear()
            dev, D, V, M = self.device, self.D, self.V, B * T
            e = lambda *s: torch.empty(*s, dtype=torch.float32, device=dev)
            pair = lambda r, c: torch.zeros(r, 2 * c, dtype=torch.float16, device=dev)
            ws = dict(x=e(B, T, D), h=pair(M, D), qkv=pair(M, 3 * D), att=pair(M, D), hid=e(M, 4 * D), hid2=pair(M, 4 * D), logits=e(B, T, V),
                      cond=torch.zeros(B * T * D, dtype=torch.float32, device=dev), ids=torch.zeros(B, T, dtype=torch.int64, device=dev),
                      tgt=torch.zeros(B, T, dtype=torch.int64, device=dev), nll=e(B * T), loss=e(()),
                      err=torch.zeros(2, dtype=torch.int32, device=dev), graphs={})
            self._pf[(B, T)] = ws
        return ws

    def _prefill_step(self, ws, B: int, T: int, Tc: int, first_row: int, n: int) -> None:
        """The full-sequence launch sequence (no host reads, capturable); n = 0: no cross-entropy."""
        D, H, V, M = self.D, self.H, self.V, B * T
        x2, h, qkv, att, hid, hid2 = ws["x"].view(M, D), ws["h"], ws["qkv"], ws["att"], ws["hid"], ws["hid2"]
        scale = 1.0 / math.sqrt(D // H)
        cond = ws["cond"][:B * Tc * D].view(B, Tc, D)
        ops.ar_embed_all(cond, self.tok_emb, self.pos_emb, ws["ids"][:, :T - Tc], ws["x"], err_flag=ws["err"][0:1])
        for lay in self.layers:
            ops.layernorm(x2, lay["g1"], lay["b1"], out=h, eps=lay["eps1"], split=True)
            ops.gemm_f16x3(h, lay["wqkv"].pair, lay["bqkv"], out=qkv, alpha=lay["wqkv"].alpha, split_out=True)  # [Qh Kh Vh | Ql Kl Vl]
            ops.attention_tc_split_causal(qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:3 * D], att[:, :D], q_lo=3 * D, k_lo=3 * D, v_lo=3 * D, o_lo=D,
                                          B=B, H=H, L=T, scale=scale, head_dim=D // H)
            ops.gemm_f16x3(att, lay["wo"].pair, lay["bo"], residual=x2, out=x2, alpha=lay["wo"].alpha)
            ops.layernorm(x2, lay["g2"], lay["b2"], out=h, eps=lay["eps2"], split=True)
            ops.gemm_f16x3(h, lay["w1"].pair, lay["bm1"], out=hid, alpha=lay["w1"].alpha)
            ops.gelu_erf_split(hid, out=hid2)
            ops.gemm_f16x3(hid2, lay["w2"].pair, lay["bm2"], residual=x2, out=x2, alpha=lay["w2"].alpha)
        ops.layernorm(x2, self.gf, self.bf, out=h, eps=self.epsf, split=True)
        ops.gemm_f16x3(h, self.whead.pair, None, out=ws["logits"].view(M, V), alpha=self.whead.alpha)
        if n:
            ops.ar_cross_entropy(ws["logits"], ws["tgt"][:, :n], first_row=first_row, nll=ws["nll"][:B * n].view(B, n), loss=ws["loss"],
                                 err_flag=ws["err"][1:2])

    @torch.no_grad()
    def prefill(self, cond: torch.Tensor, ids: torch.Tensor, targets: Optional[torch.Tensor] = None, first_row: int = 0):
        """Every position's logits in one causal pass: cond (B, Tc, D) fp32 (the embedded condition), ids (B, T - Tc) tokens.  With targets
        (B, n) int64 (ignore_index -100), also F.cross_entropy over logits rows first_row ... first_row + n - 1.  Returns (logits (B, T, V),
        loss () or None, per-row NLL (B, n) or None)."""
        self.ensure_current()
        B, Tc, _ = cond.shape
        T = Tc + ids.shape[1]
        n = 0 if targets is None else targets.shape[1]
        if targets is not None and (targets.shape[0] != B or not 0 <= first_row <= T - n):
            raise ValueError(f"targets {tuple(targets.shape)} do not fit rows {first_row} ... of {B} x {T} logits")
        ws = self.prefill_workspace(B, T)
        if Tc:
            ws["cond"][:B * Tc * self.D].view(B, Tc, self.D).copy_(cond)
        ws["ids"][:, :T - Tc].copy_(ids)
        if n:
            ws["tgt"][:, :n].copy_(targets)
        key = (Tc, first_row, n)
        g = ws["graphs"].get(key) if self.use_cuda_graph else None
        if self.use_cuda_graph and g is None:
            g = ws["graphs"][key] = capture(lambda: self._prefill_step(ws, B, T, Tc, first_row, n), self.device)
        if g is not None:
            g.replay()
        else:
            self._prefill_step(ws, B, T, Tc, first_row, n)
        err = ws["err"].tolist()  # one 8-byte read per call
        if any(err):
            ws["err"].zero_()
            if err[0]:
                raise IndexError(f"index out of range in self: a token id >= vocab_size ({self.V}) reached GPT.tok_emb")
            raise IndexError(f"Target out of bounds: a target outside [0, {self.V}) that is not ignore_index (-100)")
        if not n:
            return ws["logits"].clone(), None, None
        return ws["logits"].clone(), ws["loss"].clone(), ws["nll"][:B * n].view(B, n).clone()


def check_ar_shapes(V: int, D: int, H: int, block_size: int) -> None:
    """Refusals of the decode kernels, raised before anything is packed or launched."""
    if V > ops.AR_MAX_V:
        raise ValueError(f"vocab_size={V} too large: the autoregressive sampler takes at most {ops.AR_MAX_V} entries")
    if D % H or D // H not in ops.AR_HEAD_DIMS:
        raise ValueError(f"head_dim n_embd / n_head = {D}/{H} unsupported: the decode attention takes head_dim 32 or 64")
    if block_size > ops.AR_MAX_POS:
        raise ValueError(f"block_size={block_size} too large: the decode attention caches at most {ops.AR_MAX_POS} positions")
