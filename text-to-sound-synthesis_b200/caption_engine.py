"""Engine of the ACT audio-captioning transformer (Codebook/AudiocaptionLoss/models/TransModel.py): packs a drop-in ACT's parameters once as
split-fp16 weight pairs (every GEMM is f16x3, fp32-class) and runs

    encoder (per (B, T), one CUDA graph):  frontend (BatchNorm eval + patch split), patch GEMM, tokens (cls + pos), 12 x [LN, QKV,
        dsb_attention_tc_split, proj + residual, LN, fc1, GELU + split, fc2 + residual], LN, head (527, padded to 528), relu(encoder_linear),
        then every decoder layer's cross-attention K / V of the memory (one GEMM per batch, not per step)
    decode step (R rows):  embed, n_layer x [QKV, tree self-attention, out_proj + residual, LN, Q, cross-attention, out_proj + residual, LN,
        linear1, GELU + split, linear2 + residual, LN], dec_fc, select

The decoder layers are post-norm (nn.TransformerDecoderLayer, norm_first=False) with no final norm, so each LayerNorm runs twice: once for the
fp32 residual stream and once for the split operand of the next GEMM.  Greedy decoding is one captured step replayed per position: the select
kernel writes the next word and advances each row's position on the device.  Beam search runs the same step for the rows the host search pops.
"""
from __future__ import annotations

import math
from typing import Dict, List

import numpy as np
import torch

from . import ops
from .engine_base import PackedEngine
from .graphs import capture
from .packing import SplitWeight

MAX_POS = 2000                       # rows of PositionalEncoding.pe: the reference cannot decode a longer prefix
BEAM_SLOTS = 2002                    # slots per clip in beam search: at most 2000 expansions before qsize passes 2000 (beam_width >= 2)
HEAD_PAD = 528                       # the 527 AudioSet logits padded to a multiple of 4 (16-byte GEMM operand rows)


class CaptionEngine(PackedEngine):
    settings = ("use_cuda_graph",)

    def __init__(self, act, use_cuda_graph: bool = True):
        super().__init__(act, use_cuda_graph=use_cuda_graph)
        self.use_cuda_graph = use_cuda_graph
        self._enc: Dict[tuple, dict] = {}
        self._dec: Dict[tuple, dict] = {}
        self._last = None  # the encoder workspace of the last encode() / decode memory

    @property
    def device(self):
        return self.m.dec_fc.weight.device

    def _pack(self) -> None:
        m = self.m
        if self.device.type != "cuda":
            raise RuntimeError("CaptionEngine needs the module on a CUDA device (no CPU fallback)")
        f = lambda p: p.detach().float().contiguous()
        e = m.encoder
        bn = e.bn0
        alpha = f(bn.weight) / torch.sqrt(f(bn.running_var) + bn.eps)
        self.bn_alpha, self.bn_beta = alpha.contiguous(), (f(bn.bias) - f(bn.running_mean) * alpha).contiguous()
        self.w_patch, self.b_patch = SplitWeight(e.patch_embed.proj.weight), f(e.patch_embed.proj.bias)
        self.cls, self.pos = f(e.cls_token.reshape(-1)), f(e.pos_embedding.reshape(e.pos_embedding.shape[1], -1))
        self.E, self.EH = e.cls_token.shape[-1], e.blocks.layers[0][0].fn.heads
        self.enc_layers = []
        for attn, ff in e.blocks.layers:
            self.enc_layers.append(dict(g1=f(attn.norm.weight), b1=f(attn.norm.bias), eps1=attn.norm.eps,
                                        wqkv=SplitWeight(attn.fn.qkv.weight), bqkv=f(attn.fn.qkv.bias),
                                        wo=SplitWeight(attn.fn.proj[0].weight), bo=f(attn.fn.proj[0].bias),
                                        g2=f(ff.norm.weight), b2=f(ff.norm.bias), eps2=ff.norm.eps,
                                        w1=SplitWeight(ff.fn.mlp.fc1.weight), bm1=f(ff.fn.mlp.fc1.bias),
                                        w2=SplitWeight(ff.fn.mlp.fc2.weight), bm2=f(ff.fn.mlp.fc2.bias)))
        ln, head = e.mlp_head[0], e.mlp_head[1]
        self.gh, self.bh, self.epsh = f(ln.weight), f(ln.bias), ln.eps
        nc = head.weight.shape[0]
        wh = torch.zeros(HEAD_PAD, head.weight.shape[1], device=self.device)
        wh[:nc] = f(head.weight)
        bhd = torch.zeros(HEAD_PAD, device=self.device)
        bhd[:nc] = f(head.bias)
        self.w_head, self.b_head = SplitWeight(wh), bhd
        wl = torch.zeros(m.nhid, HEAD_PAD, device=self.device)
        wl[:, :nc] = f(m.encoder_linear.weight)
        self.w_lin, self.b_lin = SplitWeight(wl), f(m.encoder_linear.bias)
        # decoder
        self.D, self.V = m.nhid, m.ntoken
        lay0 = m.transformer_decoder.layers[0]
        self.H = lay0.self_attn.num_heads
        if self.D % self.H or self.D // self.H != ops.CAPTION_HEAD_DIM or self.D % 128:
            raise ValueError(f"decoder nhid={self.D} / nhead={self.H} unsupported: head_dim 64 and nhid a multiple of 128")
        if lay0.norm_first:
            raise ValueError("the caption engine runs post-norm decoder layers (norm_first=False)")
        ops.check_caption_vocab(self.V)
        D = self.D
        self.dec_layers, kv_w, kv_b = [], [], []
        for lay in m.transformer_decoder.layers:
            sa, ca = lay.self_attn, lay.multihead_attn
            self.dec_layers.append(dict(wsa=SplitWeight(sa.in_proj_weight), bsa=f(sa.in_proj_bias), wso=SplitWeight(sa.out_proj.weight),
                                        bso=f(sa.out_proj.bias), wq=SplitWeight(ca.in_proj_weight[:D]), bq=f(ca.in_proj_bias[:D]),
                                        wco=SplitWeight(ca.out_proj.weight), bco=f(ca.out_proj.bias),
                                        w1=SplitWeight(lay.linear1.weight), bm1=f(lay.linear1.bias), w2=SplitWeight(lay.linear2.weight),
                                        bm2=f(lay.linear2.bias), FF=lay.linear1.weight.shape[0],
                                        n=[(f(nm.weight), f(nm.bias), nm.eps) for nm in (lay.norm1, lay.norm2, lay.norm3)]))
            kv_w.append(ca.in_proj_weight[D:])
            kv_b.append(ca.in_proj_bias[D:])
        self.w_kv, self.b_kv = SplitWeight(torch.cat(kv_w, 0)), f(torch.cat(kv_b, 0))
        self.table = (f(m.word_emb.weight) * math.sqrt(m.nhid)).contiguous()  # decode(): self.word_emb(tgt) * math.sqrt(self.nhid), in fp32
        self.pe = f(m.pos_encoder.pe.reshape(m.pos_encoder.pe.shape[0], -1))
        self.w_fc, self.b_fc = SplitWeight(m.dec_fc.weight), f(m.dec_fc.bias)
        self._enc.clear()
        self._dec.clear()
        self._last = None

    # ------------------------------------------------------------------ encoder
    def _enc_ws(self, B: int, T: int) -> dict:
        ws = self._enc.get((B, T))
        if ws is None:
            dev, E, n = self.device, self.E, T // 4
            L, M, nl = n + 1, B * (n + 1), len(self.dec_layers)
            e = lambda *s: torch.empty(*s, dtype=torch.float32, device=dev)
            pair = lambda r, c: torch.zeros(r, 2 * c, dtype=torch.float16, device=dev)
            ws = dict(spec=e(B, T, 80), fe=pair(B * n, 320), patch=e(B * n, E), x=e(B, L, E), h=pair(M, E), qkv=pair(M, 3 * E), att=pair(M, E),
                      hid=e(M, 4 * E), hid2=pair(M, 4 * E), hp=pair(M, HEAD_PAD), mem=e(B, L, self.D), memp=pair(M, self.D),
                      kv=e(M, nl * 2 * self.D), graph=None)
            self._enc[(B, T)] = ws
        return ws

    def _enc_step(self, ws, B: int, T: int) -> None:
        E, n = self.E, T // 4
        L, M = n + 1, B * (n + 1)
        x2, h, qkv, att, hid, hid2 = ws["x"].view(M, E), ws["h"], ws["qkv"], ws["att"], ws["hid"], ws["hid2"]
        ops.caption_frontend(ws["spec"], self.bn_alpha, self.bn_beta, out=ws["fe"])
        ops.gemm_f16x3(ws["fe"], self.w_patch.pair, self.b_patch, out=ws["patch"], alpha=self.w_patch.alpha)
        ops.caption_tokens(ws["patch"], self.cls, self.pos, ws["x"])
        for lay in self.enc_layers:
            ops.layernorm(x2, lay["g1"], lay["b1"], out=h, eps=lay["eps1"], split=True)
            ops.gemm_f16x3(h, lay["wqkv"].pair, lay["bqkv"], out=qkv, alpha=lay["wqkv"].alpha, split_out=True)  # [Qh Kh Vh | Ql Kl Vl]
            ops.attention_tc_split(qkv[:, :E], qkv[:, E:2 * E], qkv[:, 2 * E:3 * E], att[:, :E], q_lo=3 * E, k_lo=3 * E, v_lo=3 * E, o_lo=E,
                                   B=B, H=self.EH, Lq=L, Lk=L, scale=(E // self.EH) ** -0.5, head_dim=E // self.EH)
            ops.gemm_f16x3(att, lay["wo"].pair, lay["bo"], residual=x2, out=x2, alpha=lay["wo"].alpha)
            ops.layernorm(x2, lay["g2"], lay["b2"], out=h, eps=lay["eps2"], split=True)
            ops.gemm_f16x3(h, lay["w1"].pair, lay["bm1"], out=hid, alpha=lay["w1"].alpha)
            ops.gelu_erf_split(hid, out=hid2)
            ops.gemm_f16x3(hid2, lay["w2"].pair, lay["bm2"], residual=x2, out=x2, alpha=lay["w2"].alpha)
        ops.layernorm(x2, self.gh, self.bh, out=h, eps=self.epsh, split=True)
        ops.gemm_f16x3(h, self.w_head.pair, self.b_head, out=ws["hp"], alpha=self.w_head.alpha, split_out=True)
        mem = ws["mem"].view(M, self.D)
        ops.gemm_f16x3(ws["hp"], self.w_lin.pair, self.b_lin, out=mem, alpha=self.w_lin.alpha, relu=True)
        self._project_memory(ws)

    def _project_memory(self, ws) -> None:
        mem = ws["mem"].view(-1, self.D)
        ops.split_f16(mem, out=ws["memp"])
        ops.gemm_f16x3(ws["memp"], self.w_kv.pair, self.b_kv, out=ws["kv"], alpha=self.w_kv.alpha)

    def _replay(self, ws, step) -> None:
        if not self.use_cuda_graph:
            return step()
        if ws["graph"] is None:
            ws["graph"] = capture(step, self.device)
        ws["graph"].replay()

    @torch.no_grad()
    def encode(self, spec: torch.Tensor) -> torch.Tensor:
        """spec (B, T, 80) -> the memory relu(encoder_linear(encoder(spec))) (B, T / 4 + 1, nhid) fp32; also keeps the cross-attention K / V of
        every decoder layer for the decode calls that follow with this (B, T)."""
        self.ensure_current()
        if spec.dim() != 3 or spec.shape[2] != 80 or spec.shape[1] % 4 or not 4 <= spec.shape[1] <= 4 * (self.pos.shape[0] - 1):
            raise ValueError(f"ACT encodes (B, T, 80) mels with T divisible by 4 and T <= {4 * (self.pos.shape[0] - 1)}, got {tuple(spec.shape)}")
        B, T, _ = spec.shape
        ws = self._enc_ws(B, T)
        ws["spec"].copy_(spec)
        self._replay(ws, lambda: self._enc_step(ws, B, T))
        self._last = ws
        return ws["mem"].clone()

    def _memory_ws(self, memory: torch.Tensor) -> dict:
        """The encoder workspace holding `memory` and its projected K / V: the last encode() when memory is its output, else one filled here."""
        B, Lm, D = memory.shape
        ws = self._last
        if ws is not None and ws["mem"].shape == memory.shape and torch.equal(ws["mem"], memory):
            return ws
        ws = self._enc_ws(B, 4 * (Lm - 1))
        ws["mem"].copy_(memory)
        self._project_memory(ws)
        self._last = ws
        return ws

    # ------------------------------------------------------------------ decoder
    def _dec_ws(self, B: int, S: int) -> dict:
        ws = self._dec.get((B, S))
        if ws is None:
            self._dec.clear()  # one slot pool at a time: B * S * n_layer * 2 * nhid * 4 bytes
            dev, D, V = self.device, self.D, self.V
            FF = max(l["FF"] for l in self.dec_layers)
            Vp = (V + 3) // 4 * 4
            e = lambda *s: torch.empty(*s, dtype=torch.float32, device=dev)
            pair = lambda r, c: torch.zeros(r, 2 * c, dtype=torch.float16, device=dev)
            i32 = lambda n: torch.zeros(n, dtype=torch.int32, device=dev)
            ws = dict(x=e(B, D), xp=pair(B, D), qkv=e(B, 3 * D), att=pair(B, D), t=e(B, D), q=e(B, D), hid=e(B, FF), hid2=pair(B, FF),
                      logits=e(B, Vp)[:, :V], tok=torch.zeros(B, dtype=torch.int64, device=dev), pos=i32(B), row_clip=i32(B),
                      start=torch.zeros(B, dtype=torch.int64, device=dev), path=i32(B * S), vals=e(B, ops.CAPTION_MAX_K),
                      idx=torch.zeros(B, ops.CAPTION_MAX_K, dtype=torch.int64, device=dev), err=torch.zeros(3, dtype=torch.int32, device=dev),
                      kp=[torch.zeros(B * S, D, dtype=torch.float32, device=dev) for _ in self.dec_layers],
                      vp=[torch.zeros(B * S, D, dtype=torch.float32, device=dev) for _ in self.dec_layers], graphs={})
            self._dec[(B, S)] = ws
        return ws

    def _dec_step(self, ws, enc, R: int, max_len: int) -> None:
        """One decode position for rows 0 ... R - 1 up to dec_fc's logits (no host reads, capturable)."""
        D, H = self.D, self.H
        x, xp, qkv, att, t, q = ws["x"][:R], ws["xp"][:R], ws["qkv"][:R], ws["att"][:R], ws["t"][:R], ws["q"][:R]
        Lm = enc["mem"].shape[1]
        scale = 1.0 / math.sqrt(D // H)
        ops.caption_embed(ws["tok"][:R], ws["pos"][:R], self.table, self.pe, x, err_flag=ws["err"][0:1])
        ops.split_f16(x, out=xp)
        for li, lay in enumerate(self.dec_layers):
            (g1, b1, e1), (g2, b2, e2), (g3, b3, e3) = lay["n"]
            ops.gemm_f16x3(xp, lay["wsa"].pair, lay["bsa"], out=qkv, alpha=lay["wsa"].alpha)
            ops.caption_tree_attention(qkv, ws["kp"][li], ws["vp"][li], ws["path"], ws["start"], ws["pos"], att, R=R, H=H, scale=scale, max_len=max_len,
                                        err_flag=ws["err"][2:3])
            ops.gemm_f16x3(att, lay["wso"].pair, lay["bso"], residual=x, out=t, alpha=lay["wso"].alpha)
            ops.layernorm(t, g1, b1, out=x, eps=e1)
            ops.layernorm(t, g1, b1, out=xp, eps=e1, split=True)
            ops.gemm_f16x3(xp, lay["wq"].pair, lay["bq"], out=q, alpha=lay["wq"].alpha)
            kv = enc["kv"][:, li * 2 * D:]
            ops.caption_cross_attention(q, kv, ws["row_clip"], att, R=R, H=H, Lm=Lm, v_off=D, scale=scale, err_flag=ws["err"][2:3])
            ops.gemm_f16x3(att, lay["wco"].pair, lay["bco"], residual=x, out=t, alpha=lay["wco"].alpha)
            ops.layernorm(t, g2, b2, out=x, eps=e2)
            ops.layernorm(t, g2, b2, out=xp, eps=e2, split=True)
            FF = lay["FF"]
            ops.gemm_f16x3(xp, lay["w1"].pair, lay["bm1"], out=ws["hid"][:R, :FF], alpha=lay["w1"].alpha)
            ops.gelu_erf_split(ws["hid"][:R, :FF], out=ws["hid2"][:R, :2 * FF])
            ops.gemm_f16x3(ws["hid2"][:R, :2 * FF], lay["w2"].pair, lay["bm2"], residual=x, out=t, alpha=lay["w2"].alpha)
            ops.layernorm(t, g3, b3, out=x, eps=e3)
            ops.layernorm(t, g3, b3, out=xp, eps=e3, split=True)
        ops.gemm_f16x3(xp, self.w_fc.pair, self.b_fc, out=ws["logits"][:R], alpha=self.w_fc.alpha)

    def _check_err(self, ws) -> None:
        err = ws["err"].tolist()
        if any(err):
            ws["err"].zero_()
            if err[0]:
                raise IndexError(f"index out of range: a word id outside [0, {self.V}) or a position past the {self.pe.shape[0]} rows of pe")
            if err[2]:
                raise RuntimeError("decode attention: a path outside the K / V slot pool or a clip outside the encoded batch")
            raise RuntimeError("the decoder produced NaN or infinite logits")

    def _linear_paths(self, ws, B: int, S: int) -> None:
        """Clip b's position p in slot b * S + p: path = the identity slot list, start b * S."""
        dev = self.device
        ws["path"].copy_(torch.arange(B * S, dtype=torch.int32, device=dev))
        ws["start"][:B].copy_(torch.arange(B, dtype=torch.int64, device=dev) * S)
        ws["row_clip"][:B].copy_(torch.arange(B, dtype=torch.int32, device=dev))

    @torch.no_grad()
    def decode(self, memory: torch.Tensor, tgt: torch.Tensor) -> torch.Tensor:
        """Teacher-forced ACT.decode: memory (B, Lm, nhid), tgt (B, n) -> logits (n, B, ntoken), position by position."""
        self.ensure_current()
        enc = self._memory_ws(memory)
        B, n = tgt.shape
        if n > MAX_POS:
            raise IndexError(f"a target of {n} words exceeds the {MAX_POS} rows of the positional encoding")
        ws = self._dec_ws(B, max(n, 1))
        self._linear_paths(ws, B, max(n, 1))
        out = torch.empty(n, B, self.V, dtype=torch.float32, device=self.device)
        tgt = tgt.to(self.device)
        for p in range(n):
            ws["tok"][:B].copy_(tgt[:, p])
            ws["pos"][:B].fill_(p)
            self._dec_step(ws, enc, B, n)
            out[p].copy_(ws["logits"][:B])
        self._check_err(ws)
        return out

    @torch.no_grad()
    def greedy(self, memory: torch.Tensor, sos_ind: int, max_len: int = 30) -> torch.Tensor:
        """greedy_decode: (B, max_len + 1) int64, one captured step replayed max_len times."""
        self.ensure_current()
        enc = self._memory_ws(memory)
        B = memory.shape[0]
        if max_len + 1 > MAX_POS:
            raise IndexError(f"max_len={max_len} exceeds the {MAX_POS} rows of the positional encoding")
        S = max_len + 1
        ws = self._dec_ws(B, S)
        self._linear_paths(ws, B, S)
        ys = ws.setdefault("ys", torch.zeros(B, S, dtype=torch.int64, device=self.device))

        def step():
            self._dec_step(ws, enc, B, max_len)
            ops.caption_select_greedy(ws["logits"][:B], ys, ws["tok"][:B], ws["pos"][:B], err_flag=ws["err"][1:2])

        def arm():
            ys.fill_(sos_ind)
            ws["tok"][:B].fill_(sos_ind)
            ws["pos"][:B].zero_()

        key = ("greedy", id(enc["kv"]), max_len)
        g = ws["graphs"].get(key) if self.use_cuda_graph else None
        if self.use_cuda_graph and g is None:  # the warm-up runs one step: the state is re-armed afterwards
            arm()
            g = ws["graphs"][key] = capture(step, self.device)
        arm()
        for _ in range(max_len):
            if g is not None:
                g.replay()
            else:
                step()
        self._check_err(ws)
        return ys.clone()

    @torch.no_grad()
    def beam(self, memory: torch.Tensor, sos_ind: int, eos_ind: int, beam_width: int = 5, top_k: int = 1) -> List[List[int]]:
        """beam_decode's search (evaluation.audiocaption.decode.beam_search) with every round's nodes expanded in one decode step."""
        from .evaluation.audiocaption.decode import beam_search
        self.ensure_current()
        if not 1 <= beam_width <= ops.CAPTION_MAX_K:
            raise ValueError(f"beam_width={beam_width} out of range (1 ... {ops.CAPTION_MAX_K})")
        if beam_width > self.V:
            raise RuntimeError(f"selected index k out of range: beam_width={beam_width} > vocabulary size {self.V}")
        enc = self._memory_ws(memory)
        B = memory.shape[0]
        S = BEAM_SLOTS
        ws = self._dec_ws(B, S)
        used = [0] * B
        dev = self.device

        def expand(items):
            R = len(items)
            paths, tok, pos, clip = [], np.empty(R, np.int64), np.empty(R, np.int32), np.empty(R, np.int32)
            for r, (c, n) in enumerate(items):
                if used[c] >= S:
                    raise RuntimeError(f"beam search: clip {c} expanded more than {S} nodes")
                if n.leng > MAX_POS:
                    raise IndexError(f"beam search: a prefix of {n.leng} words exceeds the {MAX_POS} rows of the positional encoding")
                n.slot = c * S + used[c]
                used[c] += 1
                n.path = np.append(n.prevNode.path, np.int32(n.slot)) if n.prevNode is not None else np.array([n.slot], np.int32)
                paths.append(n.path)
                tok[r], pos[r], clip[r] = n.wordid, n.leng - 1, c
            lens = np.array([len(p) for p in paths], np.int64)
            start = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.int64)
            flat = np.concatenate(paths)
            ws["path"][:flat.size].copy_(torch.from_numpy(flat))
            ws["start"][:R].copy_(torch.from_numpy(start))
            ws["tok"][:R].copy_(torch.from_numpy(tok))
            ws["pos"][:R].copy_(torch.from_numpy(pos))
            ws["row_clip"][:R].copy_(torch.from_numpy(clip))
            self._dec_step(ws, enc, R, int(lens.max()))
            vals = ws["vals"].view(-1)[:R * beam_width].view(R, beam_width)  # the select kernel writes (R, k) rows back to back
            idx = ws["idx"].view(-1)[:R * beam_width].view(R, beam_width)
            ops.caption_select_topk(ws["logits"], beam_width, vals, idx, R=R, err_flag=ws["err"][1:2])
            vals, idx = vals.cpu().tolist(), idx.cpu().tolist()
            self._check_err(ws)
            return vals, idx

        return beam_search(expand, B, sos_ind, eos_ind, beam_width, top_k)
