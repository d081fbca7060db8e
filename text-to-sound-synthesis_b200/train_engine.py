"""Denoiser training engine: forward with saved activations + hand-written backward of Text2ImageTransformer
(SURVEY.md section 8 row A13; reference transformer_utils.py:255-272, :421-443 differentiated by torch autograd).

Every GEMM (forward, dgrad, wgrad, the attention products) is dsb_gemm_ex on wgmma -- bf16 operands ('bf16', BASELINE config 4)
or TF32 ('tf32', the accuracy mode the parity tests use) with fp32 accumulation; the residual stream, LayerNorm statistics, softmax
inputs, all parameter gradients and the loss are fp32.  Everything else is a kernel of csrc/train.cu.  No torch arithmetic on the
path: torch supplies buffers (empty / zeros) and views only.

Layout notes
  * dgrad needs W^T as the K-major "weight" operand: transposed, cast copies of every Linear weight are rebuilt by pack() from the
    live fp32 parameters (they change every optimizer step).
  * wgrad dW (N, K) = dY^T X contracts over the M = B*L tokens: dY^T (N, Mp) and X^T (K, Mp) are produced by dsb_transpose into scratch
    (Mp = M rounded up to 8 for the 16-byte TMA stride; the GEMM's reduction length is the exact M, TMA zero-fills the tail).
  * attention, bf16 mode: fused kernels of csrc/attention_train.cu on the token-major QKV / gradient buffers in place (forward keeps only the
    log-sum-exp rows; backward = a dQ kernel and a dK/dV kernel that rebuild P).  tf32 accuracy mode: composed head-major (B*H, L, 64):
    S = alpha Q K^T, P = softmax(S) (saved), O = P V; dV = P^T dO, dP = dO V^T, dS = alpha P (dP - rowsum(dP P)), dQ = dS K, dK = dS^T Q
    as batched wgmma GEMMs.
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import torch

from . import ops
from . import train_ops as T


def _rup(n: int, m: int) -> int:
    return (n + m - 1) // m * m


class DenoiserTrainEngine:
    def __init__(self, transformer, precision: str = "bf16"):
        if precision not in ("bf16", "tf32"):
            raise ValueError("training precision must be 'bf16' or 'tf32'")
        self.m = transformer
        self.precision = precision
        self.adt = torch.bfloat16 if precision == "bf16" else torch.float32
        self.gd = ops.BF16 if precision == "bf16" else ops.TF32
        # 2-byte operands can be fed MN-major (token-major dY / X for wgrad, torch's (out, in) weights for dgrad, V / K / Q / dO as stored for
        # attention): no transposed copies at all.  The TF32 accuracy mode keeps explicit transposes (dsb_transpose).
        self.mn = precision == "bf16"
        self._ws: Dict[tuple, dict] = {}
        self._graphs: Dict[tuple, torch.cuda.CUDAGraph] = {}
        self.use_cuda_graph = True  # replay forward / backward as two CUDA graphs (~1.5k launches per step otherwise)
        self._kernel_device = "cuda"  # the kernels exist for CUDA only; tests/test_cpu_train_engine.py swaps in CPU stand-ins to check the orchestration
        self.forward_id = 0         # activations live in engine-owned buffers: backward() must follow ITS forward (checked by the caller)

    def __deepcopy__(self, memo):  # a deep copy of the module gets a fresh engine: operands, workspaces and graphs are per-instance caches
        return DenoiserTrainEngine(memo.get(id(self.m), self.m), precision=self.precision)

    # ------------------------------------------------------------------ small helpers
    @property
    def device(self):
        return self.m.to_logits[1].weight.device

    def _act(self, *shape):
        t = torch.empty(*shape, dtype=self.adt, device=self.device)
        return t

    def _f32(self, *shape):
        return torch.empty(*shape, dtype=torch.float32, device=self.device)

    def _cast_w(self, w: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
        return T.cast_scale(w.detach().contiguous(), out)

    def reset(self) -> None:
        """Drop packed operands and workspaces (the module moved to another device / dtype)."""
        self._ws.clear()
        self._graphs.clear()
        for attr in ("layers", "_layout", "_seg_plans", "_seg_names"):
            if hasattr(self, attr):
                delattr(self, attr)

    # ------------------------------------------------------------------ weights
    @torch.no_grad()
    def pack(self) -> None:
        """Cast (and transpose) the live fp32 parameters into GEMM operands.  Called at the start of every forward()."""
        m = self.m
        if self.device.type != self._kernel_device:
            raise RuntimeError("DenoiserTrainEngine needs the module on a CUDA device (no CPU fallback)")
        D, H = m.n_embd, m.n_head
        if D % 128 or D // H != 64 or D > 1024:
            raise RuntimeError(f"training kernels need head_dim 64 and n_embd a multiple of 128, <= 1024 (n_embd={D}, n_head={H})")
        self.D, self.H, self.n_layer = D, H, len(m.blocks)
        self.scale = 1.0 / math.sqrt(D // H)  # softmax(Q K^T / sqrt(head_dim)) (transformer_utils.py:50, :101)
        first = not hasattr(self, "layers")
        if first:
            self.layers = []
            Cd = m.blocks[0].attn2.key.weight.shape[1]
            self.Cd = Cd
            self.wkv_all = self._act(self.n_layer * 2 * D, Cd)
            self.bkv_all = self._f32(self.n_layer * 2 * D)
            for blk in m.blocks:
                Dh = blk.mlp[0].weight.shape[0]
                self.layers.append(dict(
                    wqkv=self._act(3 * D, D), wqkvT=self._act(D, 3 * D), bqkv=self._f32(3 * D),
                    wo1=self._act(D, D), wo1T=self._act(D, D), wq2=self._act(D, D), wq2T=self._act(D, D),
                    wo2=self._act(D, D), wo2T=self._act(D, D), w1=self._act(Dh, D), w1T=self._act(D, Dh), w2=self._act(D, Dh), w2T=self._act(Dh, D),
                    lin1T=self._f32(D, 2 * D), lin2T=self._f32(D, 2 * D)))
            self.K = m.to_logits[1].weight.shape[0]
            self.wlog, self.wlogT = self._act(self.K, D), self._act(D, self.K)
        for li, (blk, lay) in enumerate(zip(m.blocks, self.layers)):
            a1, a2 = blk.attn1, blk.attn2
            for j, lin in enumerate((a1.query, a1.key, a1.value)):
                self._cast_w(lin.weight, lay["wqkv"][j * D:(j + 1) * D])
                lay["bqkv"][j * D:(j + 1) * D].copy_(lin.bias.detach())
            if not self.mn:
                T.transpose(lay["wqkv"], lay["wqkvT"])
            for name, lin in (("wo1", a1.proj), ("wq2", a2.query), ("wo2", a2.proj), ("w1", blk.mlp[0]), ("w2", blk.mlp[2])):
                self._cast_w(lin.weight, lay[name])
                if not self.mn:
                    T.transpose(lay[name], lay[name + "T"])
            self._cast_w(a2.key.weight, self.wkv_all[li * 2 * D:li * 2 * D + D])
            self._cast_w(a2.value.weight, self.wkv_all[li * 2 * D + D:(li + 1) * 2 * D])
            self.bkv_all[li * 2 * D:li * 2 * D + D].copy_(a2.key.bias.detach())
            self.bkv_all[li * 2 * D + D:(li + 1) * 2 * D].copy_(a2.value.bias.detach())
            T.transpose(blk.ln1.linear.weight.detach(), lay["lin1T"])
            T.transpose(blk.ln1_1.linear.weight.detach(), lay["lin2T"])
        self._cast_w(m.to_logits[1].weight, self.wlog)
        if not self.mn:
            T.transpose(self.wlog, self.wlogT)

    # ------------------------------------------------------------------ workspaces (allocated once per shape; nothing is allocated per step)
    def workspace(self, B: int, L: int, Lc: int) -> dict:
        key = (B, L, Lc)
        ws = self._ws.get(key)
        if ws is not None:
            return ws
        D, H, NL, K = self.D, self.H, self.n_layer, self.K
        M, Mc, BH = B * L, B * Lc, B * H
        Dh = self.layers[0]["w1"].shape[0]
        Lp, Lcp, Mp, Mcp, Bp = _rup(L, 8), _rup(Lc, 8), _rup(M, 8), _rup(Mc, 8), _rup(B, 8)
        a, f = self._act, self._f32
        per_layer = []
        for _ in range(NL):
            per_layer.append(dict(
                x1=f(B, L, D), x2=f(B, L, D), x3=f(B, L, D),
                e1=f(B, D), s1=f(B, D), tab1=f(B, 2 * D), e2=f(B, D), s2=f(B, D), tab2=f(B, 2 * D),
                h1=a(M, D), qkv=a(M, 3 * D), att1=a(M, D), h2=a(M, D), q2=a(M, D), att2=a(M, D), h3=a(M, D), u=a(M, Dh), act=a(M, Dh)))
            if self.mn:   # fused attention: only the log-sum-exp rows are kept
                per_layer[-1].update(lse1=f(BH, L), lse2=f(BH, L))
            else:         # composed attention (tf32 accuracy mode): head-major operands and the probabilities are kept
                per_layer[-1].update(qh1=a(BH, L, 64), kh1=a(BH, L, 64), vh1=a(BH, L, 64), P1=a(BH, L, Lp),
                                     qh2=a(BH, L, 64), kh2=a(BH, Lc, 64), vh2=a(BH, Lc, 64), P2=a(BH, L, Lcp))
        ws = dict(
            layers=per_layer, x_out=f(B, L, D), hf=a(M, D), logits=f(B, L, K), cond=a(Mc, self.Cd), kv_all=a(Mc, NL * 2 * D),
            arange=torch.arange(B, dtype=torch.int64, device=self.device),
            # static inputs / outputs of the two CUDA graphs
            ids=torch.zeros(B, L, dtype=torch.int64, device=self.device), t=torch.zeros(B, dtype=torch.int64, device=self.device),
            cond_in=f(Mc, self.Cd), dlogits=f(B, L, K), scale=torch.ones(1, dtype=torch.float32, device=self.device),
            grad_flat=torch.zeros(self._grad_layout()[1], dtype=torch.float32, device=self.device),
            # scratch shared by every layer
            dx=f(B, L, D), dy=a(M, D), dbig=a(M, Dh), dbig2=a(M, Dh), dh=f(M, D), dqkv=a(M, 3 * D), dq2=a(M, D), datt=a(M, D),
            dkv_all=a(Mc, NL * 2 * D), dlog=a(M, K),
            delta=f(BH, L),
            dtab=f(B, 2 * D), dtabT=f(2 * D, Bp), sT=f(D, Bp), ds=f(B, D), de=f(B, D))
        if not self.mn:  # composed-attention / explicit-transpose scratch of the tf32 accuracy mode
            ws.update(S=f(BH, L, Lp), vT=a(BH, 64, Lp), oh=a(BH, L, 64),
                      yT=a(max(Dh, 3 * D, K), Mp), xT=a(max(Dh, D), Mp), ykvT=a(NL * 2 * D, Mcp), condT=a(self.Cd, Mcp),
                      doh=a(BH, L, 64), dP=f(BH, L, Lp), dS=a(BH, L, Lp), PT=a(BH, Lp, Lp), doT=a(BH, 64, Lp), kT=a(BH, 64, Lp), qT=a(BH, 64, Lp),
                      dST=a(BH, Lp, Lp), dqh=a(BH, L, 64), dkh=a(BH, L, 64), dvh=a(BH, L, 64))
        ws["grads"] = self._grad_views(ws["grad_flat"])
        self._ws[key] = ws
        return ws

    # ------------------------------------------------------------------ gradient storage: one flat fp32 buffer, parameters are views
    def _grad_layout(self):
        """[(key, shape, offset)], total.  attn1 q/k/v and every layer's attn2 k/v gradients come out of fused wgrad GEMMs, so they are
        slices of the fused regions '_qkv_w.{li}' / '_kv_w' rather than regions of their own."""
        if hasattr(self, "_layout"):
            return self._layout
        D, NL, Cd = self.D, self.n_layer, self.Cd
        fused = (".attn1.query.", ".attn1.key.", ".attn1.value.", ".attn2.key.", ".attn2.value.")
        specs = [(n, tuple(p.shape)) for n, p in self.m.named_parameters() if not any(f_ in n for f_ in fused)]
        for li in range(NL):
            specs += [(f"_qkv_w.{li}", (3 * D, D)), (f"_qkv_b.{li}", (3 * D,))]
        specs += [("_kv_w", (NL * 2 * D, Cd)), ("_kv_b", (NL * 2 * D,))]
        out, off = [], 0
        for k, shp in specs:
            out.append((k, shp, off))
            off += _rup(math.prod(shp), 64)
        self._layout = (out, off)
        return self._layout

    def _grad_views(self, flat: torch.Tensor) -> Dict[str, torch.Tensor]:
        D = self.D
        v = {k: flat[o:o + math.prod(shp)].view(shp) for k, shp, o in self._grad_layout()[0]}
        for li in range(self.n_layer):
            for j, nm in enumerate(("query", "key", "value")):
                v[f"blocks.{li}.attn1.{nm}.weight"] = v[f"_qkv_w.{li}"][j * D:(j + 1) * D]
                v[f"blocks.{li}.attn1.{nm}.bias"] = v[f"_qkv_b.{li}"][j * D:(j + 1) * D]
            o = li * 2 * D
            v[f"blocks.{li}.attn2.key.weight"], v[f"blocks.{li}.attn2.value.weight"] = v["_kv_w"][o:o + D], v["_kv_w"][o + D:o + 2 * D]
            v[f"blocks.{li}.attn2.key.bias"], v[f"blocks.{li}.attn2.value.bias"] = v["_kv_b"][o:o + D], v["_kv_b"][o + D:o + 2 * D]
        return v

    def _replay(self, key, fn, first_run_executes=False):
        """Run fn() through a CUDA graph captured on first use (after one eager warm-up for lazy initialisation).
        first_run_executes: fn is NOT idempotent (a backward segment accumulates into the stream gradient), so the first call runs it eagerly exactly
        once -- that run is the execution -- and only records the graph for later calls."""
        ptrs = tuple(p.data_ptr() for p in self.m.parameters())
        ent = self._graphs.get(key)
        if ent is not None and ent[1] != ptrs:
            ent = None  # a parameter was re-allocated (EMA swap, .data assignment): the captured pointers are stale
        if ent is None and first_run_executes:
            fn()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, capture_error_mode="thread_local"):
                fn()
            self._graphs[key] = (g, ptrs)
            return
        if ent is None:
            cur = torch.cuda.current_stream()
            side = torch.cuda.Stream()
            side.wait_stream(cur)
            with torch.cuda.stream(side):
                fn()
            cur.wait_stream(side)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, capture_error_mode="thread_local"):  # the backward graph is captured from autograd's worker thread; other threads (pin-memory) may touch CUDA
                fn()
            ent = self._graphs[key] = (g, ptrs)
        ent[0].replay()

    # ------------------------------------------------------------------ forward
    def _lin(self, a, w, bias, out, residual=None):
        """out = a @ w^T + bias (+ residual).  Outputs without a residual are activations that feed the next GEMM: bf16, or
        tf32-rounded fp32 in 'tf32' mode; outputs with a residual are the fp32 stream."""
        return ops.gemm(a, w, bias, residual, out, dtype=self.gd, round_out=(residual is None and out.dtype == torch.float32))

    def _ada_table(self, ln, t, e, s, tab):
        T.gather_rows(ln.emb.weight.detach(), t, e)
        ops.silu(e, out=s)
        # skinny (B rows) but K = D deep: the TF32 wgmma path reads the fp32 parameters directly (no packing) and is ~10x the SIMT GEMM here
        return ops.gemm(s, ln.linear.weight.detach(), ln.linear.bias.detach(), None, tab, dtype=ops.TF32)

    def _attn_fwd(self, q_tok, k_tok, v_tok, att_tok, qh, kh, vh, P, ws, B, Lq, Lk):
        H = self.H
        Lkp = _rup(Lk, 8)
        T.heads_split(q_tok, qh, B, H, Lq)
        T.heads_split(k_tok, kh, B, H, Lk)
        T.heads_split(v_tok, vh, B, H, Lk)
        S = ws["S"][:, :, :Lkp]
        ops.gemm(qh, kh, None, None, S, dtype=self.gd, alpha=self.scale)
        T.softmax_fwd(S, P, Lk)
        if self.mn:
            ops.gemm(P[:, :, :Lk], vh, None, None, ws["oh"], dtype=self.gd, w_mn=True)          # O = P V, V as stored (Lk, 64)
        else:
            vT = ws["vT"][:, :, :Lkp]
            T.transpose(vh, vT)
            ops.gemm(P[:, :, :Lk], vT[:, :, :Lk], None, None, ws["oh"], dtype=self.gd, round_out=True)
        T.heads_merge(ws["oh"], att_tok, B, H, Lq)

    @torch.no_grad()
    def forward(self, ids: torch.Tensor, cond_emb: torch.Tensor, t: torch.Tensor) -> torch.Tensor:
        """ids (B, L) int64, cond_emb (B, Lc, Cd) fp32, t (B,) int64 -> logits (B, L, K) fp32 (engine-owned buffer, valid until the next
        forward); activations are kept for backward()."""
        if not hasattr(self, "layers"):
            self.pack()  # allocates the packed operands; sizes the workspaces
        B, L = ids.shape
        Lc = cond_emb.shape[1]
        ws = self.workspace(B, L, Lc)
        self._shape = (B, L, Lc)
        self.forward_id += 1
        ws["ids"].copy_(ids)
        ws["t"].copy_(t)
        ws["cond_in"].copy_(cond_emb.detach().reshape(B * Lc, -1))
        if self.use_cuda_graph:
            self._replay(("fwd", B, L, Lc), lambda: self._forward_impl(ws, B, L, Lc))
        else:
            self._forward_impl(ws, B, L, Lc)
        return ws["logits"]

    def _forward_impl(self, ws, B, L, Lc):
        self.pack()
        m = self.m
        D = self.D
        self._ids, self._t = ws["ids"], ws["t"]
        ar = ws["arange"]
        T.cast_scale(ws["cond_in"], ws["cond"])
        self._lin(ws["cond"], self.wkv_all, self.bkv_all, ws["kv_all"])
        ce = m.content_emb
        x = ws["layers"][0]["x1"] if self.n_layer else ws["x_out"]
        ops.embed_tokens(self._ids, ce.emb.weight.detach(), ce.height_emb.weight.detach(), ce.width_emb.weight.detach(), out=x)
        rnd = self.adt == torch.float32
        for li, (blk, lay, sv) in enumerate(zip(m.blocks, self.layers, ws["layers"])):
            x1, x2, x3 = sv["x1"], sv["x2"], sv["x3"]
            x_next = ws["layers"][li + 1]["x1"] if li + 1 < self.n_layer else ws["x_out"]
            self._ada_table(blk.ln1, self._t, sv["e1"], sv["s1"], sv["tab1"])
            ops.ada_layernorm(x1, sv["tab1"], ar, out=sv["h1"].view(B, L, D), eps=1e-5, round_out=rnd)
            self._lin(sv["h1"], lay["wqkv"], lay["bqkv"], sv["qkv"])
            qkv = sv["qkv"]
            if self.mn:
                T.attention_train_fwd(qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:], sv["att1"], sv["lse1"], B, self.H, L, L, self.scale)
            else:
                self._attn_fwd(qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:], sv["att1"], sv["qh1"], sv["kh1"], sv["vh1"], sv["P1"], ws, B, L, L)
            self._lin(sv["att1"], lay["wo1"], blk.attn1.proj.bias.detach(), x2.view(B * L, D), residual=x1.view(B * L, D))
            self._ada_table(blk.ln1_1, self._t, sv["e2"], sv["s2"], sv["tab2"])
            ops.ada_layernorm(x2, sv["tab2"], ar, out=sv["h2"].view(B, L, D), eps=1e-5, round_out=rnd)
            self._lin(sv["h2"], lay["wq2"], blk.attn2.query.bias.detach(), sv["q2"])
            kv = ws["kv_all"][:, li * 2 * D:(li + 1) * 2 * D]
            if self.mn:
                T.attention_train_fwd(sv["q2"], kv[:, :D], kv[:, D:], sv["att2"], sv["lse2"], B, self.H, L, Lc, self.scale)
            else:
                self._attn_fwd(sv["q2"], kv[:, :D], kv[:, D:], sv["att2"], sv["qh2"], sv["kh2"], sv["vh2"], sv["P2"], ws, B, L, Lc)
            self._lin(sv["att2"], lay["wo2"], blk.attn2.proj.bias.detach(), x3.view(B * L, D), residual=x2.view(B * L, D))
            ops.layernorm(x3, blk.ln2.weight.detach(), blk.ln2.bias.detach(), out=sv["h3"].view(B, L, D), eps=blk.ln2.eps, round_out=rnd)
            self._lin(sv["h3"], lay["w1"], blk.mlp[0].bias.detach(), sv["u"])
            T.gelu2_fwd(sv["u"], sv["act"])
            self._lin(sv["act"], lay["w2"], blk.mlp[2].bias.detach(), x_next.view(B * L, D), residual=x3.view(B * L, D))
        lnf = m.to_logits[0]
        ops.layernorm(ws["x_out"], lnf.weight.detach(), lnf.bias.detach(), out=ws["hf"].view(B, L, D), eps=lnf.eps, round_out=rnd)
        ops.gemm(ws["hf"], self.wlog, m.to_logits[1].bias.detach(), None, ws["logits"].view(B * L, self.K), dtype=self.gd)
        return ws["logits"]

    # ------------------------------------------------------------------ backward
    def _linear_bwd(self, dy, x_act, w, wT, dW, db, dx_out, ws, *, yT=None, xT=None):
        """dy (M, N), x_act (M, K): dW (N, K) = dy^T x, db (N) = colsum(dy), dx_out (M, K) = dy W (if dx_out is not None).
        dx_out is either ws['dh'] (fp32, consumed by a LayerNorm backward) or an activation-typed buffer feeding another GEMM."""
        M, N = dy.shape
        Kin = x_act.shape[1]
        if self.mn:
            ops.gemm(dy, x_act, None, None, dW, dtype=self.gd, a_mn=True, w_mn=True)              # both operands token-major, read in place
        else:
            Mp = _rup(M, 8)
            yT = (ws["yT"] if yT is None else yT)[:N, :Mp]
            xT = (ws["xT"] if xT is None else xT)[:Kin, :Mp]
            T.transpose(dy, yT)
            T.transpose(x_act, xT)
            ops.gemm(yT[:, :M], xT[:, :M], None, None, dW, dtype=self.gd)
        if db is not None:
            T.colsum(dy, db)
        if dx_out is not None:
            if self.mn:
                ops.gemm(dy, w, None, None, dx_out, dtype=self.gd, w_mn=True)                      # W (N, Kin) as torch stores it
            else:
                ops.gemm(dy, wT, None, None, dx_out, dtype=self.gd, round_out=(dx_out.dtype == torch.float32 and dx_out is not ws["dh"]))

    def _attn_bwd(self, datt_tok, dq_tok, dk_tok, dv_tok, qh, kh, vh, P, ws, B, Lq, Lk):
        H = self.H
        Lkp, Lqp = _rup(Lk, 8), _rup(Lq, 8)
        scale = self.scale
        rnd = self.adt == torch.float32
        doh = ws["doh"]
        T.heads_split(datt_tok, doh, B, H, Lq)
        dP = ws["dP"][:, :, :Lkp]
        ops.gemm(doh, vh, None, None, dP, dtype=self.gd)                                  # dP = dO V^T
        dS = ws["dS"][:, :, :Lkp]
        T.softmax_bwd(P, dP, dS, Lk, scale)
        BH = B * H
        dvh = ws["dvh"].view(-1)[:BH * Lk * 64].view(BH, Lk, 64)
        dkh = ws["dkh"].view(-1)[:BH * Lk * 64].view(BH, Lk, 64)
        if self.mn:
            ops.gemm(P[:, :, :Lk], doh, None, None, dvh, dtype=self.gd, a_mn=True, w_mn=True)        # dV = P^T dO
            ops.gemm(dS[:, :, :Lk], kh, None, None, ws["dqh"], dtype=self.gd, w_mn=True)            # dQ = dS K
            ops.gemm(dS[:, :, :Lk], qh, None, None, dkh, dtype=self.gd, a_mn=True, w_mn=True)       # dK = dS^T Q
        else:
            PT, doT = ws["PT"][:, :Lk, :Lqp], ws["doT"][:, :, :Lqp]
            T.transpose(P[:, :, :Lk], PT)
            T.transpose(doh, doT)
            ops.gemm(PT[:, :, :Lq], doT[:, :, :Lq], None, None, dvh, dtype=self.gd, round_out=rnd)
            kT = ws["kT"][:, :, :Lkp]
            T.transpose(kh, kT)
            ops.gemm(dS[:, :, :Lk], kT[:, :, :Lk], None, None, ws["dqh"], dtype=self.gd, round_out=rnd)
            dST, qT = ws["dST"][:, :Lk, :Lqp], ws["qT"][:, :, :Lqp]
            T.transpose(dS[:, :, :Lk], dST)
            T.transpose(qh, qT)
            ops.gemm(dST[:, :, :Lq], qT[:, :, :Lq], None, None, dkh, dtype=self.gd, round_out=rnd)
        T.heads_merge(ws["dqh"], dq_tok, B, H, Lq)
        T.heads_merge(dkh, dk_tok, B, H, Lk)
        T.heads_merge(dvh, dv_tok, B, H, Lk)

    def _ada_bwd(self, ln, linT, x, dh, sv_e, sv_s, tab, grads, prefix, ws, B):
        """AdaLayerNorm backward incl. its timestep MLP Linear(SiLU(emb[t])) (transformer_utils.py:145-149)."""
        D = self.D
        dtab = ws["dtab"]
        dtab.zero_()
        T.ada_layernorm_bwd(x, dh.view(x.shape), ws["dx"], tab, ws["arange"], dtab, dx_act=ws["dy"])
        Bp = _rup(B, 8)
        dtabT, sT = ws["dtabT"][:, :Bp], ws["sT"][:, :Bp]
        T.transpose(dtab, dtabT)
        T.transpose(sv_s, sT)
        ops.gemm(dtabT[:, :B], sT[:, :B], None, None, grads[prefix + "linear.weight"], dtype=ops.TF32)
        T.colsum(dtab, grads[prefix + "linear.bias"])
        ops.gemm(dtab, linT, None, None, ws["ds"], dtype=ops.TF32)
        T.silu_bwd(sv_e, ws["ds"], ws["de"])
        g = grads[prefix + "emb.weight"]
        g.zero_()
        T.scatter_add_rows(g, self._t, ws["de"])

    def dlogits_buffer(self) -> torch.Tensor:
        """(B, L, K) fp32 buffer the loss kernel writes d loss / d logits into (static input of the backward graph)."""
        return self.workspace(*self._shape)["dlogits"]

    @torch.no_grad()
    def backward(self, dlogits: torch.Tensor, scale: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
        """dlogits (B, L, K) fp32 = d loss / d logits for unit upstream gradient, scale = upstream d loss (device scalar or None).
        Returns {parameter name (relative to the Text2ImageTransformer): fp32 gradient}; the tensors are views of one freshly cloned
        flat buffer, so the caller (autograd) owns them."""
        B, L, Lc = self._shape
        ws = self.workspace(B, L, Lc)
        if dlogits.data_ptr() != ws["dlogits"].data_ptr():
            ws["dlogits"].copy_(dlogits)
        if scale is None:
            ws["scale"].fill_(1.0)
        else:
            ws["scale"].copy_(scale.reshape(1))
        if self.use_cuda_graph:
            self._replay(("bwd", B, L, Lc), lambda: self._backward_impl(ws, B, L, Lc))
        else:
            self._backward_impl(ws, B, L, Lc)
        out = self._grad_views(ws["grad_flat"].clone())
        return {n: out[n] for n, _ in self.m.named_parameters()}

    # ---- segmented backward: head -> layer NL-1 ... layer 0 -> tail, one CUDA graph each.  DiffusionTransformer chains one autograd node per
    # segment, so a layer's parameter gradients reach autograd (and DistributedDataParallel's bucketed NCCL all-reduce, solver_spec.py:109) as soon
    # as that layer's backward has been launched, and the all-reduce of layer l overlaps the backward of layers l-1 ... 0.
    def segment_names(self, seg):
        """Parameter names (relative to the Text2ImageTransformer) whose gradients segment `seg` = 'head' | ('layer', li) | 'tail' produces."""
        cache = self.__dict__.setdefault("_seg_names", {})
        if seg in cache:
            return cache[seg]
        cache[seg] = self._segment_names(seg)
        return cache[seg]

    def _segment_names(self, seg):
        names = [n for n, _ in self.m.named_parameters()]
        if seg == "head":
            return [n for n in names if n.startswith("to_logits.")]
        if seg == "tail":
            return [n for n in names if n.startswith("content_emb.")]
        pre = f"blocks.{seg[1]}."
        return [n for n in names if n.startswith(pre)]

    def backward_begin(self, dlogits: torch.Tensor, scale: Optional[torch.Tensor] = None) -> None:
        B, L, Lc = self._shape
        ws = self.workspace(B, L, Lc)
        if dlogits.data_ptr() != ws["dlogits"].data_ptr():
            ws["dlogits"].copy_(dlogits)
        if scale is None:
            ws["scale"].fill_(1.0)
        else:
            ws["scale"].copy_(scale.reshape(1))

    def backward_segment(self, seg) -> Dict[str, torch.Tensor]:
        """Run one segment of the backward pass (call them in order after backward_begin) and return fresh copies of the gradients it produced."""
        B, L, Lc = self._shape
        ws = self.workspace(B, L, Lc)
        fn = {"head": lambda: self._bwd_head(ws, B, L, Lc), "tail": lambda: self._bwd_tail(ws, B, L, Lc)}.get(seg) if isinstance(seg, str) else \
            (lambda: self._bwd_layer(ws, B, L, Lc, seg[1]))
        if self.use_cuda_graph:
            self._replay(("bwd_seg", seg, B, L, Lc), fn, first_run_executes=True)
        else:
            fn()
        runs, items = self._segment_plan(seg)
        flat = ws["grad_flat"]
        copies = [flat[a:b].clone() for a, b in runs]   # one clone per contiguous run of the flat buffer (a layer: its parameters + its fused QKV region)
        return {n: copies[r][o:o + numel].view(shp) for n, r, o, numel, shp in items}

    def _segment_plan(self, seg):
        """(contiguous [start, end) runs of the flat gradient buffer, [(name, run index, offset in run, numel, shape)]), cached."""
        cache = self.__dict__.setdefault("_seg_plans", {})
        if seg in cache:
            return cache[seg]
        D, Cd = self.D, self.Cd
        layout = {k: (o, shp) for k, shp, o in self._grad_layout()[0]}
        src = {}
        for n in self.segment_names(seg):
            if n in layout:
                o, shp = layout[n]
            elif ".attn1." in n:  # a third of the layer's fused QKV wgrad / bias-gradient region
                li, j = int(n.split(".")[1]), ("query", "key", "value").index(n.split(".")[3])
                w = n.endswith("weight")
                o, shp = layout[f"_qkv_w.{li}" if w else f"_qkv_b.{li}"][0] + j * D * (D if w else 1), ((D, D) if w else (D,))
            else:                 # rows [li*2D (+D for value), +D) of the all-layer cross-attention K/V region
                li, w = int(n.split(".")[1]), n.endswith("weight")
                r0 = li * 2 * D + (0 if ".key." in n else D)
                o, shp = layout["_kv_w" if w else "_kv_b"][0] + r0 * (Cd if w else 1), ((D, Cd) if w else (D,))
            src[n] = (o, math.prod(shp), shp)
        runs = []
        for a, b in sorted((o, o + n_) for o, n_, _ in src.values()):
            if runs and a <= runs[-1][1] + 64:  # adjacent up to the 64-element alignment gaps of the layout
                runs[-1][1] = max(runs[-1][1], b)
            else:
                runs.append([a, b])
        items = []
        for n, (o, numel, shp) in src.items():
            r = max(i for i, (a, _) in enumerate(runs) if a <= o)
            items.append((n, r, o - runs[r][0], numel, shp))
        cache[seg] = ([tuple(r) for r in runs], items)
        return cache[seg]

    def _backward_impl(self, ws, B, L, Lc):
        self._bwd_head(ws, B, L, Lc)
        for li in range(self.n_layer - 1, -1, -1):
            self._bwd_layer(ws, B, L, Lc, li)
        self._bwd_tail(ws, B, L, Lc)

    def _bwd_head(self, ws, B, L, Lc):
        m = self.m
        D, K = self.D, self.K
        M = B * L
        grads = ws["grads"]
        dx = ws["dx"]
        # ---- head: logits = LN_f(x) Wlog^T + b
        T.cast_scale(ws["dlogits"].view(M, K), ws["dlog"], ws["scale"])
        self._linear_bwd(ws["dlog"], ws["hf"], self.wlog, self.wlogT, grads["to_logits.1.weight"], grads["to_logits.1.bias"], ws["dh"], ws)
        dx.zero_()
        lnf = m.to_logits[0]
        grads["to_logits.0.weight"].zero_(); grads["to_logits.0.bias"].zero_()
        T.layernorm_bwd(ws["x_out"], ws["dh"].view(B, L, D), dx, lnf.weight.detach(), grads["to_logits.0.weight"], grads["to_logits.0.bias"], lnf.eps,
                        dx_act=ws["dy"])  # every LayerNorm backward also emits the stream gradient as the next Linear backward's dY operand

    def _bwd_layer(self, ws, B, L, Lc, li):
        m = self.m
        D = self.D
        grads, dx, dkv_all = ws["grads"], ws["dx"], ws["dkv_all"]
        if True:
            blk, lay, sv = m.blocks[li], self.layers[li], ws["layers"][li]
            p = f"blocks.{li}."
            Dh = lay["w1"].shape[0]
            # ---- MLP: x_next = x3 + W2 gelu2(W1 LN2(x3))
            self._linear_bwd(ws["dy"], sv["act"], lay["w2"], lay["w2T"], grads[p + "mlp.2.weight"], grads[p + "mlp.2.bias"], ws["dbig"], ws)
            T.gelu2_bwd(sv["u"], ws["dbig"], ws["dbig2"])
            self._linear_bwd(ws["dbig2"], sv["h3"], lay["w1"], lay["w1T"], grads[p + "mlp.0.weight"], grads[p + "mlp.0.bias"], ws["dh"], ws)
            grads[p + "ln2.weight"].zero_(); grads[p + "ln2.bias"].zero_()
            T.layernorm_bwd(sv["x3"], ws["dh"].view(B, L, D), dx, blk.ln2.weight.detach(), grads[p + "ln2.weight"], grads[p + "ln2.bias"], blk.ln2.eps, dx_act=ws["dy"])
            # ---- cross-attention: x3 = x2 + Wo2 attn(q2, kv)
            self._linear_bwd(ws["dy"], sv["att2"], lay["wo2"], lay["wo2T"], grads[p + "attn2.proj.weight"], grads[p + "attn2.proj.bias"], ws["datt"], ws)
            dkv = dkv_all[:, li * 2 * D:(li + 1) * 2 * D]
            if self.mn:
                kv = ws["kv_all"][:, li * 2 * D:(li + 1) * 2 * D]
                T.attention_train_bwd(sv["q2"], kv[:, :D], kv[:, D:], sv["att2"], ws["datt"], sv["lse2"], ws["delta"], ws["dq2"], dkv[:, :D], dkv[:, D:],
                                      B, self.H, L, Lc, self.scale)
            else:
                self._attn_bwd(ws["datt"], ws["dq2"], dkv[:, :D], dkv[:, D:], sv["qh2"], sv["kh2"], sv["vh2"], sv["P2"], ws, B, L, Lc)
            # this layer's cross-attention K/V projections: kv = cond Wkv^T + b (its rows of the all-layer region; per layer, so that every parameter
            # of the layer has its gradient when the segment ends and DDP can start the layer's all-reduce)
            o_kv = li * 2 * D
            self._linear_bwd(dkv, ws["cond"], None, None, grads["_kv_w"][o_kv:o_kv + 2 * D], grads["_kv_b"][o_kv:o_kv + 2 * D], None, ws,
                             yT=ws.get("ykvT"), xT=ws.get("condT"))
            self._linear_bwd(ws["dq2"], sv["h2"], lay["wq2"], lay["wq2T"], grads[p + "attn2.query.weight"], grads[p + "attn2.query.bias"], ws["dh"], ws)
            self._ada_bwd(blk.ln1_1, lay["lin2T"], sv["x2"], ws["dh"], sv["e2"], sv["s2"], sv["tab2"], grads, p + "ln1_1.", ws, B)
            # ---- self-attention: x2 = x1 + Wo1 attn(qkv)
            self._linear_bwd(ws["dy"], sv["att1"], lay["wo1"], lay["wo1T"], grads[p + "attn1.proj.weight"], grads[p + "attn1.proj.bias"], ws["datt"], ws)
            dqkv = ws["dqkv"]
            if self.mn:
                qkv = sv["qkv"]
                T.attention_train_bwd(qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:], sv["att1"], ws["datt"], sv["lse1"], ws["delta"],
                                      dqkv[:, :D], dqkv[:, D:2 * D], dqkv[:, 2 * D:], B, self.H, L, L, self.scale)
            else:
                self._attn_bwd(ws["datt"], dqkv[:, :D], dqkv[:, D:2 * D], dqkv[:, 2 * D:], sv["qh1"], sv["kh1"], sv["vh1"], sv["P1"], ws, B, L, L)
            self._linear_bwd(dqkv, sv["h1"], lay["wqkv"], lay["wqkvT"], grads[f"_qkv_w.{li}"], grads[f"_qkv_b.{li}"], ws["dh"], ws)
            self._ada_bwd(blk.ln1, lay["lin1T"], sv["x1"], ws["dh"], sv["e1"], sv["s1"], sv["tab1"], grads, p + "ln1.", ws, B)

    def _bwd_tail(self, ws, B, L, Lc):
        grads, dx = ws["grads"], ws["dx"]
        # ---- embedding
        for n in ("content_emb.emb.weight", "content_emb.height_emb.weight", "content_emb.width_emb.weight"):
            grads[n].zero_()
        T.embed_bwd(self._ids, dx, grads["content_emb.emb.weight"], grads["content_emb.height_emb.weight"], grads["content_emb.width_emb.weight"])
