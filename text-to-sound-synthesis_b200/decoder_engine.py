"""SpecVQGAN decoder on sm_90a: every Conv2d is a wgmma implicit GEMM over a zero-padded channels-last image.

Layout: activations are fp32 (B, H+2, W+2, C) with an exact-zero one-pixel border.  Flattening (b, y, x) to a row index makes
a 3x3 tap (dy, dx) the row shift dy*(W+2)+dx, so conv3x3 = one GEMM with 9 taps, A = the padded image (rows, Cin), W packed
as (Cout, 9*Cin); the epilogue adds bias (+ residual) and re-zeroes border rows.  GroupNorm needs image-wide statistics, so
it stays a separate reduction + apply(+swish) pass that also rounds to TF32 for the next GEMM.
Reference: specvqgan/modules/diffusionmodules/model.py:92-151 (ResnetBlock), :174-226 (AttnBlock), :37-52 (Upsample), :640-671.
"""
from __future__ import annotations

import torch

from . import ops
from .engine_base import PackedEngine
from .graphs import GraphCache
from .packing import PackedConv


class DecoderEngine(PackedEngine):
    settings = ("use_cuda_graph", "max_batch")

    def __init__(self, vq, precision: str = "f16x3"):
        """precision: 'f16x3'  -- split-fp16 operands: conv inputs leave GroupNorm / upsample / the codebook gather as fp16 (hi | lo) pairs, weights are
                                   (hi | lo) pairs of 2^s * W, every product is lo*hi + hi*lo + hi*hi on fp16 wgmma with fp32 accumulation:
                                   fp32-class accuracy (1e-3 mel tolerance through ~30 conv + GroupNorm layers) at twice the TF32 MMA rate and half
                                   the operand bytes of 'tf32x3';
                      'tf32x3' -- split-TF32 operands (fp32 containers), the round-1 path; still used by the encoder and the AttnBlocks;
                      'tf32'   -- single-pass TF32 (3x fewer MMAs; mel error ~4e-3 relative)."""
        if precision not in ("f16x3", "tf32x3", "tf32"):
            raise ValueError("precision must be 'f16x3', 'tf32x3' or 'tf32'")
        super().__init__(vq, precision=precision)
        self.precision = precision
        self.launches = 0
        self.use_cuda_graph = True
        self.max_batch = 32  # clips per pass: bounds the activation memory (34.7 MB fp32 per clip per full-resolution tensor) at any caller batch
        self._graphs = GraphCache()

    def _pack_conv(self, conv, tf32x3: bool = False):
        w = conv.weight.detach().float()  # (Cout, Cin, kh, kw) -> (Cout, kh*kw*Cin), tap-major
        ntaps = w.shape[2] * w.shape[3]
        if self.precision == "f16x3" and not tf32x3:
            return PackedConv([w[:, :, ky, kx] for ky in range(w.shape[2]) for kx in range(w.shape[3])], conv.bias)
        w = w.permute(0, 2, 3, 1).reshape(w.shape[0], -1).contiguous()
        return ops.pack_split_weight(w, ntaps) if self.precision != "tf32" else ops.round_tf32(w)

    def _mm(self, a, w, bias=None, residual=None, out=None, presplit=False, **kw):
        """a: fp32 activation (rows, C) or batched (already in (hi | lo) form when presplit); w: packed weight (split-TF32 or rounded).
        (In 'f16x3' mode this serves the AttnBlocks only: 265 tokens x 512 channels, four small GEMMs kept on the split-TF32 path.)"""
        if self.precision != "tf32":
            return ops.gemm_split(a if presplit else ops.split_tf32(a), w, bias, residual, out, **kw)
        return ops.gemm(a, w, bias, residual, out, **kw)

    def _pack(self):
        vq, d = self.m, self.m.decoder
        if vq.post_quant_conv.weight.device.type != "cuda":
            raise RuntimeError("DecoderEngine needs the module on a CUDA device (no CPU fallback)")
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
                c_ = getattr(m, n)
                self.w[name + "." + n] = (self._pack_conv(c_, tf32x3=True), f(c_.bias), 1)

        conv("post_quant", vq.post_quant_conv)
        conv("conv_in", d.conv_in)
        res("mid.block_1", d.mid.block_1); attn("mid.attn_1", d.mid.attn_1); res("mid.block_2", d.mid.block_2)
        for lvl, up in enumerate(d.up):
            for j, blk in enumerate(up.block):
                res(f"up.{lvl}.block.{j}", blk)
            for j, a in enumerate(up.attn):
                attn(f"up.{lvl}.attn.{j}", a)
            if hasattr(up, "upsample"):
                conv(f"up.{lvl}.upsample", up.upsample.conv)
        gn("norm_out", d.norm_out)
        conv("conv_out", d.conv_out)
        self.codebook = f(vq.quantize.embedding.weight)
        self._graphs.clear()

    # ------------------------------------------------------------------ building blocks (all on padded NHWC tensors)
    def _conv_f16(self, x, cv, k, residual=None, pair_out=False):
        """x: fp16 pair image (B, Hp, Wp, 2*Cin) -> fp32 (B, Hp, Wp, Cout) (+ fp32 residual), or its fp16 pair when pair_out (no GroupNorm in between)."""
        B, Hp, Wp, C2 = x.shape
        Cin, R, N = C2 // 2, B * Hp * Wp, cv.N
        shifts = [dy * Wp + dx for dy in (-1, 0, 1) for dx in (-1, 0, 1)] if k == 3 else [0]
        out = torch.empty(B, Hp, Wp, 2 * N if pair_out else N, dtype=torch.float16 if pair_out else torch.float32, device=x.device)
        cv.launch(A=x.data_ptr(), out=out.data_ptr(), M=R, taps=cv.taps([(sh, 0, Cin, 0) for sh in shifts]), a_rows=R, a_cols=C2, lda=C2,
                  ldo=out.shape[-1], bias=cv.bias, flags=ops.OUT_F16_SPLIT if pair_out else 0, split_off=N if pair_out else 0,
                  residual=None if residual is None else residual.data_ptr(), ld_res=0 if residual is None else residual.shape[-1],
                  geo=(Hp * Wp, Wp, 1, Hp - 1, 1, Wp - 1))
        self.launches += 1
        return out

    def _conv(self, x, name, residual=None, round_out=False, presplit=False, pair_out=False):
        """x: padded image (B, Hp, Wp, C), or its split form (B, Hp, Wp, 2C) from a producer that fused the (hi | lo) split."""
        w, b, k = self.w[name]
        B, Hp, Wp, C = x.shape  # C counts the (hi | lo) columns when presplit; only used to flatten
        R = B * Hp * Wp
        if isinstance(w, PackedConv):
            return self._conv_f16(x, w, k, residual, pair_out)
        taps = [dy * Wp + dx for dy in (-1, 0, 1) for dx in (-1, 0, 1)] if k == 3 else [0]
        out = torch.empty(B, Hp, Wp, w.shape[0], dtype=torch.float32, device=x.device)
        self._mm(x.view(R, C), w, b, None if residual is None else residual.view(R, -1), out.view(R, -1), taps=taps, presplit=presplit,
                 geo=(Hp * Wp, Wp, 1, Hp - 1, 1, Wp - 1), round_out=round_out and self.precision == "tf32")
        self.launches += 2 if (self.precision == "tf32x3" and not presplit) else 1
        return out

    def _gn(self, x, name, swish=True, compact_len=0):
        g, b, eps = self.w[name]
        st = ops.groupnorm_stats(x)
        self.launches += 3  # memset + stats + apply
        split = self.precision == "tf32x3" and not compact_len  # conv inputs leave GroupNorm already in (hi | lo) form
        return ops.groupnorm_apply(x, st, g, b, eps=eps, swish=swish, round_out=self.precision == "tf32", compact_len=compact_len, split=split,
                                   split_f16=self.precision == "f16x3" and not compact_len)

    def _res(self, x, name):
        sp = self.precision != "tf32"
        h = self._conv(self._gn(x, name + ".norm1"), name + ".conv1", presplit=sp)
        h = self._gn(h, name + ".norm2")
        if (name + ".nin") in self.w:
            if self.precision == "f16x3":  # the 1x1 shortcut convolves the raw (un-normalised) input: one elementwise split pass, twice per decode
                B_, Hp_, Wp_, C_ = x.shape
                self.launches += 1
                x = self._conv(ops.split_f16(x.view(-1, C_)).view(B_, Hp_, Wp_, 2 * C_), name + ".nin")
            elif self.precision == "tf32":
                self.launches += 1
                x = self._conv(ops.round_tf32(x), name + ".nin")
            else:
                x = self._conv(x, name + ".nin")
        return self._conv(h, name + ".conv2", residual=x, presplit=sp)

    def _attn(self, x, name):
        """AttnBlock (model.py:202-226): single head over the H*W interior tokens, scale C^-0.5; x is updated in place."""
        B, Hp, Wp, C = x.shape
        L = (Hp - 2) * (Wp - 2)
        Lp = (L + 15) // 16 * 16  # token rows padded so every TMA stride is a multiple of 16 bytes
        h = self._gn(x, name + ".norm", swish=False, compact_len=Lp).view(B * Lp, C)
        (wq, bq, _), (wk, bk, _), (wv, bv, _), (wp, bp, _) = (self.w[name + "." + n] for n in ("q", "k", "v", "proj_out"))
        rnd = self.precision == "tf32"
        q = self._mm(h, wq, bq, round_out=rnd).view(B, Lp, C)
        k = self._mm(h, wk, bk, round_out=rnd).view(B, Lp, C)
        v = self._mm(h, wv, bv, round_out=rnd).view(B, Lp, C)
        vT = v.transpose(1, 2).contiguous()  # (B, C, Lp): data movement only (token rows >= L are masked by the softmax below)
        if self.precision != "tf32":
            s_ = ops.gemm_split(ops.split_tf32(q), ops.split_tf32(k, w_format=True), alpha=float(C) ** -0.5)  # (B, Lp, Lp)
            ops.softmax_rows_(s_, L, round_out=False)
            o = ops.gemm_split(ops.split_tf32(s_), ops.split_tf32(vT, w_format=True))  # (B, Lp, C)
        else:
            s_ = ops.gemm(q, k, alpha=float(C) ** -0.5)
            ops.softmax_rows_(s_, L)
            o = ops.gemm(s_, vT, round_out=True)
        proj = self._mm(o.view(B * Lp, C), wp, bp).view(B, Lp, C)
        ops.tokens_add_to_padded_(proj, x)
        self.launches += 8
        return x

    # ------------------------------------------------------------------ entry points
    @torch.no_grad()
    def _decode_padded(self, z):
        d = self.m.decoder
        if self.precision == "f16x3":
            z = self._conv(z, "post_quant", pair_out=True)  # 1x1 conv straight into the next conv's (hi | lo) operand: no GroupNorm between them
            h = self._conv(z, "conv_in")
        else:
            z = self._conv(z, "post_quant", round_out=True, presplit=self.precision == "tf32x3")
            h = self._conv(z, "conv_in")
        h = self._res(h, "mid.block_1")
        h = self._attn(h, "mid.attn_1")
        h = self._res(h, "mid.block_2")
        for lvl in reversed(range(d.num_resolutions)):
            for j in range(d.num_res_blocks + 1):
                h = self._res(h, f"up.{lvl}.block.{j}")
                if len(d.up[lvl].attn) > 0:
                    h = self._attn(h, f"up.{lvl}.attn.{j}")
            if lvl != 0:
                sp = self.precision == "tf32x3"
                h = self._conv(ops.upsample2x_padded(h, round_out=self.precision == "tf32", split=sp, split_f16=self.precision == "f16x3"),
                               f"up.{lvl}.upsample", presplit=sp)
                self.launches += 1
        out = self._conv(self._gn(h, "norm_out"), "conv_out", presplit=self.precision == "tf32x3")  # (B, Hp, Wp, out_ch)
        return out[:, 1:-1, 1:-1, :].permute(0, 3, 1, 2).contiguous()

    @torch.no_grad()
    def decode_tokens(self, ids, grid):
        self.ensure_current()
        H, W = grid
        ids = ids.contiguous()
        if ids.shape[0] > self.max_batch:
            return torch.cat([self.decode_tokens(ids[i:i + self.max_batch], grid) for i in range(0, ids.shape[0], self.max_batch)], 0)

        def body(ids_):
            self.launches = 1
            err = torch.zeros(1, dtype=torch.int32, device=ids_.device)
            z = ops.codebook_gather_padded(ids_, self.codebook, H, W, round_out=self.precision == "tf32", split=self.precision == "tf32x3",
                                           split_f16=self.precision == "f16x3", err_flag=err)
            return self._decode_padded(z), err

        if self.use_cuda_graph:
            mel, err = self._graphs.run(("tok", tuple(ids.shape), H, W), body, ids)
        else:
            mel, err = body(ids)
        if int(err.item()):
            raise RuntimeError("codebook index out of range")
        return mel

    @torch.no_grad()
    def decode_latents(self, quant):
        """quant (B, E, H, W) NCHW (the reference's VQModel.decode input) -> mel; layout conversion is plain data movement."""
        self.ensure_current()
        self.launches = 1
        z = torch.nn.functional.pad(quant.detach().float().permute(0, 2, 3, 1), (0, 0, 1, 1, 1, 1)).contiguous()
        if self.precision == "f16x3":
            B_, Hp_, Wp_, C_ = z.shape
            return self._decode_padded(ops.split_f16(z.view(-1, C_)).view(B_, Hp_, Wp_, 2 * C_))
        return self._decode_padded(ops.round_tf32(z) if self.precision == "tf32" else ops.split_tf32(z))
