"""MelGAN generator on sm_90a in split-fp16 ("f16x3") arithmetic: every Conv1d / ConvTranspose1d / ResnetBlock tail is ONE wgmma GEMM
over per-stage state buffers, with all the elementwise work (bias, LeakyReLU, tanh, the (hi | lo) operand split, the residual sum) in GEMM
epilogues.

Layout.  Stage i (C channels, T samples) keeps ONE state buffer S (B, P + T + P, 4C) fp16, P = 9 pad rows, whose rows are
    [raw_hi | raw_lo | act_hi | act_lo],   raw ~ hi + lo (22 significand bits),   act = LeakyReLU(0.2)(raw),
i.e. 8 bytes per element -- exactly the reference's fp32 activation plus its activated copy -- and a scratch Y (B, T, 2C) for a block's
hidden tensor.  A ResnetBlock (reference vocoder/modules.py:72-85)
    y = shortcut(x) + conv1x1(LeakyReLU(conv3_dilated(ReflectionPad(LeakyReLU(x)))))
is:  edge_pad (reflect d rows of the act columns, a few KB)  ->  G1: 3 taps x 3 passes over S.act, LeakyReLU + split epilogue -> Y
     ->  G2: ONE GEMM over two A operands (S.raw against the shortcut weights, Y against the 1x1 weights), epilogue writes the new raw pair AND
     its LeakyReLU pair back into S in place (dsb_gemm_ex: A2 / DSB_GEMM_DUAL_LRELU).
ConvTranspose1d(stride r, kernel 2r, padding r/2) runs in polyphase form (output time q*r + ph touches inputs q-1, q or q, q+1): two GEMMs
with two taps each whose N = phase*Cout + c columns are scattered by the epilogue's column groups straight into the next stage's state rows.
weight_norm (w = g * v / ||v||, :18-23) is folded once at pack time; weights are (hi | lo) fp16 pairs of 2^s * w (alpha = 2^-s in the epilogue).
Activation scales.  The shipped checkpoint's activations grow from O(10) after the first conv to O(1e8) in the last stage (its final conv has
weights of 2e-3), far beyond fp16's 65504; since every layer is positively homogeneous up to its bias (LeakyReLU(c x) = c LeakyReLU(x), c > 0),
each stored tensor carries a power-of-two scale sigma (stored = sigma * true), folded exactly into the producing GEMM's alpha and bias.  The
sigmas are calibrated ONCE at pack time on a fixed synthetic mel clip: each GEMM first runs with DSB_GEMM_NO_STORE + amax_out (the largest
magnitude it would store), sigma puts that at 2^8..2^9 -- 128x headroom below fp16's maximum, while values 1e5 times smaller than the peak still keep
>= 17 significant bits in the (hi | lo) pair.  Inputs are mels in [0, 1], so activation magnitudes cannot exceed the calibration clip's by more
than a small factor.
Every product is lo*hi + hi*lo + hi*hi on fp16 wgmma with fp32 accumulation: fp32-class accuracy (the shipped checkpoint's weights
span a wide dynamic range; single-pass 11-bit operands give 2.6e-2 waveform error) at twice the TF32 MMA rate and half the operand bytes of
the round-1 split-TF32 path, and 3 launches per ResnetBlock instead of 7.
Reference: vocoder/modules.py:72-85 (ResnetBlock), :88-130 (Generator).
"""
from __future__ import annotations

import torch

from . import ops
from .engine_base import PackedEngine
from .graphs import GraphCache
from .packing import PackedConv as _PackedConv, activation_scale

P = 9  # pad rows on either side of every clip in a state buffer (largest dilation / half kernel)


def _c8(c: int) -> int:
    """Column-block width of a state row: channels rounded up to 8 halves (TMA box coordinates must be 16-byte aligned)."""
    return (c + 7) // 8 * 8


def _fold(m) -> torch.Tensor:
    v, g = m.weight_v.detach().float(), m.weight_g.detach().float()
    return g * v / v.flatten(1).norm(dim=1).view(-1, *([1] * (v.dim() - 1)))


class VocoderEngine(PackedEngine):
    settings = ("use_cuda_graph", "max_batch")

    def __init__(self, gen, precision: str = "f16x3"):
        if precision != "f16x3":
            raise ValueError("the MelGAN engine computes in split-fp16 ('f16x3': fp32-class accuracy on the fp16 tensor pipe)")
        super().__init__(gen, precision=precision)
        self.precision = precision
        self.launches = 0
        self.use_cuda_graph = True
        self.max_batch = 32  # clips per pass (8 bytes per activation element: 55.6 MB per clip for the widest stage)
        self._graphs = GraphCache()
        self._bufs = {}

    def _pack(self):
        mods = list(self.m.model)
        dev = mods[1].bias.device
        w0 = _fold(mods[1])  # (16*ngf, n_mel, 7)
        self.n_mel = w0.shape[1]
        self.first = _PackedConv([w0[:, :, j] for j in range(w0.shape[2])], mods[1].bias)
        self.stages = []
        i = 2
        for r in self.m.ratios:
            ct = mods[i + 1]
            w = _fold(ct)  # (Cin, Cout, 2r); weight_norm dim=0 -> norm over (Cout, k) per input channel
            p = r // 2 + r % 2
            assert r % 2 == 0, "polyphase split assumes even stride (the Diffsound ratios 8,8,2,2)"
            half = r - p
            cout = w.shape[1]
            if cout > 256:
                raise NotImplementedError("the in-place ResnetBlock tail needs Cout <= 256 (one 256-wide N tile); MelGAN's widest stage is 8 * ngf = 256")
            # phases [0, half): taps (q-1 -> k=ph+p+r, q -> k=ph+p); phases [half, r): taps (q -> k=ph+p, q+1 -> k=ph+p-r); rows n = phase*Cout + c
            wa = [torch.cat([w[:, :, ph + p + r].t() for ph in range(half)], 0), torch.cat([w[:, :, ph + p].t() for ph in range(half)], 0)]
            wb = [torch.cat([w[:, :, ph + p].t() for ph in range(half, r)], 0), torch.cat([w[:, :, ph + p - r].t() for ph in range(half, r)], 0)]
            st = dict(r=r, cin=w.shape[0], cout=cout, half=half, ca=_PackedConv(wa, ct.bias.detach().repeat(half)),
                      cb=_PackedConv(wb, ct.bias.detach().repeat(r - half)), res=[])
            i += 2
            for _ in range(self.m.n_residual_layers):
                rb = mods[i]
                wd, w1, ws = _fold(rb.block[2]), _fold(rb.block[4]), _fold(rb.shortcut)
                # g2 (shortcut | 1x1) is packed during calibration: its 1x1 half absorbs the ratio of the two operands' activation scales
                st["res"].append(dict(d=rb.dilation, g1=_PackedConv([wd[:, :, j] for j in range(3)], rb.block[2].bias, fold=_c8(cout) == 32), g2=None,
                                      ws=ws[:, :, 0].contiguous(), w1=w1[:, :, 0].contiguous(),
                                      b2=(rb.shortcut.bias.detach() + rb.block[4].bias.detach()).float()))
                i += 1
            self.stages.append(st)
        last = mods[i + 2]
        wl = _fold(last)  # (1, ngf, 7)
        self.last = _PackedConv([wl[:, :, j] for j in range(wl.shape[2])], last.bias, fold=_c8(wl.shape[1]) == 32)
        # 32-channel rows, 7 taps (the shipped generator): the output conv runs on the FMA pipe straight off the state buffer (dsb_conv_out_pair)
        self.last_w = None
        if _c8(wl.shape[1]) == 32 and wl.shape[2] == 7 and wl.shape[0] == 1:
            self.last_w = torch.zeros(7, 32, dtype=torch.float32, device=dev)
            self.last_w[:, :wl.shape[1]] = wl[0].t()
        self.c0 = w0.shape[0]
        self._graphs.clear()
        self._bufs.clear()
        # ---- calibrate the power-of-two activation scales on a fixed synthetic clip (deterministic: independent of any user input)
        self.sig, self.bias_s = {}, {}
        self._amax = torch.zeros(1, dtype=torch.float32, device=dev)
        mel = torch.rand(1, self.n_mel, 32, generator=torch.Generator().manual_seed(20260923)).to(dev)
        self._forward(mel, calibrate=True)
        self._bufs.clear()
        for st in self.stages:
            for rb in st["res"]:
                rb.pop("ws"), rb.pop("w1")

    def _buffers(self, B, T0, dev):
        key = (B, T0)
        b = self._bufs.get(key)
        if b is None:
            z = lambda *s: torch.zeros(*s, dtype=torch.float16, device=dev)
            states, ys, T = [z(B, T0 + 2 * P, 4 * _c8(self.c0))], [None], T0
            for st in self.stages:
                T *= st["r"]
                states.append(z(B, T + 2 * P, 4 * _c8(st["cout"])))
                ys.append(z(B, T, 2 * _c8(st["cout"])))
            b = self._bufs[key] = (states, ys)
        return b

    @torch.no_grad()
    def forward(self, mel: torch.Tensor) -> torch.Tensor:
        if not mel.is_cuda or list(self.m.model)[1].bias.device.type != "cuda":
            raise RuntimeError("VocoderEngine.forward needs the module and its input on a CUDA device (no CPU fallback)")
        self.ensure_current()
        mel = mel.detach().float().contiguous()
        if mel.shape[0] > self.max_batch:
            return torch.cat([self.forward(mel[i:i + self.max_batch]) for i in range(0, mel.shape[0], self.max_batch)], 0)
        if self.use_cuda_graph:
            return self._graphs.run(tuple(mel.shape), self._forward, mel)
        return self._forward(mel)

    def _scaled(self, key, sig_in, calibrate, calls):
        """Launch the GEMM(s) `calls` = [(PackedConv, PackedConv.launch kwargs)] that together produce ONE stored tensor; returns that tensor's
        scale sigma_out.  stored_out = sigma_out * (alpha_w / sigma_in * (A_stored . W_packed) + bias).  Calibration: a NO_STORE pass measures the
        largest true magnitude, sigma_out = packing.activation_scale of it."""
        if calibrate:
            self._amax.zero_()
            for cv, kw in calls:
                cv.launch(**dict(kw, flags=kw["flags"] | ops.NO_STORE), alpha=1.0 / sig_in, bias=cv.bias, amax_out=self._amax)
            self.sig[key] = activation_scale(float(self._amax.item()), f"MelGAN calibration: launch site {key}")
            self.bias_s[key] = [(cv.bias * self.sig[key]).contiguous() for cv, _ in calls]
        so = self.sig[key]
        for (cv, kw), bs in zip(calls, self.bias_s[key]):
            cv.launch(**kw, alpha=so / sig_in, bias=bs)
        return so

    def _forward(self, mel: torch.Tensor, calibrate: bool = False) -> torch.Tensor:
        B, Cm, T = mel.shape
        if Cm != self.n_mel:
            raise RuntimeError(f"mel has {Cm} channels, the generator expects {self.n_mel}")
        states, ys = self._buffers(B, T, mel.device)
        SPLIT, DUAL, LRELU, TANH = ops.OUT_F16_SPLIT, ops.DUAL_LRELU, ops.LRELU, ops.TANH
        n = 0
        # ReflectionPad1d(3) + Conv1d(n_mel -> 16 ngf, k=7) + the LeakyReLU in front of the first ConvTranspose1d  ->  states[0].act
        cv = self.first
        mp = ops.mel_pack_f16(mel, 3, cv.Kp)
        S, C = states[0], self.c0
        Cs = _c8(C)
        sig = self._scaled("first", 1.0, calibrate, [(cv, dict(
            A=mp.data_ptr(), out=S.data_ptr() + 2 * (P * 4 * Cs + 2 * Cs), M=T, batch=B, taps=cv.taps([(j, 0, cv.Kp, 0) for j in range(7)]),
            a_rows=T + 6, a_cols=2 * cv.Kp, lda=2 * cv.Kp, a_batch_stride=(T + 6) * 2 * cv.Kp, ldo=4 * Cs, out_batch_stride=(T + 2 * P) * 4 * Cs,
            flags=SPLIT | LRELU, split_off=Cs))])
        n += 2
        for si, st in enumerate(self.stages):
            r, Cin, Cout, half = st["r"], st["cin"], st["cout"], st["half"]
            Sin, S, Y = states[si], states[si + 1], ys[si + 1]
            Tin, T = T, T * r
            Ci, Co = _c8(Cin), _c8(Cout)  # column-block widths of the input / output state rows
            ldin, ld = 4 * Ci, 4 * Co
            if si > 0:  # the blocks left reflected samples in the pad rows; the transposed conv's polyphase taps need zeros there
                ops.edge_pad_f16(Sin, Tin, P, 1, 2 * Ci, 2 * Ci, reflect=False)
                n += 1
            sig = self._scaled(("convT", si), sig, calibrate, [(cv, dict(
                A=Sin.data_ptr(), out=S.data_ptr() + 2 * (P * ld + col0), M=Tin, batch=B, spatial=[(sh, 2 * Ci, 3 * Ci, 0) for sh in shifts],
                a_rows=Tin + 2 * P, a_cols=ldin, lda=ldin, a_batch_stride=(Tin + 2 * P) * ldin, ldo=r * ld, out_batch_stride=(T + 2 * P) * ld,
                flags=SPLIT | DUAL, split_off=Co, dual_off=2 * Co, out_col_group=Cout, out_col_group_stride=ld))
                for cv, shifts, col0 in ((st["ca"], (P - 1, P), 0), (st["cb"], (P, P + 1), half * ld))])
            n += 2
            for ri, rb in enumerate(st["res"]):
                d, g1 = rb["d"], rb["g1"]
                ops.edge_pad_f16(S, T, P, d, 2 * Co, 2 * Co, reflect=True)
                sig_y = self._scaled(("g1", si, ri), sig, calibrate, [(g1, dict(
                    A=S.data_ptr(), out=Y.data_ptr(), M=T, batch=B, spatial=[(P + (j - 1) * d, 2 * Co, 3 * Co, 0) for j in range(3)],
                    a_rows=T + 2 * P, a_cols=ld, lda=ld, a_batch_stride=(T + 2 * P) * ld, ldo=2 * Co, out_batch_stride=T * 2 * Co,
                    flags=SPLIT | LRELU, split_off=Co))])
                if calibrate:  # x is stored at sigma, y at sigma_y: the 1x1 half of the fused weight absorbs sigma / sigma_y (a power of two)
                    rb["g2"] = _PackedConv([rb["ws"], rb["w1"] * (sig / sig_y)], rb["b2"], fold=Co == 32)
                g2 = rb["g2"]
                sig = self._scaled(("g2", si, ri), sig, calibrate, [(g2, dict(
                    A=S.data_ptr(), A2=Y.data_ptr(), out=S.data_ptr() + 2 * (P * ld), M=T, batch=B, spatial=[(P, 0, Co, 0), (0, 0, Co, 1)],
                    a_rows=T + 2 * P, a_cols=ld, lda=ld, a_batch_stride=(T + 2 * P) * ld, lda2=2 * Co, a2_rows=T, a2_cols=2 * Co,
                    a2_batch_stride=T * 2 * Co, ldo=ld, out_batch_stride=(T + 2 * P) * ld, flags=SPLIT | DUAL, split_off=Co, dual_off=2 * Co,
                    # in place: ONE N tile must cover all Cout columns (a second N tile would re-read rows the first one overwrote)
                    block_n=256 if Cout > 128 else 128))])
                n += 3
        # LeakyReLU (already in .act) + ReflectionPad1d(3) + Conv1d(ngf -> 1, k=7) + tanh
        S, C = states[-1], _c8(self.stages[-1]["cout"])
        cv = self.last
        ops.edge_pad_f16(S, T, P, 3, 2 * C, 2 * C, reflect=True)
        wav = torch.empty(B, T, 1, dtype=torch.float32, device=mel.device)
        if self.last_w is not None:
            ops.conv_out_pair(S, T, P - 3, 2 * C, self.last_w, cv.bias, 1.0 / sig, out=wav)
            self.launches = n + 2
            return wav.view(B, 1, T)
        cv.launch(A=S.data_ptr(), out=wav.data_ptr(), M=T, batch=B, spatial=[(P - 3 + j, 2 * C, 3 * C, 0) for j in range(7)], a_rows=T + 2 * P,
                  a_cols=4 * C, lda=4 * C, a_batch_stride=(T + 2 * P) * 4 * C, ldo=1, out_batch_stride=T, bias=cv.bias, flags=TANH, alpha=1.0 / sig)
        self.launches = n + 2
        return wav.view(B, 1, T)
