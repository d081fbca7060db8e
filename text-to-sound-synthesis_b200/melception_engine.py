"""Melception (Inception-v3 on 1-channel mels, the Diffsound evaluation's feature extractor) on sm_90a in split-fp16 ("f16x3") arithmetic.

Layout.  Activations are fp16 PAIR IMAGES (B, Hp, Wp, 2C): channels-last rows [hi | lo] with hi = f16(s v), lo = f16(s v - hi) (22 significand
bits), on a zero-bordered grid per resolution stage; a tensor's valid pixels are a window of its grid and every other pixel is exactly zero.
    stage A: the stem's 39 x W1 output with a 1-pixel border; the valid convs (Conv2d_2a, Conv2d_4a) keep the grid and shrink the window
             (39 x W1 -> 37 x (W1-2) -> 35 x (W1-4)), and Mixed_5b-d's 5x5 taps (radius 2) still land inside the grid;
    stage B: Mixed_6a-e at 17 x W2 with a 3-pixel border (the 1x7 / 7x1 taps);   stage C: Mixed_7a-c at 8 x W3 with a 1-pixel border.
Every convolution except the stem is ONE dsb_gemm_ex over a pair image (or three, see 5x5): taps are row shifts (dy Wp + dx), BatchNorm is folded
into the packed weights and bias (fp64), ReLU and the (hi | lo) split run in the epilogue (DSB_GEMM_RELU | DSB_GEMM_OUT_F16_SPLIT), and the geo_*
mask re-zeroes everything outside the output window.  Each branch of a block writes its channel slice of the block output directly (ldo = the
concat's row width, split_off = its channel count), so there is no concat copy.
    stride-2 valid 3x3 (Mixed_6a, Mixed_7a): dsb_pair_space_to_depth lays the input's four stride-2 phases on the next stage's grid; the conv is
        then a 9-tap GEMM with constant row shifts and per-tap A column offsets;
    5x5 (75 tap entries, over the GEMM's 32): three launches that chain the fp32 partial sum through `residual` in place; the last one adds
        the bias, ReLU after the residual (DSB_GEMM_RES_BEFORE_ACT) and writes the pair;
    pools: dsb_pair_avgpool3 (divisor 9) into a scratch pair image for the 1x1 pool branch; dsb_pair_maxpool3s2 straight into its concat slice;
    features: dsb_pair_channel_mean (adaptive_avg_pool2d) -> fp32 (B, C); fc on dsb_gemm_f32 (exact fp32).
The stem (Cin = 1, 4.8 MMAC per clip) runs on the FMA pipe (dsb_mel_stem), with the optional per-mel-bin input normalisation fused in.
Activation scales.  Each stored tensor carries a power-of-two scale sigma, folded exactly into its producers' alpha and bias (ReLU is positively
homogeneous); the branches of one block output share its sigma (the max-pool branch is moved onto it by an exact power-of-two factor).  The
sigmas are calibrated once at pack time on a fixed synthetic normalised clip: every producer runs with DSB_GEMM_NO_STORE + amax_out and sigma puts
the largest magnitude at 2^8..2^9, 2^7 below fp16's maximum.  One code path thus serves a trained checkpoint (activations ~1-100) and the
reference's own random init (~1e12 by Mixed_7c).  Features that come back non-finite raise RuntimeError.
Reference: Codebook/evaluation/feature_extractors/melception.py:23-113, torchvision models/inception.py (Inception3, InceptionA-E, BasicConv2d).
"""
from __future__ import annotations

import torch

from . import ops
from .engine_base import PackedEngine
from .graphs import GraphCache
from .packing import PackedConv, activation_scale

FEATURES = ("64", "192", "768", "2048", "logits_unbiased", "logits")
_DEPTH = {"64": 0, "192": 1, "768": 2, "2048": 3, "logits_unbiased": 3, "logits": 3}
BN_EPS = 1e-3


def _conv_names(prefix, names):
    return [f"{prefix}.{n}" for n in names]


# every BasicConv2d the forward runs on the GEMM (AuxLogits never runs; Conv2d_1a_3x3 is the stem kernel)
_A = ("branch1x1", "branch5x5_1", "branch5x5_2", "branch3x3dbl_1", "branch3x3dbl_2", "branch3x3dbl_3", "branch_pool")
_B = ("branch3x3", "branch3x3dbl_1", "branch3x3dbl_2", "branch3x3dbl_3")
_C = ("branch1x1", "branch7x7_1", "branch7x7_2", "branch7x7_3", "branch7x7dbl_1", "branch7x7dbl_2", "branch7x7dbl_3", "branch7x7dbl_4",
      "branch7x7dbl_5", "branch_pool")
_D = ("branch3x3_1", "branch3x3_2", "branch7x7x3_1", "branch7x7x3_2", "branch7x7x3_3", "branch7x7x3_4")
_E = ("branch1x1", "branch3x3_1", "branch3x3_2a", "branch3x3_2b", "branch3x3dbl_1", "branch3x3dbl_2", "branch3x3dbl_3a", "branch3x3dbl_3b",
      "branch_pool")
CONVS = ["Conv2d_2a_3x3", "Conv2d_2b_3x3", "Conv2d_3b_1x1", "Conv2d_4a_3x3"] + _conv_names("Mixed_5b", _A) + _conv_names("Mixed_5c", _A) + \
    _conv_names("Mixed_5d", _A) + _conv_names("Mixed_6a", _B) + sum((_conv_names(f"Mixed_6{c}", _C) for c in "bcde"), []) + \
    _conv_names("Mixed_7a", _D) + _conv_names("Mixed_7b", _E) + _conv_names("Mixed_7c", _E)


class _Act:
    """A stored pair image: tensor (B, Hp, Wp, 2C), channel count, scale key, window (y0, x0, H, W)."""

    def __init__(self, t, C, key, win):
        self.t, self.C, self.key, self.win = t, C, key, win



class MelceptionEngine(PackedEngine):
    settings = ("use_cuda_graph", "max_batch", "mean", "std")

    def __init__(self, module):
        super().__init__(module)
        self.use_cuda_graph = True
        self.max_batch = 64  # clips per pass: one 288-channel stage-A pair image is ~20 MB per clip at T = 848
        self._graphs = GraphCache()
        self.mean = self.std = None

    def set_normalization(self, mean=None, std=None):
        """Per-mel-bin (x - mean[f]) / std[f] fused into the stem (StandardNormalizeAudio, vggishish/transforms.py:13-40); None: inputs are
        already normalised."""
        dev = self.m.fc.weight.device
        if mean is not None and (not torch.isfinite(torch.as_tensor(std)).all() or bool((torch.as_tensor(std) == 0).any())):
            raise ValueError("normalisation std must be finite and non-zero")
        self.mean = None if mean is None else torch.as_tensor(mean, dtype=torch.float32).reshape(-1).to(dev).contiguous()
        self.std = None if std is None else torch.as_tensor(std, dtype=torch.float32).reshape(-1).to(dev).contiguous()
        self._graphs.clear()

    # ------------------------------------------------------------------------------------------------ packing
    def _fold(self, name):
        """BasicConv2d `name`: conv weight * gamma / sqrt(var + eps), beta - mean * gamma / sqrt(var + eps), in fp64."""
        c = self.m.get_submodule(name)
        w = c.conv.weight.detach().double()
        s = c.bn.weight.detach().double() / torch.sqrt(c.bn.running_var.detach().double() + BN_EPS)
        b = c.bn.bias.detach().double() - c.bn.running_mean.detach().double() * s
        return (w * s.view(-1, 1, 1, 1)).float(), b.float()

    def _pack(self):
        dev = self.m.fc.weight.device
        if dev.type != "cuda":
            raise RuntimeError("MelceptionEngine needs the module on a CUDA device (no CPU fallback)")
        w, b = self._fold("Conv2d_1a_3x3")
        self.stem = (w.reshape(w.shape[0], 9).contiguous(), b.contiguous())
        self.cv = {}
        for name in CONVS:
            w, b = self._fold(name)
            kh, kw = w.shape[2], w.shape[3]
            self.cv[name] = (PackedConv([w[:, :, y, x] for y in range(kh) for x in range(kw)], b), kh, kw, w.shape[1])
        self.fc_w = self.m.fc.weight.detach().float().contiguous()
        self.fc_b = self.m.fc.bias.detach().float().contiguous()
        self._graphs.clear()
        # ---- calibrate the power-of-two activation scales on a fixed synthetic normalised clip (independent of any user input)
        self.sig, self.amax, self._bias = {}, {}, {}
        self._amax = torch.zeros(1, dtype=torch.float32, device=dev)
        g = torch.Generator().manual_seed(20261016)
        x = (torch.rand(1, 80, 256, generator=g) * 4 - 2).to(dev)
        mean, std = self.mean, self.std
        self.mean = self.std = None
        try:
            self._forward(x, 3, calibrate=True)
        finally:
            self.mean, self.std = mean, std

    # ------------------------------------------------------------------------------------------------ producers of one stored tensor
    def _produce(self, key, prods, calibrate, extra_amax=0.0):
        """Run the launches `prods` that together write the tensor `key`; each is prod(measure): measure=True runs it unscaled with its last
        launch NO_STORE into self._amax.  Calibration measures first and sets sigma[key] = packing.activation_scale of the largest magnitude."""
        if calibrate:
            self._amax.zero_()
            for p in prods:
                p(True)
            m = max(float(self._amax.item()), extra_amax)
            self.sig[key] = activation_scale(m, f"Melception calibration: tensor {key}")
            self.amax[key] = m
        for p in prods:
            p(False)

    def _bias_for(self, name, key, measure):
        cv = self.cv[name][0]
        if measure:
            return cv.bias
        bb = self._bias.get(name)
        if bb is None:
            bb = self._bias[name] = (cv.bias * self.sig[key]).contiguous()
        return bb

    def _conv_prod(self, name, x, out, off, key, win, *, phases=None):
        """Producer of conv `name` reading pair image x (an _Act) into channels [off, off + Cout) of `out` (B, Hp, Wp, 2 Ctot) on output window
        `win`.  phases: (phase image (B, Hp, Wp, 8 Cin)) for a stride-2 conv."""
        cv, kh, kw, cin = self.cv[name]
        B, Hp, Wp, C2o = out.shape
        Ctot = C2o // 2
        M = B * Hp * Wp
        if phases is not None:
            A, lda = phases, 8 * cin
            sp = [((dy // 2) * Wp + dx // 2, (2 * (dy % 2) + dx % 2) * cin, 4 * cin + (2 * (dy % 2) + dx % 2) * cin, 0)
                  for dy in range(3) for dx in range(3)]
        else:
            A, lda = x.t, 2 * cin
            sp = [((y - kh // 2) * Wp + (xx - kw // 2), 0, cin, 0) for y in range(kh) for xx in range(kw)]
        taps = cv.taps(sp)
        y0, x0, H, W = win
        geo = (Hp * Wp, Wp, y0, y0 + H, x0, x0 + W)
        common = dict(A=A.data_ptr(), M=M, a_rows=M, a_cols=lda, lda=lda)
        optr = out.data_ptr() + 2 * off
        SPLIT, RELU = ops.OUT_F16_SPLIT, ops.RELU
        sig_in = self.sig[x.key]

        def run(measure):
            so = 1.0 if measure else self.sig[key]
            alpha = so / sig_in
            bias = self._bias_for(name, key, measure)
            last = dict(out=optr, ldo=C2o, split_off=Ctot, flags=SPLIT | RELU | (ops.NO_STORE if measure else 0), geo=geo,
                        amax_out=self._amax if measure else None)
            if len(taps) <= 32:
                cv.launch(**common, taps=taps, bias=bias, alpha=alpha, **last)
                return
            # 5x5: 25 spatial taps = 75 entries -> 27 + 24 + 24, the fp32 partial sum chained through `residual` in place
            part = torch.empty(M, cv.N, dtype=torch.float32, device=out.device)
            chunks = [taps[:27], taps[27:51], taps[51:]]
            cv.launch(**common, taps=chunks[0], alpha=alpha, out=part.data_ptr(), ldo=cv.N, flags=0)
            cv.launch(**common, taps=chunks[1], alpha=alpha, out=part.data_ptr(), ldo=cv.N, flags=0, residual=part.data_ptr(), ld_res=cv.N)
            last["flags"] |= ops.RES_BEFORE_ACT
            cv.launch(**common, taps=chunks[2], alpha=alpha, bias=bias, residual=part.data_ptr(), ld_res=cv.N, **last)
        return run

    def _conv(self, name, x, win, calibrate, *, phases=None):
        """Conv `name` into a new pair image on x's grid (or the phase image's grid)."""
        cv = self.cv[name][0]
        ref = x.t if phases is None else phases
        out = torch.empty(*ref.shape[:3], 2 * cv.N, dtype=torch.float16, device=ref.device)
        self._produce(name, [self._conv_prod(name, x, out, 0, name, win, phases=phases)], calibrate)
        return _Act(out, cv.N, name, win)

    def _concat(self, key, shape, Ctot, parts, calibrate, win, pool=None):
        """Block output: parts = [(conv name, input _Act, phases or None)], written side by side from channel 0; pool = (input _Act) for the
        stride-2 max-pool branch, written last.  shape: (B, Hp, Wp) of the output grid."""
        out = torch.empty(*shape, 2 * Ctot, dtype=torch.float16, device=parts[0][1].t.device)
        prods, off = [], 0
        for name, xa, ph in parts:
            prods.append(self._conv_prod(name, xa, out, off, key, win, phases=ph))
            off += self.cv[name][0].N
        extra = 0.0
        if pool is not None:
            xa, poff = pool, off

            def run_pool(measure):
                if not measure:
                    ops.pair_maxpool3s2(xa.t, xa.win, out, win[:2], out_ptr=out.data_ptr() + 2 * poff, ldo=2 * Ctot, lo_off=Ctot,
                                        scale=self.sig[key] / self.sig[xa.key])
            prods.append(run_pool)
            extra = self.amax[xa.key] if calibrate else 0.0  # a max pool's largest magnitude is at most its input's
            off += xa.C
        assert off == Ctot, (key, off, Ctot)
        self._produce(key, prods, calibrate, extra)
        return _Act(out, Ctot, key, win)

    def _phases(self, xa, grid_ref, origin):
        B = xa.t.shape[0]
        out = torch.empty(B, grid_ref[0], grid_ref[1], 8 * xa.C, dtype=torch.float16, device=xa.t.device)
        return ops.pair_space_to_depth(xa.t, xa.win, out, origin)

    def _avgpool(self, xa):
        return _Act(ops.pair_avgpool3(xa.t, xa.win), xa.C, xa.key, xa.win)  # same scale as its input

    # ------------------------------------------------------------------------------------------------ blocks (torchvision inception.py)
    def _block_a(self, n, x, cal):
        w = x.win
        b5 = self._conv(f"{n}.branch5x5_1", x, w, cal)
        d = self._conv(f"{n}.branch3x3dbl_2", self._conv(f"{n}.branch3x3dbl_1", x, w, cal), w, cal)
        pool = self._avgpool(x)
        parts = [(f"{n}.branch1x1", x, None), (f"{n}.branch5x5_2", b5, None), (f"{n}.branch3x3dbl_3", d, None), (f"{n}.branch_pool", pool, None)]
        return self._concat(n, x.t.shape[:3], sum(self.cv[p][0].N for p, _, _ in parts), parts, cal, w)

    def _block_b(self, n, x, grid, cal):
        origin = (3, 3)
        H, W = (x.win[2] - 3) // 2 + 1, (x.win[3] - 3) // 2 + 1
        win = (3, 3, H, W)
        d = self._conv(f"{n}.branch3x3dbl_2", self._conv(f"{n}.branch3x3dbl_1", x, x.win, cal), x.win, cal)
        px, pd = self._phases(x, grid, origin), self._phases(d, grid, origin)
        parts = [(f"{n}.branch3x3", x, px), (f"{n}.branch3x3dbl_3", d, pd)]
        return self._concat(n, (x.t.shape[0], *grid), 384 + 96 + x.C, parts, cal, win, pool=x)

    def _block_c(self, n, x, cal):
        w = x.win
        b7 = self._conv(f"{n}.branch7x7_2", self._conv(f"{n}.branch7x7_1", x, w, cal), w, cal)
        d = self._conv(f"{n}.branch7x7dbl_1", x, w, cal)
        for i in (2, 3, 4):
            d = self._conv(f"{n}.branch7x7dbl_{i}", d, w, cal)
        pool = self._avgpool(x)
        parts = [(f"{n}.branch1x1", x, None), (f"{n}.branch7x7_3", b7, None), (f"{n}.branch7x7dbl_5", d, None), (f"{n}.branch_pool", pool, None)]
        return self._concat(n, x.t.shape[:3], 768, parts, cal, w)

    def _block_d(self, n, x, grid, cal):
        origin = (1, 1)
        win = (1, 1, (x.win[2] - 3) // 2 + 1, (x.win[3] - 3) // 2 + 1)
        b3 = self._conv(f"{n}.branch3x3_1", x, x.win, cal)
        b7 = self._conv(f"{n}.branch7x7x3_1", x, x.win, cal)
        b7 = self._conv(f"{n}.branch7x7x3_3", self._conv(f"{n}.branch7x7x3_2", b7, x.win, cal), x.win, cal)
        parts = [(f"{n}.branch3x3_2", b3, self._phases(b3, grid, origin)), (f"{n}.branch7x7x3_4", b7, self._phases(b7, grid, origin))]
        return self._concat(n, (x.t.shape[0], *grid), 320 + 192 + x.C, parts, cal, win, pool=x)

    def _block_e(self, n, x, cal):
        w = x.win
        b3 = self._conv(f"{n}.branch3x3_1", x, w, cal)
        d = self._conv(f"{n}.branch3x3dbl_2", self._conv(f"{n}.branch3x3dbl_1", x, w, cal), w, cal)
        pool = self._avgpool(x)
        parts = [(f"{n}.branch1x1", x, None), (f"{n}.branch3x3_2a", b3, None), (f"{n}.branch3x3_2b", b3, None), (f"{n}.branch3x3dbl_3a", d, None),
                 (f"{n}.branch3x3dbl_3b", d, None), (f"{n}.branch_pool", pool, None)]
        return self._concat(n, x.t.shape[:3], 2048, parts, cal, w)

    # ------------------------------------------------------------------------------------------------ forward
    def _mean(self, xa):
        return ops.pair_channel_mean(xa.t, xa.win, inv_scale=1.0 / self.sig[xa.key])

    def _forward(self, x, depth, calibrate=False):
        """x (B, F, T) fp32 -> dict of the features up to `depth` (0: '64', 1: '192', 2: '768', 3: '2048' and the logits)."""
        B, Fm, T = x.shape
        H1, W1 = (Fm - 3) // 2 + 1, (T - 3) // 2 + 1
        if H1 < 11 or W1 < 11:  # Mixed_7a's stride-2 3x3 needs a 3-pixel-wide input
            raise RuntimeError(f"Melception needs at least 23 mel bins x 23 frames, got {Fm} x {T}")
        dev = x.device
        feats = {}
        # stage A: the stem's window at (1, 1) of a (H1 + 2) x (W1 + 2) grid
        Hp, Wp = H1 + 2, W1 + 2
        w0, b0 = self.stem
        t0 = torch.empty(B, Hp, Wp, 2 * w0.shape[0], dtype=torch.float16, device=dev)
        key = "Conv2d_1a_3x3"
        if calibrate:
            tmp = torch.empty_like(t0)
            ops.mel_stem(x, w0, b0, tmp, Hp=Hp, Wp=Wp, y0=1, x0=1, scale=1.0)
            m = float(tmp.float().abs().max())
            self.amax[key], self.sig[key] = m, activation_scale(m, "Melception calibration: the stem")
        ops.mel_stem(x, w0, b0, t0, Hp=Hp, Wp=Wp, y0=1, x0=1, scale=self.sig[key], mean=self.mean, std=self.std)
        h = _Act(t0, w0.shape[0], key, (1, 1, H1, W1))
        h = self._conv("Conv2d_2a_3x3", h, (2, 2, H1 - 2, W1 - 2), calibrate)
        h = self._conv("Conv2d_2b_3x3", h, h.win, calibrate)
        feats["64"] = self._mean(h)
        if depth == 0:
            return feats
        h = self._conv("Conv2d_3b_1x1", h, h.win, calibrate)
        h = self._conv("Conv2d_4a_3x3", h, (3, 3, H1 - 4, W1 - 4), calibrate)
        feats["192"] = self._mean(h)
        if depth == 1:
            return feats
        for n in ("Mixed_5b", "Mixed_5c", "Mixed_5d"):
            h = self._block_a(n, h, calibrate)
        H2, W2 = (h.win[2] - 3) // 2 + 1, (h.win[3] - 3) // 2 + 1
        h = self._block_b("Mixed_6a", h, (H2 + 6, W2 + 6), calibrate)
        for n in ("Mixed_6b", "Mixed_6c", "Mixed_6d", "Mixed_6e"):
            h = self._block_c(n, h, calibrate)
        feats["768"] = self._mean(h)
        if depth == 2:
            return feats
        H3, W3 = (H2 - 3) // 2 + 1, (W2 - 3) // 2 + 1
        h = self._block_d("Mixed_7a", h, (H3 + 2, W3 + 2), calibrate)
        h = self._block_e("Mixed_7b", h, calibrate)
        h = self._block_e("Mixed_7c", h, calibrate)
        f = self._mean(h)
        feats["2048"] = f
        feats["logits_unbiased"] = ops.gemm_f32(f, self.fc_w)
        feats["logits"] = ops.gemm_f32(f, self.fc_w, self.fc_b)
        return feats

    @torch.no_grad()
    def forward(self, x, features):
        """x (B, 80, T) fp32 CUDA -> {name: tensor} for the requested features ('64' / '192' / '768' as (B, C, 1, 1), '2048' and the logits
        as (B, C)); runs only as deep as the deepest requested feature."""
        if not x.is_cuda or self.m.fc.weight.device.type != "cuda":
            raise RuntimeError("Melception needs the module and its input on a CUDA device (no CPU fallback)")
        unknown = [f for f in features if f not in _DEPTH]
        if unknown:
            raise ValueError(f"unknown Melception features {unknown}; choose from {FEATURES}")
        if x.dim() != 3:
            raise RuntimeError(f"Melception input must be (B, n_mels, T), got {tuple(x.shape)}")
        self.ensure_current()
        x = x.detach().float().contiguous()
        depth = max(_DEPTH[f] for f in features)
        outs = []
        for i in range(0, x.shape[0], self.max_batch):
            xb = x[i:i + self.max_batch]
            keys = [f for f in FEATURES if _DEPTH[f] <= depth]
            fn = lambda xs: tuple(self._forward(xs, depth)[k] for k in keys)
            outs.append(dict(zip(keys, self._graphs.run((tuple(xb.shape), depth), fn, xb) if self.use_cuda_graph else fn(xb))))
        res = {}
        for f in features:
            v = torch.cat([o[f] for o in outs], 0) if len(outs) > 1 else outs[0][f]
            res[f] = v.view(v.shape[0], v.shape[1], 1, 1) if f in ("64", "192", "768") else v
        if not bool(torch.stack([torch.isfinite(v).all() for v in res.values()]).all()):
            raise RuntimeError("Melception produced non-finite features: the activations overflowed fp16 even after the calibrated scaling "
                               "(input far outside the normalised range the scales were calibrated on, or non-finite weights)")
        return res
