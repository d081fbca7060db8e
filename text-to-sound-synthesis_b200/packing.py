"""The host-side rules of the split-fp16 ("f16x3") GEMMs: how weights are scaled and packed into fp16 (hi | lo) pairs, how a calibrated activation
scale is chosen, and how a packed conv is handed to dsb_gemm_ex."""
from __future__ import annotations

import math

import torch

from . import ops


def k64(c: int) -> int:
    """Channels rounded up to the GEMM's 64-element fp16 k-block."""
    return (c + 63) // 64 * 64


def weight_prescale(amax: float) -> int:
    """Exponent s of the weight prescale 2^s: it puts the largest weight magnitude amax in [2^12, 2^13), so the lo halves of ordinary weights stay
    clear of fp16's subnormal range; the GEMM epilogue multiplies by alpha = 2^-s (exact).  0 for a zero or non-finite amax."""
    return 0 if amax == 0.0 or not math.isfinite(amax) else 13 - math.frexp(amax)[1]


def activation_scale(amax: float, label: str) -> float:
    """Power-of-two scale sigma of a stored activation tensor whose largest true magnitude is amax: sigma * amax lands in (2^8, 2^9], 2^7 below
    fp16's maximum.  Raises RuntimeError naming `label` when amax is not finite and positive."""
    if not (amax > 0.0 and math.isfinite(amax)):
        raise RuntimeError(f"{label} has amax = {amax} (non-finite weights or an all-zero activation)")
    return 2.0 ** (9 - math.ceil(math.log2(amax)))


class SplitWeight:
    """A Linear weight W (N, K) as the fp16 (hi | lo) pair (N, 2K) of 2^s * W (weight_prescale), plus alpha = 2^-s for the GEMM epilogue."""
    __slots__ = ("pair", "alpha")

    def __init__(self, w: torch.Tensor):
        w = w.detach().float().contiguous()
        s = weight_prescale(float(w.abs().max()))
        self.pair, self.alpha = ops.split_f16(w, 2.0 ** s), 2.0 ** (-s)

    @property
    def shape(self):
        return (self.pair.shape[0], self.pair.shape[1] // 2)


class PackedConv:
    """(N, n_blocks * 2 * Kp) fp16: per K-block j (one spatial tap of a conv, or one of several 1x1 operands), columns [j*2Kp, +Cin) hold the hi
    half and [j*2Kp + Kp, +Cin) the lo half of 2^s * W_j; everything else is zero, so an A box that reads Kp columns where only Cin exist multiplies
    the overhang by zeros.  alpha = 2^-s undoes the scale in the GEMM epilogue."""

    def __init__(self, blocks, bias, fold=False):
        """fold (Cin <= 32, operand rows laid out [hi(32) | lo(32)]): per block two 64-deep k-blocks [Wh | Wh] and [Wl | 0], so that ONE A box
        [hi | lo] yields hi*Wh + lo*Wh and hi*Wl -- the three products of the split-fp16 scheme from one staged copy of the operand."""
        N, Cin = blocks[0].shape
        Kp = k64(Cin)
        self.fold = bool(fold)
        if fold and Cin > 32:
            raise ValueError("folded packing needs Cin <= 32")
        s = weight_prescale(max(float(b.abs().max()) for b in blocks))
        w = torch.zeros(N, len(blocks), 2, Kp, dtype=torch.float16, device=blocks[0].device)
        for j, b in enumerate(blocks):
            pr = ops.split_f16(b.detach().contiguous().float(), 2.0 ** s)  # (N, 2*Cin)
            w[:, j, 0, :Cin] = pr[:, :Cin]
            if fold:
                w[:, j, 0, 32:32 + Cin] = pr[:, :Cin]
            w[:, j, 1, :Cin] = pr[:, Cin:]
        self.w = w.reshape(N, -1).contiguous()
        self.alpha, self.Kp, self.N, self.nblk = 2.0 ** (-s), Kp, N, len(blocks)
        self.bias = bias.detach().float().contiguous()

    def taps(self, spatial):
        """spatial: per K-block (row_shift, a_col_hi, a_col_lo, use_a2) -> the 3-pass tap list of dsb_gemm_ex (lo*hi, hi*lo, hi*hi)."""
        w_cols = [(j * 2 * self.Kp, j * 2 * self.Kp + self.Kp) for j in range(len(spatial))]
        if not self.fold:
            return ops.f16x3_taps(spatial, w_cols)
        out = []
        for (sh, ah, al, a2), (wh, wl) in zip(spatial, w_cols):
            if al != ah + 32:
                raise ValueError("folded packing: the lo half must follow the hi half at +32 columns")
            out += [(sh, ah, wh, a2), (sh, ah, wl, a2)]
        return out

    def taps64(self, spatial):
        """The same products as taps(), cut into 64-deep k-blocks (K = 64 per tap: dsb_gemm_ex's resident_w form); taps that
        read the same A box are adjacent so that the kernel stages it once."""
        out = []
        for sh, ac, wc, a2 in self.taps(spatial):
            out += [(sh, ac + 64 * i, wc + 64 * i, a2) for i in range(self.Kp // 64)]
        if self.Kp > 64:  # regroup: (al_i, wh_i), (ah_i, wl_i), (ah_i, wh_i) per 64-column slice i
            n = self.Kp // 64
            trip = [out[k:k + 3 * n] for k in range(0, len(out), 3 * n)]
            out = [tp[p * n + i] for tp in trip for i in range(n) for p in range(3)]
        return out

    def resident_ok(self, n_taps):
        """Use the 64-deep tap form for n_taps taps?  Narrow layers only: N <= 128 and at most 96 KB of weights (N rounded to 16 rows x 128 bytes per tap)."""
        return self.N <= 128 and n_taps <= 32 and n_taps * ((self.N + 15) // 16 * 16) * 128 <= 96 * 1024

    def launch(self, *, spatial=None, taps=None, alpha=1.0, **act):
        """One dsb_gemm_ex of this conv (ops.gemm_desc) with the activation side `act` given by the caller (A, out, M, strides, flags, bias,
        geometry, ...).  spatial: per K-block (row_shift, a_col_hi, a_col_lo, use_a2); narrow layers (resident_ok) run its 64-deep form taps64 with
        the weights resident in shared memory, the rest its 3-pass form taps.  taps: an explicit list in the 3-pass form instead, used as given.
        The epilogue scale is alpha * self.alpha."""
        resident = False
        if spatial is not None:
            taps = self.taps64(spatial)
            resident = self.resident_ok(len(taps))
            if not resident:
                taps = self.taps(spatial)
        ops.gemm_desc(**act, W=self.w.data_ptr(), N=self.N, K=64 if resident else self.Kp, taps=taps, ldw=self.w.shape[1], w_cols=self.w.shape[1],
                      alpha=self.alpha * alpha, resident_w=int(resident))
