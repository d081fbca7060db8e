"""The host-side rules of the split-fp16 ("f16x3") GEMMs (packing.py, ops.f16x3_taps), checked on CPU: the weight prescale, the calibrated activation
scale, and the tap lists handed to dsb_gemm_ex, which must have the exact form its fused split kernel recognises."""
import math

import pytest
import torch

from tests import cpu_state_gemm_emulation as E

import _pkg

_pkg.load()
from diffsound_b200 import ops, packing  # noqa: E402


@pytest.mark.parametrize("amax,s", [(0.0, 0), (math.inf, 0), (-math.inf, 0), (math.nan, 0), (1.0, 12), (2.0 ** 13, -1), (0.75, 13), (3e-3, 21),
                                    (1e-6, 32), (2.0 ** -140, 152)])
def test_weight_prescale(amax, s):
    """s = 13 - frexp(amax)[1]: 2^s * amax lands in [2^12, 2^13) (an exact power of two at 2^12), also for amax in fp16's and fp32's subnormal
    ranges; no scaling for a zero or non-finite amax."""
    assert packing.weight_prescale(amax) == s
    if amax > 0 and math.isfinite(amax):
        assert 2.0 ** 12 <= 2.0 ** s * amax < 2.0 ** 13


@pytest.mark.parametrize("amax,sigma", [(2.0 ** 9, 1.0), (2.0 ** 8, 2.0), (300.0, 1.0), (257.0, 1.0), (1.0, 2.0 ** 9), (1.5, 2.0 ** 8),
                                        (1e12, 2.0 ** -31), (1e-3, 2.0 ** 18)])
def test_activation_scale(amax, sigma):
    """sigma is the power of two that puts amax in (2^8, 2^9]: an exact 2^9 stays at 2^9, an exact 2^8 moves up to 2^9."""
    assert packing.activation_scale(amax, "site") == sigma
    assert 2.0 ** 8 < sigma * amax <= 2.0 ** 9


@pytest.mark.parametrize("amax", [0.0, -1.0, math.nan, math.inf])
def test_activation_scale_refuses_non_finite_or_non_positive(amax):
    with pytest.raises(RuntimeError, match=r"^launch site \('g1', 0, 1\) has amax = "):
        packing.activation_scale(amax, "launch site ('g1', 0, 1)")


def _fused_split_form(taps, K):
    """dsb_gemm_ex's test for the fused split-fp16 kernel (csrc/gemm_wgmma.cu, the fused3 condition), restated over the tap entries of an fp16,
    unbatched, K-major descriptor with no second A operand: triples of one row shift, (A lo, W hi), (A hi, W lo), (A hi, W hi), with the same
    positive hi -> lo column distances in A and in W throughout, and K a whole number of 64-deep k-blocks."""
    if not taps or len(taps) % 3 or K % 64 or any(t[3] for t in taps):
        return False
    lo_a, lo_w = taps[0][1] - taps[1][1], taps[1][2] - taps[0][2]
    for j in range(0, len(taps), 3):
        (s0, a0, w0, _), (s1, a1, w1, _), (s2, a2, w2, _) = taps[j:j + 3]
        if not (s0 == s1 == s2 and a1 == a2 and a0 - a1 == lo_a and w0 == w2 and w1 - w0 == lo_w):
            return False
    return lo_a > 0 and lo_w > 0


@pytest.mark.parametrize("K", [64, 512, 1024])
def test_gemm_f16x3_emits_the_fused_form(monkeypatch, K):
    seen = {}
    monkeypatch.setattr(ops, "gemm", lambda *a, **kw: seen.update(kw))
    ops.gemm_f16x3(torch.zeros(4, 2 * K, dtype=torch.float16), torch.zeros(8, 2 * K, dtype=torch.float16), out=torch.empty(4, 8))
    taps = list(zip(seen["taps"], seen["tap_acol"], seen["tap_wcol"], [0] * len(seen["taps"])))
    assert seen["dtype"] == ops.F16 and seen["k_per_tap"] == K
    assert _fused_split_form(taps, K)


@pytest.mark.parametrize("n_spatial", [1, 3, 7, 9])
@pytest.mark.parametrize("cin", [20, 64, 96, 192])
def test_packed_conv_tap_lists_emit_the_fused_form(monkeypatch, n_spatial, cin):
    """PackedConv.taps (K = Kp) and taps64 (K = 64) for an unfolded conv, with the A column layouts of the decoder ([hi | lo] at +Cin), the vocoder
    state rows (act columns at +2C / +3C) and a phase image (per-tap column offsets).  The folded form (two entries per tap) takes the plain tap
    loop on purpose and is not checked here."""
    monkeypatch.setattr(ops, "split_f16", E.split_f16)
    g = torch.Generator().manual_seed(cin)
    cv = packing.PackedConv([torch.randn(16, cin, generator=g) for _ in range(n_spatial)], torch.zeros(16))
    layouts = [[(j - n_spatial // 2, 0, cin, 0) for j in range(n_spatial)],
               [(9 + 3 * (j - 1), 2 * cin, 3 * cin, 0) for j in range(n_spatial)],
               [(j // 2, (j % 4) * cin, 4 * cin + (j % 4) * cin, 0) for j in range(n_spatial)]]
    for spatial in layouts:
        assert _fused_split_form(cv.taps(spatial), cv.Kp)
        assert _fused_split_form(cv.taps64(spatial), 64)
