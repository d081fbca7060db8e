"""ctypes binding of libdiffsound_b200.so (the C-ABI in include/diffsound_b200.h).

There is deliberately NO fallback: if the shared library is missing or a call fails, a RuntimeError is raised.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libdiffsound_b200.so")

c_vp, c_i, c_ll, c_f = C.c_void_p, C.c_int, C.c_longlong, C.c_float


class GemmDesc(C.Structure):
    """Mirror of `struct dsb_gemm_desc` (include/diffsound_b200.h)."""
    _fields_ = [
        ("A", c_vp), ("W", c_vp), ("bias", c_vp), ("residual", c_vp), ("out", c_vp),
        ("M", c_i), ("N", c_i), ("K", c_i), ("batch", c_i),
        ("a_rows", c_ll), ("lda", c_ll), ("ldw", c_ll), ("ldo", c_ll), ("ld_res", c_ll),
        ("a_batch_stride", c_ll), ("w_batch_stride", c_ll), ("out_batch_stride", c_ll), ("res_batch_stride", c_ll),
        ("dtype", c_i), ("flags", c_i), ("num_taps", c_i), ("tap_shift", c_i * 32), ("tap_acol", c_i * 32), ("a_cols", c_ll),
        ("geo_P", c_i), ("geo_Wp", c_i), ("geo_y0", c_i), ("geo_y1", c_i), ("geo_x0", c_i), ("geo_x1", c_i),
        ("alpha", c_f), ("block_n", c_i), ("max_ctas", c_i), ("cta_pair", c_i), ("a_mn_major", c_i), ("b_mn_major", c_i),
        ("use_tap_wcol", c_i), ("tap_wcol", c_i * 32), ("w_cols", c_ll), ("split_off", c_ll),
        ("dual_off", c_ll), ("out_col_group", c_i), ("out_col_group_stride", c_i), ("A2", c_vp),
        ("a2_rows", c_ll), ("a2_cols", c_ll), ("lda2", c_ll), ("a2_batch_stride", c_ll), ("tap_a2", c_i * 32), ("amax_out", c_vp), ("resident_w", c_i),
        ("schedule", c_i),
    ]


# name -> (argtypes) ; every function returns int status except the two noted
SIGNATURES = {
    "dsb_version": [],
    "dsb_device_info": [C.POINTER(c_i)] * 3,
    "dsb_gemm_ex": [C.POINTER(GemmDesc), c_vp],
    "dsb_gemm_f32": [c_vp] * 5 + [c_i] * 3 + [c_ll] * 4 + [c_i, c_vp],
    "dsb_round_tf32": [c_vp, c_vp, c_ll, c_vp],
    "dsb_f32_to_bf16": [c_vp, c_vp, c_ll, c_vp],
    "dsb_f32_to_f16": [c_vp, c_vp, c_ll, c_vp],
    "dsb_silu": [c_vp, c_vp, c_ll, c_vp],
    "dsb_split_f16": [c_vp, c_ll, c_vp, c_ll, c_ll, c_ll, c_i, c_f, c_vp],
    "dsb_attention_tc_split": [c_vp, c_ll, c_ll, c_vp, c_ll, c_ll, c_vp, c_ll, c_ll, c_vp, c_ll, c_ll, c_i, c_i, c_i, c_i, c_f, c_vp],
    "dsb_attention_tc_split_hd32": [c_vp, c_ll, c_ll, c_vp, c_ll, c_ll, c_vp, c_ll, c_ll, c_vp, c_ll, c_ll, c_i, c_i, c_i, c_i, c_f, c_vp],
    "dsb_attention_tc_split_causal": [c_vp, c_ll, c_ll, c_vp, c_ll, c_ll, c_vp, c_ll, c_ll, c_vp, c_ll, c_ll, c_i, c_i, c_i, c_i, c_f, c_i, c_vp],
    "dsb_l2_normalize_rows": [c_vp, c_ll, c_i, c_vp],
    "dsb_split_tf32": [c_vp, c_ll, c_vp, c_ll, c_ll, c_i, c_i, c_i, c_vp],
    "dsb_embed_tokens": [c_vp] * 5 + [c_i] * 6 + [c_vp, c_vp],
    "dsb_layernorm": [c_vp] * 4 + [c_i, c_i, c_f, c_i, c_vp],
    "dsb_ada_layernorm": [c_vp] * 4 + [c_i] * 4 + [c_f, c_i, c_vp],
    "dsb_attention": [c_vp, c_ll, c_vp, c_ll, c_vp, c_ll, c_vp, c_ll, c_i, c_i, c_i, c_i, c_f, c_i, c_vp],
    "dsb_attention_hd32": [c_vp, c_ll, c_vp, c_ll, c_vp, c_ll, c_vp, c_ll, c_i, c_i, c_i, c_i, c_f, c_i, c_vp],
    "dsb_codebook_gather_padded": [c_vp] * 3 + [c_i] * 6 + [c_vp, c_vp],
    "dsb_groupnorm_stats": [c_vp, c_vp] + [c_i] * 4 + [c_vp],
    "dsb_groupnorm_apply": [c_vp] * 5 + [c_i] * 5 + [c_f, c_i, c_i, c_vp],
    "dsb_upsample2x_padded": [c_vp, c_vp] + [c_i] * 5 + [c_vp],
    "dsb_softmax_rows": [c_vp, c_ll, c_i, c_i, c_i, c_vp],
    "dsb_space_to_depth_padded": [c_vp, c_vp] + [c_i] * 5 + [c_vp],
    "dsb_row_argmin": [c_vp, c_ll, c_ll, c_i, c_vp, c_vp],
    "dsb_tokens_add_to_padded": [c_vp, c_vp] + [c_i] * 5 + [c_vp],
    "dsb_lrelu_pad": [c_vp, c_vp] + [c_i] * 4 + [c_f, c_i, c_i, c_i, c_vp],
    "dsb_mel_pack_f16": [c_vp, c_vp] + [c_i] * 5 + [c_vp],
    "dsb_edge_pad_f16": [c_vp, c_ll, c_ll] + [c_i] * 7 + [c_vp],
    "dsb_conv_out_pair": [c_vp, c_ll, c_ll] + [c_i] * 6 + [c_vp, c_vp, c_f, c_vp, c_vp],
    "dsb_attention_f16": [c_vp, c_ll, c_vp, c_ll, c_vp, c_ll, c_vp, c_ll, c_i, c_i, c_i, c_i, c_f, c_i, c_vp],
    "dsb_attention_tc2": [c_vp, c_ll, c_vp, c_ll, c_vp, c_ll, c_vp, c_ll, c_i, c_i, c_i, c_i, c_f, c_vp],
    "dsb_attention_tc": [c_vp, c_ll, c_vp, c_ll, c_vp, c_ll, c_vp, c_ll, c_i, c_i, c_i, c_i, c_f, c_vp],
    "dsb_posterior_sample": [c_vp] * 8 + [c_i] * 5 + [c_f, c_i, c_i, c_vp],
    "dsb_posterior_sample_loop": [c_vp] * 8 + [c_i] * 5 + [c_f, c_i, c_vp],
    "dsb_posterior_sample_wide": [c_vp] * 8 + [c_i] * 5 + [c_f, c_i, c_i, c_vp],
    "dsb_posterior_sample_wide_loop": [c_vp] * 8 + [c_i] * 5 + [c_f, c_i, c_vp],
    "dsb_aten_uniform": [c_vp, c_ll, C.c_ulonglong, C.c_ulonglong, C.c_ulonglong, c_vp],
    "dsb_aten_exponential": [c_vp, c_ll, C.c_ulonglong, C.c_ulonglong, C.c_ulonglong, c_vp],
    # autoregressive transformer decode
    "dsb_ar_embed": [c_vp] * 4 + [c_ll, c_vp, c_vp] + [c_i] * 4 + [c_vp, c_vp],
    "dsb_ar_attention": [c_vp, c_ll, c_vp, c_vp, c_ll, c_i, c_vp, c_ll, c_ll, c_vp, c_i, c_i, c_i, c_f, c_vp],
    "dsb_ar_embed_all": [c_vp] * 4 + [c_ll, c_vp] + [c_i] * 5 + [c_vp, c_vp],
    "dsb_ar_cross_entropy": [c_vp, c_ll, c_i, c_i, c_i, c_vp, c_ll, c_vp, c_vp, c_i, c_i, c_vp, c_vp],
    "dsb_gelu_erf_split": [c_vp, c_ll, c_vp, c_ll, c_ll, c_i, c_i, c_vp],
    "dsb_ar_sample": [c_vp, c_ll, c_vp, c_ll, c_vp, c_i, c_i, c_i, c_f, c_i, c_i, c_vp, c_vp, c_ll, c_vp, c_vp],
    # Melception feature extractor
    "dsb_mel_stem": [c_vp] * 5 + [c_f, c_vp] + [c_i] * 8 + [c_vp],
    "dsb_pair_space_to_depth": [c_vp] + [c_i] * 6 + [c_vp] + [c_i] * 6 + [c_vp],
    "dsb_pair_maxpool3s2": [c_vp] + [c_i] * 6 + [c_vp, c_ll, c_ll] + [c_i] * 6 + [c_f, c_vp],
    "dsb_pair_avgpool3": [c_vp] + [c_i] * 6 + [c_vp, c_ll, c_ll, c_i, c_i, c_vp],
    "dsb_pair_channel_mean": [c_vp, c_ll, c_ll] + [c_i] * 8 + [c_f, c_vp, c_vp],
    # SpecVQGAN log-mel spectrogram
    "dsb_wav_frames_f16": [c_vp, c_ll, c_i, c_i, c_vp, c_i, c_vp, c_vp],
    "dsb_mel_log": [c_vp, c_ll, c_ll] + [c_i] * 4 + [c_vp] * 3 + [c_i, c_i, c_vp, c_vp],
    # training (A13)
    "dsb_q_sample": [c_vp] * 5 + [c_i] * 4 + [c_vp],
    "dsb_train_loss": [c_vp] * 16 + [c_i] * 4 + [c_f, c_i, c_f, c_f, c_i, c_vp],
    "dsb_transpose": [c_vp, c_ll, c_ll, c_vp, c_ll, c_ll, c_i, c_i, c_i, c_i, c_vp],
    "dsb_heads_split": [c_vp, c_ll, c_vp, c_i, c_i, c_i, c_i, c_vp],
    "dsb_heads_merge": [c_vp, c_vp, c_ll, c_i, c_i, c_i, c_i, c_vp],
    "dsb_cast_scale": [c_vp, c_vp, c_ll, c_vp, c_i, c_vp],
    "dsb_colsum": [c_vp, c_ll, c_vp, c_ll, c_i, c_i, c_vp],
    "dsb_gelu2_fwd": [c_vp, c_vp, c_ll, c_i, c_vp],
    "dsb_gelu2_bwd": [c_vp, c_vp, c_vp, c_ll, c_i, c_vp],
    "dsb_silu_bwd": [c_vp, c_vp, c_vp, c_ll, c_vp],
    "dsb_gather_rows": [c_vp, c_vp, c_vp, c_i, c_i, c_vp],
    "dsb_scatter_add_rows": [c_vp, c_vp, c_vp, c_i, c_i, c_vp],
    "dsb_layernorm_bwd": [c_vp] * 6 + [c_ll, c_i, c_f, c_vp, c_i, c_vp],
    "dsb_ada_layernorm_bwd": [c_vp] * 6 + [c_i, c_i, c_i, c_f, c_vp, c_i, c_vp],
    "dsb_softmax_fwd": [c_vp, c_ll, c_vp, c_ll, c_ll, c_i, c_i, c_vp],
    "dsb_softmax_bwd": [c_vp, c_ll, c_vp, c_ll, c_vp, c_ll, c_ll, c_i, c_f, c_i, c_vp],
    "dsb_embed_bwd": [c_vp] * 5 + [c_i] * 6 + [c_vp],
    "dsb_attention_train_fwd": [c_vp, c_ll, c_vp, c_ll, c_vp, c_ll, c_vp, c_ll, c_vp, c_i, c_i, c_i, c_i, c_f, c_vp],
    "dsb_attention_train_bwd": [c_vp, c_ll] * 5 + [c_vp, c_vp] + [c_vp, c_ll] * 3 + [c_i, c_i, c_i, c_i, c_f, c_vp],
}

_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                               "(there is no CPU / PyTorch fallback for the Diffsound hot path)")
        L = C.CDLL(LIB_PATH)
        for name, args in SIGNATURES.items():
            fn = getattr(L, name)  # AttributeError if the library does not export a declared symbol
            fn.argtypes = args
            fn.restype = c_i
        L.dsb_last_error.argtypes = []
        L.dsb_last_error.restype = C.c_char_p
        _lib = L
    return _lib


def check(status: int, what: str) -> None:
    if status != 0:
        raise RuntimeError(f"{what} failed ({status}): {lib().dsb_last_error().decode()}")
