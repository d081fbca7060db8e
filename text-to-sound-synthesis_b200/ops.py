"""torch-tensor front end of the C-ABI kernels: pointer extraction, shape checks, current-stream plumbing.

PyTorch is used here only for device memory and streams; all arithmetic happens in libdiffsound_b200.so.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Sequence

import torch

from . import _lib

TF32, BF16, F16 = 0, 1, 2
GELU2, ROUND_TF32, OUT_BF16, LRELU, TANH, GN_SWISH, GN_COMPACT, RES_BEFORE_ACT, OUT_F16, SPLIT_OUT = 1, 2, 4, 8, 16, 32, 64, 128, 256, 512
OUT_F16_SPLIT = 2048
DUAL_LRELU = 4096
SPLIT_OUT_F16 = 8192
NO_STORE = 16384
RELU = 32768


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _ptr(t: Optional[torch.Tensor]):
    return None if t is None else t.data_ptr()


def _need_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise RuntimeError("diffsound_b200 ops need CUDA tensors: this path has no CPU fallback")


def device_info():
    s, a, b = C.c_int(), C.c_int(), C.c_int()
    _lib.check(_lib.lib().dsb_device_info(C.byref(s), C.byref(a), C.byref(b)), "dsb_device_info")
    return s.value, a.value, b.value


def round_tf32(x: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    _need_cuda(x)
    x = x.contiguous()
    out = torch.empty_like(x) if out is None else out
    _lib.check(_lib.lib().dsb_round_tf32(x.data_ptr(), out.data_ptr(), x.numel(), _stream()), "dsb_round_tf32")
    return out


def to_bf16(x: torch.Tensor) -> torch.Tensor:
    _need_cuda(x)
    x = x.contiguous()
    out = torch.empty(x.shape, dtype=torch.bfloat16, device=x.device)
    _lib.check(_lib.lib().dsb_f32_to_bf16(x.data_ptr(), out.data_ptr(), x.numel(), _stream()), "dsb_f32_to_bf16")
    return out


def to_f16(x: torch.Tensor) -> torch.Tensor:
    _need_cuda(x)
    x = x.contiguous()
    out = torch.empty(x.shape, dtype=torch.float16, device=x.device)
    _lib.check(_lib.lib().dsb_f32_to_f16(x.data_ptr(), out.data_ptr(), x.numel(), _stream()), "dsb_f32_to_f16")
    return out


def split_tf32(x: torch.Tensor, w_format: bool = False) -> torch.Tensor:
    """(..., C) fp32 -> (..., 2*Cp) [hi | lo] split-TF32 A operand (or (..., 3*Cp) [hi | hi | lo] W operand), Cp = C rounded up to 32."""
    _need_cuda(x)
    C = x.shape[-1]
    Cp = (C + 31) // 32 * 32
    x2 = x.reshape(-1, C) if x.is_contiguous() else x
    if x2.dim() != 2:
        raise RuntimeError("split_tf32 needs a contiguous tensor or a 2-D row-strided view")
    nb = 3 if w_format else 2
    out = torch.empty(*x.shape[:-1], nb * Cp, dtype=torch.float32, device=x.device)
    _lib.check(_lib.lib().dsb_split_tf32(x2.data_ptr(), x2.stride(0), out.data_ptr(), nb * Cp, x2.shape[0], C, Cp, 1 if w_format else 0, _stream()),
               "dsb_split_tf32")
    return out


def pack_split_weight(w: torch.Tensor, ntaps: int) -> torch.Tensor:
    """(N, ntaps*C) fp32 tap-major weight -> (N, 3*ntaps*Cp): per tap [Whi | Whi | Wlo] (pairs with gemm_split's tap list)."""
    N = w.shape[0]
    C = w.shape[1] // ntaps
    Cp = (C + 31) // 32 * 32
    w3 = w.reshape(N, ntaps, C).float()
    hi = round_tf32(w3.contiguous())
    lo = round_tf32((w3 - hi).contiguous())
    out = torch.zeros(N, ntaps, 3, Cp, dtype=torch.float32, device=w.device)
    out[:, :, 0, :C] = hi
    out[:, :, 1, :C] = hi
    out[:, :, 2, :C] = lo
    return out.reshape(N, ntaps * 3 * Cp).contiguous()


def gemm_split(a_split: torch.Tensor, w_split: torch.Tensor, bias=None, residual=None, out=None, *, taps=None, **kw) -> torch.Tensor:
    """3xTF32 GEMM: a_split from split_tf32 (.., 2*Cp), w_split from pack_split_weight; same epilogue options as gemm()."""
    Cp = a_split.shape[-1] // 2
    taps = list(taps) if taps is not None else [0]
    t3, ac = [], []
    for s_ in taps:
        t3 += [s_, s_, s_]
        ac += [0, Cp, 0]  # hi*Whi, lo*Whi, hi*Wlo
    return gemm(a_split, w_split, bias, residual, out, dtype=TF32, taps=t3, tap_acol=ac, k_per_tap=Cp, **kw)


def split_f16(x: torch.Tensor, scale: float = 1.0, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """(rows, C) fp32 -> (rows, 2C) fp16 [hi | lo] with hi = f16(scale*x), lo = f16(scale*x - hi): one operand of a split-fp16 ("f16x3") GEMM."""
    _need_cuda(x)
    if x.dim() != 2 or x.stride(1) != 1:
        raise RuntimeError("split_f16 needs a 2-D tensor contiguous in its last dimension")
    rows, Cc = x.shape
    if out is None:
        out = torch.empty(rows, 2 * Cc, dtype=torch.float16, device=x.device)
    _lib.check(_lib.lib().dsb_split_f16(x.data_ptr(), x.stride(0), out.data_ptr(), out.stride(0), Cc, rows, Cc, float(scale), _stream()), "dsb_split_f16")
    return out


def gemm_f16x3(a_pair: torch.Tensor, w_pair: torch.Tensor, bias=None, residual=None, out=None, *, alpha: float = 1.0, gelu: bool = False,
               split_out: bool = False, **kw) -> torch.Tensor:
    """Split-fp16 GEMM at fp32-class accuracy on the fp16 tensor cores: a_pair (M, 2K) [Ahi | Alo], w_pair (N, 2K) [Whi | Wlo] (both from split_f16 or a
    split_out producer); out = epi(alpha * (Alo Whi^T + Ahi Wlo^T + Ahi Whi^T) + bias) (+ residual), fp32 accumulation over all three passes.
    split_out: write the result as an fp16 (hi | lo) pair (M, 2N) for the next split GEMM / attention instead of fp32."""
    K = a_pair.shape[-1] // 2
    if w_pair.shape[-1] != 2 * K:
        raise RuntimeError(f"gemm_f16x3: W pair has {w_pair.shape[-1]} columns, expected {2 * K}")
    N = w_pair.shape[0]
    M = a_pair.shape[0]
    if out is None:
        out = torch.empty(M, 2 * N, dtype=torch.float16, device=a_pair.device) if split_out else torch.empty(M, N, dtype=torch.float32, device=a_pair.device)
    shifts, acols, wcols, _ = zip(*f16x3_taps([(0, 0, K, 0)], [(0, K)]))
    return gemm(a_pair, w_pair, bias, residual, out, dtype=F16, taps=shifts, tap_acol=acols, tap_wcol=wcols, k_per_tap=K, alpha=alpha,
                gelu=gelu, split_out=split_out, **kw)


def f16x3_taps(spatial, w_cols):
    """The split-fp16 tap list: per K-block j, spatial[j] = (row_shift, A hi column, A lo column, use_a2) and w_cols[j] = (W hi column, W lo column)
    -> the triple (A lo . W hi), (A hi . W lo), (A hi . W hi) as (row_shift, a_col, w_col, use_a2) entries.  dsb_gemm_ex recognises exactly this
    form (same shift within a triple, constant hi -> lo distances) and runs the three products off one staged copy of the operands with a per-k-block
    fp32 promotion; any other list takes the plain tap loop, which is slower and rounds differently."""
    out = []
    for (sh, ah, al, a2), (wh, wl) in zip(spatial, w_cols):
        out += [(sh, al, wh, a2), (sh, ah, wl, a2), (sh, ah, wh, a2)]
    return out


def silu(x: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    _need_cuda(x, out)
    x = x.contiguous()
    out = torch.empty_like(x) if out is None else out
    _lib.check(_lib.lib().dsb_silu(x.data_ptr(), out.data_ptr(), x.numel(), _stream()), "dsb_silu")
    return out


def gemm(a: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None, residual: Optional[torch.Tensor] = None,
         out: Optional[torch.Tensor] = None, *, dtype: int = TF32, gelu: bool = False, round_out: bool = False, out_bf16: bool = False, out_f16: bool = False,
         lrelu: bool = False, tanh: bool = False, relu: bool = False, res_before_act: bool = False, taps: Optional[Sequence[int]] = None,
         tap_acol: Optional[Sequence[int]] = None, k_per_tap: Optional[int] = None, out_rows: Optional[int] = None, geo: Optional[Sequence[int]] = None, alpha: float = 1.0,
         block_n: int = 0, max_ctas: int = 0, cta_pair: int = 0, a_mn: bool = False, w_mn: bool = False,
         tap_wcol: Optional[Sequence[int]] = None, split_out: bool = False, schedule: int = 0) -> torch.Tensor:
    """out = epi(alpha * A @ W^T + bias) (+ residual) on the tensor cores (wgmma).  a: (M,K) or (batch,M,K); w: (N, taps*K) or (batch,N,K).
    a_mn / w_mn: that operand is given MN-major, i.e. as it lies in memory with the reduction dimension as rows -- a: (K, M), w: (K, N)
    (2-byte dtypes): out = a^T @ w with no transposed copies.
    schedule: 0 = auto (ordered stream-K when the tiles leave a partial last wave), 1 = data-parallel only; the output bits are the same."""
    _need_cuda(a, w, bias, residual, out)
    batched = a.dim() == 3
    if a.stride(-1) != 1 or w.stride(-1) != 1:
        raise RuntimeError("gemm operands must be contiguous in their last dimension")
    ntaps = 1 if taps is None else len(taps)
    batch = a.shape[0] if batched else 1
    a_rows, a_cols = (a.shape[-1], a.shape[-2]) if a_mn else (a.shape[-2], a.shape[-1])  # (M, K)
    K = a_cols if k_per_tap is None else k_per_tap  # reduction length per tap (A may hold several K blocks side by side)
    N = w.shape[-1] if w_mn else w.shape[-2]
    if tap_wcol is None and (w.shape[-2] if w_mn else w.shape[-1]) != K * ntaps:
        raise RuntimeError(f"gemm: W has reduction length {w.shape[-2] if w_mn else w.shape[-1]}, expected {K}*{ntaps}")
    M = a_rows if out_rows is None else out_rows
    odt = torch.bfloat16 if out_bf16 else (torch.float16 if out_f16 else torch.float32)
    if out is None:
        out = torch.empty((batch, M, N) if batched else (M, N), dtype=odt, device=a.device)
    out_f16 = out.dtype == torch.float16 and not split_out
    out_bf16 = out.dtype == torch.bfloat16
    if split_out and (out.dtype != torch.float16 or batched):
        raise RuntimeError("gemm: split_out writes an fp16 (hi | lo) pair and is not batched")
    flags = (GELU2 if gelu else 0) | (ROUND_TF32 if round_out else 0) | (OUT_BF16 if out_bf16 else 0) | (LRELU if lrelu else 0) | (TANH if tanh else 0) | (RELU if relu else 0) | (RES_BEFORE_ACT if res_before_act else 0) | (OUT_F16 if out_f16 else 0) | (OUT_F16_SPLIT if split_out else 0)
    shifts = taps or [0]
    _gemm_ex([(s, tap_acol[i] if tap_acol is not None else 0, tap_wcol[i] if tap_wcol is not None else 0, 0) for i, s in enumerate(shifts)],
             geo, use_tap_wcol=int(tap_wcol is not None), num_taps=ntaps,
             A=a.data_ptr(), W=w.data_ptr(), bias=_ptr(bias), residual=_ptr(residual), out=out.data_ptr(), M=M, N=N, K=K, batch=batch,
             a_rows=a_rows, a_cols=a_cols, lda=a.stride(-2), ldw=w.stride(-2), ldo=out.stride(-2), ld_res=residual.stride(-2) if residual is not None else 0,
             a_batch_stride=a.stride(0) if batched else 0, w_batch_stride=w.stride(0) if w.dim() == 3 else 0,
             out_batch_stride=out.stride(0) if batched else 0, res_batch_stride=residual.stride(0) if (residual is not None and batched) else 0,
             dtype=dtype, flags=flags, split_off=N if split_out else 0, w_cols=w.shape[-1] if tap_wcol is not None else 0, alpha=alpha,
             block_n=block_n, max_ctas=max_ctas, cta_pair=cta_pair, a_mn_major=int(a_mn), b_mn_major=int(w_mn), schedule=schedule)
    return out


def gemm_desc(*, A, W, out, M, N, K, taps, lda, ldw, ldo, dtype=F16, batch=1, a_rows=0, a_cols=0, a_batch_stride=0, w_cols=0, out_batch_stride=0,
              bias=None, flags=0, alpha=1.0, split_off=0, dual_off=0, out_col_group=0, out_col_group_stride=0, A2=None, lda2=0, a2_rows=0, a2_cols=0,
              a2_batch_stride=0, block_n=0, cta_pair=0, residual=None, ld_res=0, geo=None, amax_out=None, resident_w=0,
              schedule=0):
    """Thin front end of dsb_gemm_ex for callers that lay out their own buffers (the MelGAN / SpecVQGAN state buffers): A / W / out / A2 are
    raw device addresses (ints: tensor.data_ptr() plus a byte offset), sizes and strides in elements; taps = [(row_shift, a_col, w_col, use_a2), ...]."""
    _gemm_ex(taps, geo, use_tap_wcol=1, num_taps=len(taps), A=A, W=W, out=out, bias=_ptr(bias), A2=A2, M=M, N=N, K=K, batch=batch,
             a_rows=a_rows, a_cols=a_cols, lda=lda, ldw=ldw, ldo=ldo, a_batch_stride=a_batch_stride, out_batch_stride=out_batch_stride,
             dtype=dtype, flags=flags, alpha=alpha, w_cols=w_cols, split_off=split_off, dual_off=dual_off, out_col_group=out_col_group,
             out_col_group_stride=out_col_group_stride, lda2=lda2, a2_rows=a2_rows, a2_cols=a2_cols, a2_batch_stride=a2_batch_stride,
             block_n=block_n, cta_pair=cta_pair, residual=residual, ld_res=ld_res, amax_out=_ptr(amax_out), resident_w=int(resident_w),
             schedule=schedule)


_DESC_FIELDS = frozenset(name for name, _ in _lib.GemmDesc._fields_)


def _gemm_ex(taps, geo, **fields):
    """Fill one GemmDesc and launch dsb_gemm_ex: `fields` are GemmDesc members by name (pointers as ints or None), taps = [(row_shift, a_col,
    w_col, use_a2), ...], geo = (P, Wp, y0, y1, x0, x1) or None; every member not given stays zero."""
    d = _lib.GemmDesc()
    for name, v in fields.items():
        if name not in _DESC_FIELDS:  # a ctypes Structure would silently keep a misspelt name as a plain attribute
            raise TypeError(f"GemmDesc has no member {name!r}")
        setattr(d, name, v)
    for i, (sh, ac, wc, a2) in enumerate(taps):
        d.tap_shift[i], d.tap_acol[i], d.tap_wcol[i], d.tap_a2[i] = int(sh), int(ac), int(wc), int(a2)
    if geo is not None:
        d.geo_P, d.geo_Wp, d.geo_y0, d.geo_y1, d.geo_x0, d.geo_x1 = [int(v) for v in geo]
    _lib.check(_lib.lib().dsb_gemm_ex(C.byref(d), _stream()), "dsb_gemm_ex")


def mel_pack_f16(mel, pad, Kp):
    """mel (B, Cm, T) fp32 -> (B, T + 2 pad, 2 Kp) fp16 (hi | lo), reflection-padded in time."""
    _need_cuda(mel)
    B, Cm, T = mel.shape
    out = torch.empty(B, T + 2 * pad, 2 * Kp, dtype=torch.float16, device=mel.device)
    _lib.check(_lib.lib().dsb_mel_pack_f16(mel.data_ptr(), out.data_ptr(), B, Cm, T, pad, Kp, _stream()), "dsb_mel_pack_f16")
    return out


def edge_pad_f16(state, T, P, d, col0, ncols, reflect=True):
    """state (B, T + 2P, ld) fp16: fill pad rows P-j / P+T-1+j (j = 1..d) of columns [col0, col0+ncols) by reflection (or zeros)."""
    _need_cuda(state)
    B, Tp, ld = state.shape
    _lib.check(_lib.lib().dsb_edge_pad_f16(state.data_ptr(), ld, Tp * ld, B, T, P, d, col0, ncols, 1 if reflect else 0, _stream()), "dsb_edge_pad_f16")


def conv_out_pair(state, T, row0, col0, w, bias, scale, out=None):
    """state (B, rows, ld) fp16 with the activated (hi | lo) pair at columns [col0, col0 + 2 cs); w (kt, cs) fp32 -> tanh(scale * conv + bias) (B, T) fp32."""
    _need_cuda(state, w, bias)
    B, rows, ld = state.shape
    kt, cs = w.shape
    out = torch.empty(B, T, dtype=torch.float32, device=state.device) if out is None else out
    _lib.check(_lib.lib().dsb_conv_out_pair(state.data_ptr(), ld, rows * ld, B, T, row0, col0, cs, kt, w.data_ptr(), _ptr(bias), float(scale), out.data_ptr(),
                                            _stream()), "dsb_conv_out_pair")
    return out


def gemm_f32(a, w, bias=None, residual=None, out=None, *, gelu=False, round_out=False):
    """Exact fp32 FFMA GEMM (set-up tables, fp32-exact mode)."""
    _need_cuda(a, w, bias, residual, out)
    M, K = a.shape
    N = w.shape[0]
    out = torch.empty((M, N), dtype=torch.float32, device=a.device) if out is None else out
    flags = (GELU2 if gelu else 0) | (ROUND_TF32 if round_out else 0)
    _lib.check(_lib.lib().dsb_gemm_f32(a.data_ptr(), w.data_ptr(), _ptr(bias), _ptr(residual), out.data_ptr(), M, N, K, a.stride(0), w.stride(0),
                                       out.stride(0), residual.stride(0) if residual is not None else 0, flags, _stream()), "dsb_gemm_f32")
    return out


def embed_tokens(ids, emb, height_emb, width_emb, out=None, err_flag=None):
    _need_cuda(ids, emb, height_emb, width_emb)
    B, L = ids.shape
    D = emb.shape[1]
    H, W = height_emb.shape[0], width_emb.shape[0]
    out = torch.empty((B, L, D), dtype=torch.float32, device=ids.device) if out is None else out
    _lib.check(_lib.lib().dsb_embed_tokens(ids.data_ptr(), emb.data_ptr(), height_emb.data_ptr(), width_emb.data_ptr(), out.data_ptr(), B, L, D, H, W,
                                           emb.shape[0], _ptr(err_flag), _stream()), "dsb_embed_tokens")
    return out


def _out_flags(out, round_out, split=False):
    if split:
        return OUT_F16_SPLIT
    if out.dtype == torch.float16:
        return OUT_F16
    if out.dtype == torch.bfloat16:
        return OUT_BF16
    return ROUND_TF32 if round_out else 0


def layernorm(x, gamma, beta, out=None, *, eps=1e-5, round_out=False, out_bf16=False, split=False):
    """split: out is the fp16 (hi | lo) pair (..., 2D) of the fp32 result (the A operand of gemm_f16x3)."""
    _need_cuda(x, gamma, beta)
    D = x.shape[-1]
    rows = x.numel() // D
    if out is None:
        out = torch.empty(*x.shape[:-1], 2 * D, dtype=torch.float16, device=x.device) if split else \
            torch.empty(x.shape, dtype=torch.bfloat16 if out_bf16 else torch.float32, device=x.device)
    if split and (out.dtype != torch.float16 or out.shape[-1] != 2 * D):
        raise RuntimeError("layernorm(split=True) writes an fp16 (..., 2D) tensor")
    flags = _out_flags(out, round_out, split)
    _lib.check(_lib.lib().dsb_layernorm(x.data_ptr(), out.data_ptr(), gamma.data_ptr(), beta.data_ptr(), rows, D, eps, flags, _stream()), "dsb_layernorm")
    return out


def ada_layernorm(x, table, t, out=None, *, eps=1e-5, round_out=False, out_bf16=False, split=False):
    """x (B,L,D), table (T,2D) = Linear(SiLU(emb)) rows, t (B,) int64.  split: as layernorm()."""
    _need_cuda(x, table, t)
    B, L, D = x.shape
    if out is None:
        out = torch.empty(B, L, 2 * D, dtype=torch.float16, device=x.device) if split else \
            torch.empty(x.shape, dtype=torch.bfloat16 if out_bf16 else torch.float32, device=x.device)
    if split and (out.dtype != torch.float16 or out.shape[-1] != 2 * D):
        raise RuntimeError("ada_layernorm(split=True) writes an fp16 (..., 2D) tensor")
    flags = _out_flags(out, round_out, split)
    _lib.check(_lib.lib().dsb_ada_layernorm(x.data_ptr(), out.data_ptr(), table.data_ptr(), t.data_ptr(), B, L, D, table.shape[0], eps, flags, _stream()),
               "dsb_ada_layernorm")
    return out


def l2_normalize_rows_(x):
    """x (..., D) contiguous fp32: every row divided by its L2 norm, in place."""
    _need_cuda(x)
    D = x.shape[-1]
    _lib.check(_lib.lib().dsb_l2_normalize_rows(x.data_ptr(), x.numel() // D, D, _stream()), "dsb_l2_normalize_rows")
    return x


ATTN_CAUSAL = 1024


def _attention_head_dim(name, head_dim):
    if head_dim not in (32, 64):
        raise ValueError(f"{name}: head_dim {head_dim} unsupported (32 or 64)")


def attention(q, k, v, out, *, B, H, Lq, Lk, scale, round_out=False, causal=False, head_dim=64):
    """q/out: row-strided views with (B*Lq) rows; k/v: (B*Lk) rows; head h = columns [head_dim*h, head_dim*(h+1)), head_dim 64 or 32 (fp32
    operands only at 32).  causal (fp16 path): key j visible to query i iff j <= i."""
    _attention_head_dim("attention", head_dim)
    _need_cuda(q, k, v, out)
    for t_ in (q, k, v, out):
        if t_.stride(-1) != 1:
            raise RuntimeError("attention operands must be contiguous in the head dimension")
    if q.dtype == torch.float16:
        if k.dtype != torch.float16 or v.dtype != torch.float16:
            raise RuntimeError("attention: q, k, v must share a dtype")
        if head_dim != 64:
            raise RuntimeError(f"attention: fp16 operands need head_dim 64 (got {head_dim})")
        _lib.check(_lib.lib().dsb_attention_f16(q.data_ptr(), q.stride(0), k.data_ptr(), k.stride(0), v.data_ptr(), v.stride(0), out.data_ptr(),
                                                out.stride(0), B, H, Lq, Lk, scale, _out_flags(out, False) | (ATTN_CAUSAL if causal else 0), _stream()),
                   "dsb_attention_f16")
        return out
    if causal:
        raise RuntimeError("causal attention is implemented for fp16 operands")
    name = "dsb_attention" if head_dim == 64 else "dsb_attention_hd32"
    _lib.check(getattr(_lib.lib(), name)(q.data_ptr(), q.stride(0), k.data_ptr(), k.stride(0), v.data_ptr(), v.stride(0), out.data_ptr(), out.stride(0),
                                         B, H, Lq, Lk, scale, _out_flags(out, round_out), _stream()), name)
    return out


STAGE_INPUT_LOGPROB, STAGE_SKIP_POSTERIOR, STAGE_SKIP_SAMPLE = 1, 2, 4


def attention_tc(q, k, v, out, *, B, H, Lq, Lk, scale, pipelined=True):
    """Tensor-core attention core (fp16 in/out, K / V staged once per head by TMA); same argument conventions as attention()."""
    _need_cuda(q, k, v, out)
    if not all(t_.dtype == torch.float16 and t_.stride(-1) == 1 for t_ in (q, k, v, out)):
        raise RuntimeError("attention_tc needs fp16 tensors contiguous in the head dimension")
    fn = _lib.lib().dsb_attention_tc2 if pipelined else _lib.lib().dsb_attention_tc
    _lib.check(fn(q.data_ptr(), q.stride(0), k.data_ptr(), k.stride(0), v.data_ptr(), v.stride(0), out.data_ptr(), out.stride(0),
                  B, H, Lq, Lk, scale, _stream()), "dsb_attention_tc")
    return out


def attention_tc_split(q, k, v, out, *, q_lo, k_lo, v_lo, o_lo, B, H, Lq, Lk, scale, head_dim=64):
    """Split-fp16 tensor-core attention: q/k/v/out are the hi halves (row-strided fp16 views, head h = columns [head_dim*h, head_dim*(h+1)),
    head_dim 64 or 32); the matching lo half of every row lies *_lo elements further along the row."""
    _attention_head_dim("attention_tc_split", head_dim)
    _need_cuda(q, k, v, out)
    if not all(t_.dtype == torch.float16 and t_.stride(-1) == 1 for t_ in (q, k, v, out)):
        raise RuntimeError("attention_tc_split needs fp16 tensors contiguous in the head dimension")
    name = "dsb_attention_tc_split" if head_dim == 64 else "dsb_attention_tc_split_hd32"
    _lib.check(getattr(_lib.lib(), name)(q.data_ptr(), q.stride(0), q_lo, k.data_ptr(), k.stride(0), k_lo, v.data_ptr(), v.stride(0), v_lo,
                                         out.data_ptr(), out.stride(0), o_lo, B, H, Lq, Lk, scale, _stream()), name)
    return out


def attention_tc_split_causal(q, k, v, out, *, q_lo, k_lo, v_lo, o_lo, B, H, L, scale, head_dim=64):
    """Causal attention_tc_split (mingpt.py CausalSelfAttention, n_unmasked = 0): query row i of a sequence of L rows attends to keys 0 ... i.
    Same pair layout and arguments as attention_tc_split with Lq = Lk = L; head_dim 64 or 32."""
    _attention_head_dim("attention_tc_split_causal", head_dim)
    _need_cuda(q, k, v, out)
    if not all(t_.dtype == torch.float16 and t_.stride(-1) == 1 for t_ in (q, k, v, out)):
        raise RuntimeError("attention_tc_split_causal needs fp16 tensors contiguous in the head dimension")
    _lib.check(_lib.lib().dsb_attention_tc_split_causal(q.data_ptr(), q.stride(0), q_lo, k.data_ptr(), k.stride(0), k_lo, v.data_ptr(), v.stride(0), v_lo,
                                                        out.data_ptr(), out.stride(0), o_lo, B, H, L, L, scale, head_dim, _stream()),
               "dsb_attention_tc_split_causal")
    return out


def posterior_sample(inp, x_t, t, uniform, sched, *, T, trunc_mode=1, trunc_r=0.85, trunc_k=0, t_post=None, x_next=None, log_prob_out=None,
                     stage=0):
    """Fused p_sample tail (see dsb_posterior_sample).  inp: raw logits (B,L,K) fp32, or (B,K+1,L) log-probs with STAGE_INPUT_LOGPROB;
    x_t (B,L) int64; uniform (B,K+1,L); sched (8,T+1) -> x_next (B,L) int64 (None when sampling is skipped)."""
    return _posterior_sample("dsb_posterior_sample", inp, x_t, t, uniform, sched, T, trunc_mode, trunc_r, trunc_k, t_post, x_next, log_prob_out, stage)


def posterior_sample_wide(inp, x_t, t, uniform, sched, *, T, trunc_mode=1, trunc_r=0.85, trunc_k=0, t_post=None, x_next=None, log_prob_out=None,
                          stage=0):
    """posterior_sample for codebooks up to K = WIDE_SAMPLER_MAX_K, one CTA per column (see dsb_posterior_sample_wide)."""
    return _posterior_sample("dsb_posterior_sample_wide", inp, x_t, t, uniform, sched, T, trunc_mode, trunc_r, trunc_k, t_post, x_next, log_prob_out,
                             stage)


# Largest K of the warp-per-column sampler (posterior_sample / posterior_sample_loop) and of the CTA-per-column one (the _wide pair).
WARP_SAMPLER_MAX_K = 1055
WIDE_SAMPLER_MAX_K = 4095


def _posterior_sample(fn, inp, x_t, t, uniform, sched, T, trunc_mode, trunc_r, trunc_k, t_post, x_next, log_prob_out, stage):
    _need_cuda(inp, x_t, t, uniform, sched, log_prob_out)
    if stage & STAGE_INPUT_LOGPROB:
        B, C_, L = inp.shape
        K = C_ - 1
    else:
        B, L, K = inp.shape
    for t_ in (inp, x_t, uniform, sched, log_prob_out, t, t_post):
        if t_ is not None and not t_.is_contiguous():
            raise RuntimeError("posterior_sample needs contiguous tensors")
    if uniform is not None and tuple(uniform.shape) != (B, K + 1, L):
        raise RuntimeError(f"uniform must be (B,K+1,L)={(B, K + 1, L)}, got {tuple(uniform.shape)}")
    if sched is not None and tuple(sched.shape) != (8, T + 1):
        raise RuntimeError("sched must be (8, T+1)")
    if not (stage & STAGE_SKIP_SAMPLE) and x_next is None:
        x_next = torch.empty((B, L), dtype=torch.int64, device=inp.device)
    _lib.check(getattr(_lib.lib(), fn)(inp.data_ptr(), _ptr(x_t), _ptr(t), _ptr(t_post), _ptr(uniform), _ptr(sched), _ptr(x_next),
                                       _ptr(log_prob_out), B, K, L, T, trunc_mode, trunc_r, trunc_k, stage, _stream()), fn)
    return x_next


def aten_rand_geometry(numel: int, device=None):
    """(nthreads, counter_offset) of the kernel ATen launches for torch.rand / rand_like on a contiguous float tensor of `numel` elements
    (ATen/native/cuda/DistributionTemplates.h calc_execution_policy: block 256, grid = min(SMs * (maxThreadsPerSM // 256), ceil(numel / 256)),
    four values per curand call)."""
    pr = torch.cuda.get_device_properties(device if device is not None else torch.cuda.current_device())
    grid = min(pr.multi_processor_count * (pr.max_threads_per_multi_processor // 256), (numel + 255) // 256)
    return 256 * grid, ((numel - 1) // (256 * grid * 4) + 1) * 4


def aten_uniform(numel: int, seed: int, offset: int, device=None) -> torch.Tensor:
    """The tensor torch.rand(numel, device='cuda') would return for generator state (seed, philox offset), computed by this library's Philox."""
    out = torch.empty(numel, dtype=torch.float32, device=device if device is not None else "cuda")
    nthreads, _ = aten_rand_geometry(numel, out.device)
    _lib.check(_lib.lib().dsb_aten_uniform(out.data_ptr(), numel, seed & (2 ** 64 - 1), offset, nthreads, _stream()), "dsb_aten_uniform")
    return out


def posterior_sample_loop(logits, x, t, t_post, sched, ctrl, t_sched, t_post_sched, *, T, trunc_mode=1, trunc_r=0.85, trunc_k=0):
    """One step of the fused sampling loop (see dsb_posterior_sample_loop): in-kernel uniforms, x updated in place, t / t_post / RNG offset advanced on
    the device by the kernel itself."""
    return _posterior_sample_loop("dsb_posterior_sample_loop", logits, x, t, t_post, sched, ctrl, t_sched, t_post_sched, T, trunc_mode, trunc_r, trunc_k)


def posterior_sample_wide_loop(logits, x, t, t_post, sched, ctrl, t_sched, t_post_sched, *, T, trunc_mode=1, trunc_r=0.85, trunc_k=0):
    """posterior_sample_loop for codebooks up to K = WIDE_SAMPLER_MAX_K, one CTA per column (see dsb_posterior_sample_wide_loop)."""
    return _posterior_sample_loop("dsb_posterior_sample_wide_loop", logits, x, t, t_post, sched, ctrl, t_sched, t_post_sched, T, trunc_mode, trunc_r,
                                  trunc_k)


def _posterior_sample_loop(fn, logits, x, t, t_post, sched, ctrl, t_sched, t_post_sched, T, trunc_mode, trunc_r, trunc_k):
    _need_cuda(logits, x, t, t_post, sched, ctrl, t_sched, t_post_sched)
    B, L, K = logits.shape
    _lib.check(getattr(_lib.lib(), fn)(logits.data_ptr(), x.data_ptr(), t.data_ptr(), t_post.data_ptr(), sched.data_ptr(), ctrl.data_ptr(),
                                       t_sched.data_ptr(), t_post_sched.data_ptr(), B, K, L, T, trunc_mode, trunc_r, trunc_k, _stream()), fn)
    return x


# ---------------------------------------------------------------------------------------------- decoder / vocoder support
def codebook_gather_padded(ids, codebook, H, W, *, round_out=True, split=False, split_f16=False, err_flag=None):
    _need_cuda(ids, codebook)
    B = ids.shape[0]
    E = codebook.shape[1]
    out = torch.empty(B, H + 2, W + 2, 2 * E if (split or split_f16) else E, dtype=torch.float16 if split_f16 else torch.float32, device=ids.device)
    _lib.check(_lib.lib().dsb_codebook_gather_padded(ids.contiguous().data_ptr(), codebook.data_ptr(), out.data_ptr(), B, H, W, E, codebook.shape[0],
                                                     SPLIT_OUT_F16 if split_f16 else (SPLIT_OUT if split else (ROUND_TF32 if round_out else 0)), _ptr(err_flag), _stream()),
               "dsb_codebook_gather_padded")
    return out


def groupnorm_stats(x_pad, stats=None, groups=32):
    """x_pad (B, Hp, Wp, C) zero-bordered -> stats (B, groups, 2) fp64 (sum, sumsq)."""
    _need_cuda(x_pad)
    B, Hp, Wp, C = x_pad.shape
    stats = torch.empty(B, groups, 2, dtype=torch.float64, device=x_pad.device) if stats is None else stats
    _lib.check(_lib.lib().dsb_groupnorm_stats(x_pad.data_ptr(), stats.data_ptr(), B, Hp * Wp, C, groups, _stream()), "dsb_groupnorm_stats")
    return stats


def groupnorm_apply(x_pad, stats, gamma, beta, *, eps=1e-6, swish=True, round_out=True, compact_len=0, out=None, groups=32, split=False, split_f16=False):
    _need_cuda(x_pad, stats, gamma, beta)
    B, Hp, Wp, C = x_pad.shape
    H, W = Hp - 2, Wp - 2
    flags = (GN_SWISH if swish else 0) | (ROUND_TF32 if round_out and not (split or split_f16) else 0) | (GN_COMPACT if compact_len else 0) | \
        (SPLIT_OUT_F16 if split_f16 else (SPLIT_OUT if split else 0))
    if out is None:
        Co = 2 * C if (split or split_f16) else C
        out = torch.empty((B, compact_len, Co) if compact_len else (B, Hp, Wp, Co), dtype=torch.float16 if split_f16 else torch.float32, device=x_pad.device)
    _lib.check(_lib.lib().dsb_groupnorm_apply(x_pad.data_ptr(), stats.data_ptr(), gamma.data_ptr(), beta.data_ptr(), out.data_ptr(), B, H, W, C, groups,
                                              eps, flags, compact_len, _stream()), "dsb_groupnorm_apply")
    return out


def upsample2x_padded(x_pad, *, round_out=True, split=False, split_f16=False):
    _need_cuda(x_pad)
    B, Hp, Wp, C = x_pad.shape
    H, W = Hp - 2, Wp - 2
    out = torch.empty(B, 2 * H + 2, 2 * W + 2, 2 * C if (split or split_f16) else C, dtype=torch.float16 if split_f16 else torch.float32, device=x_pad.device)
    _lib.check(_lib.lib().dsb_upsample2x_padded(x_pad.data_ptr(), out.data_ptr(), B, H, W, C,
                                                SPLIT_OUT_F16 if split_f16 else (SPLIT_OUT if split else (ROUND_TF32 if round_out else 0)), _stream()),
               "dsb_upsample2x_padded")
    return out


def space_to_depth_padded(x_pad, *, split=False, round_out=False):
    """(B, H+2, W+2, C) zero-bordered image -> its four stride-2 phases on the half-resolution padded grid (B, H/2+2, W/2+2, 4C [8C if split])."""
    _need_cuda(x_pad)
    B, Hp, Wp, C = x_pad.shape
    H, W = Hp - 2, Wp - 2
    out = torch.empty(B, H // 2 + 2, W // 2 + 2, (8 if split else 4) * C, dtype=torch.float32, device=x_pad.device)
    _lib.check(_lib.lib().dsb_space_to_depth_padded(x_pad.data_ptr(), out.data_ptr(), B, H, W, C, SPLIT_OUT if split else (ROUND_TF32 if round_out else 0),
                                                    _stream()), "dsb_space_to_depth_padded")
    return out


def row_argmin(x, n: int):
    """x: (rows, ld) fp32 -> int64 (rows,) index of the smallest of the first n columns (first on ties)."""
    _need_cuda(x)
    out = torch.empty(x.shape[0], dtype=torch.int64, device=x.device)
    _lib.check(_lib.lib().dsb_row_argmin(x.data_ptr(), x.stride(0), x.shape[0], n, out.data_ptr(), _stream()), "dsb_row_argmin")
    return out


def softmax_rows_(x, n_valid, *, round_out=True):
    _need_cuda(x)
    assert x.is_contiguous()
    ld = x.shape[-1]
    _lib.check(_lib.lib().dsb_softmax_rows(x.data_ptr(), x.numel() // ld, n_valid, ld, ROUND_TF32 if round_out else 0, _stream()), "dsb_softmax_rows")
    return x


def tokens_add_to_padded_(tok, x_pad):
    _need_cuda(tok, x_pad)
    B, Hp, Wp, C = x_pad.shape
    _lib.check(_lib.lib().dsb_tokens_add_to_padded(tok.data_ptr(), x_pad.data_ptr(), B, Hp - 2, Wp - 2, C, tok.shape[1], _stream()),
               "dsb_tokens_add_to_padded")
    return x_pad


def lrelu_pad(x, pad, *, slope=0.2, reflect=True, channel_major=False, round_out=True, split=False):
    """x (B,T,C) channels-last, or (B,C,T) with channel_major -> (B, T+2*pad, C), or the split-TF32 operand (B, T+2*pad, 2*Cp)."""
    _need_cuda(x)
    x = x.contiguous()
    if channel_major:
        B, Cc, T = x.shape
    else:
        B, T, Cc = x.shape
    Co = 2 * ((Cc + 31) // 32 * 32) if split else Cc
    out = torch.empty(B, T + 2 * pad, Co, dtype=torch.float32, device=x.device)
    _lib.check(_lib.lib().dsb_lrelu_pad(x.data_ptr(), out.data_ptr(), B, T, Cc, pad, slope, 1 if reflect else 0, 1 if channel_major else 0,
                                        SPLIT_OUT if split else (ROUND_TF32 if round_out else 0), _stream()), "dsb_lrelu_pad")
    return out


# ---------------------------------------------------------------------------------------------- Melception support (pair images, see the header)
def mel_stem(x, w, bias, out, *, Hp, Wp, y0, x0, scale=1.0, mean=None, std=None):
    """x (B, F, T) fp32 mels -> out (B, Hp, Wp, 2 Cout) fp16 pair grid of scale * relu(conv3x3_s2((x - mean) / std) + bias), zeros outside the window."""
    _need_cuda(x, w, bias, out, mean, std)
    x = x.contiguous()
    B, F_, T = x.shape
    _lib.check(_lib.lib().dsb_mel_stem(x.data_ptr(), _ptr(mean), _ptr(std), w.data_ptr(), bias.data_ptr(), float(scale), out.data_ptr(), B, F_, T, w.shape[0],
                                       Hp, Wp, y0, x0, _stream()), "dsb_mel_stem")
    return out


def pair_space_to_depth(x, window, out, out_origin):
    """x (B, Hpi, Wpi, 2C) pair image with window (y0, x0, H, W) -> its stride-2 phases in out (B, Hpo, Wpo, 8C) at out_origin (oy0, ox0)."""
    _need_cuda(x, out)
    B, Hpi, Wpi, C2 = x.shape
    _lib.check(_lib.lib().dsb_pair_space_to_depth(x.data_ptr(), Hpi, Wpi, *window, out.data_ptr(), out.shape[1], out.shape[2], *out_origin, B, C2 // 2,
                                                  _stream()), "dsb_pair_space_to_depth")
    return out


def pair_maxpool3s2(x, window, out, out_origin, *, out_ptr=None, ldo=None, lo_off=None, scale=1.0):
    """MaxPool2d(3, 2) of x's window into out (B, Hpo, Wpo, ldo) at out_origin; out_ptr / lo_off address a channel slice of out (defaults: all of it)."""
    _need_cuda(x, out)
    B, Hpi, Wpi, C2 = x.shape
    C = C2 // 2
    _lib.check(_lib.lib().dsb_pair_maxpool3s2(x.data_ptr(), Hpi, Wpi, *window, out.data_ptr() if out_ptr is None else out_ptr, out.shape[-1] if ldo is None else ldo,
                                              C if lo_off is None else lo_off, out.shape[1], out.shape[2], *out_origin, B, C, float(scale), _stream()),
               "dsb_pair_maxpool3s2")
    return out


def pair_avgpool3(x, window, out=None):
    """AvgPool2d(3, 1, 1) (count_include_pad) of x's window (B, Hp, Wp, 2C) -> out (same shape) pair image."""
    _need_cuda(x, out)
    B, Hp, Wp, C2 = x.shape
    out = torch.empty_like(x) if out is None else out
    _lib.check(_lib.lib().dsb_pair_avgpool3(x.data_ptr(), Hp, Wp, *window, out.data_ptr(), out.shape[-1], C2 // 2, B, C2 // 2, _stream()), "dsb_pair_avgpool3")
    return out


def pair_channel_mean(x, window, *, inv_scale=1.0, out=None):
    """x (B, Hp, Wp, 2C) pair image -> (B, C) fp32 mean over the window, times inv_scale."""
    _need_cuda(x, out)
    B, Hp, Wp, C2 = x.shape
    C = C2 // 2
    out = torch.empty(B, C, dtype=torch.float32, device=x.device) if out is None else out
    _lib.check(_lib.lib().dsb_pair_channel_mean(x.data_ptr(), C2, C, Hp, Wp, *window, B, C, float(inv_scale), out.data_ptr(), _stream()),
               "dsb_pair_channel_mean")
    return out


# ---------------------------------------------------------------- autoregressive transformer decode (ar_decode.cu)
AR_MAX_V = 4096
AR_HEAD_DIMS = (32, 64)
AR_MAX_POS = 512
AR_CTRL_WORDS = 8


def aten_exponential(numel: int, seed: int, offset: int, device=None) -> torch.Tensor:
    """The tensor torch.empty(numel, device='cuda').exponential_() would return for generator state (seed, philox offset), computed by this
    library's Philox (the q that torch.multinomial(probs, 1) draws on CUDA)."""
    out = torch.empty(numel, dtype=torch.float32, device=device if device is not None else "cuda")
    nthreads, _ = aten_rand_geometry(numel, out.device)
    _lib.check(_lib.lib().dsb_aten_exponential(out.data_ptr(), numel, seed & (2 ** 64 - 1), offset, nthreads, _stream()), "dsb_aten_exponential")
    return out


def ar_embed(cond, tok_emb, pos_emb, ids, x, ctrl, *, err_flag=None):
    """x (B, D) = embedding of position ctrl[4]: cond (B, Tc, D) rows first, then tok_emb[ids (B, ids_ld)], plus pos_emb (P, D)."""
    _need_cuda(cond, tok_emb, pos_emb, ids, x, ctrl, err_flag)
    B, Tc, D = cond.shape
    _lib.check(_lib.lib().dsb_ar_embed(cond.data_ptr(), tok_emb.data_ptr(), pos_emb.data_ptr(), ids.data_ptr(), ids.stride(0), x.data_ptr(), ctrl.data_ptr(),
                                       B, Tc, tok_emb.shape[0], D, _ptr(err_flag), _stream()), "dsb_ar_embed")
    return x


def ar_embed_all(cond, tok_emb, pos_emb, ids, x, *, err_flag=None):
    """x (B, T, D) = every position's embedding: cond (B, Tc, D) rows first, then tok_emb[ids (B, T - Tc)], plus pos_emb[:T]."""
    _need_cuda(cond, tok_emb, pos_emb, ids, x, err_flag)
    B, Tc, D = cond.shape
    T = x.shape[1]
    if ids.shape != (B, T - Tc) or x.shape != (B, T, D) or not x.is_contiguous():
        raise RuntimeError(f"ar_embed_all: ids {tuple(ids.shape)} / x {tuple(x.shape)} do not match cond {tuple(cond.shape)}")
    _lib.check(_lib.lib().dsb_ar_embed_all(cond.data_ptr(), tok_emb.data_ptr(), pos_emb.data_ptr(), ids.data_ptr(), ids.stride(0), x.data_ptr(), B, T, Tc,
                                           tok_emb.shape[0], D, _ptr(err_flag), _stream()), "dsb_ar_embed_all")
    return x


def ar_cross_entropy(logits, targets, *, first_row=0, nll=None, loss=None, err_flag=None):
    """F.cross_entropy (ignore_index -100) of logits (B, T, V) rows first_row ... first_row + n - 1 against targets (B, n) int64.  Returns (loss (),
    nll (B, n)): the mean over non-ignored rows (NaN if none) and the per-row NLL (0 where ignored).  An out-of-range target sets err_flag, or
    raises IndexError when no err_flag is given (one 4-byte read)."""
    _need_cuda(logits, targets, nll, loss, err_flag)
    B, T, V = logits.shape
    n = targets.shape[1]
    if logits.dtype != torch.float32 or logits.stride(2) != 1 or logits.stride(0) != T * logits.stride(1) or targets.dtype != torch.int64 \
            or targets.stride(1) != 1 or targets.shape[0] != B:
        raise RuntimeError("ar_cross_entropy: fp32 logits (B, T, V) with uniform row stride and int64 targets (B, n)")
    if V > AR_MAX_V:
        raise ValueError(f"ar_cross_entropy: vocabulary of {V} exceeds {AR_MAX_V}")
    if not 0 <= first_row <= T - n:
        raise ValueError(f"ar_cross_entropy: rows {first_row} ... {first_row + n - 1} outside the {T} positions")
    nll = torch.empty(B, n, dtype=torch.float32, device=logits.device) if nll is None else nll
    loss = torch.empty((), dtype=torch.float32, device=logits.device) if loss is None else loss
    err = err_flag if err_flag is not None else torch.zeros(1, dtype=torch.int32, device=logits.device)
    _lib.check(_lib.lib().dsb_ar_cross_entropy(logits.data_ptr(), logits.stride(1), T, int(first_row), n, targets.data_ptr(), targets.stride(0),
                                               nll.data_ptr(), loss.data_ptr(), B, V, err.data_ptr(), _stream()), "dsb_ar_cross_entropy")
    if err_flag is None and int(err.item()):
        raise IndexError(f"Target out of bounds: a target outside [0, {V}) that is not ignore_index (-100)")
    return loss, nll


def ar_attention(qkv, k_cache, v_cache, out, ctrl, *, H, scale, lo_off=None):
    """Decode attention at position ctrl[4]: qkv (B, 3D) fp32 [Q | K | V]; k_cache / v_cache (B, P, D) fp32; out the fp16 (hi | lo) pair (B, 2D)."""
    _need_cuda(qkv, k_cache, v_cache, out, ctrl)
    B, P, D = k_cache.shape
    if D % H or D // H not in AR_HEAD_DIMS:
        raise ValueError(f"ar_attention: head_dim {D // H if D % H == 0 else D / H} unsupported (32 or 64)")
    if P > AR_MAX_POS:
        raise ValueError(f"ar_attention: {P} cache positions exceed {AR_MAX_POS}")
    if out.dtype != torch.float16 or qkv.dtype != torch.float32 or k_cache.dtype != torch.float32 or not k_cache.is_contiguous() or not v_cache.is_contiguous():
        raise RuntimeError("ar_attention: fp32 qkv and contiguous fp32 caches in, fp16 pair out")
    _lib.check(_lib.lib().dsb_ar_attention(qkv.data_ptr(), qkv.stride(0), k_cache.data_ptr(), v_cache.data_ptr(), P * D, P, out.data_ptr(), out.stride(0),
                                           D if lo_off is None else lo_off, ctrl.data_ptr(), B, H, D // H, float(scale), _stream()), "dsb_ar_attention")
    return out


def gelu_erf_split(x, out=None):
    """nn.GELU() (exact erf) of fp32 x (rows, C), written as the fp16 (hi | lo) pair (rows, 2C)."""
    _need_cuda(x, out)
    rows, Cc = x.shape
    if out is None:
        out = torch.empty(rows, 2 * Cc, dtype=torch.float16, device=x.device)
    _lib.check(_lib.lib().dsb_gelu_erf_split(x.data_ptr(), x.stride(0), out.data_ptr(), out.stride(0), Cc, rows, Cc, _stream()), "dsb_gelu_erf_split")
    return out


def ar_sample(logits, ids, ctrl, *, Tc, temperature=1.0, top_k=None, sample=True, probs_out=None, logits_hist=None, err_flag=None):
    """One sampling step at position ctrl[4] (see dsb_ar_sample): logits (B, V) fp32 -> ids[b, p - Tc + 1] when p >= ctrl[6]; top_k None = no
    truncation.  logits_hist (B, P, V) receives row p of the raw logits."""
    _need_cuda(logits, ids, ctrl, probs_out, logits_hist, err_flag)
    B, V = logits.shape
    check_ar_sampler_args(V, top_k, temperature)
    _lib.check(_lib.lib().dsb_ar_sample(logits.data_ptr(), logits.stride(0), ids.data_ptr(), ids.stride(0), ctrl.data_ptr(), B, V, Tc, float(temperature),
                                        0 if top_k is None else int(top_k), 1 if sample else 0, _ptr(probs_out), _ptr(logits_hist),
                                        0 if logits_hist is None else logits_hist.stride(0), _ptr(err_flag), _stream()), "dsb_ar_sample")
    return ids


def check_ar_sampler_args(V, top_k, temperature):
    """The sampler's refusals, raised before anything is launched."""
    if V > AR_MAX_V:
        raise ValueError(f"the autoregressive sampler takes a vocabulary of at most {AR_MAX_V} entries, got {V}")
    if top_k is not None and not 1 <= int(top_k) <= V:
        raise ValueError(f"top_k={top_k} out of range: torch.topk needs 1 <= k <= vocab size ({V})")
    if not float(temperature) == float(temperature) or float(temperature) == 0.0:
        raise ValueError("temperature must be a non-zero number")


# ---------------------------------------------------------------- SpecVQGAN log-mel spectrogram (mel.cu)
WAV_SCALE = 8192.0  # DSB_WAV_SCALE
WAV_LIMIT = 4.0     # DSB_WAV_LIMIT
MEL_HOP, MEL_PAD = 256, 512


def wav_frame_rows(length: int) -> int:
    """Rows per clip dsb_wav_frames_f16 needs: frames 1 + length // 256, frame t = rows t ... t+3."""
    return length // MEL_HOP + 4


def wav_frames_f16(wav, out=None, *, rows=None, err_flag=None):
    """wav (B, length) fp32, contiguous in time -> (B, rows, 512) fp16: the reflect-padded clip as rows of 256 samples, [hi | lo] of 2^13 x."""
    _need_cuda(wav, out, err_flag)
    if wav.dim() != 2 or wav.dtype != torch.float32 or wav.stride(1) != 1:
        raise RuntimeError("wav_frames_f16 needs a (B, length) fp32 tensor contiguous in time")
    B, length = wav.shape
    rows = wav_frame_rows(length) if rows is None else rows
    if out is None:
        out = torch.empty(B, rows, 2 * MEL_HOP, dtype=torch.float16, device=wav.device)
    _lib.check(_lib.lib().dsb_wav_frames_f16(wav.data_ptr(), wav.stride(0), B, length, out.data_ptr(), rows, _ptr(err_flag), _stream()),
               "dsb_wav_frames_f16")
    return out


def mel_log(spec, n_bins, fb_start, fb_len, fb_w, T_out, out=None):
    """spec (B, T, ld) fp32 interleaved (re, im) pairs of n_bins DFT bins -> (B, n_mels, T_out) SpecVQGAN log-mel (see dsb_mel_log)."""
    _need_cuda(spec, fb_start, fb_len, fb_w, out)
    B, T, ld = spec.shape
    n_mels, fb_ld = fb_w.shape
    if spec.stride(2) != 1 or spec.stride(1) != ld:
        raise RuntimeError("mel_log needs (B, T, ld) spectra with contiguous rows")
    if out is None:
        out = torch.empty(B, n_mels, T_out, dtype=torch.float32, device=spec.device)
    _lib.check(_lib.lib().dsb_mel_log(spec.data_ptr(), ld, spec.stride(0), B, T, T_out, n_bins, fb_start.data_ptr(), fb_len.data_ptr(), fb_w.data_ptr(),
                                      fb_ld, n_mels, out.data_ptr(), _stream()), "dsb_mel_log")
    return out
