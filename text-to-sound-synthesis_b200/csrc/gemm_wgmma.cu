// TMA + wgmma GEMM for sm_90a:  out[b][M,N] = epilogue( sum_tap A[b][m + shift_tap, :Kc] . W[n, tap*Kc : (tap+1)*Kc]^T )
//
// * A and W are K-contiguous ("TN"), i.e. torch.nn.Linear's activation (M,K) and weight (N,K) as they lie in HBM; either may instead be
//   MN-major (2-byte types, one tap), e.g. the operands of a weight-gradient GEMM dW = dY^T X.
// * operands: TF32 (fp32 containers) or BF16 / F16 (wgmma.mma_async); accumulation fp32 in registers.
// * "taps": the K loop runs over (tap, channel-block); each tap reads A rows shifted by shift_tap.  With one tap this is
//   a plain Linear layer (Text2ImageTransformer, reference transformer_utils.py:45-57,95-108,248-253,345-348); with 9 / 3 / 7
//   taps on zero-padded channels-last buffers it is the implicit-GEMM form of the SpecVQGAN decoder's 3x3 convs (reference
//   specvqgan/modules/diffusionmodules/model.py:92-151) and the MelGAN convs (reference vocoder/modules.py:72-126).
// * warp-specialised persistent kernel, 384 threads: warpgroup 0 = TMA producer (one thread), warpgroups 1-2 = consumers, each issuing
//   wgmma for 64 rows of the 128-row tile and then running the fused epilogue (registers -> XOR-swizzled smem transpose -> bias / GELU2 /
//   residual / tf32-round -> HBM) while the producer already streams the next tile's k-blocks into the smem ring.
// * split-fp16 ("f16x3") form: one stage holds the four tiles of a k-block (A hi, A lo, W hi, W lo) and the consumers run the three passes
//   lo*hi, hi*lo, hi*hi off that single staged copy.
// * tile schedule (stream_k.cuh): data-parallel, or, when the tiles leave a partial last wave, ordered stream-K -- a tile may be split
//   between two neighbouring CTAs at a k-block boundary.  The CTA holding the first k-blocks stores its fp32 accumulator to a per-device
//   workspace; the CTA holding the rest loads it and continues the same accumulation sequence (the same FADDs / wgmma accumulations in the
//   same order), then runs the epilogue.  Every output bit is what the data-parallel schedule computes.
//   Contract: the workspace is shared by all launches on a device, so at most one GEMM may be in flight per device at a time (every caller
//   issues its GEMMs on one stream; warm-up side streams are joined before and after).
#include "common.cuh"
#include "diffsound_b200.h"
#include "stream_k.cuh"
#include "wgmma.cuh"
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cstdlib>
#include <mutex>
#include <type_traits>

namespace dsb {

constexpr int BLOCK_M = 128;
constexpr int ROW_BYTES = 128;     // one swizzle-128B row of K per operand row
constexpr int GEMM_THREADS = 384;  // warpgroup 0 TMA producer, warpgroups 1-2 MMA + epilogue
constexpr int MAX_TAPS = 32;
constexpr int MN_BOX_BYTES = 64 * ROW_BYTES;  // one MN-major TMA box: 64 K rows x 64 two-byte columns
constexpr int EPI_ROWS = 16;                  // rows of one consumer warp's accumulator slab
constexpr int SMEM_BUDGET = 192 * 1024;       // operand ring; + epilogue tiles + barriers stays under the 227 KB a block may use

struct GemmParams {
  int M, N, batch;
  int tiles_m, tiles_n;
  int kb_per_tap;  // ceil(Kc / BLOCK_K)
  int block_k;     // elements per k-block (32 tf32 / 64 bf16)
  int num_taps;
  int tap_shift[MAX_TAPS];
  int tap_acol[MAX_TAPS];
  int tap_wcol[MAX_TAPS];  // W column offset per tap (default tap * Kc)
  unsigned tap_a2_mask;    // bit i set: tap i reads the SECOND A tensor map (a fused GEMM over two activation buffers)
  // fused split-fp16 form: f3_nsp spatial taps j, each with row shift tap_shift[j], hi-half columns tap_acol[j] (A) / tap_wcol[j] (W);
  // the lo halves sit lo_a / lo_w columns further right
  int f3_nsp, lo_a, lo_w;
  long long split_off;     // DSB_GEMM_OUT_F16_SPLIT: offset of the lo half inside an output row
  long long dual_off;      // DSB_GEMM_DUAL_LRELU: offset of the LeakyReLU(0.2) copy (hi at +dual_off, lo at +dual_off+split_off)
  int ocg, ocg_stride;     // output column groups: logical column n lives at (n / ocg) * ocg_stride + n % ocg (0 = plain)
  float* amax_out;         // optional: atomic max of |value stored| over the whole output (calibration of fp16 activation scales)
  int kc;          // channels per tap
  int b_batched;
  const float* bias;
  const float* residual;
  long long ld_res, res_bstride;
  void* out;
  long long ldo, out_bstride;
  int flags;
  // optional row mask (padded conv geometry): row r -> p = r % geo_P; y = p / geo_Wp; x = p % geo_Wp;
  // rows outside [y0,y1) x [x0,x1) are written as zeros.  geo_P == 0 disables.
  int geo_P, geo_Wp, geo_y0, geo_y1, geo_x0, geo_x1;
  float alpha;     // scale applied to the accumulator before bias (1.0 for Linear)
  // MN-major operands (2-byte types, one tap): the operand lies in HBM as (K rows, MN columns).  Loaded as 64-column x 64-row TMA boxes
  // (SWIZZLE_128B), consumed through MN-major (transposed) wgmma descriptors: no transposed copies.
  int a_mn, b_mn;
  // ordered stream-K (stream_k.cuh): sk_part holds one BLOCK_N / 128 x 64 KB accumulator slot per CTA, sk_flag[c] = 1 once CTA c's slot is
  // published (reset to 0 by its reader, so the workspace is clean again when the launch ends)
  int stream_k;
  float* sk_part;
  int* sk_flag;
};

constexpr int SK_SLOT_FLOATS = 128 * 128;  // one 128 x 128 fp32 accumulator; a 256-wide tile uses two
constexpr unsigned SK_SPIN_LIMIT = 1u << 24;  // ~ seconds of polling at 64 ns per try: far beyond any real wait, so only a protocol bug traps

template <int BLOCK_N, bool F3>
struct GemmSmem {
  static constexpr int A_BYTES = BLOCK_M * ROW_BYTES;
  static constexpr int B_BYTES = BLOCK_N * ROW_BYTES;
  static constexpr int STAGE_BYTES = (F3 ? 2 : 1) * (A_BYTES + B_BYTES);
  static constexpr int STAGES = SMEM_BUDGET / STAGE_BYTES;  // 6 (N 128), 4 (N 256), 3 (f16x3)
  static constexpr int EPI_BYTES = 8 * EPI_ROWS * 32 * 4;
  static constexpr int TOTAL = STAGES * STAGE_BYTES + EPI_BYTES + 256 /*barriers*/ + 1024 /*align slack*/;
};

// One 16-row x 32-column chunk of the output tile for one warp: the chunk sits in `sw` (XOR-swizzled float4 groups, row stride 32 floats);
// alpha / bias / residual / activation / rounding / border mask, then coalesced stores (lanes 0-7 cover one row's 32 columns).
// Inlined: the call (one per chunk) and its ABI register traffic cost the split-fp16 denoiser GEMMs 4-10 % of their time on an H100.
__device__ __forceinline__ void epilogue_chunk(const GemmParams& p, const float* sw, int row_base, int col0, int b, int lane, bool vec_ok) {
  const bool has_geo = p.geo_P > 0;
  const int out_mode = (p.flags & DSB_GEMM_OUT_F16_SPLIT) ? 3 : ((p.flags & DSB_GEMM_OUT_F16) ? 1 : ((p.flags & DSB_GEMM_OUT_BF16) ? 2 : 0));
  const int act = (p.flags & DSB_GEMM_GELU2) ? 1 : ((p.flags & DSB_GEMM_LRELU) ? 2 : ((p.flags & DSB_GEMM_TANH) ? 3 : ((p.flags & DSB_GEMM_RELU) ? 4 : 0)));
  const bool do_round = (p.flags & DSB_GEMM_ROUND_TF32) != 0;
  const bool dual = (p.flags & DSB_GEMM_DUAL_LRELU) != 0;
  const bool res_first = (p.flags & DSB_GEMM_RES_BEFORE_ACT) != 0;
  const int c4 = lane & 7;    // float4 column slot inside the 32-column chunk
  const int rsub = lane >> 3; // row inside each group of 4 rows
  constexpr int NI = EPI_ROWS / 4;
  uint32_t ok_mask = 0, in_mask = 0;  // bit i: row (row_base + i*4 + rsub) exists / is an interior row
#pragma unroll
  for (int i = 0; i < NI; ++i) {
    const int row = row_base + i * 4 + rsub;
    if (row < p.M) ok_mask |= 1u << i;
    bool interior = true;
    if (has_geo) {
      const int pp = row % p.geo_P;
      const int y = pp / p.geo_Wp, x = pp - y * p.geo_Wp;
      interior = (y >= p.geo_y0) && (y < p.geo_y1) && (x >= p.geo_x0) && (x < p.geo_x1);
    }
    if (interior) in_mask |= 1u << i;
  }
  const long long out_boff = (long long)b * p.out_bstride;
  const float* res_b = p.residual ? p.residual + (long long)b * p.res_bstride : nullptr;
  const int col = col0 + c4 * 4;
  if (vec_ok && (col0 + 32 <= p.N)) {
    // ---------------- fast path: whole chunk in range, 16-byte aligned everywhere
    float x[4 * NI];
    const float4 bz = p.bias ? __ldg(reinterpret_cast<const float4*>(p.bias + col)) : make_float4(0.f, 0.f, 0.f, 0.f);
    float4 rz[NI];
#pragma unroll
    for (int i = 0; i < NI; ++i) {
      const int r = i * 4 + rsub;
      const float4 a4 = *reinterpret_cast<const float4*>(sw + r * 32 + ((c4 ^ (r & 7)) << 2));
      rz[i] = (res_b && ((ok_mask >> i) & 1u)) ? *reinterpret_cast<const float4*>(res_b + (long long)(row_base + r) * p.ld_res + col)
                                              : make_float4(0.f, 0.f, 0.f, 0.f);
      x[4 * i + 0] = fmaf(a4.x, p.alpha, bz.x); x[4 * i + 1] = fmaf(a4.y, p.alpha, bz.y);
      x[4 * i + 2] = fmaf(a4.z, p.alpha, bz.z); x[4 * i + 3] = fmaf(a4.w, p.alpha, bz.w);
    }
    if (res_b && res_first) {
#pragma unroll
      for (int i = 0; i < NI; ++i) { x[4 * i] += rz[i].x; x[4 * i + 1] += rz[i].y; x[4 * i + 2] += rz[i].z; x[4 * i + 3] += rz[i].w; }
    }
    if (act == 1) {
#pragma unroll
      for (int e = 0; e < 4 * NI; ++e) x[e] = __fdividef(x[e], 1.0f + __expf(-1.702f * x[e]));
    } else if (act == 2) {
#pragma unroll
      for (int e = 0; e < 4 * NI; ++e) x[e] = x[e] > 0.f ? x[e] : 0.2f * x[e];
    } else if (act == 3) {
#pragma unroll
      for (int e = 0; e < 4 * NI; ++e) {  // tanh(x) = 1 - 2 / (1 + exp(2x)), clamped so exp stays finite
        const float z = fminf(fmaxf(x[e], -15.f), 15.f);
        x[e] = 1.0f - __fdividef(2.0f, 1.0f + __expf(2.0f * z));
      }
    } else if (act == 4) {
#pragma unroll
      for (int e = 0; e < 4 * NI; ++e) x[e] = x[e] < 0.f ? 0.f : x[e];  // a NaN passes through, as in torch.relu
    }
    if (res_b && !res_first) {
#pragma unroll
      for (int i = 0; i < NI; ++i) { x[4 * i] += rz[i].x; x[4 * i + 1] += rz[i].y; x[4 * i + 2] += rz[i].z; x[4 * i + 3] += rz[i].w; }
    }
    if (do_round) {
#pragma unroll
      for (int e = 0; e < 4 * NI; ++e) x[e] = round_tf32(x[e]);
    }
    if (has_geo) {
#pragma unroll
      for (int i = 0; i < NI; ++i)
        if (!((in_mask >> i) & 1u)) { x[4 * i] = 0.f; x[4 * i + 1] = 0.f; x[4 * i + 2] = 0.f; x[4 * i + 3] = 0.f; }
    }
    if (p.amax_out) {  // calibration runs only: largest magnitude this launch would store
      // integer max over the bit patterns of |x|: non-negative floats order like their bits and a NaN (sign cleared by fabsf) sorts above
      // +inf, so a NaN survives into amax_out exactly as in the scalar path's atomicMax (fmaxf would drop it and calibration would pass)
      int mi = 0;
#pragma unroll
      for (int i = 0; i < NI; ++i)
        if ((ok_mask >> i) & 1u)
#pragma unroll
          for (int e = 0; e < 4; ++e) mi = max(mi, __float_as_int(fabsf(x[4 * i + e])));
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) mi = max(mi, __shfl_xor_sync(0xffffffffu, mi, o));
      if (lane == 0) atomicMax(reinterpret_cast<int*>(p.amax_out), mi);
    }
    if (p.flags & DSB_GEMM_NO_STORE) {
    } else if (out_mode == 0) {
      float* op = reinterpret_cast<float*>(p.out) + out_boff + (long long)(row_base + rsub) * p.ldo + col;
#pragma unroll
      for (int i = 0; i < NI; ++i)
        if ((ok_mask >> i) & 1u) *reinterpret_cast<float4*>(op + (long long)i * 4 * p.ldo) = make_float4(x[4 * i], x[4 * i + 1], x[4 * i + 2], x[4 * i + 3]);
    } else if (out_mode == 1) {
      __half* op = reinterpret_cast<__half*>(p.out) + out_boff + (long long)(row_base + rsub) * p.ldo + col;
#pragma unroll
      for (int i = 0; i < NI; ++i)
        if ((ok_mask >> i) & 1u) {
          __half2 h0 = __floats2half2_rn(x[4 * i], x[4 * i + 1]), h1 = __floats2half2_rn(x[4 * i + 2], x[4 * i + 3]);
          uint2 u;
          u.x = *reinterpret_cast<uint32_t*>(&h0); u.y = *reinterpret_cast<uint32_t*>(&h1);
          *reinterpret_cast<uint2*>(op + (long long)i * 4 * p.ldo) = u;
        }
    } else if (out_mode == 3) {  // fp16 (hi | lo) pair: the A operand of a split-fp16 GEMM / attention
      const int ocol = p.ocg > 0 ? (col / p.ocg) * p.ocg_stride + col % p.ocg : col;
      __half* op = reinterpret_cast<__half*>(p.out) + out_boff + (long long)(row_base + rsub) * p.ldo + ocol;
#pragma unroll 1
      for (int pass = 0; pass < (dual ? 2 : 1); ++pass) {
#pragma unroll
        for (int i = 0; i < NI; ++i)
          if ((ok_mask >> i) & 1u) {
            const __half2 h0 = __floats2half2_rn(x[4 * i], x[4 * i + 1]), h1 = __floats2half2_rn(x[4 * i + 2], x[4 * i + 3]);
            const __half2 l0 = __floats2half2_rn(x[4 * i] - __low2float(h0), x[4 * i + 1] - __high2float(h0));
            const __half2 l1 = __floats2half2_rn(x[4 * i + 2] - __low2float(h1), x[4 * i + 3] - __high2float(h1));
            uint2 u, w;
            u.x = *reinterpret_cast<const uint32_t*>(&h0); u.y = *reinterpret_cast<const uint32_t*>(&h1);
            w.x = *reinterpret_cast<const uint32_t*>(&l0); w.y = *reinterpret_cast<const uint32_t*>(&l1);
            *reinterpret_cast<uint2*>(op + (long long)i * 4 * p.ldo) = u;
            *reinterpret_cast<uint2*>(op + (long long)i * 4 * p.ldo + p.split_off) = w;
          }
        if (dual) {  // second copy: LeakyReLU(0.2) of the value just stored (the next conv's input; the raw copy feeds the 1x1 shortcut)
#pragma unroll
          for (int e = 0; e < 4 * NI; ++e) x[e] = x[e] > 0.f ? x[e] : 0.2f * x[e];
          op += p.dual_off;
        }
      }
    } else {
      __nv_bfloat16* op = reinterpret_cast<__nv_bfloat16*>(p.out) + out_boff + (long long)(row_base + rsub) * p.ldo + col;
#pragma unroll
      for (int i = 0; i < NI; ++i)
        if ((ok_mask >> i) & 1u) {
          __nv_bfloat162 h0 = __floats2bfloat162_rn(x[4 * i], x[4 * i + 1]), h1 = __floats2bfloat162_rn(x[4 * i + 2], x[4 * i + 3]);
          uint2 u;
          u.x = *reinterpret_cast<uint32_t*>(&h0); u.y = *reinterpret_cast<uint32_t*>(&h1);
          *reinterpret_cast<uint2*>(op + (long long)i * 4 * p.ldo) = u;
        }
    }
  } else {
    // ---------------- slow path (N tail, unaligned leading dimensions): rolled scalar loops, rarely taken
#pragma unroll 1
    for (int i = 0; i < NI; ++i) {
      if (!((ok_mask >> i) & 1u)) continue;
      const int r = i * 4 + rsub;
      const long long row = row_base + r;
      const float4 a4 = *reinterpret_cast<const float4*>(sw + r * 32 + ((c4 ^ (r & 7)) << 2));
      const float av[4] = {a4.x, a4.y, a4.z, a4.w};
#pragma unroll 1
      for (int k = 0; k < 4; ++k) {
        if (col + k >= p.N) break;
        float xv = av[k] * p.alpha + (p.bias ? __ldg(p.bias + col + k) : 0.f);
        const float rv = res_b ? res_b[row * p.ld_res + col + k] : 0.f;
        if (res_first) xv += rv;
        if (act == 1) xv = __fdividef(xv, 1.0f + __expf(-1.702f * xv));
        else if (act == 2) xv = xv > 0.f ? xv : 0.2f * xv;
        else if (act == 3) { const float z = fminf(fmaxf(xv, -15.f), 15.f); xv = 1.0f - __fdividef(2.0f, 1.0f + __expf(2.0f * z)); }
        else if (act == 4) xv = xv < 0.f ? 0.f : xv;
        if (!res_first) xv += rv;
        if (do_round) xv = round_tf32(xv);
        if (!((in_mask >> i) & 1u)) xv = 0.f;
        const long long o = out_boff + row * p.ldo + col + k;
        if (p.amax_out) atomicMax(reinterpret_cast<int*>(p.amax_out), __float_as_int(fabsf(xv)));
        if (p.flags & DSB_GEMM_NO_STORE) continue;
        if (out_mode == 0) reinterpret_cast<float*>(p.out)[o] = xv;
        else if (out_mode == 1) reinterpret_cast<__half*>(p.out)[o] = __float2half_rn(xv);
        else if (out_mode == 3) {
          const int cc = col + k;
          const long long o3 = out_boff + row * p.ldo + (p.ocg > 0 ? (cc / p.ocg) * p.ocg_stride + cc % p.ocg : cc);
          __half hv = __float2half_rn(xv);
          reinterpret_cast<__half*>(p.out)[o3] = hv;
          reinterpret_cast<__half*>(p.out)[o3 + p.split_off] = __float2half_rn(xv - __half2float(hv));
          if (dual) {
            const float yv = xv > 0.f ? xv : 0.2f * xv;
            hv = __float2half_rn(yv);
            reinterpret_cast<__half*>(p.out)[o3 + p.dual_off] = hv;
            reinterpret_cast<__half*>(p.out)[o3 + p.dual_off + p.split_off] = __float2half_rn(yv - __half2float(hv));
          }
        }
        else reinterpret_cast<__nv_bfloat16*>(p.out)[o] = __float2bfloat16(xv);
      }
    }
  }
}

// One k-block of MMAs for this consumer warpgroup's 64 rows: NH halves of 128 columns, 4 K slices of 32 bytes (K-major) / 16 rows (MN-major).
template <int KIND, int TA, int TB, int NH, bool F3>
__device__ __forceinline__ void mma_kblock(float (&acc)[NH][64], uint32_t sa, int wg, uint32_t first) {
  using S = GemmSmem<NH * 128, F3>;
  // A: this warpgroup's 64 rows (K-major: 64 rows x 128 B further; MN-major: the second 64-column box)
  const uint32_t a_off = TA ? wg * MN_BOX_BYTES : wg * 64 * ROW_BYTES;
  const uint32_t b_base = sa + (F3 ? 2 : 1) * S::A_BYTES;
  constexpr uint32_t a_step = TA ? (16 * ROW_BYTES) >> 4 : 2, b_step = TB ? (16 * ROW_BYTES) >> 4 : 2;
  const uint32_t lbo_a = TA ? MN_BOX_BYTES : 16, lbo_b = TB ? MN_BOX_BYTES : 16;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
#pragma unroll
    for (int h = 0; h < NH; ++h) {
      // the second 128 columns of B: 128 K-major rows, or two 64-column MN-major boxes, further = 16 KB either way
      const uint64_t db = make_sw128_desc(b_base + h * 128 * ROW_BYTES, lbo_b) + b_step * k;
      const uint64_t da = make_sw128_desc(sa + a_off, lbo_a) + a_step * k;
      if constexpr (F3) {  // lo*hi, hi*lo, hi*hi off one staged copy of [A hi | A lo | W hi | W lo]
        const uint64_t da_lo = make_sw128_desc(sa + S::A_BYTES + a_off, lbo_a) + a_step * k;
        const uint64_t db_lo = make_sw128_desc(b_base + S::B_BYTES + h * 128 * ROW_BYTES, lbo_b) + b_step * k;
        wgmma_m64n128<KIND, TA, TB>(acc[h], da_lo, db, (first | k) != 0 ? 1u : 0u);
        wgmma_m64n128<KIND, TA, TB>(acc[h], da, db_lo, 1u);
        wgmma_m64n128<KIND, TA, TB>(acc[h], da, db, 1u);
      } else {
        wgmma_m64n128<KIND, TA, TB>(acc[h], da, db, (first | k) != 0 ? 1u : 0u);
      }
    }
  }
}

template <int BLOCK_N, int KIND, bool F3>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_a2, const __grid_constant__ CUtensorMap tmap_b,
                  const __grid_constant__ GemmParams p) {
  using S = GemmSmem<BLOCK_N, F3>;
  constexpr int STAGES = S::STAGES;
  constexpr int NH = BLOCK_N / 128;
  static_assert(!F3 || NH == 1, "the split-fp16 form runs 128-wide tiles");
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  float* epi_smem = reinterpret_cast<float*>(smem + STAGES * S::STAGE_BYTES);  // 8 consumer warps x 16 x 32 floats (XOR-swizzled)
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * S::STAGE_BYTES + S::EPI_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int num_tiles = p.tiles_m * p.tiles_n * p.batch;
  // k-blocks per tile: (tap, channel block) pairs; the f16x3 form runs kb_per_tap blocks for each spatial tap
  const int num_kb = F3 ? p.kb_per_tap * p.f3_nsp : p.kb_per_tap * p.num_taps;
  const dsb_sk::Work work = dsb_sk::cta_work(num_tiles, num_kb, gridDim.x, blockIdx.x, p.stream_k != 0);
  const int n_pieces = dsb_sk::num_pieces(work);

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmap_a);
    prefetch_tmap(&tmap_a2);
    prefetch_tmap(&tmap_b);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 8);  // one arrive per consumer warp, after its own wgmma wait
    }
    fence_barrier_init();
  }
  __syncthreads();
  // everything above (barrier init, tensor-map prefetch) overlapped the predecessor's tail
  pdl_wait();
  pdl_trigger();

  if (warp < 4) {
    // ------------------------------------------------------------ TMA producer
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int pi = 0; pi < n_pieces; ++pi) {
        const dsb_sk::Piece pc = dsb_sk::piece(work, num_kb, pi);
        const int m_blk = pc.tile % p.tiles_m;
        const int n_blk = (pc.tile / p.tiles_m) % p.tiles_n;
        const int b = pc.tile / (p.tiles_m * p.tiles_n);
        for (int kb = pc.kb0; kb < pc.kb1; ++kb) {
          const int tap = kb / p.kb_per_tap;
          const int c0 = (kb - tap * p.kb_per_tap) * p.block_k;
          mbar_wait(&empty_bar[stage], phase ^ 1);
          mbar_arrive_expect_tx(&full_bar[stage], S::STAGE_BYTES);
          uint8_t* sa = smem + stage * S::STAGE_BYTES;
          if constexpr (F3) {
            const int arow = m_blk * BLOCK_M + p.tap_shift[tap], acol = p.tap_acol[tap] + c0, wcol = p.tap_wcol[tap] + c0;
            tma_load_3d(&tmap_a, &full_bar[stage], sa, acol, arow, b);
            tma_load_3d(&tmap_a, &full_bar[stage], sa + S::A_BYTES, acol + p.lo_a, arow, b);
            tma_load_3d(&tmap_b, &full_bar[stage], sa + 2 * S::A_BYTES, wcol, n_blk * BLOCK_N, 0);
            tma_load_3d(&tmap_b, &full_bar[stage], sa + 2 * S::A_BYTES + S::B_BYTES, wcol + p.lo_w, n_blk * BLOCK_N, 0);
          } else {
            if (p.a_mn) {
#pragma unroll
              for (int j = 0; j < BLOCK_M / 64; ++j) tma_load_3d(&tmap_a, &full_bar[stage], sa + j * MN_BOX_BYTES, m_blk * BLOCK_M + j * 64, c0, b);
            } else {
              tma_load_3d(((p.tap_a2_mask >> tap) & 1u) ? &tmap_a2 : &tmap_a, &full_bar[stage], sa, c0 + p.tap_acol[tap], m_blk * BLOCK_M + p.tap_shift[tap], b);
            }
            if (p.b_mn) {
#pragma unroll
              for (int j = 0; j < BLOCK_N / 64; ++j)
                tma_load_3d(&tmap_b, &full_bar[stage], sa + S::A_BYTES + j * MN_BOX_BYTES, n_blk * BLOCK_N + j * 64, c0, p.b_batched ? b : 0);
            } else {
              tma_load_3d(&tmap_b, &full_bar[stage], sa + S::A_BYTES, p.tap_wcol[tap] + c0, n_blk * BLOCK_N, p.b_batched ? b : 0);
            }
          }
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ------------------------------------------------------------ consumers: warpgroup wg owns rows [64 wg, 64 wg + 64) of every tile
    setmaxnreg_inc<232>();
    const int wg = (warp >> 2) - 1;
    const int wq = warp & 3;  // 16-row slab of the warpgroup's 64 rows
    float* sw = epi_smem + (warp - 4) * (EPI_ROWS * 32);
    const bool vec_ok = ((p.ldo & 3) == 0) && ((p.out_bstride & 3) == 0) && ((p.split_off & 3) == 0) && ((p.dual_off & 3) == 0) && ((p.ocg & 3) == 0) &&
                        ((p.ocg_stride & 3) == 0) &&
                        ((reinterpret_cast<uintptr_t>(p.out) & (4 * ((p.flags & (DSB_GEMM_OUT_F16_SPLIT | DSB_GEMM_OUT_F16 | DSB_GEMM_OUT_BF16)) ? 2 : 4) - 1)) == 0) &&
                        (!p.residual || (((p.ld_res & 3) == 0) && ((p.res_bstride & 3) == 0) && ((reinterpret_cast<uintptr_t>(p.residual) & 15) == 0))) &&
                        (!p.bias || ((reinterpret_cast<uintptr_t>(p.bias) & 15) == 0));
    const int ct = threadIdx.x - 128;  // consumer thread 0..255: its accumulator fragment's place in a stream-K slot
    int stage = 0;
    uint32_t phase = 0;
    for (int pi = 0; pi < n_pieces; ++pi) {
      const dsb_sk::Piece pc = dsb_sk::piece(work, num_kb, pi);
      const int m_blk = pc.tile % p.tiles_m;
      const int n_blk = (pc.tile / p.tiles_m) % p.tiles_n;
      const int b = pc.tile / (p.tiles_m * p.tiles_n);
      float acc[NH][64];
      const bool tail = pc.kb0 > 0;  // stream-K tail: continue from the accumulator CTA blockIdx.x - 1 published for k-blocks [0, kb0)
      if (tail) {
        if (ct == 0) {
          int* flag = p.sk_flag + blockIdx.x - 1;
          unsigned spins = 0;
          while (ld_acquire_gpu(flag) == 0) {
            if (++spins > SK_SPIN_LIMIT) __trap();
            __nanosleep(64);
          }
          *flag = 0;  // consumed: the next launch finds the flag clear
        }
        named_bar_sync(1, 256);
      }
      {
        const float4* slot = reinterpret_cast<const float4*>(p.sk_part + (size_t)(blockIdx.x - 1) * NH * SK_SLOT_FLOATS);
#pragma unroll
        for (int h = 0; h < NH; ++h)
#pragma unroll
          for (int q = 0; q < 16; ++q) {
            const float4 v = tail ? __ldcg(slot + (h * 16 + q) * 256 + ct) : make_float4(0.f, 0.f, 0.f, 0.f);  // __ldcg: L2, not a stale L1 line
            acc[h][4 * q] = v.x; acc[h][4 * q + 1] = v.y; acc[h][4 * q + 2] = v.z; acc[h][4 * q + 3] = v.w;
          }
      }
      int prev_stage = -1;
      if constexpr (F3) {
        // parity-grade form: the wgmma accumulator does not round every addition like an fp32 FADD, which over K = 4096 costs more than
        // the 22-bit operands allow; each k-block's 3 x 64-deep partial sum is therefore promoted into the fp32 accumulator with FADDs.
        // The pipe drains once per k-block for this.  Overlapping the promotion with the next k-block (two partial accumulators,
        // wgmma_wait<1>) measured slower on an H100, see DESIGN section 4.
        float part[64];
        for (int kb = pc.kb0; kb < pc.kb1; ++kb) {
          mbar_wait(&full_bar[stage], phase);
          const uint32_t sa = smem_u32(smem + stage * S::STAGE_BYTES);
          wgmma_fence_regs(part);
          wgmma_fence();
          float(&pp)[1][64] = *reinterpret_cast<float(*)[1][64]>(&part);
          mma_kblock<KIND, 0, 0, 1, true>(pp, sa, wg, 0);
          wgmma_commit();
          wgmma_wait<0>();
          wgmma_fence_regs(part);
          if (lane == 0) mbar_arrive(&empty_bar[stage]);
#pragma unroll
          for (int i = 0; i < 64; ++i) acc[0][i] += part[i];
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      } else {
        // the MN-major choice is made once per tile, outside the wgmma window: a branch between wgmma_fence and commit makes
        // ptxas inject warpgroup.arrive (C7519) around every MMA
        // kb is absolute, so a stream-K tail's first k-block accumulates onto the loaded partial (scale-d = 1)
        auto mainloop = [&](auto ta, auto tb) {
          for (int kb = pc.kb0; kb < pc.kb1; ++kb) {
            mbar_wait(&full_bar[stage], phase);
            const uint32_t sa = smem_u32(smem + stage * S::STAGE_BYTES);
#pragma unroll
            for (int h = 0; h < NH; ++h) wgmma_fence_regs(acc[h]);
            wgmma_fence();
            mma_kblock<KIND, decltype(ta)::value, decltype(tb)::value, NH, false>(acc, sa, wg, kb);
            wgmma_commit();
#pragma unroll
            for (int h = 0; h < NH; ++h) wgmma_fence_regs(acc[h]);
            // keep one k-block of MMAs in flight: the previous one has retired, so its smem slot goes back to the producer
            wgmma_wait<1>();
            if (prev_stage >= 0 && lane == 0) mbar_arrive(&empty_bar[prev_stage]);
            prev_stage = stage;
            if (++stage == STAGES) { stage = 0; phase ^= 1; }
          }
        };
        using K0 = std::integral_constant<int, 0>;
        using K1 = std::integral_constant<int, 1>;
        if constexpr (KIND == DSB_DTYPE_TF32) mainloop(K0{}, K0{});
        else if (!p.a_mn && !p.b_mn) mainloop(K0{}, K0{});
        else if (p.a_mn && !p.b_mn) mainloop(K1{}, K0{});
        else if (!p.a_mn) mainloop(K0{}, K1{});
        else mainloop(K1{}, K1{});
      }
      wgmma_wait<0>();
#pragma unroll
      for (int h = 0; h < NH; ++h) wgmma_fence_regs(acc[h]);
      if (prev_stage >= 0 && lane == 0) mbar_arrive(&empty_bar[prev_stage]);

      if (pc.kb1 < num_kb) {
        // stream-K head (this CTA's first piece): publish the partial accumulator to slot blockIdx.x for CTA blockIdx.x + 1
        float4* slot = reinterpret_cast<float4*>(p.sk_part + (size_t)blockIdx.x * NH * SK_SLOT_FLOATS);
#pragma unroll
        for (int h = 0; h < NH; ++h)
#pragma unroll
          for (int q = 0; q < 16; ++q) __stcg(slot + (h * 16 + q) * 256 + ct, make_float4(acc[h][4 * q], acc[h][4 * q + 1], acc[h][4 * q + 2], acc[h][4 * q + 3]));
        __threadfence();
        named_bar_sync(1, 256);
        if (ct == 0) st_release_gpu(p.sk_flag + blockIdx.x, 1);
        continue;
      }

      // ---- epilogue: accumulator fragment (rows lane/4 and lane/4 + 8 of this warp's 16, columns 8j + 2(lane%4) + {0,1}) -> smem chunk -> stores
      const int row_base = m_blk * BLOCK_M + wg * 64 + wq * 16;
      const int n_chunks = min(BLOCK_N / 32, (p.N - n_blk * BLOCK_N + 31) / 32);
      const int r0 = lane >> 2, cc = 2 * (lane & 3);
#pragma unroll
      for (int c = 0; c < BLOCK_N / 32; ++c) {
        if (c < n_chunks) {
          const int h = c >> 2, j0 = (c & 3) * 4;
#pragma unroll
          for (int jj = 0; jj < 4; ++jj) {
            const int col = 8 * jj + cc;
            *reinterpret_cast<float2*>(sw + r0 * 32 + (((col >> 2) ^ (r0 & 7)) << 2) + (col & 3)) =
                make_float2(acc[h][4 * (j0 + jj)], acc[h][4 * (j0 + jj) + 1]);
            *reinterpret_cast<float2*>(sw + (r0 + 8) * 32 + (((col >> 2) ^ ((r0 + 8) & 7)) << 2) + (col & 3)) =
                make_float2(acc[h][4 * (j0 + jj) + 2], acc[h][4 * (j0 + jj) + 3]);
          }
          __syncwarp();
          epilogue_chunk(p, sw, row_base, n_blk * BLOCK_N + c * 32, b, lane, vec_ok);
          __syncwarp();  // the smem tile is rewritten by the next chunk
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------ host side
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess && qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(p);
  }
  return fn;
}

// 3-D map (K, rows, batch) over a K-contiguous matrix; box = (128 bytes of K, box_rows, 1); SWIZZLE_128B; OOB -> 0
int make_operand_map(CUtensorMap* map, const void* ptr, int kind, long long kdim, long long rows, long long batch,
                            long long ld_elems, long long bstride_elems, int box_rows, int l2_promo_128, int box_bytes) {
  PFN_encodeTiled enc = get_encode();
  DSB_REQUIRE(enc != nullptr, "cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
  DSB_REQUIRE(box_bytes == ROW_BYTES || box_bytes == 64, "make_operand_map: box_bytes must be 128 or 64 (got %d)", box_bytes);
  const int es = kind == DSB_DTYPE_TF32 ? 4 : 2;
  DSB_REQUIRE((reinterpret_cast<uintptr_t>(ptr) & 15) == 0, "GEMM operand pointer must be 16-byte aligned");
  DSB_REQUIRE((ld_elems * es) % 16 == 0, "GEMM operand leading dimension must be a multiple of 16 bytes (ld=%lld)", ld_elems);
  DSB_REQUIRE(batch == 1 || (bstride_elems * es) % 16 == 0, "GEMM batch stride must be a multiple of 16 bytes");
  cuuint64_t gdim[3] = {(cuuint64_t)kdim, (cuuint64_t)rows, (cuuint64_t)batch};
  cuuint64_t gstr[2] = {(cuuint64_t)(ld_elems * es), (cuuint64_t)((batch == 1 ? ld_elems * rows : bstride_elems) * es)};
  cuuint32_t box[3] = {(cuuint32_t)(box_bytes / es), (cuuint32_t)box_rows, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(map, kind == DSB_DTYPE_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : (kind == DSB_DTYPE_F16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32), 3, const_cast<void*>(ptr), gdim, gstr,
                   box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, box_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B,
                   // state rows [raw pair | activated pair] are read one 128-byte half at a time: a 256-byte promotion would fetch the other half too
                   l2_promo_128 ? CU_TENSOR_MAP_L2_PROMOTION_L2_128B : CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  DSB_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed (%d): k=%lld rows=%lld batch=%lld ld=%lld", (int)r, kdim, rows, batch, ld_elems);
  return 0;
}

// 3-D map (MN, K rows, batch) over an MN-contiguous operand; box = (64 columns = 128 bytes, 64 K rows, 1); SWIZZLE_128B; OOB -> 0
int make_operand_map_mn(CUtensorMap* map, const void* ptr, int kind, long long mn, long long krows, long long batch, long long ld_elems,
                        long long bstride_elems) {
  PFN_encodeTiled enc = get_encode();
  DSB_REQUIRE(enc != nullptr, "cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
  DSB_REQUIRE(kind != DSB_DTYPE_TF32, "MN-major GEMM operands are implemented for the 2-byte types only");
  DSB_REQUIRE((reinterpret_cast<uintptr_t>(ptr) & 15) == 0, "GEMM operand pointer must be 16-byte aligned");
  DSB_REQUIRE((ld_elems * 2) % 16 == 0, "GEMM operand leading dimension must be a multiple of 16 bytes (ld=%lld)", ld_elems);
  DSB_REQUIRE(batch == 1 || (bstride_elems * 2) % 16 == 0, "GEMM batch stride must be a multiple of 16 bytes");
  cuuint64_t gdim[3] = {(cuuint64_t)mn, (cuuint64_t)krows, (cuuint64_t)batch};
  cuuint64_t gstr[2] = {(cuuint64_t)(ld_elems * 2), (cuuint64_t)((batch == 1 ? ld_elems * krows : bstride_elems) * 2)};
  cuuint32_t box[3] = {64, 64, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(map, kind == DSB_DTYPE_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, const_cast<void*>(ptr), gdim, gstr,
                   box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  DSB_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled (MN-major) failed (%d): mn=%lld k=%lld batch=%lld ld=%lld", (int)r, mn, krows, batch, ld_elems);
  return 0;
}

// The stream-K workspace of the current device: one 256-wide accumulator slot per SM, then one flag per SM.  Allocated zeroed on the first
// call that is not being captured into a CUDA graph; until then (a first call inside a capture) the caller runs data-parallel.
static int sk_workspace(cudaStream_t st, float** part, int** flag) {
  static std::mutex mu;
  static void* ws[64] = {};
  int dev = 0;
  DSB_CHECK_CUDA(cudaGetDevice(&dev));
  DSB_REQUIRE(dev < 64, "dsb_gemm_ex: device %d out of range for the stream-K workspace", dev);
  std::lock_guard<std::mutex> lock(mu);
  if (!ws[dev]) {
    cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
    DSB_CHECK_CUDA(cudaStreamIsCapturing(st, &cap));
    if (cap != cudaStreamCaptureStatusNone) return 0;
    const size_t bytes = (size_t)sm_count() * (2 * SK_SLOT_FLOATS * sizeof(float) + sizeof(int));
    void* w = nullptr;
    DSB_CHECK_CUDA(cudaMalloc(&w, bytes));
    DSB_CHECK_CUDA(cudaMemsetAsync(w, 0, bytes, st));
    ws[dev] = w;
  }
  *part = static_cast<float*>(ws[dev]);
  *flag = reinterpret_cast<int*>(*part + (size_t)sm_count() * 2 * SK_SLOT_FLOATS);
  return 0;
}

template <int BLOCK_N, int KIND, bool F3>
static int launch(const CUtensorMap& ma, const CUtensorMap& ma2, const CUtensorMap& mb, GemmParams& p, int max_ctas, int schedule, cudaStream_t st) {
  using S = GemmSmem<BLOCK_N, F3>;
  auto kern = gemm_wgmma_kernel<BLOCK_N, KIND, F3>;
  static bool attr_done = false;
  if (!attr_done) {
    DSB_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, S::TOTAL));
    attr_done = true;
  }
  const int tiles = p.tiles_m * p.tiles_n * p.batch;
  int grid = tiles < max_ctas ? tiles : max_ctas;
  const int num_kb = F3 ? p.kb_per_tap * p.f3_nsp : p.kb_per_tap * p.num_taps;
  p.stream_k = 0;
  if (schedule == 0 && dsb_sk::stream_k_applies(tiles, num_kb, grid, sm_count())) {
    if (int r = sk_workspace(st, &p.sk_part, &p.sk_flag)) return r;
    p.stream_k = p.sk_part != nullptr;
  }
  DSB_CHECK_CUDA(launch_pdl(kern, dim3(grid), dim3(GEMM_THREADS), S::TOTAL, st, ma, ma2, mb, p));
  return 0;
}

}  // namespace dsb

using namespace dsb;

extern "C" int dsb_gemm_ex(const dsb_gemm_desc* d, void* stream) {
  DSB_REQUIRE(d != nullptr, "dsb_gemm_ex: null descriptor");
  DSB_REQUIRE(d->M > 0 && d->N > 0 && d->K > 0 && d->batch > 0, "dsb_gemm_ex: bad shape M=%d N=%d K=%d batch=%d", d->M, d->N, d->K, d->batch);
  DSB_REQUIRE(d->num_taps >= 1 && d->num_taps <= MAX_TAPS, "dsb_gemm_ex: num_taps=%d out of range", d->num_taps);
  DSB_REQUIRE(d->dtype == DSB_DTYPE_TF32 || d->dtype == DSB_DTYPE_BF16 || d->dtype == DSB_DTYPE_F16,
              "dsb_gemm_ex: dtype must be TF32, BF16 or F16 (use dsb_gemm_f32 for exact fp32)");
  const int kind = d->dtype;
  const int block_k = kind == DSB_DTYPE_TF32 ? 32 : 64;
  GemmParams p{};
  p.M = d->M; p.N = d->N; p.batch = d->batch;
  p.tiles_m = (d->M + BLOCK_M - 1) / BLOCK_M;
  p.kb_per_tap = (d->K + block_k - 1) / block_k;
  p.block_k = block_k;
  p.num_taps = d->num_taps;
  for (int i = 0; i < MAX_TAPS; ++i) {
    p.tap_shift[i] = i < d->num_taps ? d->tap_shift[i] : 0;
    p.tap_acol[i] = i < d->num_taps ? d->tap_acol[i] : 0;
    p.tap_wcol[i] = i < d->num_taps ? (d->use_tap_wcol ? d->tap_wcol[i] : i * d->K) : 0;
  }
  {
    const int es_ = kind == DSB_DTYPE_TF32 ? 4 : 2;
    for (int i = 0; i < d->num_taps; ++i)
      DSB_REQUIRE((p.tap_acol[i] * es_) % 16 == 0 && (p.tap_wcol[i] * es_) % 16 == 0,
                  "dsb_gemm_ex: tap %d starts at A column %d / W column %d: TMA box coordinates must be multiples of 16 bytes", i, p.tap_acol[i], p.tap_wcol[i]);
  }
  p.split_off = d->split_off > 0 ? d->split_off : d->N;
  p.dual_off = d->dual_off;
  p.amax_out = d->amax_out;
  p.ocg = d->out_col_group; p.ocg_stride = d->out_col_group_stride;
  p.tap_a2_mask = 0;
  if (d->A2) {
    for (int i = 0; i < d->num_taps; ++i)
      if (d->tap_a2[i]) p.tap_a2_mask |= 1u << i;
  }
  DSB_REQUIRE(!(d->flags & DSB_GEMM_DUAL_LRELU) || ((d->flags & DSB_GEMM_OUT_F16_SPLIT) && d->dual_off > 0),
              "dsb_gemm_ex: DSB_GEMM_DUAL_LRELU needs DSB_GEMM_OUT_F16_SPLIT and dual_off > 0");
  DSB_REQUIRE(d->out_col_group == 0 || ((d->flags & DSB_GEMM_OUT_F16_SPLIT) && d->out_col_group % 4 == 0 && d->out_col_group_stride % 4 == 0 && !d->residual),
              "dsb_gemm_ex: output column groups need the split-fp16 output, multiples of 4 and no residual");
  p.kc = d->K;
  p.b_batched = d->w_batch_stride != 0;
  p.bias = d->bias; p.residual = d->residual; p.ld_res = d->ld_res; p.res_bstride = d->res_batch_stride;
  p.out = d->out; p.ldo = d->ldo; p.out_bstride = d->out_batch_stride;
  p.flags = d->flags;
  p.geo_P = d->geo_P; p.geo_Wp = d->geo_Wp; p.geo_y0 = d->geo_y0; p.geo_y1 = d->geo_y1; p.geo_x0 = d->geo_x0; p.geo_x1 = d->geo_x1;
  p.alpha = d->alpha == 0.0f ? 1.0f : d->alpha;
  p.a_mn = d->a_mn_major != 0;
  p.b_mn = d->b_mn_major != 0;
  const bool any_mn = p.a_mn || p.b_mn;
  DSB_REQUIRE(!any_mn || (kind != DSB_DTYPE_TF32 && d->num_taps == 1 && d->tap_shift[0] == 0 && d->tap_acol[0] == 0),
              "dsb_gemm_ex: MN-major operands need a 2-byte dtype and a single unshifted tap");
  if (d->resident_w)
    DSB_REQUIRE(kind != DSB_DTYPE_TF32 && !any_mn && !p.b_batched && d->K == 64 && d->N <= 128 && d->use_tap_wcol,
                "dsb_gemm_ex: resident_w needs a 2-byte dtype, K-major operands, K == 64 per tap, N <= 128, explicit tap_wcol and an unbatched W");
  DSB_REQUIRE(!(any_mn && d->cta_pair > 0), "dsb_gemm_ex: 256 x 256 pair tiles take K-major operands only");
  DSB_REQUIRE(d->schedule == 0 || d->schedule == 1, "dsb_gemm_ex: schedule must be 0 (auto) or 1 (data-parallel only)");

  const int sms = sm_count();
  const int max_ctas = d->max_ctas > 0 ? d->max_ctas : sms;
  // tile-N choice: fewest waves (a 256-wide tile costs two 128-wide ones), then the wider tile (less A re-read)
  int block_n = d->block_n;
  if (block_n == 0 && d->cta_pair > 0) block_n = 256;
  if (block_n == 0) {
    if (d->N <= 128) block_n = 128;
    else {
      const long long t256 = (long long)p.tiles_m * ((d->N + 255) / 256) * d->batch;
      const long long t128 = (long long)p.tiles_m * ((d->N + 127) / 128) * d->batch;
      const long long cost256 = ((t256 + sms - 1) / sms) * 2, cost128 = ((t128 + sms - 1) / sms);
      block_n = cost128 < cost256 ? 128 : 256;
    }
  }
  DSB_REQUIRE(block_n == 128 || block_n == 256, "dsb_gemm_ex: block_n must be 0, 128 or 256");
  // split-fp16 tap list -- per spatial tap j the triple (shift_j, A lo, W hi), (shift_j, A hi, W lo), (shift_j, A hi, W hi) with constant hi -> lo column
  // distances: run the three passes off ONE staged copy of the four tiles (Linear layers: one unshifted triple; convs: 9 / 3 / 2 shifted triples).
  // cta_pair = -1 keeps the plain tap loop (same products, one staged tile pair per tap).
  bool fused3 = kind == DSB_DTYPE_F16 && d->cta_pair >= 0 && d->num_taps % 3 == 0 && !p.tap_a2_mask && !p.b_batched && !any_mn && d->K % 64 == 0;
  int f3_lo_a = 0, f3_lo_w = 0;
  if (fused3) {
    f3_lo_a = p.tap_acol[0] - p.tap_acol[1];
    f3_lo_w = p.tap_wcol[1] - p.tap_wcol[0];
    for (int j = 0; j < d->num_taps && fused3; j += 3)
      fused3 = p.tap_shift[j] == p.tap_shift[j + 1] && p.tap_shift[j] == p.tap_shift[j + 2] && p.tap_acol[j + 1] == p.tap_acol[j + 2] &&
               p.tap_acol[j] - p.tap_acol[j + 1] == f3_lo_a && p.tap_wcol[j] == p.tap_wcol[j + 2] && p.tap_wcol[j + 1] - p.tap_wcol[j] == f3_lo_w;
    fused3 = fused3 && f3_lo_a > 0 && f3_lo_w > 0;
  }
  if (fused3) block_n = 128;  // four tiles per stage: 64 KB at N = 128 leaves room for a 3-deep ring
  p.tiles_n = (d->N + block_n - 1) / block_n;

  CUtensorMap ma, mb;
  const long long a_rows = d->a_rows > 0 ? d->a_rows : d->M;
  if (p.a_mn) {
    if (make_operand_map_mn(&ma, d->A, kind, a_rows, d->K, d->batch, d->lda, d->a_batch_stride)) return 3;
  } else if (make_operand_map(&ma, d->A, kind, d->a_cols > 0 ? d->a_cols : d->K, a_rows, d->batch, d->lda, d->a_batch_stride, BLOCK_M)) return 3;
  if (p.b_mn) {
    if (make_operand_map_mn(&mb, d->W, kind, d->N, d->K, p.b_batched ? d->batch : 1, d->ldw, d->w_batch_stride)) return 3;
  } else if (make_operand_map(&mb, d->W, kind, d->w_cols > 0 ? d->w_cols : (long long)d->K * d->num_taps, d->N, p.b_batched ? d->batch : 1, d->ldw,
                              d->w_batch_stride, block_n)) return 3;
  CUtensorMap ma2 = ma;
  if (p.tap_a2_mask) {
    DSB_REQUIRE(!any_mn, "dsb_gemm_ex: a second A operand is K-major only");
    if (make_operand_map(&ma2, d->A2, kind, d->a2_cols > 0 ? d->a2_cols : d->K, d->a2_rows > 0 ? d->a2_rows : d->M, d->batch, d->lda2, d->a2_batch_stride, BLOCK_M)) return 3;
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (fused3) {
    p.f3_nsp = d->num_taps / 3;
    p.lo_a = f3_lo_a;
    p.lo_w = f3_lo_w;
    for (int j = 0; j < p.f3_nsp; ++j) {  // triple j -> spatial tap j: (row shift, hi-half column of A, hi-half column of W)
      const int sh = p.tap_shift[3 * j], ac = p.tap_acol[3 * j + 1], wc = p.tap_wcol[3 * j];
      p.tap_shift[j] = sh; p.tap_acol[j] = ac; p.tap_wcol[j] = wc;
    }
    return launch<128, DSB_DTYPE_F16, true>(ma, ma2, mb, p, max_ctas, d->schedule, st);
  }
  if (block_n == 256) {
    if (kind == DSB_DTYPE_TF32) return launch<256, DSB_DTYPE_TF32, false>(ma, ma2, mb, p, max_ctas, d->schedule, st);
    if (kind == DSB_DTYPE_BF16) return launch<256, DSB_DTYPE_BF16, false>(ma, ma2, mb, p, max_ctas, d->schedule, st);
    return launch<256, DSB_DTYPE_F16, false>(ma, ma2, mb, p, max_ctas, d->schedule, st);
  }
  if (kind == DSB_DTYPE_TF32) return launch<128, DSB_DTYPE_TF32, false>(ma, ma2, mb, p, max_ctas, d->schedule, st);
  if (kind == DSB_DTYPE_BF16) return launch<128, DSB_DTYPE_BF16, false>(ma, ma2, mb, p, max_ctas, d->schedule, st);
  return launch<128, DSB_DTYPE_F16, false>(ma, ma2, mb, p, max_ctas, d->schedule, st);
}
