// Split-fp16 ("f16x3") attention core, templated on the head dimension (64 or 32) -- the parity-grade twin of attention_tc.cu
// (reference transformer_utils.py:48-54 FullAttention, :99-105 CrossAttention: softmax(Q K^T / sqrt(head_dim)) V).
//
// Every operand is an fp16 (hi | lo) pair (x ~ hi + lo, 22 significand bits) produced by the split GEMM epilogue:
//   S = Qlo Khi^T + Qhi Klo^T + Qhi Khi^T : 3 x HD/16 wgmma m64n64k16 (SS) per 64-key chunk into one fp32 accumulator;
//   softmax: flash-style (online max / exp2 / sum) over the chunks in fp32; P is split into (hi | lo) in registers;
//   O += Plo Vhi + Phi Vlo + Phi Vhi      : 12 wgmma m64nHDk16 (RS: P from the S accumulator's registers, V read MN-major) into a
//                                           zeroed partial, folded into the fp32 O with FADDs after the rescale;
//   epilogue: O / rowsum -> (hi | lo) fp16 pair -> shared memory -> 16-byte stores (the A operand of the output projection's split GEMM).
// Persistent, warp-specialised CTAs: one TMA producer warp and two consumer warpgroups.  A unit is (batch, head, pair of 64-row query
// tiles); consumer warpgroup w owns tile 2 * pair + w.  Both consumers read the same K / V chunks from a ring of stages, so each chunk is
// loaded once per pair and the next chunks (and the next unit's first ones) load under the current MMAs.
//
// A head row is HD fp16 = 2 * HD bytes, and that is the swizzle width of every tile: SWIZZLE_128B at head_dim 64, SWIZZLE_64B at 32 (TMA
// boxes of HD columns x 64 rows, wgmma descriptors of the same layout).  Each instantiation lives in its own translation unit:
// attention_tc_split.cu (64) and attention_tc_split_hd32.cu (32); attention_tc_split_causal.cu holds both with CAUSAL set (the autoregressive
// transformer's masked self-attention, Lq == Lk).
#pragma once
#include "common.cuh"
#include "diffsound_b200.h"
#include "wgmma.cuh"
#include <cuda_fp16.h>

namespace dsb {
namespace {
template <int HD>
struct AtCfg {
  static_assert(HD == 64 || HD == 32, "split attention is built for head_dim 64 and 32");
  static constexpr int ROW = 2 * HD;                      // bytes of one head row = swizzle width
  static constexpr int TILE = 64 * ROW;                   // 64 rows x HD fp16: one TMA box
  static constexpr int LCH = HD == 64 ? 3 : 2;            // log2 of the 16-byte chunks per row
  // K/V ring depth, in 64-key chunks.  At head_dim 32 a stage is half as large, but a deeper ring (6, 8, 10) measured within noise of 4
  // (DESIGN.md section 4e), so both keep 4.
  static constexpr int STAGES = 4;
  static constexpr int STAGE_BYTES = 4 * TILE;            // K hi, K lo, V hi, V lo
  static constexpr int Q_BYTES = 2 * TILE;                // Q hi, Q lo of one 64-row tile
  static constexpr int THREADS = 384;                     // warpgroup 0: producer (one thread issues TMA), 1 and 2: consumers
  static constexpr int SMEM = STAGES * STAGE_BYTES + 4 * Q_BYTES + 4 * STAGES * 8 + 1024;
  static constexpr int ACC = HD / 2;                      // fp32 registers per thread of an m64nHD accumulator
  // 16-byte chunk j of row r sits at chunk j ^ swz(r) (the TMA / wgmma swizzle of ROW-byte rows)
  static __device__ __forceinline__ int swz(int r) { return HD == 64 ? (r & 7) : ((r >> 1) & 3); }
  // K-major descriptor (Q, K: ROW-byte rows, 8-row groups 8 * ROW bytes apart)
  static __device__ __forceinline__ uint64_t kmajor(uint32_t a) {
    if constexpr (HD == 64) return make_sw128_kmajor_desc(a);
    else return make_sw64_kmajor_desc(a);
  }
  // MN-major descriptor (V: one box of 64 key rows x HD columns)
  static __device__ __forceinline__ uint64_t mnmajor(uint32_t a) {
    if constexpr (HD == 64) return make_sw128_desc(a, TILE);
    else return make_sw64_desc(a, TILE);
  }
};

struct AtParams {
  int H, Lq, Lk;
  int n_chunks, n_tiles, n_pairs, n_units;  // 64-key chunks, 64-row query tiles per (batch, head), tile pairs, (batch, head, pair) units
  int q_lo_col, k_lo_col, v_lo_col;         // column (element) offset of the lo halves inside the tensor maps
  long long ldo, o_lo_off;
  __half* o;
  float scale_log2e;
};

__device__ __forceinline__ float at_ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ void at_pack_pair(float a, float b, uint32_t& hi, uint32_t& lo) {
  const __half2 h = __floats2half2_rn(a, b);
  const __half2 l = __floats2half2_rn(a - __low2float(h), b - __high2float(h));
  hi = *reinterpret_cast<const uint32_t*>(&h);
  lo = *reinterpret_cast<const uint32_t*>(&l);
}

// O partial += P (A fragment, registers) * V chunk rows [16kk, 16kk + 16) (MN-major)
template <int HD>
__device__ __forceinline__ void at_pv(float (&part)[HD / 2], const uint32_t (&a)[4], uint64_t dv, uint32_t scale_d) {
  if constexpr (HD == 64) wgmma_m64n64_f16_rs<1>(part, a, dv, scale_d);
  else wgmma_m64n32_f16_rs<1>(part, a, dv, scale_d);
}

// One consumer warpgroup, one 64-row query tile (Q hi / lo staged at sq) against every K / V chunk of its (batch, head).
// Accumulator fragment: this thread's rows are wq*16 + lane/4 (r0) and + 8 (r1); entry 4j + {0,1} / {2,3} is column 8j + 2(lane%4) + {0,1}.
// CAUSAL (Lq == Lk): the tile multiplies chunks 0 ... tile only and masks key > row on the diagonal chunk.
template <int HD, bool CAUSAL>
__device__ __forceinline__ void at_tile(const AtParams& p, uint8_t* ring, uint64_t* full, uint64_t* empty, int& stage, uint32_t& phase, uint8_t* sq,
                                        int b, int h, int tile, int wg, int wq, int lane) {
  using C = AtCfg<HD>;
  const int t = lane & 3;
  const uint32_t sq_u = smem_u32(sq);
  float o[C::ACC], s[32], part[C::ACC];
#pragma unroll
  for (int i = 0; i < C::ACC; ++i) o[i] = 0.f;
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
  for (int c = 0; c < (CAUSAL ? tile + 1 : p.n_chunks); ++c) {
    mbar_wait(&full[stage], phase);
    const uint32_t sk = smem_u32(ring + stage * C::STAGE_BYTES);
    wgmma_fence_regs(s);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < HD / 16; ++k) {  // 16 head-dim columns (32 bytes of the swizzled row) per step
      const uint64_t dqh = C::kmajor(sq_u) + 2 * k, dql = C::kmajor(sq_u + C::TILE) + 2 * k;
      const uint64_t dkh = C::kmajor(sk) + 2 * k, dkl = C::kmajor(sk + C::TILE) + 2 * k;
      wgmma_m64n64_f16_ss<0, 0>(s, dql, dkh, k != 0 ? 1u : 0u);
      wgmma_m64n64_f16_ss<0, 0>(s, dqh, dkl, 1u);
      wgmma_m64n64_f16_ss<0, 0>(s, dqh, dkh, 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(s);

    if constexpr (CAUSAL) {
      // only the diagonal chunk (c == tile) holds keys past a row; they include every key past Lk of a stored row (row < Lq = Lk)
      if (c == tile) {
        const int r0 = wq * 16 + (lane >> 2), r1 = r0 + 8;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int key = j * 8 + 2 * t;
          if (key > r0) s[4 * j] = -INFINITY;
          if (key + 1 > r0) s[4 * j + 1] = -INFINITY;
          if (key > r1) s[4 * j + 2] = -INFINITY;
          if (key + 1 > r1) s[4 * j + 3] = -INFINITY;
        }
      }
    } else if ((c + 1) * 64 > p.Lk) {  // keys past Lk (zero rows from the TMA bounds) never enter the softmax
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int key = c * 64 + j * 8 + 2 * t;
        if (key >= p.Lk) { s[4 * j] = -INFINITY; s[4 * j + 2] = -INFINITY; }
        if (key + 1 >= p.Lk) { s[4 * j + 1] = -INFINITY; s[4 * j + 3] = -INFINITY; }
      }
    }
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      mx0 = fmaxf(mx0, fmaxf(s[4 * j], s[4 * j + 1]));
      mx1 = fmaxf(mx1, fmaxf(s[4 * j + 2], s[4 * j + 3]));
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    const float mn0 = fmaxf(m0, mx0), mn1 = fmaxf(m1, mx1);
    const float c0 = at_ex2((m0 - mn0) * p.scale_log2e), c1 = at_ex2((m1 - mn1) * p.scale_log2e);
    const float ms0 = mn0 * p.scale_log2e, ms1 = mn1 * p.scale_log2e;
    m0 = mn0; m1 = mn1;
    l0 *= c0; l1 *= c1;
#pragma unroll
    for (int j = 0; j < HD / 8; ++j) { o[4 * j] *= c0; o[4 * j + 1] *= c0; o[4 * j + 2] *= c1; o[4 * j + 3] *= c1; }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      s[4 * j] = at_ex2(fmaf(s[4 * j], p.scale_log2e, -ms0)); s[4 * j + 1] = at_ex2(fmaf(s[4 * j + 1], p.scale_log2e, -ms0));
      s[4 * j + 2] = at_ex2(fmaf(s[4 * j + 2], p.scale_log2e, -ms1)); s[4 * j + 3] = at_ex2(fmaf(s[4 * j + 3], p.scale_log2e, -ms1));
      l0 += s[4 * j] + s[4 * j + 1];
      l1 += s[4 * j + 2] + s[4 * j + 3];
    }
    // P as A fragments: keys [16kk, 16kk + 16) are accumulator columns 8(2kk) .. 8(2kk + 1) + 7
    uint32_t ph[4][4], pl[4][4];
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      at_pack_pair(s[8 * kk], s[8 * kk + 1], ph[kk][0], pl[kk][0]);
      at_pack_pair(s[8 * kk + 2], s[8 * kk + 3], ph[kk][1], pl[kk][1]);
      at_pack_pair(s[8 * kk + 4], s[8 * kk + 5], ph[kk][2], pl[kk][2]);
      at_pack_pair(s[8 * kk + 6], s[8 * kk + 7], ph[kk][3], pl[kk][3]);
    }
    // the wgmma accumulator does not round every addition like an fp32 FADD: each chunk's 3 x 64-deep P V goes into a fresh partial, then
    // into O with FADDs (the split GEMM promotes per k-block the same way)
    wgmma_fence_regs(part);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {  // 16 keys (16 rows of the MN-major V chunk, 16 * ROW bytes) per step
      const uint64_t dvh = C::mnmajor(sk + 2 * C::TILE) + C::ROW * kk, dvl = C::mnmajor(sk + 3 * C::TILE) + C::ROW * kk;
      at_pv<HD>(part, pl[kk], dvh, kk != 0 ? 1u : 0u);
      at_pv<HD>(part, ph[kk], dvl, 1u);
      at_pv<HD>(part, ph[kk], dvh, 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(part);
    if (lane == 0) mbar_arrive(&empty[stage]);
#pragma unroll
    for (int i = 0; i < C::ACC; ++i) o[i] += part[i];
    if (++stage == C::STAGES) { stage = 0; phase ^= 1; }
  }

  l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const float i0 = __fdividef(1.0f, l0), i1 = __fdividef(1.0f, l1);  // l >= 1 (the row maximum contributes exp2(0)): no IEEE slow path needed
  // the Q tile is dead once every warp's last S has retired: stage the O pair there ([hi tile | lo tile], same swizzle)
  named_bar_sync(1 + wg, 128);
  const int r0 = wq * 16 + (lane >> 2), r1 = r0 + 8;
#pragma unroll
  for (int j = 0; j < HD / 8; ++j) {
    uint32_t hi, lo;
    at_pack_pair(o[4 * j] * i0, o[4 * j + 1] * i0, hi, lo);
    *reinterpret_cast<uint32_t*>(sq + r0 * C::ROW + ((j ^ C::swz(r0)) << 4) + 4 * t) = hi;
    *reinterpret_cast<uint32_t*>(sq + C::TILE + r0 * C::ROW + ((j ^ C::swz(r0)) << 4) + 4 * t) = lo;
    at_pack_pair(o[4 * j + 2] * i1, o[4 * j + 3] * i1, hi, lo);
    *reinterpret_cast<uint32_t*>(sq + r1 * C::ROW + ((j ^ C::swz(r1)) << 4) + 4 * t) = hi;
    *reinterpret_cast<uint32_t*>(sq + C::TILE + r1 * C::ROW + ((j ^ C::swz(r1)) << 4) + 4 * t) = lo;
  }
  named_bar_sync(1 + wg, 128);
  const int ct = wq * 32 + lane;
  __half* ob = p.o + (long long)b * p.Lq * p.ldo + h * HD;
#pragma unroll
  for (int i = 0; i < HD / 8; ++i) {  // 2 halves x 64 rows x HD/8 sixteen-byte chunks over 128 threads
    const int idx = ct + 128 * i, half = idx >> (6 + C::LCH), r = (idx >> C::LCH) & 63, ch = idx & ((1 << C::LCH) - 1);
    const int row = tile * 64 + r;
    if (row < p.Lq)
      *reinterpret_cast<uint4*>(ob + (long long)row * p.ldo + half * p.o_lo_off + ch * 8) =
          *reinterpret_cast<const uint4*>(sq + half * C::TILE + r * C::ROW + ((ch ^ C::swz(r)) << 4));
  }
  fence_proxy_async_smem();  // these generic reads / writes come before the TMA that refills the tile
}

// Unit u -> (batch, head, tile pair).  Non-causal units run head-major: u = bh * n_pairs + pair.  Causal units run heaviest pair first,
// u = (n_pairs - 1 - pair) * (B * H) + bh, so the persistent CTAs start on the longest key streams and end on the shortest (DESIGN.md
// section 4g); a causal unit streams the K / V chunks up to the diagonal of its pair's odd tile.  Written as constexpr-selected initialisers
// rather than a helper so that the non-causal instantiations compile to the same instructions as before CAUSAL existed.
#define DSB_AT_UNIT(u)                                                                                                           \
  const int bh = CAUSAL ? (u) % (p.n_units / p.n_pairs) : (u) / p.n_pairs,                                                       \
            pair = CAUSAL ? p.n_pairs - 1 - (u) / (p.n_units / p.n_pairs) : (u) - bh * p.n_pairs, b = bh / p.H, h = bh - b * p.H; \
  const int n_stream = CAUSAL ? min(p.n_chunks, 2 * pair + 2) : p.n_chunks

template <int HD, bool CAUSAL>
__global__ void __launch_bounds__(AtCfg<HD>::THREADS, 1)
attention_tc_split_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k, const __grid_constant__ CUtensorMap map_v,
                          const __grid_constant__ AtParams p) {
  using C = AtCfg<HD>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* ring = smem;
  uint8_t* qbuf = ring + C::STAGES * C::STAGE_BYTES;  // [consumer warpgroup][slot]: Q double-buffered, so the next unit's Q loads early
  uint64_t* full = reinterpret_cast<uint64_t*>(qbuf + 4 * C::Q_BYTES);
  uint64_t* empty = full + C::STAGES;
  uint64_t* q_full = empty + C::STAGES;  // [2 * wg + slot]
  uint64_t* q_empty = q_full + 4;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int s = 0; s < C::STAGES; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 8);  // every consumer warp, including those of a warpgroup with no tile in the unit
    }
    for (int i = 0; i < 4; ++i) {
      mbar_init(&q_full[i], 1);
      mbar_init(&q_empty[i], 4);
    }
    fence_barrier_init();
    prefetch_tmap(&map_q); prefetch_tmap(&map_k); prefetch_tmap(&map_v);
  }
  __syncthreads();
  pdl_wait();
  pdl_trigger();

  if (warp < 4) {
    // ------------------------------------------------------------ TMA producer
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      int stage = 0, qn[2] = {0, 0};
      uint32_t phase = 0;
      for (int u = blockIdx.x; u < p.n_units; u += gridDim.x) {
        DSB_AT_UNIT(u);
#pragma unroll
        for (int w = 0; w < 2; ++w) {
          const int tile = 2 * pair + w;
          if (tile >= p.n_tiles) continue;
          const int q = 2 * w + (qn[w] & 1);
          mbar_wait(&q_empty[q], ((qn[w] >> 1) & 1) ^ 1);
          mbar_arrive_expect_tx(&q_full[q], C::Q_BYTES);
          uint8_t* dst = qbuf + q * C::Q_BYTES;
          tma_load_3d(&map_q, &q_full[q], dst, h * HD, tile * 64, b);
          tma_load_3d(&map_q, &q_full[q], dst + C::TILE, p.q_lo_col + h * HD, tile * 64, b);
          ++qn[w];
        }
        for (int c = 0; c < n_stream; ++c) {
          mbar_wait(&empty[stage], phase ^ 1);
          mbar_arrive_expect_tx(&full[stage], C::STAGE_BYTES);
          uint8_t* st = ring + stage * C::STAGE_BYTES;
          tma_load_3d(&map_k, &full[stage], st, h * HD, c * 64, b);
          tma_load_3d(&map_k, &full[stage], st + C::TILE, p.k_lo_col + h * HD, c * 64, b);
          tma_load_3d(&map_v, &full[stage], st + 2 * C::TILE, h * HD, c * 64, b);
          tma_load_3d(&map_v, &full[stage], st + 3 * C::TILE, p.v_lo_col + h * HD, c * 64, b);
          if (++stage == C::STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ------------------------------------------------------------ consumers: warpgroup wg runs query tile 2 * pair + wg of every unit
    setmaxnreg_inc<232>();
    const int wg = (warp >> 2) - 1, wq = warp & 3;
    int stage = 0, qn = 0;
    uint32_t phase = 0;
    for (int u = blockIdx.x; u < p.n_units; u += gridDim.x) {
      DSB_AT_UNIT(u);
      const int tile = 2 * pair + wg;
      if (tile < p.n_tiles) {
        const int q = 2 * wg + (qn & 1);
        mbar_wait(&q_full[q], (qn >> 1) & 1);
        at_tile<HD, CAUSAL>(p, ring, full, empty, stage, phase, qbuf + q * C::Q_BYTES, b, h, tile, wg, wq, lane);
        __syncwarp();
        if (lane == 0) mbar_arrive(&q_empty[q]);
        ++qn;
        if constexpr (CAUSAL) {
          for (int c = tile + 1; c < n_stream; ++c) {  // the pair's odd tile's diagonal chunk: released unread by the even tile
            mbar_wait(&full[stage], phase);
            if (lane == 0) mbar_arrive(&empty[stage]);
            if (++stage == C::STAGES) { stage = 0; phase ^= 1; }
          }
        }
      } else {
        // the odd last tile of a head: this warpgroup only passes the chunks on (waiting for each, so it never runs a ring lap ahead)
        for (int c = 0; c < n_stream; ++c) {
          mbar_wait(&full[stage], phase);
          if (lane == 0) mbar_arrive(&empty[stage]);
          if (++stage == C::STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  }
}

#undef DSB_AT_UNIT

// Host side of dsb_attention_tc_split (HD 64), dsb_attention_tc_split_hd32 (HD 32) and dsb_attention_tc_split_causal (both, CAUSAL);
// `name` prefixes every error message.
template <int HD, bool CAUSAL = false>
int attention_tc_split_launch(const char* name, const void* q, long long ldq, long long q_lo_off, const void* k, long long ldk, long long k_lo_off,
                              const void* v, long long ldv, long long v_lo_off, void* o, long long ldo, long long o_lo_off, int B, int H, int Lq,
                              int Lk, float scale, void* stream) {
  using C = AtCfg<HD>;
  DSB_REQUIRE(B > 0 && H > 0 && Lq > 0 && Lk > 0, "%s: need B, H, Lq, Lk > 0", name);
  DSB_REQUIRE(!CAUSAL || Lq == Lk, "%s: causal attention needs Lq == Lk (got %d, %d)", name, Lq, Lk);
  DSB_REQUIRE(ldo % 8 == 0 && o_lo_off % 8 == 0 && (reinterpret_cast<uintptr_t>(o) & 15) == 0, "%s: o must be 16-byte aligned, ldo / o_lo_off %% 8 == 0",
              name);
  DSB_REQUIRE(q_lo_off >= (long long)H * HD && k_lo_off >= (long long)H * HD && v_lo_off >= (long long)H * HD && o_lo_off >= (long long)H * HD,
              "%s: the lo halves must not overlap the hi halves", name);
  DSB_REQUIRE(q_lo_off + (long long)H * HD <= ldq && k_lo_off + (long long)H * HD <= ldk && v_lo_off + (long long)H * HD <= ldv,
              "%s: lo halves must lie inside a row (lo_off + H*%d <= ld)", name, HD);
  DSB_REQUIRE(ldq % 8 == 0 && (reinterpret_cast<uintptr_t>(q) & 15) == 0, "%s: q must be 16-byte aligned, ldq %% 8 == 0 (TMA)", name);
  AtParams p{};
  p.H = H; p.Lq = Lq; p.Lk = Lk;
  p.n_chunks = (Lk + 63) / 64;
  p.n_tiles = (Lq + 63) / 64;
  // an odd last tile (265 rows: tiles 0-3 full, tile 4 nine rows) runs alone in its unit: pairing it with another head's tile would need a
  // second K / V stream in the ring for 9 useful rows of 64
  p.n_pairs = (p.n_tiles + 1) / 2;
  const long long units = (long long)B * H * p.n_pairs;
  DSB_REQUIRE(units < (1LL << 31), "%s: too many (batch, head, tile pair) units", name);
  p.n_units = (int)units;
  p.q_lo_col = (int)q_lo_off; p.k_lo_col = (int)k_lo_off; p.v_lo_col = (int)v_lo_off;
  p.ldo = ldo; p.o_lo_off = o_lo_off; p.o = (__half*)o;
  p.scale_log2e = scale * 1.4426950408889634f;
  // (columns, rows of one batch, batch) maps with HD-column boxes: rows past Lq / Lk read as zeros instead of the next batch's rows
  CUtensorMap mq, mk, mv;
  if (make_operand_map(&mq, q, DSB_DTYPE_F16, q_lo_off + (long long)H * HD, Lq, B, ldq, (long long)Lq * ldq, 64, 0, C::ROW)) return 3;
  if (make_operand_map(&mk, k, DSB_DTYPE_F16, k_lo_off + (long long)H * HD, Lk, B, ldk, (long long)Lk * ldk, 64, 0, C::ROW)) return 3;
  if (make_operand_map(&mv, v, DSB_DTYPE_F16, v_lo_off + (long long)H * HD, Lk, B, ldv, (long long)Lk * ldv, 64, 0, C::ROW)) return 3;
  static bool attr_set = false;
  if (!attr_set) {
    DSB_CHECK_CUDA(cudaFuncSetAttribute(attention_tc_split_kernel<HD, CAUSAL>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM));
    attr_set = true;
  }
  const int grid = min(p.n_units, sm_count());
  DSB_CHECK_CUDA(launch_pdl(attention_tc_split_kernel<HD, CAUSAL>, dim3(grid), dim3(C::THREADS), C::SMEM, (cudaStream_t)stream, mq, mk, mv, p));
  return 0;
}
}  // namespace
}  // namespace dsb
