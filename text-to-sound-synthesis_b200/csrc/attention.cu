// softmax(Q K^T * scale) V for head_dim 64 and 32, no mask / dropout: FullAttention and CrossAttention cores
// (reference transformer_utils.py:48-54, :99-105; head_dim 32 is Diffsound's caps_small_transformer.yaml).  The (B,16,265,265) score tensor and the discarded head-mean `att`
// (:54, :105) never exist: scores live in registers (online softmax over 64-key chunks staged in shared memory).
// Warp-level mma.sync m16n8k8 TF32.
#include "common.cuh"
#include "diffsound_b200.h"
#include <cuda_fp16.h>

namespace dsb {
constexpr int QT = 64, KT = 64;

__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t tf32_bits(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return r;
}

// KS = HD + 4: padded smem row stride (floats) -> conflict-free fragment loads at both head dims
template <int HD>
__global__ void __launch_bounds__(128)
attention_kernel(const float* __restrict__ q, long long ldq, const float* __restrict__ k, long long ldk, const float* __restrict__ v,
                 long long ldv, float* __restrict__ o, long long ldo, int Lq, int Lk, float scale_log2e, int flags) {
  constexpr int KS = HD + 4, NK = HD / 8, LC4 = HD == 64 ? 4 : 3;  // NK: 8-wide k-steps / output column blocks; 1 << LC4 float4 per row
  __shared__ __align__(16) uint32_t Ks[KT * KS];
  __shared__ __align__(16) uint32_t Vs[KT * KS];
  const int qt = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int r0 = qt * QT + warp * 16;
  const float* qb = q + (long long)b * Lq * ldq + h * HD;
  const float* kb = k + (long long)b * Lk * ldk + h * HD;
  const float* vb = v + (long long)b * Lk * ldv + h * HD;

  pdl_wait();
  pdl_trigger();
  uint32_t a[NK][4];
#pragma unroll
  for (int ks = 0; ks < NK; ++ks) {
    const int ra = r0 + g, rb = r0 + g + 8;
    a[ks][0] = ra < Lq ? tf32_bits(qb[(long long)ra * ldq + ks * 8 + t]) : 0u;
    a[ks][1] = rb < Lq ? tf32_bits(qb[(long long)rb * ldq + ks * 8 + t]) : 0u;
    a[ks][2] = ra < Lq ? tf32_bits(qb[(long long)ra * ldq + ks * 8 + t + 4]) : 0u;
    a[ks][3] = rb < Lq ? tf32_bits(qb[(long long)rb * ldq + ks * 8 + t + 4]) : 0u;
  }
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
  float oacc[NK][4];
#pragma unroll
  for (int i = 0; i < NK; ++i) oacc[i][0] = oacc[i][1] = oacc[i][2] = oacc[i][3] = 0.f;

  const int nchunks = (Lk + KT - 1) / KT;
  for (int kc = 0; kc < nchunks; ++kc) {
    __syncthreads();
    for (int idx = threadIdx.x; idx < KT * (HD / 4); idx += 128) {
      const int row = idx >> LC4, c4 = (idx & ((1 << LC4) - 1)) * 4;
      const int key = kc * KT + row;
      float4 kv = make_float4(0.f, 0.f, 0.f, 0.f), vv = kv;
      if (key < Lk) {
        kv = *reinterpret_cast<const float4*>(kb + (long long)key * ldk + c4);
        vv = *reinterpret_cast<const float4*>(vb + (long long)key * ldv + c4);
      }
      *reinterpret_cast<uint4*>(&Ks[row * KS + c4]) = make_uint4(tf32_bits(kv.x), tf32_bits(kv.y), tf32_bits(kv.z), tf32_bits(kv.w));
      *reinterpret_cast<uint4*>(&Vs[row * KS + c4]) = make_uint4(tf32_bits(vv.x), tf32_bits(vv.y), tf32_bits(vv.z), tf32_bits(vv.w));
    }
    __syncthreads();

    float s[8][4];
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f;
#pragma unroll
      for (int ks = 0; ks < NK; ++ks) {
        const uint32_t b0 = Ks[(nt * 8 + g) * KS + ks * 8 + t];
        const uint32_t b1 = Ks[(nt * 8 + g) * KS + ks * 8 + t + 4];
        mma_tf32(s[nt], a[ks], b0, b1);
      }
    }
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      const int key = kc * KT + nt * 8 + 2 * t;
      if (key >= Lk) { s[nt][0] = -INFINITY; s[nt][2] = -INFINITY; }
      if (key + 1 >= Lk) { s[nt][1] = -INFINITY; s[nt][3] = -INFINITY; }
      mx0 = fmaxf(mx0, fmaxf(s[nt][0], s[nt][1]));
      mx1 = fmaxf(mx1, fmaxf(s[nt][2], s[nt][3]));
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    const float mn0 = fmaxf(m0, mx0), mn1 = fmaxf(m1, mx1);
    const float c0 = exp2f((m0 - mn0) * scale_log2e), c1 = exp2f((m1 - mn1) * scale_log2e);
    m0 = mn0; m1 = mn1;
    l0 *= c0; l1 *= c1;
#pragma unroll
    for (int nd = 0; nd < NK; ++nd) { oacc[nd][0] *= c0; oacc[nd][1] *= c0; oacc[nd][2] *= c1; oacc[nd][3] *= c1; }
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      s[nt][0] = exp2f((s[nt][0] - mn0) * scale_log2e); s[nt][1] = exp2f((s[nt][1] - mn0) * scale_log2e);
      s[nt][2] = exp2f((s[nt][2] - mn1) * scale_log2e); s[nt][3] = exp2f((s[nt][3] - mn1) * scale_log2e);
      l0 += s[nt][0] + s[nt][1];
      l1 += s[nt][2] + s[nt][3];
    }
    // O += P V.  The C fragment of S is reused as the A fragment of P with the key permutation
    // k-slot t <-> key 2t, k-slot t+4 <-> key 2t+1 (the sum over keys is order-free); V rows are read to match.
#pragma unroll
    for (int ks = 0; ks < 8; ++ks) {
      const uint32_t pa[4] = {tf32_bits(s[ks][0]), tf32_bits(s[ks][2]), tf32_bits(s[ks][1]), tf32_bits(s[ks][3])};
#pragma unroll
      for (int nd = 0; nd < NK; ++nd) {
        const uint32_t b0 = Vs[(ks * 8 + 2 * t) * KS + nd * 8 + g];
        const uint32_t b1 = Vs[(ks * 8 + 2 * t + 1) * KS + nd * 8 + g];
        mma_tf32(oacc[nd], pa, b0, b1);
      }
    }
  }
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const float i0 = 1.0f / l0, i1 = 1.0f / l1;
  const bool rnd = (flags & DSB_GEMM_ROUND_TF32) != 0;
  float* ob = o + (long long)b * Lq * ldo + h * HD;
  const int ra = r0 + g, rb = r0 + g + 8;
  if (flags & DSB_GEMM_OUT_F16) {  // `o` is an fp16 buffer with row stride ldo (elements)
    __half* oh = reinterpret_cast<__half*>(o) + (long long)b * Lq * ldo + h * HD;
#pragma unroll
    for (int nd = 0; nd < NK; ++nd) {
      if (ra < Lq) *reinterpret_cast<__half2*>(oh + (long long)ra * ldo + nd * 8 + 2 * t) = __floats2half2_rn(oacc[nd][0] * i0, oacc[nd][1] * i0);
      if (rb < Lq) *reinterpret_cast<__half2*>(oh + (long long)rb * ldo + nd * 8 + 2 * t) = __floats2half2_rn(oacc[nd][2] * i1, oacc[nd][3] * i1);
    }
    return;
  }
#pragma unroll
  for (int nd = 0; nd < NK; ++nd) {
    float2 x = make_float2(oacc[nd][0] * i0, oacc[nd][1] * i0), y = make_float2(oacc[nd][2] * i1, oacc[nd][3] * i1);
    if (rnd) { x.x = round_tf32(x.x); x.y = round_tf32(x.y); y.x = round_tf32(y.x); y.y = round_tf32(y.y); }
    if (ra < Lq) *reinterpret_cast<float2*>(ob + (long long)ra * ldo + nd * 8 + 2 * t) = x;
    if (rb < Lq) *reinterpret_cast<float2*>(ob + (long long)rb * ldo + nd * 8 + 2 * t) = y;
  }
}
}  // namespace dsb
using namespace dsb;

template <int HD>
static int attention_launch(const char* name, const float* q, long long ldq, const float* k, long long ldk, const float* v, long long ldv, float* o,
                            long long ldo, int B, int H, int Lq, int Lk, float scale, int flags, void* stream) {
  DSB_REQUIRE(B > 0 && H > 0 && Lq > 0 && Lk > 0, "%s: bad shape", name);
  DSB_REQUIRE(ldk % 4 == 0 && ldv % 4 == 0 && ldo % 2 == 0, "%s: ldk/ldv must be multiples of 4, ldo of 2", name);
  DSB_REQUIRE(((reinterpret_cast<uintptr_t>(k) | reinterpret_cast<uintptr_t>(v)) & 15) == 0 && (reinterpret_cast<uintptr_t>(o) & 3) == 0,
              "%s: k/v must be 16-byte aligned, o 8-byte aligned", name);
  dim3 grid((Lq + QT - 1) / QT, H, B);
  DSB_CHECK_CUDA(launch_pdl(attention_kernel<HD>, grid, dim3(128), 0, (cudaStream_t)stream, q, ldq, k, ldk, v, ldv, o, ldo, Lq, Lk,
                            scale * 1.4426950408889634f, flags));
  return 0;
}

extern "C" int dsb_attention(const float* q, long long ldq, const float* k, long long ldk, const float* v, long long ldv, float* o, long long ldo,
                             int B, int H, int Lq, int Lk, float scale, int flags, void* stream) {
  return attention_launch<64>("dsb_attention", q, ldq, k, ldk, v, ldv, o, ldo, B, H, Lq, Lk, scale, flags, stream);
}

extern "C" int dsb_attention_hd32(const float* q, long long ldq, const float* k, long long ldk, const float* v, long long ldv, float* o, long long ldo,
                                  int B, int H, int Lq, int Lk, float scale, int flags, void* stream) {
  return attention_launch<32>("dsb_attention_hd32", q, ldq, k, ldk, v, ldv, o, ldo, B, H, Lq, Lk, scale, flags, stream);
}
