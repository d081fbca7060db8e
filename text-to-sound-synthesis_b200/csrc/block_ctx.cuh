// CTA-per-column lane context for codebooks above K = 1055, where one column no longer fits one warp's registers.
// Element k of a column lives in thread k % NT at slot j = k / NT (k = tid + NT j), so a row read by ascending k coalesces.
//
// Every reduction runs in one fixed order that depends on NT alone (never on B, L or other columns), so results are
// batch-invariant and a test can restate them:
//   1. each thread combines its own values in ascending j (done by the caller's loop);
//   2. a warp xor butterfly over offsets 16, 8, 4, 2, 1 (every lane of the warp ends with the same value);
//   3. lane 0 of each warp stores its partial; after one __syncthreads every thread reads the NW partials and combines them
//      in ascending warp order, starting from warp 0's partial.
// Two scratch buffers are used alternately, so one __syncthreads per reduction suffices: a thread can only overwrite a buffer
// after passing the barrier of the next reduction, which every thread reaches after it finished reading the previous one.
// Every thread of the CTA must call every reduction (they contain __syncthreads).
#pragma once
#include <cuda_runtime.h>

namespace dsb {

template <int NT>
struct BlockCtx {
  static_assert(NT % 32 == 0 && NT >= 64 && NT <= 1024, "NT must be a multiple of 32 warps, 64..1024");
  static constexpr int NW = NT / 32;
  double* red;      // shared, 2 * NW doubles
  int tid;
  mutable int par;  // which of the two buffers the next reduction writes

  __device__ __forceinline__ int lane() const { return tid; }
  __device__ __forceinline__ int lanes() const { return NT; }

  template <class V, class Op>
  __device__ __forceinline__ V reduce(V v, Op op) const {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = op(v, __shfl_xor_sync(0xffffffffu, v, o));
    V* slot = reinterpret_cast<V*>(red + par * NW);
    par ^= 1;
    if ((tid & 31) == 0) slot[tid >> 5] = v;
    __syncthreads();
    V r = slot[0];
#pragma unroll
    for (int w = 1; w < NW; ++w) r = op(r, slot[w]);
    return r;
  }
  __device__ __forceinline__ float sumf(float v) const { return reduce(v, [](float a, float b) { return a + b; }); }
  __device__ __forceinline__ double sumd(double v) const { return reduce(v, [](double a, double b) { return a + b; }); }
  __device__ __forceinline__ float maxf(float v) const { return reduce(v, [](float a, float b) { return fmaxf(a, b); }); }
  __device__ __forceinline__ int mini(int v) const { return reduce(v, [](int a, int b) { return min(a, b); }); }
  __device__ __forceinline__ unsigned long long maxu(unsigned long long v) const {
    return reduce(v, [](unsigned long long a, unsigned long long b) { return a > b ? a : b; });
  }
};

}  // namespace dsb
