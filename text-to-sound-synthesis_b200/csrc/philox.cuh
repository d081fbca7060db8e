// In-kernel replay of ATen's CUDA Philox streams (torch.rand_like, Tensor.exponential_), shared by the diffusion sampler (sampler.cu) and the
// autoregressive sampler (ar_decode.cu).
// ATen fills a contiguous float tensor with distribution_elementwise_grid_stride_kernel (ATen/native/cuda/DistributionTemplates.h): thread
// tid of `nthreads` = 256 * grid runs curand_init(seed, tid, offset) and its c-th curand_uniform4 call yields elements
// tid + nthreads * (4 c + ii), ii = 0..3.  With offset a multiple of 4 (always, for ATen) that is Philox4x32-10 on counter
// (offset / 4 + c, tid) under key = seed, component ii, mapped by curand's _curand_uniform to (0, 1].
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace dsb {

__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
    c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
    k.x += 0x9E3779B9u; k.y += 0xBB67AE85u;
  }
  return c;
}
// curand_uniform4's (0, 1] value for element li of the tensor
__device__ __forceinline__ float aten_curand_uniform(unsigned long long seed, unsigned long long offset, unsigned long long nthreads, unsigned long long li) {
  const unsigned long long tid = li % nthreads, q = li / nthreads;
  const unsigned long long ctr = (offset >> 2) + (q >> 2);
  const uint4 r = philox4x32_10(make_uint4((uint32_t)ctr, (uint32_t)(ctr >> 32), (uint32_t)tid, (uint32_t)(tid >> 32)),
                                make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)));
  const uint32_t ii = (uint32_t)(q & 3ull);
  const uint32_t x = ii == 0 ? r.x : (ii == 1 ? r.y : (ii == 2 ? r.z : r.w));
  return x * 2.3283064e-10f + (2.3283064e-10f / 2.0f);  // _curand_uniform (curand_uniform.h:69-72), same expression / same contraction
}
// torch.rand: uniform_kernel's reverse_bound_value maps (0, 1] to [0, 1) (DistributionTemplates.h:494-502).  The body restates
// aten_curand_uniform instead of calling it so that the diffusion sampler's kernels keep the exact instruction sequence they had.
__device__ __forceinline__ float aten_uniform(unsigned long long seed, unsigned long long offset, unsigned long long nthreads, unsigned long long li) {
  const unsigned long long tid = li % nthreads, q = li / nthreads;
  const unsigned long long ctr = (offset >> 2) + (q >> 2);
  const uint4 r = philox4x32_10(make_uint4((uint32_t)ctr, (uint32_t)(ctr >> 32), (uint32_t)tid, (uint32_t)(tid >> 32)),
                                make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)));
  const uint32_t ii = (uint32_t)(q & 3ull);
  const uint32_t x = ii == 0 ? r.x : (ii == 1 ? r.y : (ii == 2 ? r.z : r.w));
  const float u = x * 2.3283064e-10f + (2.3283064e-10f / 2.0f);
  return u == 1.0f ? 0.0f : u;
}
// Tensor.exponential_(1) on a float tensor: exponential_kernel -> uniform_and_transform (the same stream, no flip) -> transformation::exponential
// (ATen/core/TransformationHelper.h): at::log(u), which is __logf in device code (ATen/NumericUtils.h), except that u >= 1 - eps/2 gives
// -eps/2, then -1 / lambda * log with lambda = 1.
__device__ __forceinline__ float aten_exponential(unsigned long long seed, unsigned long long offset, unsigned long long nthreads, unsigned long long li) {
  const float u = aten_curand_uniform(seed, offset, nthreads, li);
  const float eps_half = 5.9604645e-08f;  // std::numeric_limits<float>::epsilon() / 2
  const float lg = u >= 1.0f - eps_half ? -eps_half : __logf(u);
  return -1.0f / 1.0f * lg;
}

}  // namespace dsb
