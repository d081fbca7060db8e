// Shared device/host helpers for the Diffsound kernels (sm_90a, Hopper).
// Raw PTX wrappers for mbarrier / TMA / wgmma -- no CUTLASS dependency.
#pragma once
#include <cuda_runtime.h>
#include <cuda.h>
#include <cstdint>
#include <cstdio>

namespace dsb {

// ---------------------------------------------------------------- error plumbing (host)
void set_error(const char* fmt, ...);
#define DSB_CHECK_CUDA(expr)                                                                    \
  do {                                                                                          \
    cudaError_t _e = (expr);                                                                    \
    if (_e != cudaSuccess) {                                                                    \
      dsb::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e));     \
      return 1;                                                                                 \
    }                                                                                           \
  } while (0)
#define DSB_REQUIRE(cond, ...)                                                                  \
  do {                                                                                          \
    if (!(cond)) {                                                                              \
      dsb::set_error(__VA_ARGS__);                                                              \
      return 2;                                                                                 \
    }                                                                                           \
  } while (0)

int sm_count();
// 3-D TMA map (K, rows, batch) over a K-contiguous matrix; box = (box_bytes of K, box_rows, 1); SWIZZLE_128B for 128-byte boxes, SWIZZLE_64B
// for 64-byte ones; OOB reads give zeros.  kind: DSB_DTYPE_TF32 (fp32 elements) / BF16 / F16.  Returns non-zero and sets the error string on
// failure.  (gemm_wgmma.cu)
int make_operand_map(CUtensorMap* map, const void* ptr, int kind, long long kdim, long long rows, long long batch, long long ld_elems,
                     long long bstride_elems, int box_rows, int l2_promo_128 = 0, int box_bytes = 128);
bool pdl_enabled();  // programmatic dependent launch (env DSB_PDL=0 disables)

// Launch with the programmatic-stream-serialization attribute: the grid may be scheduled while its predecessor drains; the
// kernel calls pdl_wait() before touching anything the predecessor wrote.
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kern, KArgs(args)...);
}

// ---------------------------------------------------------------- small device utils
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31; }

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t}"
      : "=r"(pred));
  return pred != 0;
}

// round-to-nearest fp32 -> tf32 (kept in an fp32 container; low 13 mantissa bits zero)
__device__ __forceinline__ float round_tf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}

// programmatic dependent launch: wait for the predecessor grid(s) to complete and flush; let the successor start launching
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug traps (=> launch error reported to the host) instead of hanging the GPU.
// No printf on the timeout path: it compiles to a call, and ptxas serialises every wgmma of a mainloop that can reach a call
// (C7510).  Build with -DDSB_MBAR_DEBUG to print the waiting block / thread before the trap, at that cost.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > (1u << 26)) {
#ifdef DSB_MBAR_DEBUG
      printf("dsb: mbarrier wait timeout (block %d thread %d)\n", blockIdx.x, threadIdx.x);
#endif
      __trap();
    }
  }
}

// ---------------------------------------------------------------- inter-CTA flags (global memory, GPU scope)
__device__ __forceinline__ int ld_acquire_gpu(const int* p) {
  int v;
  asm volatile("ld.acquire.gpu.global.b32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_gpu(int* p, int v) { asm volatile("st.release.gpu.global.b32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
// barrier over a subset of the block's warps (id 0 is __syncthreads)
__device__ __forceinline__ void named_bar_sync(int id, int threads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory"); }

// ---------------------------------------------------------------- TMA (cp.async.bulk.tensor)
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_3d(const CUtensorMap* m, uint64_t* bar, void* dst, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}

// ---------------------------------------------------------------- wgmma (warpgroup MMA, accumulators in registers)
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across an in-flight wgmma
template <int N>
__device__ __forceinline__ void wgmma_fence_regs(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
template <uint32_t R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
template <uint32_t R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }

// wgmma shared-memory matrix descriptor, SWIZZLE_128B (layout type 1 @62), 1024-byte aligned tiles (base offset 0):
//   [0,14) start>>4 | [16,30) LBO>>4 | [32,46) SBO>>4
// K-major (128-byte rows, 8-row groups 1024 B apart): LBO unused (1), SBO = 1024 B.  Advancing K by 32 bytes inside the swizzle row = +2.
// MN-major (64 two-byte MN columns per 128-byte row, one TMA box of 64 K rows = 8 KB per 64 MN columns): LBO = 8 KB between 64-column
// blocks, SBO = 1024 B between groups of 8 K rows.  Advancing K by 16 rows = +128.
__device__ __forceinline__ uint64_t make_sw128_desc(uint32_t smem_addr, uint32_t lbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>(lbo_bytes >> 4) << 16;
  d |= static_cast<uint64_t>(1024 >> 4) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}
__device__ __forceinline__ uint64_t make_sw128_kmajor_desc(uint32_t smem_addr) { return make_sw128_desc(smem_addr, 16); }
// The same for SWIZZLE_64B (layout type 2 @62): 64-byte rows, 8-row groups 512 B apart.  K-major: advancing K by 32 bytes = +2.
// MN-major (32 two-byte MN columns per 64-byte row, 64 K rows = 4 KB per 32 MN columns): LBO between 32-column blocks, SBO = 512 B between
// groups of 8 K rows.  Advancing K by 16 rows = +64.
__device__ __forceinline__ uint64_t make_sw64_desc(uint32_t smem_addr, uint32_t lbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>(lbo_bytes >> 4) << 16;
  d |= static_cast<uint64_t>(512 >> 4) << 32;
  d |= static_cast<uint64_t>(2) << 62;
  return d;
}
__device__ __forceinline__ uint64_t make_sw64_kmajor_desc(uint32_t smem_addr) { return make_sw64_desc(smem_addr, 16); }

}  // namespace dsb
