// Training-side kernels of the denoiser (SURVEY.md section 8 row A13): q_sample, the fused _train_loss forward + logit gradient, and
// the backward passes of every non-GEMM op of Text2ImageTransformer.  GEMM gradients reuse dsb_gemm_ex (dgrad with transposed
// weight copies, wgrad with the transposed operands produced by dsb_transpose below).
//   reference: sound_synthesis/modeling/transformers/diffusion_transformer.py:370-377 (q_sample), :408-476 (_train_loss);
//              transformer_utils.py:43-58, :91-109 (attention), :111-115 (GELU2), :134-149 (AdaLayerNorm), :255-272 (Block);
//              embeddings/dalle_mask_image_embedding.py:36-58.  The reference gets all of these gradients from torch autograd.
// Activation storage type "T": float (tf32-rounded on store; DSB_DTYPE_TF32) or bf16 (DSB_DTYPE_BF16).
#include "block_ctx.cuh"
#include "common.cuh"
#include "diffsound_b200.h"
#include "train_loss_math.cuh"
#include <cuda_bf16.h>

namespace dsb {

// ---------------------------------------------------------------------------------------------- small helpers
__device__ __forceinline__ float t_wsum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float t_wmax(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
template <class T> __device__ __forceinline__ float ld_act(const T* p);
template <> __device__ __forceinline__ float ld_act<float>(const float* p) { return *p; }
template <> __device__ __forceinline__ float ld_act<__nv_bfloat16>(const __nv_bfloat16* p) { return __bfloat162float(*p); }
template <class T> __device__ __forceinline__ void st_act(T* p, float v);
template <> __device__ __forceinline__ void st_act<float>(float* p, float v) { *p = round_tf32(v); }
template <> __device__ __forceinline__ void st_act<__nv_bfloat16>(__nv_bfloat16* p, float v) { *p = __float2bfloat16_rn(v); }

// 8 consecutive activations <-> 8 floats (16-byte access for bf16, 2 x 16 bytes for fp32); p must be 8-element aligned
template <class T> __device__ __forceinline__ void ld_act8(const T* p, float (&v)[8]);
template <> __device__ __forceinline__ void ld_act8<float>(const float* p, float (&v)[8]) {
  const float4 a = reinterpret_cast<const float4*>(p)[0], b = reinterpret_cast<const float4*>(p)[1];
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
template <> __device__ __forceinline__ void ld_act8<__nv_bfloat16>(const __nv_bfloat16* p, float (&v)[8]) {
  const uint4 u = *reinterpret_cast<const uint4*>(p);
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    v[2 * i] = __uint_as_float(w[i] << 16);
    v[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
  }
}
template <class T> __device__ __forceinline__ void st_act8(T* p, const float (&v)[8]);
template <> __device__ __forceinline__ void st_act8<float>(float* p, const float (&v)[8]) {
  reinterpret_cast<float4*>(p)[0] = make_float4(round_tf32(v[0]), round_tf32(v[1]), round_tf32(v[2]), round_tf32(v[3]));
  reinterpret_cast<float4*>(p)[1] = make_float4(round_tf32(v[4]), round_tf32(v[5]), round_tf32(v[6]), round_tf32(v[7]));
}
template <> __device__ __forceinline__ void st_act8<__nv_bfloat16>(__nv_bfloat16* p, const float (&v)[8]) {
  uint4 u;
  __nv_bfloat162 h;
  h = __floats2bfloat162_rn(v[0], v[1]); u.x = *reinterpret_cast<uint32_t*>(&h);
  h = __floats2bfloat162_rn(v[2], v[3]); u.y = *reinterpret_cast<uint32_t*>(&h);
  h = __floats2bfloat162_rn(v[4], v[5]); u.z = *reinterpret_cast<uint32_t*>(&h);
  h = __floats2bfloat162_rn(v[6], v[7]); u.w = *reinterpret_cast<uint32_t*>(&h);
  *reinterpret_cast<uint4*>(p) = u;
}

struct WarpCtx {  // lane context of train_loss_math.cuh: one warp per column
  int ln;
  __device__ __forceinline__ int lane() const { return ln; }
  __device__ __forceinline__ int lanes() const { return 32; }
  __device__ __forceinline__ float sumf(float v) const { return t_wsum(v); }
  __device__ __forceinline__ float maxf(float v) const { return t_wmax(v); }
  __device__ __forceinline__ double sumd(double v) const {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
  }
  __device__ __forceinline__ int mini(int v) const {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = min(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
  }
};

// ---------------------------------------------------------------------------------------------- q_sample
// x_t[b,l] = argmax_k( gumbel(u[b,k,l]) + q_pred(log_onehot(x0), t)[k] )   (diffusion_transformer.py:370-377, :253-267, :359-365)
__global__ void __launch_bounds__(256)
q_sample_kernel(const int64_t* __restrict__ x0, const int64_t* __restrict__ t, const float* __restrict__ uniform,
                const float* __restrict__ sched, int64_t* __restrict__ x_t, int B, int K, int L, int T) {
  const int col = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (col >= B * L) return;
  const int lane = threadIdx.x & 31;
  const int b = col / L, l = col - b * L;
  const int C = K + 1, S1 = T + 1;
  long long tt = t[b];
  tt = ((tt % S1) + S1) % S1;
  const float cA = sched[4 * S1 + tt], cB = sched[5 * S1 + tt], cC = sched[6 * S1 + tt], cC1 = sched[7 * S1 + tt];
  const int x = (int)x0[col];
  const float* u = uniform + (long long)b * C * L + l;
  float best = -INFINITY;
  int bi = 0x7fffffff;
  for (int k = lane; k < C; k += 32) {
    const float X = (k == x) ? 0.f : dsb_loss::LOGZ;
    const float v = (k < K) ? dsb_loss::lae(X + cA, cB) : dsb_loss::lae(X + cC1, cC);
    const float g = -logf(-logf(u[(long long)k * L] + 1e-30f) + 1e-30f);
    const float val = g + v;
    if (val > best) { best = val; bi = k; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
  }
  if (lane == 0) x_t[col] = bi;
}

// ---------------------------------------------------------------------------------------------- fused _train_loss
template <int NJ>
__global__ void __launch_bounds__(256)
train_loss_kernel(const float* __restrict__ logits, const int64_t* __restrict__ x0, const int64_t* __restrict__ xt,
                  const int64_t* __restrict__ t, const float* __restrict__ pt, const float* __restrict__ sched, float* __restrict__ dlogits,
                  float* __restrict__ prob_out, float* __restrict__ col_out, int* __restrict__ hits, int B, int K, int L, int T, float aux_w,
                  int adaptive, float mw0, float mw1, int prob_exp) {
  const int col = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (col >= B * L) return;
  const int b = col / L, l = col - b * L;
  WarpCtx c{(int)(threadIdx.x & 31)};
  const long long tb = t[b];
  const dsb_loss::Sched s = dsb_loss::load_sched(sched, T, tb);
  dsb_loss::ColumnIn in;
  in.K = K; in.x0 = (int)x0[col]; in.xt = (int)xt[col]; in.is0 = tb == 0;
  in.g_main = 1.f / (pt[b] * (float)(B * L));
  in.g_aux = aux_w != 0.f ? in.g_main * aux_w * (adaptive ? ((float)tb / (float)T + 1.0f) : 1.0f) : 0.f;
  in.mw0 = mw0; in.mw1 = mw1;
  const dsb_loss::ColumnOut o = dsb_loss::column_loss<WarpCtx, NJ>(
      c, logits + (long long)col * K, dlogits ? dlogits + (long long)col * K : nullptr,
      prob_out ? prob_out + (long long)b * (K + 1) * L + l : nullptr, L, prob_exp != 0, in, s);
  if (c.ln == 0) {
    col_out[2 * (long long)col] = o.main;
    col_out[2 * (long long)col + 1] = o.aux;
    if (hits) { hits[2 * (long long)col] = o.x0_hit; hits[2 * (long long)col + 1] = o.keep_hit; }
  }
}

// Wide form for K + 1 > 32 * 33: one CTA of WIDE_LOSS_NT threads per column, CAP = ceil((K+1) / WIDE_LOSS_NT) values per thread, the
// same column_loss on a block context (reductions in the fixed order of block_ctx.cuh).
constexpr int WIDE_LOSS_NT = 256;
constexpr int WIDE_LOSS_MAX_CAP = 16;  // K + 1 <= 4096

template <int CAP>
__global__ void __launch_bounds__(WIDE_LOSS_NT, CAP <= 9 ? 2 : 1)
train_loss_wide_kernel(const float* __restrict__ logits, const int64_t* __restrict__ x0, const int64_t* __restrict__ xt,
                       const int64_t* __restrict__ t, const float* __restrict__ pt, const float* __restrict__ sched, float* __restrict__ dlogits,
                       float* __restrict__ prob_out, float* __restrict__ col_out, int* __restrict__ hits, int B, int K, int L, int T, float aux_w,
                       int adaptive, float mw0, float mw1, int prob_exp) {
  __shared__ double red[2 * (WIDE_LOSS_NT / 32)];
  const long long col = blockIdx.x;
  const int b = (int)(col / L), l = (int)(col - (long long)b * L);
  const BlockCtx<WIDE_LOSS_NT> c{red, (int)threadIdx.x, 0};
  const long long tb = t[b];
  const dsb_loss::Sched s = dsb_loss::load_sched(sched, T, tb);
  dsb_loss::ColumnIn in;
  in.K = K; in.x0 = (int)x0[col]; in.xt = (int)xt[col]; in.is0 = tb == 0;
  in.g_main = 1.f / (pt[b] * (float)(B * L));
  in.g_aux = aux_w != 0.f ? in.g_main * aux_w * (adaptive ? ((float)tb / (float)T + 1.0f) : 1.0f) : 0.f;
  in.mw0 = mw0; in.mw1 = mw1;
  const dsb_loss::ColumnOut o = dsb_loss::column_loss<BlockCtx<WIDE_LOSS_NT>, CAP>(
      c, logits + col * K, dlogits ? dlogits + col * K : nullptr,
      prob_out ? prob_out + (long long)b * (K + 1) * L + l : nullptr, L, prob_exp != 0, in, s);
  if (threadIdx.x == 0) {
    col_out[2 * col] = o.main;
    col_out[2 * col + 1] = o.aux;
    if (hits) { hits[2 * col] = o.x0_hit; hits[2 * col + 1] = o.keep_hit; }
  }
}

// one CTA: per-batch sums in a fixed order (deterministic), vb_loss, the scalar loss of forward() (:568-569) and the Lt_history /
// Lt_count bookkeeping (:448-454: gather the old history for every b first, then scatter in batch order).
__global__ void __launch_bounds__(256)
train_loss_finalize_kernel(const float* __restrict__ col, const int64_t* __restrict__ t, const float* __restrict__ pt, float* __restrict__ kl_loss,
                           float* __restrict__ vb_loss, float* __restrict__ loss, float* __restrict__ lt_history, float* __restrict__ lt_count,
                           float* __restrict__ new_hist, int B, int L, int T, float aux_w, int adaptive) {
  __shared__ float red[2][8];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  float total = 0.f;
  for (int b = 0; b < B; ++b) {
    float m = 0.f, a = 0.f;
    for (int l = tid; l < L; l += 256) {
      m += col[2 * ((long long)b * L + l)];
      a += col[2 * ((long long)b * L + l) + 1];
    }
    m = t_wsum(m); a = t_wsum(a);
    if (lane == 0) { red[0][warp] = m; red[1][warp] = a; }
    __syncthreads();
    if (tid == 0) {
      float ms = 0.f, as = 0.f;
      for (int w = 0; w < 8; ++w) { ms += red[0][w]; as += red[1][w]; }
      const long long tb = t[b];
      float vb = ms / pt[b];
      if (aux_w != 0.f) vb += (adaptive ? ((float)tb / (float)T + 1.0f) : 1.0f) * aux_w * as / pt[b];
      kl_loss[b] = ms;
      vb_loss[b] = vb;
      total += vb;
      if (lt_history) new_hist[b] = 0.1f * ms * ms + 0.9f * lt_history[tb];
    }
    __syncthreads();
  }
  if (tid == 0) {
    loss[0] = total / (float)((long long)B * L);
    if (lt_history)
      for (int b = 0; b < B; ++b) {
        lt_history[t[b]] = new_hist[b];
        lt_count[t[b]] += 1.f;
      }
  }
}

// ---------------------------------------------------------------------------------------------- layout kernels
// out[c][r] = in[r][c] per batch; 32x32 tiles through shared memory, any 2- or 4-byte element
template <class E>
__global__ void __launch_bounds__(256)
transpose_kernel(const E* __restrict__ in, long long ld_in, long long in_bs, E* __restrict__ out, long long ld_out, long long out_bs, int rows,
                 int cols) {
  __shared__ E tile[32][33];
  in += (long long)blockIdx.z * in_bs;
  out += (long long)blockIdx.z * out_bs;
  const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int r = r0 + ty + 8 * i, c = c0 + tx;
    if (r < rows && c < cols) tile[ty + 8 * i][tx] = in[(long long)r * ld_in + c];
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int c = c0 + ty + 8 * i, r = r0 + tx;
    if (r < rows && c < cols) out[(long long)c * ld_out + r] = tile[tx][ty + 8 * i];
  }
}

// 2-byte elements, 64x64 tiles, 16-byte global accesses on both sides (the wgrad operand copies are the bulk of the backward's
// non-GEMM traffic).  Requires 16-byte aligned bases / leading dimensions / batch strides; ragged edges fall back to element accesses.
__global__ void __launch_bounds__(256)
transpose16_kernel(const uint16_t* __restrict__ in, long long ld_in, long long in_bs, uint16_t* __restrict__ out, long long ld_out, long long out_bs,
                   int rows, int cols) {
  constexpr int PITCH = 66;  // elements; 33 words: the 8 row-groups a warp reads per column land on 4 banks (2-way conflict at worst)
  __shared__ __align__(16) uint16_t tile[64 * PITCH];
  in += (long long)blockIdx.z * in_bs;
  out += (long long)blockIdx.z * out_bs;
  const int c0 = blockIdx.x * 64, r0 = blockIdx.y * 64;
#pragma unroll
  for (int it = 0; it < 2; ++it) {
    const int q = threadIdx.x + 256 * it;
    const int r = q >> 3, cc = (q & 7) * 8;
    const int gr = r0 + r, gc = c0 + cc;
    uint32_t* dst = reinterpret_cast<uint32_t*>(tile + r * PITCH + cc);
    if (gr < rows && gc + 7 < cols) {
      const uint4 v = *reinterpret_cast<const uint4*>(in + (long long)gr * ld_in + gc);
      dst[0] = v.x; dst[1] = v.y; dst[2] = v.z; dst[3] = v.w;
    } else {
#pragma unroll
      for (int i = 0; i < 8; ++i) tile[r * PITCH + cc + i] = (gr < rows && gc + i < cols) ? in[(long long)gr * ld_in + gc + i] : (uint16_t)0;
    }
  }
  __syncthreads();
#pragma unroll
  for (int it = 0; it < 2; ++it) {
    const int q = threadIdx.x + 256 * it;
    const int c = q >> 3, rg = (q & 7) * 8;   // output row c (= input column), 8 consecutive input rows
    const int gc = c0 + c, gr = r0 + rg;
    if (gc >= cols) continue;
    uint16_t e[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) e[i] = tile[(rg + i) * PITCH + c];
    uint16_t* dst = out + (long long)gc * ld_out + gr;
    if (gr + 7 < rows) {
      uint4 v;
      v.x = e[0] | ((uint32_t)e[1] << 16); v.y = e[2] | ((uint32_t)e[3] << 16);
      v.z = e[4] | ((uint32_t)e[5] << 16); v.w = e[6] | ((uint32_t)e[7] << 16);
      *reinterpret_cast<uint4*>(dst) = v;
    } else {
#pragma unroll
      for (int i = 0; i < 8; ++i)
        if (gr + i < rows) dst[i] = e[i];
    }
  }
}

// heads: token-major (B*Lx, ld) columns [h*64, h*64+64)  <->  head-major (B*H, Lx, 64); 16-byte chunks
template <int TO_HEADS>
__global__ void __launch_bounds__(256)
heads_kernel(uint4* __restrict__ tok, long long ld16, uint4* __restrict__ hm, int B, int H, int Lx, int chunks) {
  const long long n = (long long)B * H * Lx * chunks;
  for (long long i = blockIdx.x * 256LL + threadIdx.x; i < n; i += 256LL * gridDim.x) {
    const int ch = (int)(i % chunks);
    long long r = i / chunks;
    const int l = (int)(r % Lx); r /= Lx;
    const int h = (int)(r % H);
    const int b = (int)(r / H);
    uint4* tp = tok + ((long long)b * Lx + l) * ld16 + (long long)h * chunks + ch;
    if (TO_HEADS) hm[i] = *tp; else *tp = hm[i];
  }
}

// out = T(in * (scale ? *scale : 1))
template <class T>
__global__ void __launch_bounds__(256)
cast_scale_kernel(const float* __restrict__ in, T* __restrict__ out, long long n, const float* __restrict__ scale) {
  const float s = scale ? *scale : 1.f;
  const bool vec = ((reinterpret_cast<uintptr_t>(in) | reinterpret_cast<uintptr_t>(out)) & 15) == 0;
  const long long n4 = vec ? n / 4 : 0;
  for (long long i = blockIdx.x * 256LL + threadIdx.x; i < n4; i += 256LL * gridDim.x) {
    const float4 v = reinterpret_cast<const float4*>(in)[i];
    st_act<T>(out + 4 * i, v.x * s); st_act<T>(out + 4 * i + 1, v.y * s); st_act<T>(out + 4 * i + 2, v.z * s); st_act<T>(out + 4 * i + 3, v.w * s);
  }
  for (long long i = n4 * 4 + blockIdx.x * 256LL + threadIdx.x; i < n; i += 256LL * gridDim.x) st_act<T>(out + i, in[i] * s);
}

// column sums of a (rows, N) matrix into fp32 out[N] (atomic accumulation; out zeroed by the host wrapper).
// VEC: each thread owns 8 consecutive columns (16-byte loads: a warp row covers 256 columns); otherwise one column per thread.
template <class T, bool VEC>
__global__ void __launch_bounds__(256)
colsum_kernel(const T* __restrict__ in, long long ld, float* __restrict__ out, long long rows, int N, int rows_per_cta) {
  constexpr int CPT = VEC ? 8 : 1;
  __shared__ float red[8][32 * CPT];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int c = (blockIdx.x * 32 + tx) * CPT;
  const long long r0 = (long long)blockIdx.y * rows_per_cta;
  const long long r1 = r0 + rows_per_cta < rows ? r0 + rows_per_cta : rows;
  float acc[CPT];
#pragma unroll
  for (int i = 0; i < CPT; ++i) acc[i] = 0.f;
  if (c < N) {
    for (long long r = r0 + ty; r < r1; r += 8) {
      if (VEC) {
        float v[8];
        ld_act8<T>(in + r * ld + c, v);
#pragma unroll
        for (int i = 0; i < CPT; ++i) acc[i] += v[i];
      } else {
        acc[0] += ld_act<T>(in + r * ld + c);
      }
    }
  }
#pragma unroll
  for (int i = 0; i < CPT; ++i) red[ty][tx * CPT + i] = acc[i];
  __syncthreads();
  for (int j = threadIdx.x; j < 32 * CPT; j += 256) {
    const int cg = blockIdx.x * 32 * CPT + j;
    if (cg < N) {
      float sacc = 0.f;
#pragma unroll
      for (int w = 0; w < 8; ++w) sacc += red[w][j];
      atomicAdd(out + cg, sacc);
    }
  }
}

// ---------------------------------------------------------------------------------------------- GELU2  (transformer_utils.py:111-115)
template <class T>
__global__ void __launch_bounds__(256)
gelu2_fwd_kernel(const T* __restrict__ u, T* __restrict__ a, long long n) {  // n % 8 == 0, 16-byte aligned (checked by the host wrapper)
  for (long long i = (blockIdx.x * 256LL + threadIdx.x) * 8; i < n; i += 256LL * 8 * gridDim.x) {
    float x[8];
    ld_act8<T>(u + i, x);
#pragma unroll
    for (int j = 0; j < 8; ++j) x[j] = x[j] / (1.f + __expf(-1.702f * x[j]));
    st_act8<T>(a + i, x);
  }
}
template <class T>
__global__ void __launch_bounds__(256)
gelu2_bwd_kernel(const T* __restrict__ u, const T* __restrict__ da, T* __restrict__ du, long long n) {
  for (long long i = (blockIdx.x * 256LL + threadIdx.x) * 8; i < n; i += 256LL * 8 * gridDim.x) {
    float x[8], d[8];
    ld_act8<T>(u + i, x);
    ld_act8<T>(da + i, d);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float sg = 1.f / (1.f + __expf(-1.702f * x[j]));
      d[j] *= sg + 1.702f * x[j] * sg * (1.f - sg);
    }
    st_act8<T>(du + i, d);
  }
}
__global__ void __launch_bounds__(256)
silu_bwd_kernel(const float* __restrict__ x, const float* __restrict__ dy, float* __restrict__ dx, long long n) {
  for (long long i = blockIdx.x * 256LL + threadIdx.x; i < n; i += 256LL * gridDim.x) {
    const float v = x[i];
    const float s = 1.f / (1.f + expf(-v));
    dx[i] = dy[i] * (s + v * s * (1.f - s));
  }
}
// out[i, :] = table[idx[i], :]   /   table[idx[i], :] += src[i, :]
__global__ void __launch_bounds__(256)
gather_rows_kernel(const float* __restrict__ table, const int64_t* __restrict__ idx, float* __restrict__ out, int n, int D) {
  for (long long i = blockIdx.x * 256LL + threadIdx.x; i < (long long)n * D; i += 256LL * gridDim.x) out[i] = table[idx[i / D] * D + i % D];
}
__global__ void __launch_bounds__(256)
scatter_add_rows_kernel(float* __restrict__ table, const int64_t* __restrict__ idx, const float* __restrict__ src, int n, int D) {
  for (long long i = blockIdx.x * 256LL + threadIdx.x; i < (long long)n * D; i += 256LL * gridDim.x) atomicAdd(table + idx[i / D] * D + i % D, src[i]);
}

// ---------------------------------------------------------------------------------------------- LayerNorm / AdaLayerNorm backward
// y = xhat * g + beta with g = gamma (MODE 0) or 1 + table[idx[b], 0:D] (MODE 1, beta = table[idx[b], D:2D]).
//   dx    = rstd * (dy g - mean(dy g) - xhat mean(dy g xhat));   dx_io += dx   (the residual branch's gradient is already in dx_io)
//   dg   += sum_rows dy xhat ;  dbeta += sum_rows dy                 (MODE 0: dgamma[D], dbeta[D];  MODE 1: dtable[idx[b]] = (dscale | dshift))
// grid (ceil(L / 32), B): a CTA never straddles two batch elements; 8 warps x 4 rows (enough CTAs to fill 132 SMs at B = 20).
constexpr int LNB_ROWS = 32;
template <int MODE, int NV>
__global__ void __launch_bounds__(256)
layernorm_bwd_kernel(const float* __restrict__ x, const float* __restrict__ dy, float* __restrict__ dx_io, const float* __restrict__ p0,
                     const int64_t* __restrict__ idx, float* __restrict__ dg_out, float* __restrict__ db_out, int L, int D, float eps,
                     void* __restrict__ dx_act, int act_mode /*0 none, 1 fp32 tf32-rounded, 2 bf16*/) {
  __shared__ float red[2][8][128];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int b = blockIdx.y;
  const long long pi = MODE == 1 ? idx[b] : 0;
  const float4* g4 = reinterpret_cast<const float4*>(MODE == 1 ? p0 + pi * 2LL * D : p0);
  float4 dg[NV], db[NV];
#pragma unroll
  for (int j = 0; j < NV; ++j) dg[j] = db[j] = make_float4(0.f, 0.f, 0.f, 0.f);
  const int l_end = min(L, (int)(blockIdx.x + 1) * LNB_ROWS);
  for (int l = blockIdx.x * LNB_ROWS + warp; l < l_end; l += 8) {
    const long long row = (long long)b * L + l;
    const float4* xr = reinterpret_cast<const float4*>(x + row * D);
    const float4* dr = reinterpret_cast<const float4*>(dy + row * D);
    float4* dxr = reinterpret_cast<float4*>(dx_io + row * D);
    float4 v[NV], d[NV];
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < NV; ++j) {
      v[j] = xr[lane + 32 * j];
      d[j] = dr[lane + 32 * j];
      s += (v[j].x + v[j].y) + (v[j].z + v[j].w);
    }
    const float mean = t_wsum(s) / (float)D;
    float q = 0.f;
#pragma unroll
    for (int j = 0; j < NV; ++j) {
      v[j].x -= mean; v[j].y -= mean; v[j].z -= mean; v[j].w -= mean;
      q += (v[j].x * v[j].x + v[j].y * v[j].y) + (v[j].z * v[j].z + v[j].w * v[j].w);
    }
    const float rstd = rsqrtf(t_wsum(q) / (float)D + eps);
    float m1 = 0.f, m2 = 0.f;
#pragma unroll
    for (int j = 0; j < NV; ++j) {
      float4 g = __ldg(g4 + lane + 32 * j);
      if (MODE == 1) { g.x += 1.f; g.y += 1.f; g.z += 1.f; g.w += 1.f; }
      v[j].x *= rstd; v[j].y *= rstd; v[j].z *= rstd; v[j].w *= rstd;  // xhat
      dg[j].x += d[j].x * v[j].x; dg[j].y += d[j].y * v[j].y; dg[j].z += d[j].z * v[j].z; dg[j].w += d[j].w * v[j].w;
      db[j].x += d[j].x; db[j].y += d[j].y; db[j].z += d[j].z; db[j].w += d[j].w;
      d[j].x *= g.x; d[j].y *= g.y; d[j].z *= g.z; d[j].w *= g.w;      // dxhat
      m1 += (d[j].x + d[j].y) + (d[j].z + d[j].w);
      m2 += (d[j].x * v[j].x + d[j].y * v[j].y) + (d[j].z * v[j].z + d[j].w * v[j].w);
    }
    m1 = t_wsum(m1) / (float)D;
    m2 = t_wsum(m2) / (float)D;
#pragma unroll
    for (int j = 0; j < NV; ++j) {
      float4 o = dxr[lane + 32 * j];
      o.x += rstd * (d[j].x - m1 - v[j].x * m2); o.y += rstd * (d[j].y - m1 - v[j].y * m2);
      o.z += rstd * (d[j].z - m1 - v[j].z * m2); o.w += rstd * (d[j].w - m1 - v[j].w * m2);
      dxr[lane + 32 * j] = o;
      // the updated stream gradient is the next Linear backward's dY: emit its GEMM-operand copy here instead of a separate cast pass
      if (act_mode == 2) {
        __nv_bfloat162 h0 = __floats2bfloat162_rn(o.x, o.y), h1 = __floats2bfloat162_rn(o.z, o.w);
        uint2 u;
        u.x = *reinterpret_cast<uint32_t*>(&h0); u.y = *reinterpret_cast<uint32_t*>(&h1);
        reinterpret_cast<uint2*>(reinterpret_cast<__nv_bfloat16*>(dx_act) + row * D)[lane + 32 * j] = u;
      } else if (act_mode == 1) {
        reinterpret_cast<float4*>(reinterpret_cast<float*>(dx_act) + row * D)[lane + 32 * j] =
            make_float4(round_tf32(o.x), round_tf32(o.y), round_tf32(o.z), round_tf32(o.w));
      }
    }
  }
  // cross-warp reduction of the parameter gradients, 128 columns (one float4 slot j) at a time
  float* dgo = MODE == 1 ? dg_out + pi * 2LL * D : dg_out;
  float* dbo = MODE == 1 ? dg_out + pi * 2LL * D + D : db_out;
#pragma unroll
  for (int j = 0; j < NV; ++j) {
    __syncthreads();
    reinterpret_cast<float4*>(&red[0][warp][0])[lane] = dg[j];
    reinterpret_cast<float4*>(&red[1][warp][0])[lane] = db[j];
    __syncthreads();
    const int which = threadIdx.x >> 7, cc = threadIdx.x & 127;
    float sacc = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) sacc += red[which][w][cc];
    // slot j of lane ln holds columns (ln + 32 j) * 4 .. +3  ->  smem column cc = ln * 4 + e
    const int colg = ((cc >> 2) + 32 * j) * 4 + (cc & 3);
    atomicAdd((which == 0 ? dgo : dbo) + colg, sacc);
  }
}

// ---------------------------------------------------------------------------------------------- softmax rows (attention)
// P[r, 0:n] = softmax(S[r, 0:n]);  S fp32 (already scaled by the GEMM's alpha), P in T
template <class T>
__global__ void __launch_bounds__(256)
softmax_fwd_kernel(const float* __restrict__ S, long long ld_s, T* __restrict__ P, long long ld_p, long long rows, int n) {
  const long long r = blockIdx.x * 8LL + (threadIdx.x >> 5);
  if (r >= rows) return;
  const int lane = threadIdx.x & 31;
  const float* s = S + r * ld_s;
  float mx = -INFINITY;
  for (int k = lane; k < n; k += 32) mx = fmaxf(mx, s[k]);
  mx = t_wmax(mx);
  float sum = 0.f;
  for (int k = lane; k < n; k += 32) sum += __expf(s[k] - mx);
  sum = t_wsum(sum);
  const float inv = 1.f / sum;
  for (int k = lane; k < n; k += 32) st_act<T>(P + r * ld_p + k, __expf(s[k] - mx) * inv);
}
// dS[r, k] = alpha * P[r, k] * (dP[r, k] - sum_j dP[r, j] P[r, j])
template <class T>
__global__ void __launch_bounds__(256)
softmax_bwd_kernel(const T* __restrict__ P, long long ld_p, const float* __restrict__ dP, long long ld_dp, T* __restrict__ dS, long long ld_ds,
                   long long rows, int n, float alpha) {
  const long long r = blockIdx.x * 8LL + (threadIdx.x >> 5);
  if (r >= rows) return;
  const int lane = threadIdx.x & 31;
  float dot = 0.f;
  for (int k = lane; k < n; k += 32) dot += ld_act<T>(P + r * ld_p + k) * dP[r * ld_dp + k];
  dot = t_wsum(dot);
  for (int k = lane; k < n; k += 32) st_act<T>(dS + r * ld_ds + k, alpha * ld_act<T>(P + r * ld_p + k) * (dP[r * ld_dp + k] - dot));
}

// ---------------------------------------------------------------------------------------------- embedding backward
// demb[ids[row]] += dx[row]   (atomics);   dheight / dwidth: fixed-order sums over the batch and the other grid axis
__global__ void __launch_bounds__(256)
embed_bwd_tokens_kernel(const int64_t* __restrict__ ids, const float* __restrict__ dx, float* __restrict__ demb, long long rows, int D, int num_embed) {
  for (long long i = blockIdx.x * 256LL + threadIdx.x; i < rows * D; i += 256LL * gridDim.x) {
    long long id = ids[i / D];
    id = id < 0 ? 0 : (id >= num_embed ? num_embed - 1 : id);
    atomicAdd(demb + id * D + i % D, dx[i]);
  }
}
__global__ void __launch_bounds__(256)
embed_bwd_pos_kernel(const float* __restrict__ dx, float* __restrict__ dheight, float* __restrict__ dwidth, int B, int L, int D, int H, int W) {
  const int r = blockIdx.y;  // 0..H-1: height rows, H..H+W-1: width rows
  const int c = blockIdx.x * 256 + threadIdx.x;
  if (c >= D) return;
  float acc = 0.f;
  if (r < H) {
    for (int b = 0; b < B; ++b)
      for (int w = 0; w < W; ++w) {
        const int l = r * W + w;
        if (l < L) acc += dx[((long long)b * L + l) * D + c];
      }
    dheight[(long long)r * D + c] += acc;
  } else {
    const int w = r - H;
    for (int b = 0; b < B; ++b)
      for (int h = 0; h < H; ++h) {
        const int l = h * W + w;
        if (l < L) acc += dx[((long long)b * L + l) * D + c];
      }
    dwidth[(long long)w * D + c] += acc;
  }
}

static inline int grid_for(long long n) {
  long long g = (n + 255) / 256;
  const long long cap = (long long)sm_count() * 16;
  return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}
}  // namespace dsb
using namespace dsb;

namespace dsb {
template <class T> static void run_cast_scale(const float* in, void* out, long long n, const float* scale, cudaStream_t st) {
  cast_scale_kernel<T><<<grid_for(n), 256, 0, st>>>(in, (T*)out, n, scale);
}
template <class T> static void run_colsum(const void* in, long long ld, float* out, long long rows, int N, int rpc, cudaStream_t st) {
  const bool vec = N % 8 == 0 && ld % 8 == 0 && ((uintptr_t)in & 31) == 0;
  if (vec) {
    dim3 grid((N + 255) / 256, (unsigned)((rows + rpc - 1) / rpc));
    colsum_kernel<T, true><<<grid, 256, 0, st>>>((const T*)in, ld, out, rows, N, rpc);
  } else {
    dim3 grid((N + 31) / 32, (unsigned)((rows + rpc - 1) / rpc));
    colsum_kernel<T, false><<<grid, 256, 0, st>>>((const T*)in, ld, out, rows, N, rpc);
  }
}
template <class T> static void run_gelu2_fwd(const void* u, void* a, long long n, cudaStream_t st) {
  gelu2_fwd_kernel<T><<<grid_for(n / 8), 256, 0, st>>>((const T*)u, (T*)a, n);
}
template <class T> static void run_gelu2_bwd(const void* u, const void* da, void* du, long long n, cudaStream_t st) {
  gelu2_bwd_kernel<T><<<grid_for(n / 8), 256, 0, st>>>((const T*)u, (const T*)da, (T*)du, n);
}
template <class T> static void run_softmax_fwd(const float* S, long long ld_s, void* P, long long ld_p, long long rows, int n, cudaStream_t st) {
  softmax_fwd_kernel<T><<<(unsigned)((rows + 7) / 8), 256, 0, st>>>(S, ld_s, (T*)P, ld_p, rows, n);
}
template <class T> static void run_softmax_bwd(const void* P, long long ld_p, const float* dP, long long ld_dp, void* dS, long long ld_ds, long long rows,
                                               int n, float alpha, cudaStream_t st) {
  softmax_bwd_kernel<T><<<(unsigned)((rows + 7) / 8), 256, 0, st>>>((const T*)P, ld_p, dP, ld_dp, (T*)dS, ld_ds, rows, n, alpha);
}
}  // namespace dsb

#define DSB_ACT_CALL(dtype, FN, ...)                                                              \
  do {                                                                                            \
    if ((dtype) == DSB_DTYPE_TF32) FN<float>(__VA_ARGS__);                                        \
    else if ((dtype) == DSB_DTYPE_BF16) FN<__nv_bfloat16>(__VA_ARGS__);                           \
    else { dsb::set_error("%s: dtype must be DSB_DTYPE_TF32 or DSB_DTYPE_BF16", __func__); return 2; } \
    DSB_CHECK_CUDA(cudaGetLastError());                                                           \
  } while (0)

extern "C" int dsb_q_sample(const int64_t* x0, const int64_t* t, const float* uniform, const float* sched, int64_t* x_t, int B, int K, int L, int T,
                            void* stream) {
  DSB_REQUIRE(B > 0 && K > 0 && L > 0 && T > 0, "dsb_q_sample: bad shape");
  q_sample_kernel<<<(B * L + 7) / 8, 256, 0, (cudaStream_t)stream>>>(x0, t, uniform, sched, x_t, B, K, L, T);
  DSB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dsb_train_loss(const float* logits, const int64_t* x0, const int64_t* x_t, const int64_t* t, const float* pt, const float* sched,
                              float* dlogits, float* log_model_prob, float* col_loss, int* hits, float* kl_loss, float* vb_loss, float* loss,
                              float* lt_history, float* lt_count, float* scratch_b, int B, int K, int L, int T, float aux_weight, int adaptive,
                              float mw0, float mw1, int prob_as_exp, void* stream) {
  DSB_REQUIRE(B > 0 && K > 0 && L > 0 && T > 0, "dsb_train_loss: bad shape");
  DSB_REQUIRE(K + 1 <= WIDE_LOSS_NT * WIDE_LOSS_MAX_CAP, "dsb_train_loss: K=%d too large (max %d)", K, WIDE_LOSS_NT * WIDE_LOSS_MAX_CAP - 1);
  DSB_REQUIRE(logits && x0 && x_t && t && pt && sched && col_loss && kl_loss && vb_loss && loss, "dsb_train_loss: null argument");
  DSB_REQUIRE(!lt_history || (lt_count && scratch_b), "dsb_train_loss: Lt bookkeeping needs lt_count and a B-float scratch");
  cudaStream_t st = (cudaStream_t)stream;
  const int nj = (K + 1 + 31) / 32;
  const int grid = (B * L + 7) / 8;
  const int cap = (K + 1 + WIDE_LOSS_NT - 1) / WIDE_LOSS_NT;
#define DSB_LOSS_CASE(N)                                                                                                               \
  if (nj <= N) {                                                                                                                       \
    train_loss_kernel<N><<<grid, 256, 0, st>>>(logits, x0, x_t, t, pt, sched, dlogits, log_model_prob, col_loss, hits, B, K, L, T,      \
                                               aux_weight, adaptive, mw0, mw1, prob_as_exp);                                           \
  } else
#define DSB_WIDE_LOSS_CASE(N)                                                                                                          \
  if (cap <= N) {                                                                                                                      \
    train_loss_wide_kernel<N><<<B * L, WIDE_LOSS_NT, 0, st>>>(logits, x0, x_t, t, pt, sched, dlogits, log_model_prob, col_loss, hits, B, \
                                                              K, L, T, aux_weight, adaptive, mw0, mw1, prob_as_exp);                   \
  } else
  DSB_LOSS_CASE(2) DSB_LOSS_CASE(5) DSB_LOSS_CASE(9) DSB_LOSS_CASE(17) DSB_LOSS_CASE(33)
  DSB_WIDE_LOSS_CASE(9) DSB_WIDE_LOSS_CASE(WIDE_LOSS_MAX_CAP) { return 2; }
#undef DSB_LOSS_CASE
#undef DSB_WIDE_LOSS_CASE
  DSB_CHECK_CUDA(cudaGetLastError());
  train_loss_finalize_kernel<<<1, 256, 0, st>>>(col_loss, t, pt, kl_loss, vb_loss, loss, lt_history, lt_count, scratch_b, B, L, T, aux_weight, adaptive);
  DSB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dsb_transpose(const void* in, long long ld_in, long long in_batch_stride, void* out, long long ld_out, long long out_batch_stride,
                             int rows, int cols, int batch, int elem_bytes, void* stream) {
  DSB_REQUIRE(rows > 0 && cols > 0 && batch > 0, "dsb_transpose: bad shape");
  DSB_REQUIRE(elem_bytes == 2 || elem_bytes == 4, "dsb_transpose: elem_bytes must be 2 or 4");
  DSB_REQUIRE(batch <= 65535, "dsb_transpose: batch=%d exceeds 65535", batch);
  dim3 grid((cols + 31) / 32, (rows + 31) / 32, batch);
  const bool vec_ok = elem_bytes == 2 && ((uintptr_t)in & 15) == 0 && ((uintptr_t)out & 15) == 0 && ld_in % 8 == 0 && ld_out % 8 == 0 &&
                      (batch == 1 || (in_batch_stride % 8 == 0 && out_batch_stride % 8 == 0));
  if (vec_ok)
    transpose16_kernel<<<dim3((cols + 63) / 64, (rows + 63) / 64, batch), 256, 0, (cudaStream_t)stream>>>(
        (const uint16_t*)in, ld_in, in_batch_stride, (uint16_t*)out, ld_out, out_batch_stride, rows, cols);
  else if (elem_bytes == 2)
    transpose_kernel<uint16_t><<<grid, 256, 0, (cudaStream_t)stream>>>((const uint16_t*)in, ld_in, in_batch_stride, (uint16_t*)out, ld_out, out_batch_stride, rows, cols);
  else
    transpose_kernel<uint32_t><<<grid, 256, 0, (cudaStream_t)stream>>>((const uint32_t*)in, ld_in, in_batch_stride, (uint32_t*)out, ld_out, out_batch_stride, rows, cols);
  DSB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dsb_heads_split(const void* tok, long long ld, void* heads, int B, int H, int Lx, int elem_bytes, void* stream) {
  DSB_REQUIRE(elem_bytes == 2 || elem_bytes == 4, "dsb_heads_split: elem_bytes must be 2 or 4");
  DSB_REQUIRE((ld * elem_bytes) % 16 == 0 && ((uintptr_t)tok & 15) == 0 && ((uintptr_t)heads & 15) == 0, "dsb_heads_split: 16-byte alignment required");
  const int chunks = 64 * elem_bytes / 16;
  heads_kernel<1><<<grid_for((long long)B * H * Lx * chunks), 256, 0, (cudaStream_t)stream>>>((uint4*)tok, ld * elem_bytes / 16, (uint4*)heads, B, H, Lx, chunks);
  DSB_CHECK_CUDA(cudaGetLastError());
  return 0;
}
extern "C" int dsb_heads_merge(const void* heads, void* tok, long long ld, int B, int H, int Lx, int elem_bytes, void* stream) {
  DSB_REQUIRE(elem_bytes == 2 || elem_bytes == 4, "dsb_heads_merge: elem_bytes must be 2 or 4");
  DSB_REQUIRE((ld * elem_bytes) % 16 == 0 && ((uintptr_t)tok & 15) == 0 && ((uintptr_t)heads & 15) == 0, "dsb_heads_merge: 16-byte alignment required");
  const int chunks = 64 * elem_bytes / 16;
  heads_kernel<0><<<grid_for((long long)B * H * Lx * chunks), 256, 0, (cudaStream_t)stream>>>((uint4*)tok, ld * elem_bytes / 16, (uint4*)heads, B, H, Lx, chunks);
  DSB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dsb_cast_scale(const float* in, void* out, long long n, const float* scale, int dtype, void* stream) {
  DSB_ACT_CALL(dtype, run_cast_scale, in, out, n, scale, (cudaStream_t)stream);
  return 0;
}

extern "C" int dsb_colsum(const void* in, long long ld, float* out, long long rows, int N, int dtype, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  DSB_REQUIRE(rows > 0 && N > 0, "dsb_colsum: bad shape");
  DSB_CHECK_CUDA(cudaMemsetAsync(out, 0, (size_t)N * sizeof(float), st));
  DSB_ACT_CALL(dtype, run_colsum, in, ld, out, rows, N, 64, st);
  return 0;
}

extern "C" int dsb_gelu2_fwd(const void* u, void* a, long long n, int dtype, void* stream) {
  DSB_REQUIRE(n % 8 == 0 && (((uintptr_t)u | (uintptr_t)a) & 31) == 0, "dsb_gelu2_fwd: n must be a multiple of 8 and the buffers 32-byte aligned");
  DSB_ACT_CALL(dtype, run_gelu2_fwd, u, a, n, (cudaStream_t)stream);
  return 0;
}
extern "C" int dsb_gelu2_bwd(const void* u, const void* da, void* du, long long n, int dtype, void* stream) {
  DSB_REQUIRE(n % 8 == 0 && (((uintptr_t)u | (uintptr_t)da | (uintptr_t)du) & 31) == 0, "dsb_gelu2_bwd: n must be a multiple of 8 and the buffers 32-byte aligned");
  DSB_ACT_CALL(dtype, run_gelu2_bwd, u, da, du, n, (cudaStream_t)stream);
  return 0;
}
extern "C" int dsb_silu_bwd(const float* x, const float* dy, float* dx, long long n, void* stream) {
  silu_bwd_kernel<<<grid_for(n), 256, 0, (cudaStream_t)stream>>>(x, dy, dx, n);
  DSB_CHECK_CUDA(cudaGetLastError());
  return 0;
}
extern "C" int dsb_gather_rows(const float* table, const int64_t* idx, float* out, int n, int D, void* stream) {
  gather_rows_kernel<<<grid_for((long long)n * D), 256, 0, (cudaStream_t)stream>>>(table, idx, out, n, D);
  DSB_CHECK_CUDA(cudaGetLastError());
  return 0;
}
extern "C" int dsb_scatter_add_rows(float* table, const int64_t* idx, const float* src, int n, int D, void* stream) {
  scatter_add_rows_kernel<<<grid_for((long long)n * D), 256, 0, (cudaStream_t)stream>>>(table, idx, src, n, D);
  DSB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

template <int MODE>
static int launch_ln_bwd(const float* x, const float* dy, float* dx_io, const float* p0, const int64_t* idx, float* dg, float* db, int B, int L, int D,
                         float eps, void* dx_act, int dtype, cudaStream_t st) {
  const int act_mode = dx_act ? (dtype == DSB_DTYPE_BF16 ? 2 : 1) : 0;
  DSB_REQUIRE(!dx_act || dtype == DSB_DTYPE_BF16 || dtype == DSB_DTYPE_TF32, "layernorm_bwd: dx_act dtype must be DSB_DTYPE_TF32 or DSB_DTYPE_BF16");
  dim3 grid((L + LNB_ROWS - 1) / LNB_ROWS, B);
  switch (D / 128) {
#define DSB_LNB_CASE(N) case N: layernorm_bwd_kernel<MODE, N><<<grid, 256, 0, st>>>(x, dy, dx_io, p0, idx, dg, db, L, D, eps, dx_act, act_mode); break;
    DSB_LNB_CASE(1) DSB_LNB_CASE(2) DSB_LNB_CASE(3) DSB_LNB_CASE(4) DSB_LNB_CASE(5) DSB_LNB_CASE(6) DSB_LNB_CASE(7) DSB_LNB_CASE(8)
#undef DSB_LNB_CASE
    default: set_error("layernorm_bwd: D=%d unsupported (need D %% 128 == 0 and D <= 1024)", D); return 2;
  }
  DSB_CHECK_CUDA(cudaGetLastError());
  return 0;
}
extern "C" int dsb_layernorm_bwd(const float* x, const float* dy, float* dx_io, const float* gamma, float* dgamma, float* dbeta, long long rows, int D,
                                 float eps, void* dx_act, int dtype, void* stream) {
  DSB_REQUIRE(D % 128 == 0 && rows > 0 && rows < (1LL << 31), "dsb_layernorm_bwd: bad shape");
  return launch_ln_bwd<0>(x, dy, dx_io, gamma, nullptr, dgamma, dbeta, 1, (int)rows, D, eps, dx_act, dtype, (cudaStream_t)stream);
}
extern "C" int dsb_ada_layernorm_bwd(const float* x, const float* dy, float* dx_io, const float* table, const int64_t* idx, float* dtable, int B, int L,
                                     int D, float eps, void* dx_act, int dtype, void* stream) {
  DSB_REQUIRE(D % 128 == 0 && B > 0 && L > 0 && B <= 65535, "dsb_ada_layernorm_bwd: bad shape");
  return launch_ln_bwd<1>(x, dy, dx_io, table, idx, dtable, nullptr, B, L, D, eps, dx_act, dtype, (cudaStream_t)stream);
}

extern "C" int dsb_softmax_fwd(const float* S, long long ld_s, void* P, long long ld_p, long long rows, int n, int dtype, void* stream) {
  DSB_ACT_CALL(dtype, run_softmax_fwd, S, ld_s, P, ld_p, rows, n, (cudaStream_t)stream);
  return 0;
}
extern "C" int dsb_softmax_bwd(const void* P, long long ld_p, const float* dP, long long ld_dp, void* dS, long long ld_ds, long long rows, int n,
                               float alpha, int dtype, void* stream) {
  DSB_ACT_CALL(dtype, run_softmax_bwd, P, ld_p, dP, ld_dp, dS, ld_ds, rows, n, alpha, (cudaStream_t)stream);
  return 0;
}

extern "C" int dsb_embed_bwd(const int64_t* ids, const float* dx, float* demb, float* dheight, float* dwidth, int B, int L, int D, int H, int W,
                             int num_embed, void* stream) {
  DSB_REQUIRE(L <= H * W, "dsb_embed_bwd: L=%d exceeds the %dx%d grid", L, H, W);
  cudaStream_t st = (cudaStream_t)stream;
  const long long rows = (long long)B * L;
  embed_bwd_tokens_kernel<<<grid_for(rows * D), 256, 0, st>>>(ids, dx, demb, rows, D, num_embed);
  DSB_CHECK_CUDA(cudaGetLastError());
  embed_bwd_pos_kernel<<<dim3((D + 255) / 256, H + W), 256, 0, st>>>(dx, dheight, dwidth, B, L, D, H, W);
  DSB_CHECK_CUDA(cudaGetLastError());
  return 0;
}
