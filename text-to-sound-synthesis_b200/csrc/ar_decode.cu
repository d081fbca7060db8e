// KV-cached decode of the autoregressive SpecVQGAN transformer (Codebook/specvqgan/modules/transformer/mingpt.py GPTFeats / GPT / Block,
// Codebook/specvqgan/models/cond_transformer.py:124-194 Net2NetTransformer.sample): one position of one batch of rows per launch sequence.
//   embed -> n_layer x [LayerNorm, QKV GEMM, decode attention, proj GEMM + residual, LayerNorm, MLP1 GEMM, GELU(erf) + split, MLP2 GEMM + residual]
//   -> ln_f -> head GEMM -> sampler step
// The GEMMs and LayerNorms are the existing split-fp16 entry points with M = B rows; this file holds the pieces that are specific to the
// decode loop.  Every kernel reads the current position p from a device loop-control block (64-bit words), and the sampler's last CTA
// advances it, so one captured step replays for every position without host work between replays:
//   [0] seed  [1] philox offset  [2] offset increment per sampled position  [3] ATen's thread count (256 * grid)  [4] position p
//   [5] number of positions  [6] first position that samples  [7] CTA ticket
// A position at or past [5] is a no-op in every kernel (a replay past the end writes nothing).
// The full-sequence forward (scoring: Net2NetTransformer.shared_step) uses dsb_ar_embed_all for every position at once and dsb_ar_cross_entropy
// on the head's logits; its attention is dsb_attention_tc_split_causal.
#include "common.cuh"
#include "diffsound_b200.h"
#include "philox.cuh"
#include <cuda_fp16.h>

namespace dsb {
namespace {
constexpr int AR_SEED = 0, AR_OFFSET = 1, AR_OFFSET_INC = 2, AR_NTHREADS = 3, AR_POS = 4, AR_NPOS = 5, AR_FIRST = 6, AR_TICKET = 7;
constexpr int ANT = 256;   // threads of the attention and sampler CTAs
constexpr int ANW = ANT / 32;
constexpr int AR_MAX_CAP = 16;  // sampler: V <= 256 * 16

__device__ __forceinline__ void store_pair(__half* hi, __half* lo, float v) {  // the dsb_split_f16 pair: hi = f16(v), lo = f16(v - hi)
  const __half h = __float2half_rn(v);
  *hi = h;
  *lo = __float2half_rn(v - __half2float(h));
}

// Fixed-order CTA reductions: each thread's own value, a warp xor butterfly 16 ... 1, then the ANW warp partials in ascending warp order.
// `red` is a shared scratch of ANW words; the leading barrier lets the caller reuse it back to back.
template <class V, class Op>
__device__ __forceinline__ V cta_reduce(V v, V* red, Op op) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = op(v, __shfl_xor_sync(0xffffffffu, v, o));
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  V r = red[0];
#pragma unroll
  for (int w = 1; w < ANW; ++w) r = op(r, red[w]);
  return r;
}
__device__ __forceinline__ uint32_t ord_key(float v) {
  const uint32_t bits = __float_as_uint(v + 0.0f);  // -0 and +0 compare equal in the reference: one key
  return (bits & 0x80000000u) ? ~bits : (bits | 0x80000000u);
}
__device__ __forceinline__ void pick(float& best, int& besti, float ob, int oi) {
  if (ob > best || (ob == best && oi < besti)) { best = ob; besti = oi; }
}
}  // namespace

// ---- embed: x[b] = (p < Tc ? cond[b, p] : tok_emb[ids[b, p - Tc]]) + pos_emb[p]     (mingpt.py:167-176, GPTFeats.forward :276-293)
__global__ void ar_embed_kernel(const float* __restrict__ cond, const float* __restrict__ tok_emb, const float* __restrict__ pos_emb,
                                const int64_t* __restrict__ ids, long long ids_ld, float* __restrict__ x, const unsigned long long* ctrl, int Tc, int V,
                                int D, int* err) {
  const long long p = (long long)ctrl[AR_POS];
  if (p >= (long long)ctrl[AR_NPOS]) return;
  const int b = blockIdx.x;
  const float* src;
  if (p < Tc) {
    src = cond + ((long long)b * Tc + p) * D;
  } else {
    long long id = ids[(long long)b * ids_ld + (p - Tc)];
    if (id < 0 || id >= V) {
      if (threadIdx.x == 0 && err) atomicExch(err, 1);
      id = 0;
    }
    src = tok_emb + id * D;
  }
  const float* pe = pos_emb + p * D;
  for (int d = threadIdx.x; d < D; d += blockDim.x) x[(long long)b * D + d] = src[d] + pe[d];
}

// ---- embed of every position: x[b, t] = (t < Tc ? cond[b, t] : tok_emb[ids[b, t - Tc]]) + pos_emb[t], t < T  (the same fp32 sum as ar_embed)
__global__ void ar_embed_all_kernel(const float* __restrict__ cond, const float* __restrict__ tok_emb, const float* __restrict__ pos_emb,
                                    const int64_t* __restrict__ ids, long long ids_ld, float* __restrict__ x, int T, int Tc, int V, int D, int* err) {
  const int t = blockIdx.x, b = blockIdx.y;
  const float* src;
  if (t < Tc) {
    src = cond + ((long long)b * Tc + t) * D;
  } else {
    long long id = ids[(long long)b * ids_ld + (t - Tc)];
    if (id < 0 || id >= V) {
      if (threadIdx.x == 0 && err) atomicExch(err, 1);
      id = 0;
    }
    src = tok_emb + id * D;
  }
  const float* pe = pos_emb + (long long)t * D;
  float* xr = x + ((long long)b * T + t) * D;
  for (int d = threadIdx.x; d < D; d += blockDim.x) xr[d] = src[d] + pe[d];
}

// ---- cross-entropy of one logits row per CTA (F.cross_entropy, reduction 'none', ignore_index -100), rows r0 ... r0 + n - 1 of every batch item:
//   m = max_k l_k;  S = sum_k expf(l_k - m) (thread-strided ascending k, then cta_reduce);  nll = logf(S) - (l_y - m);  an ignored row is 0.
// A target outside [0, V) (other than -100) sets err and writes NaN.  Nothing depends on B.
__global__ void __launch_bounds__(ANT) ar_xent_rows_kernel(const float* __restrict__ logits, long long ld, int T, int r0, int n,
                                                           const int64_t* __restrict__ targets, long long tgt_ld, float* __restrict__ nll, int V, int* err) {
  __shared__ float red[ANW];
  const int i = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
  const long long y = targets[(long long)b * tgt_ld + i];
  float* out = nll + (long long)b * n + i;
  if (y == -100) {
    if (tid == 0) *out = 0.f;
    return;
  }
  if (y < 0 || y >= V) {
    if (tid == 0) {
      *out = NAN;
      if (err) atomicExch(err, 1);
    }
    return;
  }
  const float* row = logits + ((long long)b * T + r0 + i) * ld;
  float mx = -INFINITY;
  for (int k = tid; k < V; k += ANT) mx = fmaxf(mx, row[k]);
  mx = cta_reduce(mx, red, [](float a, float c) { return fmaxf(a, c); });
  float se = 0.f;
  for (int k = tid; k < V; k += ANT) se += expf(row[k] - mx);
  se = cta_reduce(se, red, [](float a, float c) { return a + c; });
  if (tid == 0) *out = logf(se) - (row[y] - mx);
}

// ---- mean over the non-ignored rows: the fp64 NLLs added by one thread in ascending row order (b-major), staged through shared memory in chunks
// (an ignored row enters as +0.0, which leaves every partial sum unchanged); the count is an integer sum.  0 rows give 0 / 0 = NaN, as
// F.cross_entropy does.
constexpr int XENT_CHUNK = 2048;
__global__ void __launch_bounds__(ANT) ar_xent_mean_kernel(const float* __restrict__ nll, const int64_t* __restrict__ targets, long long tgt_ld, int B,
                                                           int n, float* loss) {
  __shared__ double vals[XENT_CHUNK];
  __shared__ int redi[ANW];
  const long long rows = (long long)B * n;
  double sum = 0.0;
  int cnt = 0;
  for (long long c0 = 0; c0 < rows; c0 += XENT_CHUNK) {
    const int len = (int)min((long long)XENT_CHUNK, rows - c0);
    for (int i = threadIdx.x; i < len; i += ANT) {
      const long long r = c0 + i, b = r / n;
      const bool keep = targets[b * tgt_ld + (r - b * n)] != -100;
      vals[i] = keep ? (double)nll[r] : 0.0;
      cnt += keep ? 1 : 0;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
#pragma unroll 8
      for (int i = 0; i < len; ++i) sum += vals[i];
    }
    __syncthreads();
  }
  cnt = cta_reduce(cnt, redi, [](int a, int e) { return a + e; });
  if (threadIdx.x == 0) *loss = (float)(sum / (double)cnt);
}

// ---- decode attention for one (head, b) at position p  (mingpt.py:76-94 with a KV cache)
// Copies K / V of position p from the QKV GEMM's fp32 output into the layer's cache, then over cache rows j = 0 ... p:
//   s_j = (sum_d q_d k_jd, ascending d, FMA) * scale;  m = max_j s_j;  e_j = expf(s_j - m);  S = sum_j e_j;  p_j = e_j / S;
//   o_d = sum_j p_j v_jd  (each of ANT / HD thread groups sums a contiguous j chunk in ascending j, the chunks are added in ascending order)
// and writes o as the fp16 (hi | lo) pair the proj GEMM reads.  Max and sum use cta_reduce.  Nothing depends on B.
template <int HD>
__global__ void __launch_bounds__(ANT) ar_attention_kernel(const float* __restrict__ qkv, long long ld_qkv, float* kc, float* vc, long long cache_ld,
                                                           __half* __restrict__ out, long long ld_out, long long lo_off, const unsigned long long* ctrl,
                                                           int H, float scale, int max_pos) {
  extern __shared__ float sm[];
  constexpr int KS = HD + 1;  // padded K row: thread j reading its own row hits 32 distinct banks
  constexpr int G = ANT / HD;
  const unsigned long long pos = ctrl[AR_POS];
  // shared memory and the cache rows hold max_pos positions: a position past them (a control block the caller armed beyond the cache) is a no-op
  if (pos >= ctrl[AR_NPOS] || pos >= (unsigned long long)max_pos) return;
  const int p = (int)pos;
  const int h = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
  const int D = H * HD;
  const int n = p + 1;
  float* q_s = sm;                // [HD]
  float* pr_s = q_s + HD;         // [n] probabilities
  float* part = pr_s + n;         // [G][HD] partial outputs
  float* red = part + G * HD;     // [ANW]
  float* k_s = red + ANW;         // [n][KS]
  const float* row = qkv + (long long)b * ld_qkv + h * HD;
  float* kb = kc + (long long)b * cache_ld + h * HD;  // row j at kb + j * D
  float* vb = vc + (long long)b * cache_ld + h * HD;
  if (tid < HD) {
    q_s[tid] = row[tid];
    kb[(long long)p * D + tid] = row[D + tid];
    vb[(long long)p * D + tid] = row[2 * D + tid];
  }
  __syncthreads();  // the cache rows written above are read below by other threads of this CTA
  for (int i = tid; i < n * HD; i += ANT) {
    const int j = i / HD, d = i - j * HD;
    k_s[j * KS + d] = kb[(long long)j * D + d];
  }
  __syncthreads();
  float s[2];  // n <= 512
  float mx = -INFINITY;
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int j = tid + ANT * r;
    float acc = -INFINITY;
    if (j < n) {
      acc = 0.f;
#pragma unroll
      for (int d = 0; d < HD; ++d) acc = fmaf(q_s[d], k_s[j * KS + d], acc);
      acc = acc * scale;
    }
    s[r] = acc;
    mx = fmaxf(mx, acc);
  }
  mx = cta_reduce(mx, red, [](float a, float c) { return fmaxf(a, c); });
  float se = 0.f;
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int j = tid + ANT * r;
    s[r] = j < n ? expf(s[r] - mx) : 0.f;
    se += s[r];
  }
  se = cta_reduce(se, red, [](float a, float c) { return a + c; });
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int j = tid + ANT * r;
    if (j < n) pr_s[j] = s[r] / se;
  }
  __syncthreads();
  const int g = tid / HD, d = tid - g * HD;
  const int chunk = (n + G - 1) / G;
  const int j0 = g * chunk, j1 = min(n, j0 + chunk);
  float acc = 0.f;
  for (int j = j0; j < j1; ++j) acc = fmaf(pr_s[j], vb[(long long)j * D + d], acc);
  part[g * HD + d] = acc;
  __syncthreads();
  if (tid < HD) {
    float o = part[tid];
#pragma unroll
    for (int gg = 1; gg < G; ++gg) o += part[gg * HD + tid];
    __half* orow = out + (long long)b * ld_out + h * HD + tid;
    store_pair(orow, orow + lo_off, o);
  }
}

// ---- GELU (exact erf form, torch.nn.GELU()) + split: out[r, c] = hi, out[r, lo_off + c] = lo of x * 0.5 * (1 + erf(x / sqrt(2)))
__global__ void ar_gelu_split_kernel(const float* __restrict__ in, long long ld_in, __half* __restrict__ out, long long ld_out, long long lo_off, int rows,
                                     int C) {
  const long long n = (long long)rows * C;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / C, c = i - r * C;
    const float x = in[r * ld_in + c];
    const float y = x * 0.5f * (1.0f + erff(x * 0.70710678118654752440f));
    __half* o = out + r * ld_out + c;
    store_pair(o, o + lo_off, y);
  }
}

// ---- sampler step, one CTA per row b  (cond_transformer.py:118-122 top_k_logits, :171-186)
// Element k = tid + ANT * j.  l_k = logits_k / temperature (fp32 division);  top-k: keep l_k >= the k-th largest value (ties at it kept), found
// by bisection over the order-preserving 32-bit key of the value (count of keys >= t, cta_reduce);  fp32 softmax over the kept entries (max and
// sum by cta_reduce, p_k = expf(l_k - m) / S);  sampling: torch.multinomial(probs, 1)'s fast path, argmax of p_k / q_k with q the replayed
// exponential_(1) of the (B, V) tensor;  greedy: argmax p_k.  Ties go to the lowest index.

template <int CAP>
__global__ void __launch_bounds__(ANT) ar_sample_kernel(const float* __restrict__ logits, long long ld_logits, int64_t* ids, long long ids_ld,
                                                        unsigned long long* ctrl, int V, int Tc, float temperature, int top_k, int do_sample,
                                                        float* __restrict__ probs_out, float* __restrict__ hist, long long hist_ld, int* err) {
  __shared__ float redf[ANW];
  __shared__ int redi[ANW];
  const int b = blockIdx.x, tid = threadIdx.x;
  const unsigned long long p = ctrl[AR_POS];
  const bool live = p < ctrl[AR_NPOS];
  const bool sampled = live && p >= ctrl[AR_FIRST];
  const unsigned long long rng_seed = ctrl[AR_SEED], rng_off = ctrl[AR_OFFSET], rng_n = ctrl[AR_NTHREADS];
  if (live) {
    const float* row = logits + (long long)b * ld_logits;
    float l[CAP];
#pragma unroll
    for (int j = 0; j < CAP; ++j) {
      const int k = tid + ANT * j;
      const float raw = k < V ? row[k] : 0.f;
      if (hist && k < V) hist[(long long)b * hist_ld + (long long)p * V + k] = raw;
      l[j] = k < V ? __fdiv_rn(raw, temperature) : -INFINITY;
    }
    if (top_k > 0 && top_k < V) {
      // kth = the largest key t with #{key_k >= t} >= top_k (the top_k-th largest value, counted with multiplicity)
      uint32_t key[CAP];
#pragma unroll
      for (int j = 0; j < CAP; ++j) key[j] = (tid + ANT * j < V) ? ord_key(l[j]) : 0u;  // padding below every real key (NaN aside)
      uint32_t lo = 0u, hi = 0xFFFFFFFFu;  // invariant: count(>= lo) >= top_k, count(>= hi + 1) < top_k when hi < max
      while (lo < hi) {
        const uint32_t mid = (uint32_t)(((unsigned long long)lo + hi + 1ull) >> 1);  // 64-bit sum: hi - lo + 1 overflows at the start
        int c = 0;
#pragma unroll
        for (int j = 0; j < CAP; ++j) c += (tid + ANT * j < V && key[j] >= mid) ? 1 : 0;
        c = cta_reduce(c, redi, [](int a, int e) { return a + e; });
        if (c >= top_k) lo = mid; else hi = mid - 1u;
      }
#pragma unroll
      for (int j = 0; j < CAP; ++j)
        if (tid + ANT * j < V && key[j] < lo) l[j] = -INFINITY;
    }
    float mx = -INFINITY;
#pragma unroll
    for (int j = 0; j < CAP; ++j) mx = fmaxf(mx, l[j]);
    mx = cta_reduce(mx, redf, [](float a, float e) { return fmaxf(a, e); });
    float e[CAP];
    float se = 0.f;
#pragma unroll
    for (int j = 0; j < CAP; ++j) {
      e[j] = (tid + ANT * j < V) ? expf(l[j] - mx) : 0.f;
      se += e[j];
    }
    se = cta_reduce(se, redf, [](float a, float c) { return a + c; });
    float best = -INFINITY;
    int besti = 0x7fffffff;
    int bad = 0;
#pragma unroll
    for (int j = 0; j < CAP; ++j) {
      const int k = tid + ANT * j;
      if (k < V) {
        const float pk = e[j] / se;
        if (isnan(pk)) bad = 1;
        if (probs_out) probs_out[(long long)b * V + k] = pk;
        float val = pk;
        if (do_sample) val = __fdiv_rn(pk, aten_exponential(rng_seed, rng_off, rng_n, (unsigned long long)b * V + k));
        if (val > best) { best = val; besti = k; }  // ascending k per thread: keeps the first maximum
      }
    }
    if (bad && err) atomicExch(err, 1);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) pick(best, besti, __shfl_xor_sync(0xffffffffu, best, o), __shfl_xor_sync(0xffffffffu, besti, o));
    __syncthreads();
    if ((tid & 31) == 0) { redf[tid >> 5] = best; redi[tid >> 5] = besti; }
    __syncthreads();
    if (tid == 0 && sampled) {
      best = redf[0];
      besti = redi[0];
      for (int w = 1; w < ANW; ++w) pick(best, besti, redf[w], redi[w]);
      if (besti >= V) besti = 0;  // every value NaN (already flagged)
      ids[(long long)b * ids_ld + (long long)(p - Tc + 1)] = besti;
    }
  }
  __syncthreads();
  if (tid == 0) {  // the last CTA to retire (every CTA has read p and the offset by then) moves the loop to the next position
    __threadfence();
    if (atomicAdd(&ctrl[AR_TICKET], 1ull) == (unsigned long long)gridDim.x - 1ull) {
      ctrl[AR_TICKET] = 0ull;
      if (live) {
        ctrl[AR_POS] = p + 1ull;
        if (sampled && do_sample) ctrl[AR_OFFSET] = rng_off + ctrl[AR_OFFSET_INC];
      }
      __threadfence();
    }
  }
}

__global__ void aten_exponential_fill_kernel(float* out, long long n, unsigned long long seed, unsigned long long offset, unsigned long long nthreads) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    out[i] = aten_exponential(seed, offset, nthreads, (unsigned long long)i);
}

template <int CAP>
static int launch_ar_sample(const float* logits, long long ld_logits, int64_t* ids, long long ids_ld, unsigned long long* ctrl, int B, int V, int Tc,
                     float temperature, int top_k, int do_sample, float* probs_out, float* hist, long long hist_ld, int* err, cudaStream_t st) {
  ar_sample_kernel<CAP><<<B, ANT, 0, st>>>(logits, ld_logits, ids, ids_ld, ctrl, V, Tc, temperature, top_k, do_sample, probs_out, hist, hist_ld, err);
  DSB_CHECK_CUDA(cudaGetLastError());
  return 0;
}
}  // namespace dsb
using namespace dsb;

extern "C" int dsb_ar_embed(const float* cond, const float* tok_emb, const float* pos_emb, const int64_t* ids, long long ids_ld, float* x,
                            const unsigned long long* ctrl, int B, int Tc, int V, int D, int* err_flag, void* stream) {
  DSB_REQUIRE(B > 0 && Tc >= 0 && V > 0 && D > 0, "dsb_ar_embed: bad shape");
  DSB_REQUIRE((cond || Tc == 0) && tok_emb && pos_emb && ids && x && ctrl, "dsb_ar_embed: null argument");  // no condition rows: cond unused
  ar_embed_kernel<<<B, 256, 0, (cudaStream_t)stream>>>(cond, tok_emb, pos_emb, ids, ids_ld, x, ctrl, Tc, V, D, err_flag);
  DSB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dsb_ar_embed_all(const float* cond, const float* tok_emb, const float* pos_emb, const int64_t* ids, long long ids_ld, float* x, int B,
                                int T, int Tc, int V, int D, int* err_flag, void* stream) {
  DSB_REQUIRE(B > 0 && B <= 65535 && T > 0 && Tc >= 0 && Tc <= T && V > 0 && D > 0, "dsb_ar_embed_all: bad shape (B=%d T=%d Tc=%d)", B, T, Tc);
  DSB_REQUIRE((cond || Tc == 0) && tok_emb && pos_emb && (ids || Tc == T) && x, "dsb_ar_embed_all: null argument");
  ar_embed_all_kernel<<<dim3(T, B), 256, 0, (cudaStream_t)stream>>>(cond, tok_emb, pos_emb, ids, ids_ld, x, T, Tc, V, D, err_flag);
  DSB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dsb_ar_cross_entropy(const float* logits, long long ld, int T, int r0, int n, const int64_t* targets, long long tgt_ld, float* nll,
                                    float* loss, int B, int V, int* err_flag, void* stream) {
  DSB_REQUIRE(B > 0 && B <= 65535 && n > 0 && r0 >= 0 && r0 + n <= T && V > 0 && ld >= V, "dsb_ar_cross_entropy: bad shape (B=%d T=%d r0=%d n=%d V=%d)",
              B, T, r0, n, V);
  DSB_REQUIRE(V <= ANT * AR_MAX_CAP, "dsb_ar_cross_entropy: V=%d too large (max %d)", V, ANT * AR_MAX_CAP);
  DSB_REQUIRE(logits && targets && nll && loss, "dsb_ar_cross_entropy: null argument");
  cudaStream_t st = (cudaStream_t)stream;
  ar_xent_rows_kernel<<<dim3(n, B), ANT, 0, st>>>(logits, ld, T, r0, n, targets, tgt_ld, nll, V, err_flag);
  DSB_CHECK_CUDA(cudaGetLastError());
  ar_xent_mean_kernel<<<1, ANT, 0, st>>>(nll, targets, tgt_ld, B, n, loss);
  DSB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dsb_ar_attention(const float* qkv, long long ld_qkv, float* k_cache, float* v_cache, long long cache_ld, int max_pos, void* out,
                                long long ld_out, long long lo_off, const unsigned long long* ctrl, int B, int H, int head_dim, float scale, void* stream) {
  DSB_REQUIRE(head_dim == 32 || head_dim == 64, "dsb_ar_attention: head_dim=%d unsupported (32 or 64)", head_dim);
  DSB_REQUIRE(B > 0 && B <= 65535 && H > 0 && max_pos > 0 && max_pos <= 2 * ANT, "dsb_ar_attention: bad shape (B=%d H=%d max_pos=%d, max_pos <= %d)",
              B, H, max_pos, 2 * ANT);
  DSB_REQUIRE(qkv && k_cache && v_cache && out && ctrl, "dsb_ar_attention: null argument");
  const int KS = head_dim + 1, G = ANT / head_dim;
  const size_t smem = sizeof(float) * ((size_t)head_dim + max_pos + (size_t)G * head_dim + ANW + (size_t)max_pos * KS);
  cudaStream_t st = (cudaStream_t)stream;
  const dim3 grid(H, B);
  if (head_dim == 64) {
    DSB_CHECK_CUDA(cudaFuncSetAttribute(ar_attention_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    ar_attention_kernel<64><<<grid, ANT, smem, st>>>(qkv, ld_qkv, k_cache, v_cache, cache_ld, (__half*)out, ld_out, lo_off, ctrl, H, scale, max_pos);
  } else {
    DSB_CHECK_CUDA(cudaFuncSetAttribute(ar_attention_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    ar_attention_kernel<32><<<grid, ANT, smem, st>>>(qkv, ld_qkv, k_cache, v_cache, cache_ld, (__half*)out, ld_out, lo_off, ctrl, H, scale, max_pos);
  }
  DSB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dsb_gelu_erf_split(const float* in, long long ld_in, void* out, long long ld_out, long long lo_off, int rows, int C, void* stream) {
  DSB_REQUIRE(rows > 0 && C > 0 && in && out, "dsb_gelu_erf_split: bad argument");
  const long long n = (long long)rows * C;
  long long g = (n + 255) / 256;
  const long long cap = (long long)sm_count() * 8;
  ar_gelu_split_kernel<<<(unsigned)(g > cap ? cap : g), 256, 0, (cudaStream_t)stream>>>(in, ld_in, (__half*)out, ld_out, lo_off, rows, C);
  DSB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dsb_ar_sample(const float* logits, long long ld_logits, int64_t* ids, long long ids_ld, unsigned long long* ctrl, int B, int V, int Tc,
                             float temperature, int top_k, int do_sample, float* probs_out, float* logits_hist, long long hist_ld, int* err_flag,
                             void* stream) {
  DSB_REQUIRE(B > 0 && V > 0 && Tc >= 0, "dsb_ar_sample: bad shape");
  DSB_REQUIRE(V <= ANT * AR_MAX_CAP, "dsb_ar_sample: V=%d too large (max %d)", V, ANT * AR_MAX_CAP);
  DSB_REQUIRE(top_k >= 0 && top_k <= V, "dsb_ar_sample: top_k=%d out of range (0 = no truncation, else 1 ... V=%d)", top_k, V);
  DSB_REQUIRE(temperature == temperature && temperature != 0.f, "dsb_ar_sample: temperature must be a non-zero number");
  DSB_REQUIRE(logits && ids && ctrl, "dsb_ar_sample: null argument");
  cudaStream_t st = (cudaStream_t)stream;
  const int cap = (V + ANT - 1) / ANT;
#define DSB_AR_CASE(N) \
  if (cap <= N) return launch_ar_sample<N>(logits, ld_logits, ids, ids_ld, ctrl, B, V, Tc, temperature, top_k, do_sample, probs_out, logits_hist, hist_ld, err_flag, st)
  DSB_AR_CASE(1);
  DSB_AR_CASE(2);
  DSB_AR_CASE(4);
  DSB_AR_CASE(8);
  DSB_AR_CASE(AR_MAX_CAP);
#undef DSB_AR_CASE
  return 2;
}

extern "C" int dsb_aten_exponential(float* out, long long n, unsigned long long seed, unsigned long long offset, unsigned long long nthreads,
                                    void* stream) {
  DSB_REQUIRE(n > 0 && nthreads > 0 && offset % 4 == 0, "dsb_aten_exponential: need n > 0, nthreads > 0 and a philox offset that is a multiple of 4");
  long long g = (n + 255) / 256;
  const long long cap = (long long)sm_count() * 8;
  aten_exponential_fill_kernel<<<(unsigned)(g > cap ? cap : g), 256, 0, (cudaStream_t)stream>>>(out, n, seed, offset, nthreads);
  DSB_CHECK_CUDA(cudaGetLastError());
  return 0;
}
