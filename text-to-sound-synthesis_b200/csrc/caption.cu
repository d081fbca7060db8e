// ACT audio-captioning transformer (Codebook/AudiocaptionLoss/models/TransModel.py ACT, models/AudioTransformer.py AudioTransformer_80,
// tools/utils.py greedy_decode, tools/beam.py beam_decode): the pieces of the encoder front end and of one decode step that the split-fp16
// GEMMs, dsb_layernorm, dsb_attention_tc_split and dsb_gelu_erf_split do not cover.
//   encoder:  frontend (BatchNorm2d eval affine + split of the 4 x 80 patch rows) -> patch GEMM -> tokens (cls + positional embedding) -> ...
//   decode step (R rows, each row one node of its own clip):
//     embed -> n_layer x [split, QKV GEMM, tree self-attention, out_proj + residual, LayerNorm, Q GEMM, cross-attention, out_proj + residual,
//     LayerNorm, FF1, GELU + split, FF2 + residual, LayerNorm] -> dec_fc -> select
// Every kernel works in fp32 with a reduction order that depends neither on R nor on which other rows are present.
#include "common.cuh"
#include "diffsound_b200.h"
#include <cuda_fp16.h>

namespace dsb {
namespace {
constexpr int CT = 256;        // threads of the attention and select CTAs
constexpr int CW = CT / 32;
constexpr int HD = 64;         // the decoder's head_dim (nhid 512 / nhead 8)
constexpr int CG = CT / HD;    // P.V thread groups
constexpr int CAP_MAX_LEN = 16384;
constexpr int CAP_MAX_V = 16384;
constexpr int CAP_MAX_K = 16;

__device__ __forceinline__ void cap_store_pair(__half* hi, long long lo_off, float v) {  // the dsb_split_f16 pair
  const __half h = __float2half_rn(v);
  hi[0] = h;
  hi[lo_off] = __float2half_rn(v - __half2float(h));
}

// Fixed-order CTA reduction: a warp xor butterfly 16 ... 1, then the CW warp partials in ascending warp order (leading barrier: `red` reusable).
template <class V, class Op>
__device__ __forceinline__ V cap_reduce(V v, V* red, Op op) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = op(v, __shfl_xor_sync(0xffffffffu, v, o));
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  V r = red[0];
#pragma unroll
  for (int w = 1; w < CW; ++w) r = op(r, red[w]);
  return r;
}

// (value desc, index asc): true when (v, i) comes before (bv, bi)
__device__ __forceinline__ bool cap_before(float v, int i, float bv, int bi) { return v > bv || (v == bv && i < bi); }

__device__ __forceinline__ void cap_pick_cta(float& best, int& besti, float* redf, int* redi) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, besti, o);
    if (cap_before(ov, oi, best, besti)) { best = ov; besti = oi; }
  }
  __syncthreads();
  if ((threadIdx.x & 31) == 0) { redf[threadIdx.x >> 5] = best; redi[threadIdx.x >> 5] = besti; }
  __syncthreads();
  best = redf[0];
  besti = redi[0];
  for (int w = 1; w < CW; ++w)
    if (cap_before(redf[w], redi[w], best, besti)) { best = redf[w]; besti = redi[w]; }
}

// One query row of one head against n keys (key j of this head at k + koff(j), its value at v + koff(j)), fp32:
//   s_j = (q_2l k_2l + q_2l+1 k_2l+1 per lane, xor butterfly 16 ... 1) * scale;  m = max_j s_j;  e_j = expf(s_j - m);  S = sum_j e_j
//   (thread-strided ascending j, then cap_reduce);  p_j = e_j / S;  o_d = sum_j p_j v_jd (CG groups of contiguous ascending j, added in group order).
// o goes out as the fp16 (hi | lo) pair.  Shared memory: q[HD], part[CG * HD], red[CW], p[n].
template <class KOff>
__device__ __forceinline__ void cap_attend(const float* __restrict__ q, const float* k, const float* v, KOff koff, int n, float scale, float* sm,
                                           __half* out, long long lo_off) {
  float* q_s = sm;
  float* part = q_s + HD;
  float* red = part + CG * HD;
  float* p_s = red + CW;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid < HD) q_s[tid] = q[tid];
  __syncthreads();
  const float q0 = q_s[2 * lane], q1 = q_s[2 * lane + 1];
  for (int j = warp; j < n; j += CW) {
    const float2 kk = *reinterpret_cast<const float2*>(k + koff(j) + 2 * lane);
    float d = fmaf(q1, kk.y, q0 * kk.x);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
    if (lane == 0) p_s[j] = d * scale;
  }
  __syncthreads();
  float mx = -INFINITY;
  for (int j = tid; j < n; j += CT) mx = fmaxf(mx, p_s[j]);
  mx = cap_reduce(mx, red, [](float a, float b) { return fmaxf(a, b); });
  float se = 0.f;
  for (int j = tid; j < n; j += CT) {
    const float e = expf(p_s[j] - mx);
    p_s[j] = e;
    se += e;
  }
  se = cap_reduce(se, red, [](float a, float b) { return a + b; });
  for (int j = tid; j < n; j += CT) p_s[j] = p_s[j] / se;
  __syncthreads();
  const int g = tid / HD, d = tid - g * HD;
  const int chunk = (n + CG - 1) / CG;
  const int j0 = g * chunk, j1 = min(n, j0 + chunk);
  float acc = 0.f;
  for (int j = j0; j < j1; ++j) acc = fmaf(p_s[j], v[koff(j) + d], acc);
  part[g * HD + d] = acc;
  __syncthreads();
  if (tid < HD) {
    float o = part[tid];
#pragma unroll
    for (int gg = 1; gg < CG; ++gg) o += part[gg * HD + tid];
    cap_store_pair(out + tid, lo_off, o);
  }
}
}  // namespace

// ---- encoder front end: BatchNorm2d(80) eval affine y = x * alpha[f] + beta[f] (mul, then add) and the 4 x 80 patch rearrange, which is the
// plain reshape of (T, 80) into (T / 4, 320); out row r = b * T / 4 + h is the split pair [hi(320) | lo(320)].
__global__ void cap_frontend_kernel(const float* __restrict__ spec, long long spec_bs, int T, const float* __restrict__ alpha,
                                    const float* __restrict__ beta, __half* __restrict__ out, long long rows) {
  const int n = T / 4;
  const long long total = rows * 320;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / 320;
    const int c = (int)(i - r * 320);
    const long long b = r / n;
    const int h = (int)(r - b * n), f = c % 80;
    const float x = spec[b * spec_bs + (long long)(4 * h) * 80 + c];
    cap_store_pair(out + r * 640 + c, 320, __fadd_rn(__fmul_rn(x, alpha[f]), beta[f]));
  }
}

// ---- tokens: x[b, 0] = cls + pos[0];  x[b, i] = patch[b * n + i - 1] + pos[i]  (torch.cat((cls_token, x), 1); x += pos_embedding[:, :n + 1])
__global__ void cap_tokens_kernel(const float* __restrict__ patch, const float* __restrict__ cls, const float* __restrict__ pos, float* __restrict__ x,
                                  int n, int D) {
  const int i = blockIdx.x, b = blockIdx.y;
  const float* src = i == 0 ? cls : patch + ((long long)b * n + i - 1) * D;
  float* dst = x + ((long long)b * (n + 1) + i) * D;
  for (int d = threadIdx.x; d < D; d += blockDim.x) dst[d] = src[d] + pos[(long long)i * D + d];
}

// ---- decode embed: x[r] = table[tok[r]] + pe[pos[r]]  (table = word_emb * sqrt(nhid), so this is decode()'s fp32 emb * sqrt(d) + pe[p])
__global__ void cap_embed_kernel(const int64_t* __restrict__ tok, const int* __restrict__ pos, const float* __restrict__ table,
                                 const float* __restrict__ pe, float* __restrict__ x, int V, int D, int max_pos, int* err) {
  const int r = blockIdx.x;
  long long id = tok[r];
  int p = pos[r];
  if (id < 0 || id >= V || p < 0 || p >= max_pos) {
    if (threadIdx.x == 0 && err) atomicExch(err, 1);
    id = id < 0 || id >= V ? 0 : id;
    p = p < 0 || p >= max_pos ? 0 : p;
  }
  for (int d = threadIdx.x; d < D; d += blockDim.x) x[(long long)r * D + d] = table[id * D + d] + pe[(long long)p * D + d];
}

// ---- tree self-attention, one CTA per (head, row): the row's node owns slot path[start + pos] of the pool; its K / V (from the QKV GEMM) are
// written there, then it attends over the pos + 1 slots path[start ... start + pos], its ancestors' slots from the root down.
// A row whose path does not fit (pos + 1 outside [1, max_len], the list outside [0, path_len), a slot outside [0, n_slots)) sets *err and
// writes nothing.
__global__ void __launch_bounds__(CT) cap_tree_attention_kernel(const float* __restrict__ qkv, long long ld_qkv, float* kp, float* vp, long long pool_ld,
                                                                long long n_slots, const int* __restrict__ path, long long path_len,
                                                                const long long* __restrict__ start, const int* __restrict__ pos, int max_len,
                                                                __half* __restrict__ out, long long ld_out, long long lo_off, int H, float scale,
                                                                int* err) {
  extern __shared__ float sm[];
  __shared__ int redi[CW];
  const int h = blockIdx.x, r = blockIdx.y, tid = threadIdx.x;
  const int D = H * HD;
  const int n = pos[r] + 1;
  const long long st = start[r];
  if (n < 1 || n > max_len || st < 0 || st + n > path_len) {  // uniform over the CTA
    if (tid == 0 && err) atomicExch(err, 1);
    return;
  }
  const int* pr = path + st;
  int bad = 0;
  for (int j = tid; j < n; j += CT) bad |= pr[j] < 0 || (long long)pr[j] >= n_slots;
  bad = cap_reduce(bad, redi, [](int a, int b) { return a | b; });
  if (bad) {
    if (tid == 0 && err) atomicExch(err, 1);
    return;
  }
  const float* row = qkv + (long long)r * ld_qkv + h * HD;
  if (tid < HD) {
    const long long s = (long long)pr[n - 1] * pool_ld + h * HD + tid;
    kp[s] = row[D + tid];
    vp[s] = row[2 * D + tid];
  }
  __syncthreads();  // the slot written above is read below by other threads of this CTA
  cap_attend(row, kp + h * HD, vp + h * HD, [=](int j) { return (long long)pr[j] * pool_ld; }, n, scale, sm,
             out + (long long)r * ld_out + h * HD, lo_off);
}

// ---- cross-attention, one CTA per (head, row): row r's query against the Lm memory rows of clip row_clip[r] (K at kv + (c * Lm + j) * ld_kv,
// V v_off further).  A clip outside [0, n_clips) sets *err and writes nothing.
__global__ void __launch_bounds__(CT) cap_cross_attention_kernel(const float* __restrict__ q, long long ldq, const float* __restrict__ kv,
                                                                 long long ld_kv, long long v_off, int Lm, const int* __restrict__ row_clip, int n_clips,
                                                                 __half* __restrict__ out, long long ld_out, long long lo_off, float scale, int* err) {
  extern __shared__ float sm[];
  const int h = blockIdx.x, r = blockIdx.y;
  const int c = row_clip[r];
  if (c < 0 || c >= n_clips) {
    if (threadIdx.x == 0 && err) atomicExch(err, 1);
    return;
  }
  const long long base = (long long)c * Lm;
  cap_attend(q + (long long)r * ldq + h * HD, kv + h * HD, kv + v_off + h * HD, [=](int j) { return (base + j) * ld_kv; }, Lm, scale, sm,
             out + (long long)r * ld_out + h * HD, lo_off);
}

// ---- row select, one CTA per row.  m = max_k l_k;  S = sum_k expf(l_k - m) (thread-strided ascending k, cap_reduce).
//   k_top > 0 (beam): ls_k = (l_k - m) - logf(S) (F.log_softmax); the k_top largest ls_k in descending order, ties to the lowest index, found
//   as k_top successive maxima of the (value desc, index asc) order below the previous pick -> vals / idx (R, k_top).
//   k_top = 0 (greedy): argmax_k expf(l_k - m) / S (F.softmax then argmax, ties to the lowest index) -> ys[r, pos[r] + 1], tok[r]; pos[r] += 1.
// A NaN or infinite logit sets *err.
__global__ void __launch_bounds__(CT) cap_select_kernel(const float* __restrict__ logits, long long ld, int V, int k_top, float* vals, int64_t* idx,
                                                        int64_t* ys, long long ys_ld, int64_t* tok, int* pos, int* err) {
  __shared__ float redf[CW];
  __shared__ int redi[CW];
  const int r = blockIdx.x, tid = threadIdx.x;
  const float* row = logits + (long long)r * ld;
  float mx = -INFINITY;
  int bad = 0;
  for (int k = tid; k < V; k += CT) {
    const float l = row[k];
    bad |= !isfinite(l);
    mx = fmaxf(mx, l);
  }
  mx = cap_reduce(mx, redf, [](float a, float b) { return fmaxf(a, b); });
  bad = cap_reduce(bad, redi, [](int a, int b) { return a | b; });
  if (bad && tid == 0 && err) atomicExch(err, 1);
  float se = 0.f;
  for (int k = tid; k < V; k += CT) se += expf(row[k] - mx);
  se = cap_reduce(se, redf, [](float a, float b) { return a + b; });
  if (k_top == 0) {
    float best = -INFINITY;
    int besti = 0x7fffffff;
    for (int k = tid; k < V; k += CT) {
      const float p = expf(row[k] - mx) / se;
      if (cap_before(p, k, best, besti)) { best = p; besti = k; }
    }
    cap_pick_cta(best, besti, redf, redi);
    if (tid == 0) {
      const int p = pos[r];
      const int64_t w = besti < V ? besti : 0;  // every value NaN (already flagged)
      ys[(long long)r * ys_ld + p + 1] = w;
      tok[r] = w;
      pos[r] = p + 1;
    }
    return;
  }
  const float lse = logf(se);
  float pv = INFINITY;
  int pi = -1;
  for (int t = 0; t < k_top; ++t) {
    float best = -INFINITY;
    int besti = 0x7fffffff;
    for (int k = tid; k < V; k += CT) {
      const float ls = (row[k] - mx) - lse;
      if (cap_before(pv, pi, ls, k) && cap_before(ls, k, best, besti)) { best = ls; besti = k; }
    }
    cap_pick_cta(best, besti, redf, redi);
    if (tid == 0) {
      vals[(long long)r * k_top + t] = best;
      idx[(long long)r * k_top + t] = besti < V ? besti : 0;
    }
    pv = best;
    pi = besti;
  }
}
}  // namespace dsb
using namespace dsb;

static size_t cap_attend_smem(int n) { return sizeof(float) * ((size_t)HD + (size_t)CG * HD + CW + (size_t)n); }

extern "C" int dsb_caption_frontend(const float* spec, long long spec_bs, int B, int T, const float* alpha, const float* beta, void* out, void* stream) {
  DSB_REQUIRE(B > 0 && T > 0 && T % 4 == 0 && spec_bs >= (long long)T * 80, "dsb_caption_frontend: bad shape (B=%d T=%d, T %% 4 == 0)", B, T);
  DSB_REQUIRE(spec && alpha && beta && out, "dsb_caption_frontend: null argument");
  const long long rows = (long long)B * (T / 4);
  long long g = (rows * 320 + 255) / 256;
  const long long cap = (long long)sm_count() * 8;
  cap_frontend_kernel<<<(unsigned)(g > cap ? cap : g), 256, 0, (cudaStream_t)stream>>>(spec, spec_bs, T, alpha, beta, (__half*)out, rows);
  DSB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dsb_caption_tokens(const float* patch, const float* cls, const float* pos, float* x, int B, int n, int D, void* stream) {
  DSB_REQUIRE(B > 0 && B <= 65535 && n > 0 && D > 0, "dsb_caption_tokens: bad shape (B=%d n=%d D=%d)", B, n, D);
  DSB_REQUIRE(patch && cls && pos && x, "dsb_caption_tokens: null argument");
  cap_tokens_kernel<<<dim3(n + 1, B), 256, 0, (cudaStream_t)stream>>>(patch, cls, pos, x, n, D);
  DSB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dsb_caption_embed(const int64_t* tok, const int* pos, const float* table, const float* pe, float* x, int R, int V, int D, int max_pos,
                                 int* err_flag, void* stream) {
  DSB_REQUIRE(R > 0 && V > 0 && D > 0 && max_pos > 0, "dsb_caption_embed: bad shape (R=%d V=%d D=%d)", R, V, D);
  DSB_REQUIRE(tok && pos && table && pe && x, "dsb_caption_embed: null argument");
  cap_embed_kernel<<<R, 256, 0, (cudaStream_t)stream>>>(tok, pos, table, pe, x, V, D, max_pos, err_flag);
  DSB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dsb_caption_tree_attention(const float* qkv, long long ld_qkv, float* k_pool, float* v_pool, long long pool_ld, long long n_slots,
                                          const int* path, long long path_len, const long long* path_start, const int* pos, int max_len, void* out,
                                          long long ld_out, long long lo_off, int R, int H, int head_dim, float scale, int* err_flag, void* stream) {
  DSB_REQUIRE(head_dim == HD, "dsb_caption_tree_attention: head_dim=%d unsupported (64)", head_dim);
  DSB_REQUIRE(R > 0 && R <= 65535 && H > 0 && max_len > 0 && max_len <= CAP_MAX_LEN,
              "dsb_caption_tree_attention: bad shape (R=%d H=%d max_len=%d, max_len <= %d)", R, H, max_len, CAP_MAX_LEN);
  DSB_REQUIRE(pool_ld >= (long long)H * HD && pool_ld % 2 == 0 && ld_qkv >= 3LL * H * HD, "dsb_caption_tree_attention: bad leading dimension");
  DSB_REQUIRE(n_slots > 0 && path_len > 0, "dsb_caption_tree_attention: empty pool or path list");
  DSB_REQUIRE(qkv && k_pool && v_pool && path && path_start && pos && out, "dsb_caption_tree_attention: null argument");
  const size_t smem = cap_attend_smem(max_len);
  DSB_CHECK_CUDA(cudaFuncSetAttribute(cap_tree_attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  cap_tree_attention_kernel<<<dim3(H, R), CT, smem, (cudaStream_t)stream>>>(qkv, ld_qkv, k_pool, v_pool, pool_ld, n_slots, path, path_len, path_start,
                                                                            pos, max_len, (__half*)out, ld_out, lo_off, H, scale, err_flag);
  DSB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dsb_caption_cross_attention(const float* q, long long ldq, const float* kv, long long ld_kv, long long v_off, int Lm, const int* row_clip,
                                           int n_clips, void* out, long long ld_out, long long lo_off, int R, int H, int head_dim, float scale, int* err_flag,
                                           void* stream) {
  DSB_REQUIRE(head_dim == HD, "dsb_caption_cross_attention: head_dim=%d unsupported (64)", head_dim);
  DSB_REQUIRE(R > 0 && R <= 65535 && H > 0 && Lm > 0 && Lm <= CAP_MAX_LEN, "dsb_caption_cross_attention: bad shape (R=%d H=%d Lm=%d)", R, H, Lm);
  DSB_REQUIRE(ld_kv % 2 == 0 && v_off % 2 == 0 && ld_kv >= (long long)H * HD, "dsb_caption_cross_attention: bad leading dimension");
  DSB_REQUIRE(n_clips > 0, "dsb_caption_cross_attention: n_clips=%d", n_clips);
  DSB_REQUIRE(q && kv && row_clip && out, "dsb_caption_cross_attention: null argument");
  const size_t smem = cap_attend_smem(Lm);
  DSB_CHECK_CUDA(cudaFuncSetAttribute(cap_cross_attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  cap_cross_attention_kernel<<<dim3(H, R), CT, smem, (cudaStream_t)stream>>>(q, ldq, kv, ld_kv, v_off, Lm, row_clip, n_clips, (__half*)out, ld_out,
                                                                             lo_off, scale, err_flag);
  DSB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dsb_caption_select(const float* logits, long long ld, int R, int V, int k_top, float* vals, int64_t* idx, int64_t* ys, long long ys_ld,
                                  int64_t* tok, int* pos, int* err_flag, void* stream) {
  DSB_REQUIRE(R > 0 && V > 0 && ld >= V, "dsb_caption_select: bad shape (R=%d V=%d)", R, V);
  DSB_REQUIRE(V <= CAP_MAX_V, "dsb_caption_select: V=%d too large (max %d)", V, CAP_MAX_V);
  DSB_REQUIRE(k_top >= 0 && k_top <= CAP_MAX_K && k_top <= V, "dsb_caption_select: k_top=%d out of range (0 ... min(%d, V))", k_top, CAP_MAX_K);
  DSB_REQUIRE(logits && (k_top == 0 ? (ys && tok && pos) : (vals && idx)), "dsb_caption_select: null argument");
  cap_select_kernel<<<R, CT, 0, (cudaStream_t)stream>>>(logits, ld, V, k_top, vals, idx, ys, ys_ld, tok, pos, err_flag);
  DSB_CHECK_CUDA(cudaGetLastError());
  return 0;
}
