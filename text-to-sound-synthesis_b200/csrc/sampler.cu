// Fused p_sample tail: fp64 log_softmax + clamp  ->  top-k / nucleus truncation  ->  closed-form q_posterior  ->
// Gumbel-argmax, one warp per (batch, position) column, token ids in / token ids out.  Codebooks above K = 1055 use the wide form
// below (one CTA per column, dsb_posterior_sample_wide).
//   reference: diffusion_transformer.py:285-289 (predict_start tail), models/dalle_spec.py:146-174 (truncation wrappers),
//              diffusion_transformer.py:28-30,241-267,293-339 (q_posterior), :359-368 (log_sample_categorical).
// Numerics follow the reference's CPU path op by op: fp64 exactly where it uses fp64 (log_softmax; torch's CPU cumsum
// accumulates fp32 in fp64), fp32 expf/logf elsewhere.  Nucleus membership is computed by rank instead of a sort: element
// k is kept iff the fp64 sum of exp(v_i) over all i ordered before k (v_i > v_k, ties by lower index = stable descending
// sort) rounds to an fp32 below r -- the same predicate as sort + cumsum + shift-by-one + gather(argsort).
// HBM-bound: reads K + (K+1) floats and writes one id per column.
#include "block_ctx.cuh"
#include "common.cuh"
#include "diffsound_b200.h"
#include "philox.cuh"

namespace dsb {
constexpr int SW = 8;  // warps (= columns) per CTA

__device__ __forceinline__ float lae(float a, float b) {  // log_add_exp, diffusion_transformer.py:28-30
  const float m = fmaxf(a, b);
  return m + logf(expf(a - m) + expf(b - m));
}
__device__ __forceinline__ float wmaxf(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float wsumf(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double wsumd(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ---- in-kernel replay of torch.rand_like's CUDA stream (diffusion_transformer.py:360 draws uniform = torch.rand_like(logits)): aten_uniform,
// philox.cuh.
__global__ void aten_uniform_fill_kernel(float* out, long long n, unsigned long long seed, unsigned long long offset, unsigned long long nthreads) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    out[i] = aten_uniform(seed, offset, nthreads, (unsigned long long)i);
}

// Loop control block (device memory, 64-bit words) of the fused sampling loop: the kernel draws its own uniforms and, when its last CTA retires,
// advances the RNG offset and writes the NEXT step's timesteps, so a whole diffusion step is a fixed launch sequence with no host-side updates.
//   [0] seed  [1] philox offset  [2] offset increment per step  [3] ATen's thread count (256 * grid)  [4] step index  [5] number of steps  [6] CTA ticket
constexpr int CTRL_SEED = 0, CTRL_OFFSET = 1, CTRL_OFFSET_INC = 2, CTRL_NTHREADS = 3, CTRL_STEP = 4, CTRL_NSTEPS = 5, CTRL_TICKET = 6;

// NJ = ceil((K+1)/32): elements per lane; element index k = lane + 32*j
template <int NJ>
__global__ void __launch_bounds__(SW * 32)
posterior_sample_kernel(const float* __restrict__ logits, const int64_t* x_t, int64_t* t,
                        int64_t* t_post, const float* __restrict__ uniform, const float* __restrict__ sched,
                        int64_t* x_next, float* __restrict__ log_prob_out, int K, int L, int T, int trunc_mode, float trunc_r,
                        int trunc_k, int stage, unsigned long long* ctrl, const int64_t* __restrict__ t_sched, const int64_t* __restrict__ tp_sched, int B) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int C = K + 1;
  float* u_s = reinterpret_cast<float*>(smem_raw);                    // [C][SW]  uniforms, later reused for log_prob_out
  float* v_s = u_s + C * SW;                                          // [SW][C]  truncation keys (log-probs)
  double* e_s = reinterpret_cast<double*>(v_s + ((SW * C + 1) & ~1)); // [SW][C]  exp(v) in fp64
  float* in_s = reinterpret_cast<float*>(e_s + SW * C);               // [C][SW]  input tile when it arrives as (B, K+1, L) log-probs
  const bool in_logprob = (stage & DSB_STAGE_INPUT_LOGPROB) != 0;
  const bool do_post = (stage & DSB_STAGE_SKIP_POSTERIOR) == 0;
  const bool do_sample = (stage & DSB_STAGE_SKIP_SAMPLE) == 0;
  const int b = blockIdx.y;
  const int l0 = blockIdx.x * SW;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int l = l0 + warp;
  const bool active = l < L;
  pdl_wait();
  pdl_trigger();

  unsigned long long rng_seed = 0ull, rng_off = 0ull, rng_n = 1ull;
  if (ctrl) { rng_seed = ctrl[CTRL_SEED]; rng_off = ctrl[CTRL_OFFSET]; rng_n = ctrl[CTRL_NTHREADS]; }
  // stage the (C x SW) tile of uniforms: u[b, k, l0 + j]
  if (do_sample && !ctrl) {
    const float* ub = uniform + (long long)b * C * L;
    for (int idx = threadIdx.x; idx < C * SW; idx += SW * 32) {
      const int k = idx / SW, j = idx - k * SW;
      u_s[idx] = (l0 + j < L) ? ub[(long long)k * L + l0 + j] : 0.5f;
    }
  }
  if (in_logprob) {
    const float* ib = logits + (long long)b * C * L;
    for (int idx = threadIdx.x; idx < C * SW; idx += SW * 32) {
      const int k = idx / SW, j = idx - k * SW;
      in_s[idx] = (l0 + j < L) ? ib[(long long)k * L + l0 + j] : -70.f;
    }
  }
  __syncthreads();

  float lp[NJ];
  int xt = 0;
  if (active) {
    if (in_logprob) {
#pragma unroll
      for (int j = 0; j < NJ; ++j) {
        const int k = lane + 32 * j;
        lp[j] = k < C ? in_s[k * SW + warp] : -70.f;
      }
    } else {
    const float* row = logits + ((long long)b * L + l) * K;
    float x[NJ];
    float mx = -INFINITY;
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      const int k = lane + 32 * j;
      x[j] = k < K ? row[k] : -INFINITY;
      mx = fmaxf(mx, x[j]);
    }
    mx = wmaxf(mx);
    // A.1: log_softmax in fp64, cast to fp32, clamp to [-70, 0]; class K (mask) = -70
    double se = 0.0;
#pragma unroll
    for (int j = 0; j < NJ; ++j)
      if (lane + 32 * j < K) se += exp((double)x[j] - (double)mx);
    se = wsumd(se);
    const double lse = log(se);
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      const int k = lane + 32 * j;
      float vlp = -70.f;
      if (k < K) vlp = fminf(fmaxf((float)(((double)x[j] - (double)mx) - lse), -70.f), 0.f);
      lp[j] = vlp;
    }
    }  // !in_logprob
    // A.2: truncation
    if (trunc_mode != 0) {
      // Keep-set = a prefix of the (value desc, index asc) order: element k is kept iff P(key_k), with key = (orderable value bits,
      // 0xFFFF - index) a strict total order, T(key) = fp64 sum of exp(v_i) over keys_i > key, and
      //   nucleus:  P = (float)T(key) < r  (top element always kept)      top-k:  P = #{keys_i > key} < k.
      // P is monotone in key, so the boundary is found by bisection over the 48-bit key space (48 warp-wide reductions) instead
      // of ranking every element against every other one (O(K^2)); the predicate itself is unchanged.
      unsigned long long key[NJ];
      double ex[NJ];
      unsigned long long kmax = 0ull;
#pragma unroll
      for (int j = 0; j < NJ; ++j) {
        const int k = lane + 32 * j;
        if (k < C) {
          const uint32_t bits = __float_as_uint(lp[j] + 0.0f);
          const uint32_t u = (bits & 0x80000000u) ? ~bits : (bits | 0x80000000u);
          key[j] = ((unsigned long long)u << 16) | (unsigned long long)(0xFFFF - k);
          ex[j] = (double)expf(lp[j]);
        } else {
          key[j] = 0ull;  // below every real key (real keys have index bits <= 0xFFFF and u >= 1 for finite values)
          ex[j] = 0.0;
        }
        kmax = key[j] > kmax ? key[j] : kmax;
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long other = __shfl_xor_sync(0xffffffffu, kmax, o);
        kmax = other > kmax ? other : kmax;
      }
      // invariant: P(hi) true (the top key: nothing ahead of it), P(lo) false or lo below all keys
      unsigned long long lo = 0ull, hi = kmax;
      while (hi - lo > 1ull) {
        const unsigned long long mid = lo + ((hi - lo) >> 1);
        double tsum = 0.0;
        int tcnt = 0;
#pragma unroll
        for (int j = 0; j < NJ; ++j)
          if (key[j] > mid) { tsum += ex[j]; tcnt += 1; }
        tsum = wsumd(tsum);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) tcnt += __shfl_xor_sync(0xffffffffu, tcnt, o);
        const bool pm = (trunc_mode == 1) ? ((float)tsum < trunc_r) : (tcnt < trunc_k);
        if (pm) hi = mid; else lo = mid;
      }
#pragma unroll
      for (int j = 0; j < NJ; ++j) {
        const bool keep = key[j] >= hi;  // includes the top element (key == kmax >= hi)
        if (!keep) lp[j] = -70.f;
      }
    }
    if (do_post || do_sample) {
    // A.3: q_posterior closed form
    float qv[NJ], lq1[NJ];
    float slse = 0.f, pA = 0.f, pB = 0.f, pC = 0.f, pC1 = 0.f;
    if (do_post) {
      xt = (int)x_t[(long long)b * L + l];
      const bool masked = (xt == K);
      long long tp = t_post ? t_post[b] : t[b];
      tp = tp < 0 ? 0 : (tp >= T ? T - 1 : tp);
      const int tm1 = (int)((tp - 1 + (T + 1)) % (T + 1));
      const int S1 = T + 1;
      const float la = sched[0 * S1 + tp], lb = sched[1 * S1 + tp], lc = sched[2 * S1 + tp];
      const float cA = sched[4 * S1 + tp], cB = sched[5 * S1 + tp], cC = sched[6 * S1 + tp];
      pA = sched[4 * S1 + tm1]; pB = sched[5 * S1 + tm1]; pC = sched[6 * S1 + tm1]; pC1 = sched[7 * S1 + tm1];
      const float LOGZ = -69.07755279f;  // log(1e-30) in fp32
      float qmax = -INFINITY;
#pragma unroll
      for (int j = 0; j < NJ; ++j) {
        const int k = lane + 32 * j;
        float lqt, l1;
        if (k < K) {
          if (masked) { lqt = cC; l1 = lc; }
          else {
            const float oh = (k == xt) ? 0.f : LOGZ;
            lqt = lae(oh + cA, cB);
            l1 = lae(oh + la, lb);
          }
        } else {  // k == K (and padding lanes, ignored below)
          lqt = masked ? 0.f : LOGZ;
          l1 = lqt;
        }
        lq1[j] = l1;
        qv[j] = (k < C) ? lp[j] - lqt : -INFINITY;
        qmax = fmaxf(qmax, qv[j]);
      }
      qmax = wmaxf(qmax);
      float ssum = 0.f;
#pragma unroll
      for (int j = 0; j < NJ; ++j)
        if (lane + 32 * j < C) ssum += expf(qv[j] - qmax);
      ssum = wsumf(ssum);
      slse = logf(ssum) + qmax;  // torch.logsumexp
    }
    // A.4: Gumbel-argmax (first index wins ties)
    float best = -INFINITY;
    int besti = 0x7fffffff;
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      const int k = lane + 32 * j;
      if (k < C) {
        float outv = lp[j];
        if (do_post) {
          const float qn = qv[j] - slse;
          const float r = (k < K) ? lae(qn + pA, pB) : lae(qn + pC1, pC);
          outv = fminf(fmaxf(r + lq1[j] + slse, -70.f), 0.f);
          lp[j] = outv;
        }
        const float u = !do_sample ? 0.5f : (ctrl ? aten_uniform(rng_seed, rng_off, rng_n, ((unsigned long long)b * C + k) * L + l) : u_s[k * SW + warp]);
        const float gmb = -logf(-logf(u + 1e-30f) + 1e-30f);
        const float val = gmb + outv;
        if (val > best) { best = val; besti = k; }  // ascending k per lane -> keeps the first maximum
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ob = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, besti, o);
      if (ob > best || (ob == best && oi < besti)) { best = ob; besti = oi; }
    }
    if (lane == 0 && do_sample) x_next[(long long)b * L + l] = besti;
    }  // do_post || do_sample
  }
  if (log_prob_out) {  // optional model_log_prob (B, K+1, L): stage through smem for coalesced rows
    __syncthreads();
    if (active) {
#pragma unroll
      for (int j = 0; j < NJ; ++j) {
        const int k = lane + 32 * j;
        if (k < C) u_s[k * SW + warp] = lp[j];
      }
    }
    __syncthreads();
    float* ob = log_prob_out + (long long)b * C * L;
    for (int idx = threadIdx.x; idx < C * SW; idx += SW * 32) {
      const int k = idx / SW, j = idx - k * SW;
      if (l0 + j < L) ob[(long long)k * L + l0 + j] = u_s[idx];
    }
  }
  if (ctrl) {  // the last CTA to retire (every CTA has read offset / t by then) prepares the next step
    __syncthreads();
    if (threadIdx.x == 0) {
      __threadfence();
      const unsigned long long n_cta = (unsigned long long)gridDim.x * gridDim.y;
      if (atomicAdd(&ctrl[CTRL_TICKET], 1ull) == n_cta - 1ull) {
        ctrl[CTRL_TICKET] = 0ull;
        ctrl[CTRL_OFFSET] = rng_off + ctrl[CTRL_OFFSET_INC];
        const unsigned long long step = ctrl[CTRL_STEP] + 1ull;
        ctrl[CTRL_STEP] = step;
        if (step < ctrl[CTRL_NSTEPS]) {
          const int64_t tn = t_sched[step], tpn = tp_sched[step];
          for (int i = 0; i < B; ++i) { t[i] = tn; if (t_post) t_post[i] = tpn; }
        }
        __threadfence();
      }
    }
  }
}

template <int NJ>
static int launch_sampler(const float* logits, const int64_t* x_t, int64_t* t, int64_t* t_post, const float* uniform,
                          const float* sched, int64_t* x_next, float* lpo, int B, int K, int L, int T, int mode, float r, int kk, int stage, cudaStream_t st,
                          unsigned long long* ctrl = nullptr, const int64_t* t_sched = nullptr, const int64_t* tp_sched = nullptr) {
  const int C = K + 1;
  const size_t smem = (size_t)C * SW * 4 + (((size_t)SW * C + 1) & ~(size_t)1) * 4 + (size_t)SW * C * 8 + (size_t)C * SW * 4;
  auto kern = posterior_sample_kernel<NJ>;
  if (smem > 48 * 1024) DSB_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  dim3 grid((L + SW - 1) / SW, B);
  DSB_CHECK_CUDA(launch_pdl(kern, grid, dim3(SW * 32), smem, st, logits, x_t, t, t_post, uniform, sched, x_next, lpo, K, L, T, mode, r, kk, stage, ctrl, t_sched,
                            tp_sched, B));
  return 0;
}

// ---- wide form: one CTA of WNT threads per (b, l) column, for codebooks whose column does not fit one warp (K + 1 > 32 * 33).
// Element k = tid + WNT * j, CAP = ceil((K+1) / WNT) values per thread.  The contract is the warp kernel's, item by item (A.1 - A.4,
// stage flags, key and bisection predicate, first-index ties, t_post and the clamp of t, log_prob_out, the in-kernel Philox replay
// indexed by the same global element, the loop-control block); only the reduction order differs, and it is fixed (block_ctx.cuh):
// each thread in ascending j, then a warp xor butterfly 16 ... 1, then the WNT / 32 warp partials in ascending warp order.  The
// bisection's fp64 sum and count, and the Gumbel (value, index) argmax, use the same three steps.
// Logits (B, L, K) are one contiguous row per CTA.  The (B, K+1, L) tensors (log-prob input, explicit uniforms, log_prob_out) are
// read and written with stride L: only the staged, reference-named methods use them; the sampling loop reads logits and draws
// its uniforms in-kernel.
constexpr int WNT = 256;
constexpr int WIDE_MAX_CAP = 16;  // K + 1 <= 4096

__device__ __forceinline__ void wide_pick(float& best, int& besti, float ob, int oi) {
  if (ob > best || (ob == best && oi < besti)) { best = ob; besti = oi; }
}

template <int CAP>
__global__ void __launch_bounds__(WNT, CAP <= 9 ? 3 : 2)
posterior_sample_wide_kernel(const float* __restrict__ logits, const int64_t* x_t, int64_t* t, int64_t* t_post, const float* __restrict__ uniform,
                             const float* __restrict__ sched, int64_t* x_next, float* __restrict__ log_prob_out, int K, int L, int T, int trunc_mode,
                             float trunc_r, int trunc_k, int stage, unsigned long long* ctrl, const int64_t* __restrict__ t_sched,
                             const int64_t* __restrict__ tp_sched, int B) {
  constexpr int NW = WNT / 32;
  __shared__ double red[2 * NW];
  __shared__ double red_sum[2][NW];
  __shared__ int red_cnt[2][NW];
  __shared__ float red_best[NW];
  __shared__ int red_idx[NW];
  const BlockCtx<WNT> c{red, (int)threadIdx.x, 0};
  const int C = K + 1;
  const int l = blockIdx.x, b = blockIdx.y, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const bool in_logprob = (stage & DSB_STAGE_INPUT_LOGPROB) != 0;
  const bool do_post = (stage & DSB_STAGE_SKIP_POSTERIOR) == 0;
  const bool do_sample = (stage & DSB_STAGE_SKIP_SAMPLE) == 0;
  pdl_wait();
  pdl_trigger();

  unsigned long long rng_seed = 0ull, rng_off = 0ull, rng_n = 1ull;
  if (ctrl) { rng_seed = ctrl[CTRL_SEED]; rng_off = ctrl[CTRL_OFFSET]; rng_n = ctrl[CTRL_NTHREADS]; }

  float lp[CAP];
  if (in_logprob) {
    const float* col = logits + (long long)b * C * L + l;
#pragma unroll
    for (int j = 0; j < CAP; ++j) {
      const int k = tid + WNT * j;
      lp[j] = k < C ? col[(long long)k * L] : -70.f;
    }
  } else {
    const float* row = logits + ((long long)b * L + l) * K;
    float x[CAP];
    float mx = -INFINITY;
#pragma unroll
    for (int j = 0; j < CAP; ++j) {
      const int k = tid + WNT * j;
      x[j] = k < K ? row[k] : -INFINITY;
      mx = fmaxf(mx, x[j]);
    }
    mx = c.maxf(mx);
    // A.1: log_softmax in fp64, cast to fp32, clamp to [-70, 0]; class K (mask) = -70
    double se = 0.0;
#pragma unroll
    for (int j = 0; j < CAP; ++j)
      if (tid + WNT * j < K) se += exp((double)x[j] - (double)mx);
    se = c.sumd(se);
    const double lse = log(se);
#pragma unroll
    for (int j = 0; j < CAP; ++j) {
      const int k = tid + WNT * j;
      float vlp = -70.f;
      if (k < K) vlp = fminf(fmaxf((float)(((double)x[j] - (double)mx) - lse), -70.f), 0.f);
      lp[j] = vlp;
    }
  }
  // A.2: truncation, the warp kernel's key and bisection predicate (see posterior_sample_kernel)
  if (trunc_mode != 0) {
    unsigned long long key[CAP];
    double ex[CAP];
    unsigned long long kmax = 0ull;
#pragma unroll
    for (int j = 0; j < CAP; ++j) {
      const int k = tid + WNT * j;
      if (k < C) {
        const uint32_t bits = __float_as_uint(lp[j] + 0.0f);
        const uint32_t u = (bits & 0x80000000u) ? ~bits : (bits | 0x80000000u);
        key[j] = ((unsigned long long)u << 16) | (unsigned long long)(0xFFFF - k);
        ex[j] = (double)expf(lp[j]);
      } else {
        key[j] = 0ull;
        ex[j] = 0.0;
      }
      kmax = key[j] > kmax ? key[j] : kmax;
    }
    kmax = c.maxu(kmax);
    unsigned long long lo = 0ull, hi = kmax;
    int par = 0;
    while (hi - lo > 1ull) {  // every thread holds the same lo / hi, so the barriers inside are uniform
      const unsigned long long mid = lo + ((hi - lo) >> 1);
      double tsum = 0.0;
      int tcnt = 0;
#pragma unroll
      for (int j = 0; j < CAP; ++j)
        if (key[j] > mid) { tsum += ex[j]; tcnt += 1; }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        tsum += __shfl_xor_sync(0xffffffffu, tsum, o);
        tcnt += __shfl_xor_sync(0xffffffffu, tcnt, o);
      }
      if (lane == 0) { red_sum[par][warp] = tsum; red_cnt[par][warp] = tcnt; }
      __syncthreads();
      tsum = red_sum[par][0];
      tcnt = red_cnt[par][0];
#pragma unroll
      for (int w = 1; w < NW; ++w) { tsum += red_sum[par][w]; tcnt += red_cnt[par][w]; }
      par ^= 1;
      const bool pm = (trunc_mode == 1) ? ((float)tsum < trunc_r) : (tcnt < trunc_k);
      if (pm) hi = mid; else lo = mid;
    }
#pragma unroll
    for (int j = 0; j < CAP; ++j)
      if (!(key[j] >= hi)) lp[j] = -70.f;
  }
  if (do_post || do_sample) {
    // A.3: q_posterior closed form
    float qv[CAP], lq1[CAP];
    float slse = 0.f, pA = 0.f, pB = 0.f, pC = 0.f, pC1 = 0.f;
    if (do_post) {
      const int xt = (int)x_t[(long long)b * L + l];
      const bool masked = (xt == K);
      long long tp = t_post ? t_post[b] : t[b];
      tp = tp < 0 ? 0 : (tp >= T ? T - 1 : tp);
      const int tm1 = (int)((tp - 1 + (T + 1)) % (T + 1));
      const int S1 = T + 1;
      const float la = sched[0 * S1 + tp], lb = sched[1 * S1 + tp], lc = sched[2 * S1 + tp];
      const float cA = sched[4 * S1 + tp], cB = sched[5 * S1 + tp], cC = sched[6 * S1 + tp];
      pA = sched[4 * S1 + tm1]; pB = sched[5 * S1 + tm1]; pC = sched[6 * S1 + tm1]; pC1 = sched[7 * S1 + tm1];
      const float LOGZ = -69.07755279f;
      float qmax = -INFINITY;
#pragma unroll
      for (int j = 0; j < CAP; ++j) {
        const int k = tid + WNT * j;
        float lqt, l1;
        if (k < K) {
          if (masked) { lqt = cC; l1 = lc; }
          else {
            const float oh = (k == xt) ? 0.f : LOGZ;
            lqt = lae(oh + cA, cB);
            l1 = lae(oh + la, lb);
          }
        } else {
          lqt = masked ? 0.f : LOGZ;
          l1 = lqt;
        }
        lq1[j] = l1;
        qv[j] = (k < C) ? lp[j] - lqt : -INFINITY;
        qmax = fmaxf(qmax, qv[j]);
      }
      qmax = c.maxf(qmax);
      float ssum = 0.f;
#pragma unroll
      for (int j = 0; j < CAP; ++j)
        if (tid + WNT * j < C) ssum += expf(qv[j] - qmax);
      ssum = c.sumf(ssum);
      slse = logf(ssum) + qmax;
#pragma unroll
      for (int j = 0; j < CAP; ++j) {
        const int k = tid + WNT * j;
        if (k < C) {
          const float qn = qv[j] - slse;
          const float r = (k < K) ? lae(qn + pA, pB) : lae(qn + pC1, pC);
          lp[j] = fminf(fmaxf(r + lq1[j] + slse, -70.f), 0.f);
        }
      }
    }
    // A.4: Gumbel-argmax (first index wins ties)
    if (do_sample) {
      float best = -INFINITY;
      int besti = 0x7fffffff;
#pragma unroll
      for (int j = 0; j < CAP; ++j) {
        const int k = tid + WNT * j;
        if (k < C) {
          const long long gi = ((long long)b * C + k) * L + l;
          const float u = ctrl ? aten_uniform(rng_seed, rng_off, rng_n, (unsigned long long)gi) : uniform[gi];
          const float gmb = -logf(-logf(u + 1e-30f) + 1e-30f);
          const float val = gmb + lp[j];
          if (val > best) { best = val; besti = k; }  // ascending k per thread -> keeps the first maximum
        }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) wide_pick(best, besti, __shfl_xor_sync(0xffffffffu, best, o), __shfl_xor_sync(0xffffffffu, besti, o));
      if (lane == 0) { red_best[warp] = best; red_idx[warp] = besti; }
      __syncthreads();  // also orders every thread's read of x_t before the in-place write below
      if (tid == 0) {
        best = red_best[0];
        besti = red_idx[0];
        for (int w = 1; w < NW; ++w) wide_pick(best, besti, red_best[w], red_idx[w]);
        x_next[(long long)b * L + l] = besti;
      }
    }
  }
  if (log_prob_out) {
#pragma unroll
    for (int j = 0; j < CAP; ++j) {
      const int k = tid + WNT * j;
      if (k < C) log_prob_out[((long long)b * C + k) * L + l] = lp[j];
    }
  }
  if (ctrl) {  // the last CTA to retire (every CTA has read offset / t by then) prepares the next step
    __syncthreads();
    if (tid == 0) {
      __threadfence();
      const unsigned long long n_cta = (unsigned long long)gridDim.x * gridDim.y;
      if (atomicAdd(&ctrl[CTRL_TICKET], 1ull) == n_cta - 1ull) {
        ctrl[CTRL_TICKET] = 0ull;
        ctrl[CTRL_OFFSET] = rng_off + ctrl[CTRL_OFFSET_INC];
        const unsigned long long step = ctrl[CTRL_STEP] + 1ull;
        ctrl[CTRL_STEP] = step;
        if (step < ctrl[CTRL_NSTEPS]) {
          const int64_t tn = t_sched[step], tpn = tp_sched[step];
          for (int i = 0; i < B; ++i) { t[i] = tn; if (t_post) t_post[i] = tpn; }
        }
        __threadfence();
      }
    }
  }
}

template <int CAP>
static int launch_sampler_wide(const float* logits, const int64_t* x_t, int64_t* t, int64_t* t_post, const float* uniform, const float* sched,
                               int64_t* x_next, float* lpo, int B, int K, int L, int T, int mode, float r, int kk, int stage, cudaStream_t st,
                               unsigned long long* ctrl, const int64_t* t_sched, const int64_t* tp_sched) {
  DSB_CHECK_CUDA(launch_pdl(posterior_sample_wide_kernel<CAP>, dim3(L, B), dim3(WNT), 0, st, logits, x_t, t, t_post, uniform, sched, x_next, lpo, K, L, T,
                            mode, r, kk, stage, ctrl, t_sched, tp_sched, B));
  return 0;
}

// CAP buckets of the wide kernel: K + 1 <= 512, 1024, 2304 (covers the 2048-code codebook), 4096
static int dispatch_sampler_wide(const float* logits, const int64_t* x_t, int64_t* t, int64_t* t_post, const float* uniform, const float* sched,
                                 int64_t* x_next, float* lpo, int B, int K, int L, int T, int mode, float r, int kk, int stage, cudaStream_t st,
                                 unsigned long long* ctrl, const int64_t* t_sched, const int64_t* tp_sched) {
  const int cap = (K + 1 + WNT - 1) / WNT;
#define DSB_WIDE_CASE(N) \
  if (cap <= N) return launch_sampler_wide<N>(logits, x_t, t, t_post, uniform, sched, x_next, lpo, B, K, L, T, mode, r, kk, stage, st, ctrl, t_sched, tp_sched)
  DSB_WIDE_CASE(2);
  DSB_WIDE_CASE(4);
  DSB_WIDE_CASE(9);
  DSB_WIDE_CASE(WIDE_MAX_CAP);
#undef DSB_WIDE_CASE
  return 2;
}
}  // namespace dsb
using namespace dsb;

extern "C" int dsb_posterior_sample(const float* logits, const int64_t* x_t, const int64_t* t, const int64_t* t_post, const float* uniform,
                                    const float* sched, int64_t* x_next, float* log_prob_out, int B, int K, int L, int T, int trunc_mode,
                                    float trunc_r, int trunc_k, int stage_flags, void* stream) {
  DSB_REQUIRE(B > 0 && K > 0 && L > 0 && T > 0, "dsb_posterior_sample: bad shape");
  DSB_REQUIRE(trunc_mode >= 0 && trunc_mode <= 2, "dsb_posterior_sample: trunc_mode must be 0, 1 or 2");
  DSB_REQUIRE(K + 1 <= 32 * 33, "dsb_posterior_sample: K=%d too large (max 1055; dsb_posterior_sample_wide takes larger K)", K);
  DSB_REQUIRE((stage_flags & DSB_STAGE_SKIP_SAMPLE) || (uniform && x_next), "dsb_posterior_sample: sampling needs uniform and x_next");
  DSB_REQUIRE((stage_flags & DSB_STAGE_SKIP_POSTERIOR) || (x_t && t && sched), "dsb_posterior_sample: the posterior needs x_t, t and sched");
  cudaStream_t st = (cudaStream_t)stream;
  const int nj = (K + 1 + 31) / 32;
#define DSB_SAMPLER_CASE(N) \
  if (nj <= N) return launch_sampler<N>(logits, x_t, const_cast<int64_t*>(t), const_cast<int64_t*>(t_post), uniform, sched, x_next, log_prob_out, B, K, L, T, trunc_mode, trunc_r, trunc_k, stage_flags, st)
  DSB_SAMPLER_CASE(2);
  DSB_SAMPLER_CASE(5);
  DSB_SAMPLER_CASE(9);
  DSB_SAMPLER_CASE(17);
  DSB_SAMPLER_CASE(33);
#undef DSB_SAMPLER_CASE
  return 2;
}

extern "C" int dsb_posterior_sample_loop(const float* logits, int64_t* x, int64_t* t, int64_t* t_post, const float* sched, unsigned long long* ctrl,
                                         const int64_t* t_sched, const int64_t* t_post_sched, int B, int K, int L, int T, int trunc_mode, float trunc_r,
                                         int trunc_k, void* stream) {
  DSB_REQUIRE(B > 0 && K > 0 && L > 0 && T > 0 && K + 1 <= 32 * 33, "dsb_posterior_sample_loop: bad shape");
  DSB_REQUIRE(logits && x && t && t_post && sched && ctrl && t_sched && t_post_sched, "dsb_posterior_sample_loop: null argument");
  DSB_REQUIRE(trunc_mode >= 0 && trunc_mode <= 2, "dsb_posterior_sample_loop: trunc_mode must be 0, 1 or 2");
  cudaStream_t st = (cudaStream_t)stream;
  const int nj = (K + 1 + 31) / 32;
#define DSB_SAMPLER_CASE(N) \
  if (nj <= N) return launch_sampler<N>(logits, x, t, t_post, nullptr, sched, x, nullptr, B, K, L, T, trunc_mode, trunc_r, trunc_k, 0, st, ctrl, t_sched, t_post_sched)
  DSB_SAMPLER_CASE(2);
  DSB_SAMPLER_CASE(5);
  DSB_SAMPLER_CASE(9);
  DSB_SAMPLER_CASE(17);
  DSB_SAMPLER_CASE(33);
#undef DSB_SAMPLER_CASE
  return 2;
}

extern "C" int dsb_posterior_sample_wide(const float* logits, const int64_t* x_t, const int64_t* t, const int64_t* t_post, const float* uniform,
                                         const float* sched, int64_t* x_next, float* log_prob_out, int B, int K, int L, int T, int trunc_mode,
                                         float trunc_r, int trunc_k, int stage_flags, void* stream) {
  DSB_REQUIRE(B > 0 && K > 0 && L > 0 && T > 0 && B <= 65535, "dsb_posterior_sample_wide: bad shape");
  DSB_REQUIRE(trunc_mode >= 0 && trunc_mode <= 2, "dsb_posterior_sample_wide: trunc_mode must be 0, 1 or 2");
  DSB_REQUIRE(K + 1 <= WNT * WIDE_MAX_CAP, "dsb_posterior_sample_wide: K=%d too large (max %d)", K, WNT * WIDE_MAX_CAP - 1);
  DSB_REQUIRE((stage_flags & DSB_STAGE_SKIP_SAMPLE) || (uniform && x_next), "dsb_posterior_sample_wide: sampling needs uniform and x_next");
  DSB_REQUIRE((stage_flags & DSB_STAGE_SKIP_POSTERIOR) || (x_t && t && sched), "dsb_posterior_sample_wide: the posterior needs x_t, t and sched");
  return dispatch_sampler_wide(logits, x_t, const_cast<int64_t*>(t), const_cast<int64_t*>(t_post), uniform, sched, x_next, log_prob_out, B, K, L, T,
                               trunc_mode, trunc_r, trunc_k, stage_flags, (cudaStream_t)stream, nullptr, nullptr, nullptr);
}

extern "C" int dsb_posterior_sample_wide_loop(const float* logits, int64_t* x, int64_t* t, int64_t* t_post, const float* sched, unsigned long long* ctrl,
                                              const int64_t* t_sched, const int64_t* t_post_sched, int B, int K, int L, int T, int trunc_mode,
                                              float trunc_r, int trunc_k, void* stream) {
  DSB_REQUIRE(B > 0 && K > 0 && L > 0 && T > 0 && B <= 65535, "dsb_posterior_sample_wide_loop: bad shape");
  DSB_REQUIRE(K + 1 <= WNT * WIDE_MAX_CAP, "dsb_posterior_sample_wide_loop: K=%d too large (max %d)", K, WNT * WIDE_MAX_CAP - 1);
  DSB_REQUIRE(logits && x && t && t_post && sched && ctrl && t_sched && t_post_sched, "dsb_posterior_sample_wide_loop: null argument");
  DSB_REQUIRE(trunc_mode >= 0 && trunc_mode <= 2, "dsb_posterior_sample_wide_loop: trunc_mode must be 0, 1 or 2");
  return dispatch_sampler_wide(logits, x, t, t_post, nullptr, sched, x, nullptr, B, K, L, T, trunc_mode, trunc_r, trunc_k, 0, (cudaStream_t)stream, ctrl,
                               t_sched, t_post_sched);
}

extern "C" int dsb_aten_uniform(float* out, long long n, unsigned long long seed, unsigned long long offset, unsigned long long nthreads, void* stream) {
  DSB_REQUIRE(n > 0 && nthreads > 0 && offset % 4 == 0, "dsb_aten_uniform: need n > 0, nthreads > 0 and a philox offset that is a multiple of 4");
  long long g = (n + 255) / 256;
  const long long cap = (long long)sm_count() * 8;
  aten_uniform_fill_kernel<<<(unsigned)(g > cap ? cap : g), 256, 0, (cudaStream_t)stream>>>(out, n, seed, offset, nthreads);
  DSB_CHECK_CUDA(cudaGetLastError());
  return 0;
}
