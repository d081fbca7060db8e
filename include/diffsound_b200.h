/* diffsound_b200.h -- C-ABI of libdiffsound_b200.so (hand-written sm_90a kernels for the Diffsound hot path).
 *
 * The reference (yangdongchao/Text-to-sound-Synthesis) is pure PyTorch and has NO native / FFI interface to mirror
 * (SURVEY.md section 2.1, 8b): the seam it offers is Python classes built by instantiate_from_config
 * (Diffsound/sound_synthesis/utils/misc.py:125-132).  This header is therefore the boundary a maintainer would bind
 * with ctypes from those classes; every entry point names the reference code it replaces.  INTEGRATION.md shows the
 * binding stub.
 *
 * Conventions
 *   - plain pointers and sizes only; every pointer is a DEVICE pointer unless it says "host".
 *   - the caller (PyTorch) owns all memory; the library never allocates, frees or retains caller pointers.
 *   - `stream` is a cudaStream_t passed as void*; every call is asynchronous on that stream, performs no
 *     synchronisation and no allocation, and is CUDA-graph capturable.
 *   - return 0 on success, non-zero on error; dsb_last_error() returns a thread-local message.  No C++ exceptions
 *     cross this boundary.
 */
#ifndef DIFFSOUND_B200_H
#define DIFFSOUND_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DSB_VERSION 100

/* operand types of the tensor-core GEMM */
#define DSB_DTYPE_TF32 0 /* fp32 containers, TF32 wgmma (inputs should be pre-rounded with dsb_round_tf32) */
#define DSB_DTYPE_BF16 1 /* bf16 containers, BF16 wgmma */
#define DSB_DTYPE_F16 2  /* fp16 containers, FP16 wgmma: same 11-bit significand as TF32 at twice the MMA rate */

/* epilogue flags */
#define DSB_GEMM_GELU2 1      /* x * sigmoid(1.702 x)           (reference transformer_utils.py:111-115) */
#define DSB_GEMM_ROUND_TF32 2 /* round the fp32 output to tf32 (it feeds another tf32 GEMM) */
#define DSB_GEMM_OUT_BF16 4   /* store bf16 instead of fp32 */
#define DSB_GEMM_LRELU 8      /* LeakyReLU(0.2)                 (reference vocoder/modules.py:76,79) */
#define DSB_GEMM_TANH 16      /* tanh                           (reference vocoder/modules.py:123) */
#define DSB_GEMM_OUT_F16 256   /* store fp16 instead of fp32 */
#define DSB_GEMM_RES_BEFORE_ACT 128 /* add the residual before the activation (default: after) */
#define DSB_GEMM_DUAL_LRELU 4096 /* with OUT_F16_SPLIT: also store the pair of LeakyReLU(0.2)(x) at +dual_off (reference vocoder/modules.py:76: the
                                   next ResnetBlock convolves the activated signal while its 1x1 shortcut reads the raw one) */
#define DSB_GEMM_NO_STORE 16384 /* run the GEMM and its epilogue but store nothing (amax_out calibration pass) */
#define DSB_GEMM_RELU 32768   /* max(x, 0), NaN passes through     (torchvision inception.py BasicConv2d, Melception's every conv) */
#define DSB_GEMM_OUT_F16_SPLIT 2048 /* store the fp16 (hi | lo) pair of the fp32 result: hi = f16(x) at out[r*ldo + c], lo = f16(x - hi) at
                                       out[r*ldo + split_off + c] -- the A operand of a split-fp16 ("f16x3") GEMM, see dsb_split_f16 */
/* GroupNorm-apply flags (share the ROUND_TF32 bit) */
#define DSB_GN_SWISH 32       /* x * sigmoid(x) after the affine (reference model.py:29-31) */
#define DSB_GN_COMPACT 64     /* write (B, Lp, C) tokens instead of the zero-padded image */
#define DSB_SPLIT_OUT_F16 8192 /* elementwise producers: write the fp16 (hi | lo) pair, 2*C halves per row (out is then a __half buffer): the A
                                  operand of a split-fp16 conv GEMM (codebook gather, GroupNorm apply, upsample) */
#define DSB_SPLIT_OUT 512     /* elementwise producers: write the split-TF32 operand (hi | lo), 2*Cp floats per row (see dsb_split_tf32) */

const char* dsb_last_error(void);
int dsb_version(void);
/* host out-params; returns non-zero when no CUDA device is usable */
int dsb_device_info(int* sm_count, int* cc_major, int* cc_minor);

/* ---------------------------------------------------------------------------------------------------------------
 * Tensor-core GEMM (TMA -> smem -> wgmma -> register accumulators -> fused epilogue).
 *   out[b][m, n] = epi( alpha * sum_{tap, k} A[b][m + tap_shift[tap], k] * W[b?][n, tap*K + k] + bias[n] ) (+ residual[b][m, n])
 * Replaces torch.nn.Linear / addmm on the hot path (reference transformer_utils.py:45-47,57,95-97,108,248-253,347) and,
 * with taps on zero-padded channels-last buffers, Conv2d 3x3/1x1 (specvqgan/modules/diffusionmodules/model.py:92-151,174-226)
 * and Conv1d/ConvTranspose1d (vocoder/modules.py:72-126).
 * A: (a_rows, K) row-major, leading dimension lda (elements); W: (N, num_taps*K) row-major, ldw.  Rows read outside
 * [0, a_rows) are zeros (TMA out-of-bounds fill).  16-byte alignment of pointers and leading dimensions is required.
 * ------------------------------------------------------------------------------------------------------------- */
typedef struct dsb_gemm_desc {
  const void* A;
  const void* W;
  const float* bias;     /* [N] or NULL */
  const float* residual; /* fp32 (M, N) with ld_res, or NULL; may alias out */
  void* out;             /* fp32 or bf16 (M, N) with ldo */
  int M, N, K;           /* K = reduction length per tap */
  int batch;             /* >= 1 */
  long long a_rows;      /* rows of A that exist (0 -> M) */
  long long lda, ldw, ldo, ld_res;
  long long a_batch_stride, w_batch_stride /* 0 = shared W */, out_batch_stride, res_batch_stride;
  int dtype;             /* DSB_DTYPE_* */
  int flags;             /* DSB_GEMM_* */
  int num_taps;          /* 1..32 */
  int tap_shift[32];     /* A row shift per tap */
  int tap_acol[32];      /* A column offset per tap (elements); with a_cols this lets one A buffer hold several K-blocks side by
                            side, e.g. the (hi | lo) halves of a split-TF32 operand */
  long long a_cols;      /* columns of A that exist (0 -> K) */
  int geo_P, geo_Wp, geo_y0, geo_y1, geo_x0, geo_x1; /* optional zero-border row mask, geo_P = 0 disables */
  float alpha;           /* 0 -> 1 */
  int block_n;           /* 0 = auto, 128, 256 */
  int max_ctas;          /* 0 = one per SM */
  int cta_pair;          /* 0 = auto, 1 = 256-wide tiles (K-major operands), -1 = never fuse split-fp16 tap triples (plain tap loop) */
  int a_mn_major;        /* 1: A lies in memory as (K rows, M columns), lda = row stride: out[m, n] = sum_k A[k, m] W[n, k]; 2-byte dtypes, 1 tap */
  int b_mn_major;        /* 1: W lies in memory as (K rows, N columns), ldw = row stride (e.g. dW = dY^T X with both operands token-major,
                            dX = dY W with torch's (out, in) weight as stored) */
  int use_tap_wcol;      /* 1: tap i reads W columns [tap_wcol[i], tap_wcol[i] + K) instead of [i*K, (i+1)*K) */
  int tap_wcol[32];
  long long w_cols;      /* columns of W that exist (0 -> num_taps*K) */
  long long split_off;   /* DSB_GEMM_OUT_F16_SPLIT: element offset of the lo half inside an output row (0 -> N) */
  long long dual_off;    /* DSB_GEMM_DUAL_LRELU: element offset of the LeakyReLU(0.2) copy of the output pair */
  int out_col_group;     /* > 0: logical output column n is stored at (n / group) * out_col_group_stride + n % group -- lets the polyphase
                            ConvTranspose1d GEMM (columns = phase * Cout + c) write straight into rows of [raw pair | activated pair] */
  int out_col_group_stride;
  const void* A2;        /* optional second A operand (same dtype, K-major): taps with tap_a2[i] != 0 read it instead of A -- one GEMM over two
                            activation buffers, e.g. MelGAN's ResnetBlock tail  shortcut(x) + conv1x1(y)  (vocoder/modules.py:84-85) */
  long long a2_rows, a2_cols, lda2, a2_batch_stride;
  int tap_a2[32];
  float* amax_out;       /* optional device float (caller zero-initialises): atomic max of |value| over everything this launch stores (or would store,
                            with DSB_GEMM_NO_STORE) -- used once, at pack time, to calibrate the power-of-two activation scales of the fp16 MelGAN path */
  int resident_w;        /* 1: narrow-channel conv form (MelGAN's 64- and 32-channel stages, vocoder/modules.py:104-126): every tap is ONE 64-deep
                            k-block (K == 64), N <= 128.  2-byte dtypes, K-major operands, W not batched; runs on the same kernel as every other GEMM */
  int schedule;          /* 0 = auto, 1 = data-parallel only.  Auto splits tiles between neighbouring CTAs (ordered stream-K) when the tiles leave a
                            partial last wave; the output bits are the same either way.  Stream-K uses a per-device workspace, so at most one
                            dsb_gemm_ex launch may be in flight per device at a time. */
} dsb_gemm_desc;
int dsb_gemm_ex(const dsb_gemm_desc* desc, void* stream);

/* Exact fp32 (FFMA) GEMM with the same epilogue: out = epi(A W^T + bias) (+ residual).  Used for set-up time tables and
 * as the "fp32-exact" mode that proves free-running token parity (SURVEY.md section 7.2). */
int dsb_gemm_f32(const float* A, const float* W, const float* bias, const float* residual, float* out, int M, int N, int K,
                 long long lda, long long ldw, long long ldo, long long ld_res, int flags, void* stream);

/* elementwise helpers */
int dsb_round_tf32(const float* in, float* out, long long n, void* stream);
int dsb_f32_to_bf16(const float* in, void* out_bf16, long long n, void* stream);
int dsb_f32_to_f16(const float* in, void* out_f16, long long n, void* stream);
/* Split-fp16 operand ("f16x3", the parity-grade tensor-core mode of the denoiser): hi = f16(scale * in), lo = f16(scale * in - hi);
 * out[r, c] = hi, out[r, lo_off + c] = lo (fp16, ld_out elements per row).  A W^T ~ Ahi Whi^T + Alo Whi^T + Ahi Wlo^T with fp32
 * accumulation carries 22 significand bits per operand: three kind::f16 passes replace the reference's fp32 nn.Linear
 * (transformer_utils.py:45-57,95-108,248-253,345-348) at fp32-class accuracy.  scale is a power of two that lifts small weights
 * out of fp16's subnormal range (undone exactly by the GEMM's alpha). */
int dsb_split_f16(const float* in, long long ld_in, void* out_f16, long long ld_out, long long lo_off, long long rows, int C, float scale,
                  void* stream);
/* Split-TF32 operand: out[r, c] = hi = tf32(in[r, c]), out[r, Cp + c] = lo = tf32(in[r, c] - hi), zeros in the padding columns
 * [C, Cp); out has 2*Cp columns (ld_out elements per row).  A*W ~ hi*Whi + lo*Whi + hi*Wlo recovers fp32-class accuracy on
 * the TF32 tensor pipe (three K passes), used for the SpecVQGAN decoder / MelGAN convolutions.  w_format = 1 writes the
 * weight-side layout [hi | hi | lo] (3*Cp columns) for an activation that is the W operand of a GEMM (attention K, V^T). */
int dsb_split_tf32(const float* in, long long ld_in, float* out, long long ld_out, long long rows, int C, int Cp, int w_format, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Denoiser pieces (reference sound_synthesis/modeling/transformers/transformer_utils.py,
 *                  sound_synthesis/modeling/embeddings/dalle_mask_image_embedding.py)
 * ------------------------------------------------------------------------------------------------------------- */
/* DalleMaskImageEmbedding.forward (dalle_mask_image_embedding.py:36-58): out[b,l,:] = emb[max(ids,0)] + height[l / W] + width[l % W].
 * Returns an error through *err_flag (device int, may be NULL) if an id >= num_embed. */
int dsb_embed_tokens(const int64_t* ids, const float* emb, const float* height_emb, const float* width_emb, float* out, int B, int L,
                     int D, int H, int W, int num_embed, int* err_flag, void* stream);

/* nn.LayerNorm(D) with affine (transformer_utils.py:197 ln2, :345 to_logits.0): out = LN(x) * gamma + beta. flags: DSB_GEMM_ROUND_TF32 | DSB_GEMM_OUT_BF16 |
 * DSB_GEMM_OUT_F16 | DSB_GEMM_OUT_F16_SPLIT (then out has 2*D fp16 columns per row: hi | lo) */
int dsb_layernorm(const float* x, void* out, const float* gamma, const float* beta, int rows, int D, float eps, int flags, void* stream);

/* AdaLayerNorm.forward (transformer_utils.py:145-149) with the timestep MLP hoisted into a table:
 * table[t] = Linear(SiLU(emb[t])) = (scale | shift), shape (T, 2D); out[b,l,:] = LN(x[b,l,:]) * (1 + scale[t[b]]) + shift[t[b]]. */
int dsb_ada_layernorm(const float* x, void* out, const float* table, const int64_t* t, int B, int L, int D, int T, float eps, int flags,
                      void* stream);

/* x[r, :] /= ||x[r, :]||_2 in place: the per-token normalisation of CLIPTextEmbedding.forward (embeddings/clip_text_embedding.py:78-79) */
int dsb_l2_normalize_rows(float* x, long long rows, int D, void* stream);

/* SiLU on a (rows, D) table (set-up of the AdaLN table) */
int dsb_silu(const float* in, float* out, long long n, void* stream);

/* softmax(Q K^T * scale) V per (batch, head), head_dim 64, no mask, no dropout (FullAttention / CrossAttention,
 * transformer_utils.py:48-54, :99-105).  q/k/v/o are fp32 with row strides ld* (elements); head h occupies columns
 * [64h, 64h+64).  Rows of batch b start at b*Lq (q, o) and b*Lk (k, v).  flags: DSB_GEMM_ROUND_TF32 on the output. */
int dsb_attention(const float* q, long long ldq, const float* k, long long ldk, const float* v, long long ldv, float* o, long long ldo,
                  int B, int H, int Lq, int Lk, float scale, int flags, void* stream);

/* dsb_attention for head_dim 32 (Diffsound caps_small_transformer.yaml: n_embd 512, 16 heads; transformer_utils.py:48-54, :99-105): the same
 * arguments and layout, head h occupies columns [32h, 32h+32). */
int dsb_attention_hd32(const float* q, long long ldq, const float* k, long long ldk, const float* v, long long ldv, float* o, long long ldo,
                       int B, int H, int Lq, int Lk, float scale, int flags, void* stream);

/* Same attention core with fp16 q/k/v (row strides in halves, multiples of 8); o is fp16 (DSB_GEMM_OUT_F16) or fp32.
 * flags | DSB_ATTN_CAUSAL: key j is visible to query i only if j <= i (the CLIP text transformer's mask, clip/model.py build_attention_mask). */
#define DSB_ATTN_CAUSAL 1024
int dsb_attention_f16(const void* q, long long ldq, const void* k, long long ldk, const void* v, long long ldv, void* o, long long ldo,
                      int B, int H, int Lq, int Lk, float scale, int flags, void* stream);

/* Tensor-core version of the same core: K and V of a (batch, head) are staged once by TMA, every warp runs 16 query rows with mma.sync
 * (S = Q K^T, fp32 online softmax, O = P V), one CTA per (batch, head) (two above 256 query rows), Lk <= 272.  q/k/v/o fp16. */
int dsb_attention_tc(const void* q, long long ldq, const void* k, long long ldk, const void* v, long long ldv, void* o, long long ldo,
                     int B, int H, int Lq, int Lk, float scale, void* stream);
/* the same kernel under the name of the former pipelined variant */
int dsb_attention_tc2(const void* q, long long ldq, const void* k, long long ldk, const void* v, long long ldv, void* o, long long ldo,
                      int B, int H, int Lq, int Lk, float scale, void* stream);
/* split-fp16 ("f16x3") version of the same core for the parity-grade mode: q / k / v / o are fp16 (hi | lo) pairs -- the lo half of a row
 * lies *_lo_off elements after its hi half -- S = Qhi Khi^T + Qlo Khi^T + Qhi Klo^T and O = Phi Vhi + Plo Vhi + Phi Vlo with wgmma and fp32
 * accumulation; P = exp2(...) is split into (hi | lo) in registers.  q / k / v / o 16-byte aligned (TMA), any Lk. */
int dsb_attention_tc_split(const void* q, long long ldq, long long q_lo_off, const void* k, long long ldk, long long k_lo_off, const void* v,
                           long long ldv, long long v_lo_off, void* o, long long ldo, long long o_lo_off, int B, int H, int Lq, int Lk,
                           float scale, void* stream);
/* dsb_attention_tc_split for head_dim 32 (caps_small_transformer.yaml; transformer_utils.py:48-54, :99-105): the same arguments and pair
 * layout, head h occupies columns [32h, 32h+32) of each half; 64-byte swizzled tiles, S = 6 and P V = 12 wgmma per 64-key chunk. */
int dsb_attention_tc_split_hd32(const void* q, long long ldq, long long q_lo_off, const void* k, long long ldk, long long k_lo_off, const void* v,
                                long long ldv, long long v_lo_off, void* o, long long ldo, long long o_lo_off, int B, int H, int Lq, int Lk,
                                float scale, void* stream);
/* Causal dsb_attention_tc_split (Codebook/specvqgan/modules/transformer/mingpt.py:76-94 CausalSelfAttention, n_unmasked = 0:
 *   att = att.masked_fill(self.mask[:,:,:T,:T] == 0, float('-inf'))  -- key j of query row i is dropped when j > i, condition rows included)
 * for head_dim 64 or 32 (the arguments of dsb_attention_tc_split / _hd32 plus head_dim).  Lq must equal Lk.  A 64-row query tile t multiplies the
 * 64-key chunks 0 ... t only; chunks past the diagonal are neither loaded nor multiplied. */
int dsb_attention_tc_split_causal(const void* q, long long ldq, long long q_lo_off, const void* k, long long ldk, long long k_lo_off, const void* v,
                                  long long ldv, long long v_lo_off, void* o, long long ldo, long long o_lo_off, int B, int H, int Lq, int Lk,
                                  float scale, int head_dim, void* stream);


/* ---------------------------------------------------------------------------------------------------------------
 * Posterior + truncation + Gumbel-argmax sampler, one kernel (reference diffusion_transformer.py:285-289 predict_start tail,
 * models/dalle_spec.py:146-174 top-k / nucleus truncation, diffusion_transformer.py:293-339 q_posterior,
 * :359-368 log_sample_categorical).  ids are carried instead of log-one-hot tensors.
 *   logits  (B, L, K) fp32  -- denoiser output BEFORE the reference's 'b l c -> b c l' view
 *   x_t     (B, L) int64, values in [0, K]; K is [MASK]
 *   t       (B,) int64 timestep fed to the denoiser;  t_post (B,) int64 timestep used by q_posterior (NULL -> t)
 *   uniform (B, K+1, L) fp32 in [0,1) -- the tensor torch.rand_like(logits) would have produced
 *   sched   (8, T+1) fp32: rows log_at, log_bt, log_ct, log_1_min_ct (T entries used), log_cumprod_at, log_cumprod_bt,
 *           log_cumprod_ct, log_1_min_cumprod_ct (T+1 entries)      (diffusion_transformer.py:224-231)
 *   trunc_mode 0 none, 1 nucleus 'top{r}r' (trunc_r), 2 top-k 'top{k}p' (trunc_k)
 *   x_next  (B, L) int64;  log_prob_out optional (B, K+1, L) fp32 (NULL to skip): the last stage's log-probabilities
 *   stage_flags select a sub-range of the pipeline so the reference's separately callable (and monkey-patchable,
 *   dalle_spec.py:207-210) methods map onto the same kernel:
 *     predict_start          = 0 | SKIP_POSTERIOR | SKIP_SAMPLE           (log_prob_out = log_pred)
 *     q_posterior            = INPUT_LOGPROB | SKIP_SAMPLE, trunc_mode 0  (log_prob_out = model_log_prob)
 *     log_sample_categorical = INPUT_LOGPROB | SKIP_POSTERIOR, trunc_mode 0
 *     p_sample (fused)       = 0
 *   With INPUT_LOGPROB, `logits` is a (B, K+1, L) log-probability tensor instead of raw (B, L, K) logits.
 * ------------------------------------------------------------------------------------------------------------- */
#define DSB_STAGE_INPUT_LOGPROB 1
#define DSB_STAGE_SKIP_POSTERIOR 2
#define DSB_STAGE_SKIP_SAMPLE 4
int dsb_posterior_sample(const float* logits, const int64_t* x_t, const int64_t* t, const int64_t* t_post, const float* uniform,
                         const float* sched, int64_t* x_next, float* log_prob_out, int B, int K, int L, int T, int trunc_mode,
                         float trunc_r, int trunc_k, int stage_flags, void* stream);

/* Loop form of the same kernel for DiffusionTransformer.sample's 100-step loop (diffusion_transformer.py:638-641): no uniform tensor, no host
 * update between steps.  The kernel draws the uniforms itself, replaying the CUDA stream of the reference's `torch.rand_like(logits)` (:360) bit for
 * bit (Philox4x32-10, ATen's element -> (thread, call, component) mapping for a contiguous (B, K+1, L) float tensor), samples x IN PLACE (a column is
 * read and written by the same warp), and its last CTA advances the philox offset and writes the next step's timesteps into t / t_post:
 *   ctrl (device, 7 x uint64): [0] seed  [1] philox offset (multiple of 4)  [2] offset increment per step = ATen's counter_offset
 *                              [3] ATen's thread count 256 * grid  [4] step index  [5] number of steps  [6] CTA ticket (0)
 *   t_sched / t_post_sched (device, n_steps int64): denoiser / posterior timestep of every step; t, t_post (B,) hold step 0's values at entry. */
int dsb_posterior_sample_loop(const float* logits, int64_t* x, int64_t* t, int64_t* t_post, const float* sched, unsigned long long* ctrl,
                              const int64_t* t_sched, const int64_t* t_post_sched, int B, int K, int L, int T, int trunc_mode, float trunc_r,
                              int trunc_k, void* stream);
/* Wide forms of the two entry points above, for codebooks up to K = 4095 (the 2048-code AudioSet codebook has K + 1 = 2049 classes), with
 * identical argument lists and the same contract: diffusion_transformer.py:285-289 (predict_start tail), dalle_spec.py:146-174 (top-k /
 * nucleus truncation), diffusion_transformer.py:293-339 (q_posterior), :359-368 (log_sample_categorical); same stage flags, layouts,
 * truncation key and predicate, first-index ties, t_post and clamp of t, log_prob_out, in-kernel replay of torch.rand_like and loop-control
 * block.  One CTA of 256 threads per (b, l) column instead of one warp; the fp64 / fp32 reductions run in a fixed order that depends on
 * nothing but the column (each thread in ascending k, a warp xor butterfly 16 ... 1, then the 8 warp partials in ascending warp order), so
 * log-probs can differ from the warp kernel's in the last bit of a near-midpoint value and ids only at near ties.  Every K in [1, 4095] is
 * accepted; K > 4095 is refused ("too large") before anything is launched.  B <= 65535. */
int dsb_posterior_sample_wide(const float* logits, const int64_t* x_t, const int64_t* t, const int64_t* t_post, const float* uniform,
                              const float* sched, int64_t* x_next, float* log_prob_out, int B, int K, int L, int T, int trunc_mode,
                              float trunc_r, int trunc_k, int stage_flags, void* stream);
int dsb_posterior_sample_wide_loop(const float* logits, int64_t* x, int64_t* t, int64_t* t_post, const float* sched, unsigned long long* ctrl,
                                   const int64_t* t_sched, const int64_t* t_post_sched, int B, int K, int L, int T, int trunc_mode, float trunc_r,
                                   int trunc_k, void* stream);
/* out[i] = the i-th element torch.rand(n, device='cuda') would hold for generator state (seed, philox offset) with ATen's launch geometry
 * nthreads = 256 * min(SMs * (maxThreadsPerSM / 256), ceil(n / 256)); used by the tests to pin the replay against torch.rand itself. */
int dsb_aten_uniform(float* out, long long n, unsigned long long seed, unsigned long long offset, unsigned long long nthreads, void* stream);
/* out[i] = the i-th element torch.empty(n, device='cuda').exponential_() would hold for generator state (seed, philox offset): the same Philox
 * stream and geometry as dsb_aten_uniform, curand's (0, 1] value u, then -__logf(u) with ATen's clamp near 1 (TransformationHelper.h exponential(),
 * DistributionTemplates.h exponential_kernel).  The draw torch.multinomial(probs, 1) makes on CUDA. */
int dsb_aten_exponential(float* out, long long n, unsigned long long seed, unsigned long long offset, unsigned long long nthreads, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Autoregressive SpecVQGAN transformer, KV-cached decode (reference Codebook/specvqgan/modules/transformer/mingpt.py GPTFeats / GPT,
 * Codebook/specvqgan/models/cond_transformer.py Net2NetTransformer.sample).  One position of B rows per launch sequence; the current position p
 * and the RNG state live in a device loop-control block of 8 uint64 words, advanced by dsb_ar_sample's last CTA, so one captured step replays
 * for every position:
 *   [0] seed  [1] philox offset  [2] offset increment per sampled position (ATen's counter_offset(B * V))  [3] ATen's thread count (256 * grid)
 *   [4] position p  [5] number of positions  [6] first position that samples  [7] CTA ticket (0)
 * Every kernel is a no-op at p >= [5].  The GEMMs between them are dsb_gemm_ex split-fp16 calls and the LayerNorms dsb_layernorm, unchanged.
 * ------------------------------------------------------------------------------------------------------------- */
/* mingpt.py:167-176 + :276-293 (embedder output prepended, tok_emb lookup, + pos_emb[:, :t]) at one position:
 * x[b, :] = (p < Tc ? cond[b, p, :] : tok_emb[ids[b * ids_ld + p - Tc], :]) + pos_emb[p, :]; cond (B, Tc, D) is the Conv1d(k=1) embedding.
 * An id outside [0, V) sets *err_flag (nn.Embedding's index error) and reads row 0.  With Tc = 0 (GPT without a condition) cond may be NULL. */
int dsb_ar_embed(const float* cond, const float* tok_emb, const float* pos_emb, const int64_t* ids, long long ids_ld, float* x,
                 const unsigned long long* ctrl, int B, int Tc, int V, int D, int* err_flag, void* stream);
/* CausalSelfAttention (mingpt.py:76-94) for the one query row of position p, per (b, head): copies K / V of row b of qkv (fp32 (B, 3D) =
 * [Q | K | V], row stride ld_qkv) bit-exactly into k_cache / v_cache (fp32, row b at b * cache_ld, position j at + j * D), then attends over
 * cache rows 0 ... p in fp32 FMA arithmetic with a fixed reduction order: s_j = (q . k_j, ascending d) * scale, softmax with expf, o = sum_j
 * p_j v_j.  o is written as the fp16 (hi | lo) pair of the proj GEMM's A operand (hi at out[b * ld_out + c], lo lo_off halves further).
 * head_dim must be 32 or 64 (refused otherwise); max_pos (the cache capacity, sizes shared memory) <= 512.  A position p >= max_pos writes and
 * reads nothing. */
int dsb_ar_attention(const float* qkv, long long ld_qkv, float* k_cache, float* v_cache, long long cache_ld, int max_pos, void* out, long long ld_out,
                     long long lo_off, const unsigned long long* ctrl, int B, int H, int head_dim, float scale, void* stream);
/* The full-sequence forward (scoring) of the same model, every position at once (mingpt.py:161-169):
 *   token_embeddings = self.tok_emb(idx); token_embeddings = torch.cat((embeddings, token_embeddings), dim=1)
 *   x = self.drop(token_embeddings + position_embeddings)
 * x[b, t, :] = (t < Tc ? cond[b, t, :] : tok_emb[ids[b * ids_ld + t - Tc], :]) + pos_emb[t, :] for t < T, x (B, T, D) fp32, the fp32 sum of
 * dsb_ar_embed.  An id outside [0, V) sets *err_flag and reads row 0. */
int dsb_ar_embed_all(const float* cond, const float* tok_emb, const float* pos_emb, const int64_t* ids, long long ids_ld, float* x, int B, int T,
                     int Tc, int V, int D, int* err_flag, void* stream);
/* GPT.forward's loss (mingpt.py:183-185) and Net2NetTransformer.shared_step's (cond_transformer.py:106, :358-359):
 *   logits = logits[:, cond_size-1:];  loss = F.cross_entropy(logits.reshape(-1, logits.size(-1)), target.reshape(-1))
 * logits fp32 (B, T, V), row (b, t) at logits + (b * T + t) * ld; the window is rows r0 ... r0 + n - 1 of every batch item; targets int64 (B, n)
 * (row stride tgt_ld).  nll (B, n): the per-row -log_softmax at the target (0 at ignore_index -100), each row reduced by one CTA in a fixed
 * order (independent of B); loss (1): the mean of the non-ignored rows, summed in fp64 in ascending row order (NaN when every row is ignored).
 * A target outside [0, V) other than -100 sets *err_flag (its nll is NaN).  V <= 4096. */
int dsb_ar_cross_entropy(const float* logits, long long ld, int T, int r0, int n, const int64_t* targets, long long tgt_ld, float* nll, float* loss,
                         int B, int V, int* err_flag, void* stream);
/* nn.GELU() (exact erf form, mingpt.py:104-109) between the MLP GEMMs: y = x * 0.5 * (1 + erff(x / sqrt(2))) of fp32 in (rows, C), written
 * as the fp16 (hi | lo) pair (hi at out[r * ld_out + c], lo lo_off halves further). */
int dsb_gelu_erf_split(const float* in, long long ld_in, void* out, long long ld_out, long long lo_off, int rows, int C, void* stream);
/* One sampling step of Net2NetTransformer.sample (cond_transformer.py:118-122, :171-186), one CTA per row b, V <= 4096:
 * logits / temperature (fp32 division); top_k (1 ... V; 0 = None): entries below the top_k-th largest value become -inf (ties kept), by a
 * bisection over the value's order-preserving key; fp32 softmax in a fixed order; do_sample: argmax(p / q) with q the replayed
 * exponential_(1) of the (B, V) tensor at the control block's RNG state (torch.multinomial(probs, 1)'s CUDA fast path), else argmax(p); ties
 * go to the lowest index.  At p >= ctrl[6] the id is written to ids[b * ids_ld + p - Tc + 1]; the last CTA advances p and, when it sampled,
 * the philox offset.  A NaN probability (NaN / inf logits, all entries -inf) sets *err_flag.  Optional: probs_out (B, V) and logits_hist
 * (raw logits of row b at position p written to logits_hist[b * hist_ld + p * V + k]). */
int dsb_ar_sample(const float* logits, long long ld_logits, int64_t* ids, long long ids_ld, unsigned long long* ctrl, int B, int V, int Tc,
                  float temperature, int top_k, int do_sample, float* probs_out, float* logits_hist, long long hist_ld, int* err_flag, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * SpecVQGAN decoder support (reference Diffsound/specvqgan/modules/diffusionmodules/model.py:570-671 Decoder and its
 * blocks; sound_synthesis/modeling/models/dalle_spec.py:80-91 decode_to_img).  Activations are fp32 channels-last images
 * with a one-pixel zero border, (B, H+2, W+2, C); the convolutions themselves are dsb_gemm_ex calls with 9 (3x3) or 1 (1x1)
 * taps and the geo_* border mask.
 * ------------------------------------------------------------------------------------------------------------- */
/* ColumnMajor(reverse=True) + get_codebook_entry (permuter.py:46-49, quantize.py:88-103): ids (B, H*W) int64 in column-major
 * token order -> padded z (B, H+2, W+2, E). */
int dsb_codebook_gather_padded(const int64_t* ids, const float* codebook, float* out, int B, int H, int W, int E, int n_codes, int flags,
                               int* err_flag, void* stream);
/* GroupNorm statistics: stats (B, groups, 2) fp64 = (sum, sum of squares) over the P = (H+2)(W+2) rows of each image */
int dsb_groupnorm_stats(const float* x, double* stats, int B, int P, int C, int groups, void* stream);
/* GroupNorm affine (+swish) from those statistics (model.py:34-35, :29-31); border stays zero.  flags: DSB_GN_SWISH,
 * DSB_GEMM_ROUND_TF32, DSB_GN_COMPACT (then out is (B, Lp, C) tokens in row-major pixel order, rows >= H*W zero). */
int dsb_groupnorm_apply(const float* x, const double* stats, const float* gamma, const float* beta, float* out, int B, int H, int W, int C,
                        int groups, float eps, int flags, int Lp, void* stream);
/* nearest-neighbour x2 (model.py:48-52): (B, H+2, W+2, C) -> (B, 2H+2, 2W+2, C) */
int dsb_upsample2x_padded(const float* in, float* out, int B, int H, int W, int C, int flags, void* stream);
/* AttnBlock plumbing (model.py:202-226): in-place masked row softmax; scatter-add of (B, Lp, C) tokens into the padded image */
int dsb_softmax_rows(float* x, long long rows, int n_valid, int ld, int flags, void* stream);
/* Encoder side of the SpecVQGAN codec (training-time tokeniser, SURVEY.md section 8f N4):
 * Downsample (specvqgan/modules/diffusionmodules/model.py:55-75: zero pad (0,1,0,1) + 3x3 stride-2 conv) = this phase rearrangement of the
 * padded image (B,H+2,W+2,C) into (B,H/2+2,W/2+2,4C) [DSB_SPLIT_OUT: (hi | lo), 8C columns] followed by a 9-tap dsb_gemm_ex with row shifts
 * (dy/2)(W/2+2) + dx/2 and A column offsets (2(dy%2) + dx%2) C. */
int dsb_space_to_depth_padded(const float* in, float* out, int B, int H, int W, int C, int flags, void* stream);
/* VectorQuantizer.forward's nearest code (specvqgan/modules/vqvae/quantize.py:56-63): out[r] = argmin_k x[r, k], first index on ties;
 * x = |e|^2 - 2 z.e from a GEMM with alpha = -2 and bias = |e|^2. */
int dsb_row_argmin(const float* x, long long ld, long long rows, int n, int64_t* out, void* stream);
int dsb_tokens_add_to_padded(const float* tok, float* xpad, int B, int H, int W, int C, int Lp, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * MelGAN generator support (reference Diffsound/vocoder/modules.py:72-130): LeakyReLU(slope) + reflection / zero padding
 * into a channels-last (B, T+2*pad, C) buffer; in_channel_major reads a (B, C, T) input (the mel spectrogram).
 * ------------------------------------------------------------------------------------------------------------- */
int dsb_lrelu_pad(const float* in, float* out, int B, int T, int C, int pad, float slope, int reflect, int in_channel_major, int flags,
                  void* stream);
/* Split-fp16 ("f16x3") MelGAN path.  Activations live in per-stage STATE buffers (B, P + T + P, 4C) fp16 whose rows are
 * [raw_hi | raw_lo | act_hi | act_lo], act = LeakyReLU(0.2)(raw); every Conv1d / ConvTranspose1d / ResnetBlock tail is one dsb_gemm_ex over
 * them (taps = row shifts into the P pad rows; DSB_GEMM_OUT_F16_SPLIT | DSB_GEMM_DUAL_LRELU writes the next state's rows).
 * dsb_mel_pack_f16: mel (B, Cm, T) fp32 (Generator.forward's input, vocoder/modules.py:129) -> (B, T + 2 pad, 2 Kp) fp16 [hi | lo],
 *   ReflectionPad1d(pad) applied in time (:96), channel columns [Cm, Kp) zero (Kp = K rounded up to the GEMM's 64-wide k-block).
 * dsb_edge_pad_f16: fills pad rows P-j and P+T-1+j (j = 1..d) of columns [col0, col0 + ncols) of every clip with the reflection of rows
 *   P+j / P+T-1-j (ReflectionPad1d(dilation), :77; ReflectionPad1d(3), :121) or with zeros (the zero-extended input of the polyphase
 *   ConvTranspose1d taps). */
int dsb_mel_pack_f16(const float* mel, void* out_f16, int B, int Cm, int T, int pad, int Kp, void* stream);
int dsb_edge_pad_f16(void* state_f16, long long ld, long long batch_stride, int B, int T, int P, int d, int col0, int ncols, int reflect,
                     void* stream);
/* MelGAN output layer on the FMA pipe (reference vocoder/modules.py:121-126: LeakyReLU -> ReflectionPad1d(3) -> Conv1d(ngf, 1, kernel 7) -> tanh):
   out[b, t] = tanh(scale * sum_{j < kt, c < cs} x[b, row0 + t + j, c] * w[j, c] + bias[0]),  x = hi + lo of the fp16 pair stored at columns
   [col0, col0 + cs) and [col0 + cs, col0 + 2 cs) of state rows (ld halves per row); the pad rows already hold the reflected samples
   (dsb_edge_pad_f16).  w (kt, cs) fp32, out (B, T) fp32.  Built for cs == 32, kt == 7; other shapes go through dsb_gemm_ex. */
int dsb_conv_out_pair(const void* state, long long ld, long long batch_stride, int B, int T, int row0, int col0, int cs, int kt, const float* w,
                      const float* bias, float scale, float* out, void* stream);


/* ---------------------------------------------------------------------------------------------------------------
 * Melception feature extractor support (reference Codebook/evaluation/feature_extractors/melception.py:23-113 over torchvision's Inception3).
 * Activations are split-fp16 PAIR IMAGES: channels-last fp16 (B, Hp, Wp, ld) whose pixel rows hold hi = f16(v) at [0, C) and lo = f16(v - hi)
 * at [lo_off, lo_off + C), on a zero-bordered grid; a tensor's valid pixels are a window [y0, y0 + H) x [x0, x0 + W) of that grid and every
 * other pixel is zero.  Where an argument list has no ld / lo_off for a tensor, its rows are [hi C | lo C].  Every convolution except the stem
 * is a dsb_gemm_ex over such images (row-shift taps, the geo_* window mask, DSB_GEMM_RELU, DSB_GEMM_OUT_F16_SPLIT into a channel slice).
 * ------------------------------------------------------------------------------------------------------------- */
/* Conv2d_1a_3x3 (1 -> Cout, 3x3, stride 2, valid) with its BatchNorm folded into w (Cout, 9) / bias (Cout), ReLU, times the power of two `scale`:
 * x (B, F, T) fp32 mels, optionally normalised per mel bin first, (x - mean[f]) / stdv[f] (mean = stdv = NULL: none).  Writes the whole
 * (B, Hp, Wp, 2 Cout) pair grid: the ((F-3)/2+1) x ((T-3)/2+1) output window at (y0, x0), zeros elsewhere. */
int dsb_mel_stem(const float* x, const float* mean, const float* stdv, const float* w, const float* bias, float scale, void* out, int B, int F, int T,
                 int Cout, int Hp, int Wp, int y0, int x0, void* stream);
/* Stride-2 phases of a pair image (the fp16-pair form of dsb_space_to_depth_padded, for 3x3 stride-2 VALID convs): in (B, Hpi, Wpi, 2C), window
 * (y0, x0, H, W) -> out (B, Hpo, Wpo, 8C), rows [hi of phases 0..3 | lo of phases 0..3], phase ph = 2 py + px of pixel (oy0 + u, ox0 + v) holding
 * window pixel (2u + py, 2v + px) (zero outside the window).  The conv is then a 9-tap GEMM with row shifts (dy/2) Wpo + dx/2 and A column
 * offsets (2 (dy%2) + dx%2) C.  A pure copy: bit-exact.  C % 8 == 0. */
int dsb_pair_space_to_depth(const void* in, int Hpi, int Wpi, int y0, int x0, int H, int W, void* out, int Hpo, int Wpo, int oy0, int ox0, int B, int C,
                            void* stream);
/* MaxPool2d(3, stride 2) of the window (y0, x0, H, W) of in (B, Hpi, Wpi, 2C) into the output window at (oy0, ox0) of the grid (B, Hpo, Wpo, ldo)
 * (hi at column c, lo at lo_off + c; out may point into a channel slice of a concat), zeros elsewhere in that slice.  The winning pixel's pair is
 * copied (times the power of two `scale`, which moves it to the concat's activation scale): exact. */
int dsb_pair_maxpool3s2(const void* in, int Hpi, int Wpi, int y0, int x0, int H, int W, void* out, long long ldo, long long lo_off, int Hpo, int Wpo,
                        int oy0, int ox0, int B, int C, float scale, void* stream);
/* AvgPool2d(3, stride 1, padding 1, count_include_pad) over the window of in (B, Hp, Wp, 2C): sum of the nine (hi + lo) in fp32, / 9, re-split,
 * into out (same grid, row stride ldo, lo at lo_off); zeros outside the window.  C % 4 == 0. */
int dsb_pair_avgpool3(const void* in, int Hp, int Wp, int y0, int x0, int H, int W, void* out, long long ldo, long long lo_off, int B, int C, void* stream);
/* adaptive_avg_pool2d(., 1) of a pair image: out (B, C) fp32 = inv_scale * mean over the window of (hi + lo), fp64 partial sums in a fixed order
 * (deterministic).  inv_scale undoes the tensor's power-of-two activation scale exactly. */
int dsb_pair_channel_mean(const void* in, long long ld, long long lo_off, int Hp, int Wp, int y0, int x0, int H, int W, int B, int C, float inv_scale,
                          float* out, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * SpecVQGAN log-mel spectrogram (reference Codebook/feature_extraction/extract_mel_spectrogram.py: MelSpectrogram :15-38, the transforms
 * :40-139, TRANSFORMS :141-151, get_spectrogram :166-187; librosa 0.8.0: stft(n_fft 1024, hop 256, center, reflect, periodic Hann),
 * filters.mel(22050, 1024, fmin 125, fmax 7600, 80 mels, Slaney) in float32).  The DFT between the two entry points is a dsb_gemm_ex
 * split-fp16 4-tap conv over the frames buffer: frame t = rows t ... t+3, K = 256 per tap, W = windowed cos / -sin pairs of the bins that
 * any filter covers, fp32 out.
 * ------------------------------------------------------------------------------------------------------------- */
#define DSB_WAV_SCALE 8192.0f /* 2^13: samples are stored scaled so that lo halves stay in fp16's normal range; the GEMM alpha undoes it */
#define DSB_WAV_LIMIT 4.0f    /* |x| must be below this (x * 2^13 < 2^15 stays finite in fp16) */
/* wav (B, length) fp32, row stride ld_wav -> out (B, rows, 512) fp16: row r holds padded samples [256 r, 256 r + 256) of the clip
 * reflect-padded by 512 on each side (numpy.pad mode='reflect', librosa.stft center=True), as hi = f16(2^13 x) at [0, 256) and
 * lo = f16(2^13 x - hi) at [256, 512); samples past the padded end are zero.  rows >= length / 256 + 4 (frames 1 + length / 256 need rows up to
 * length / 256 + 3).  length > 512.  A sample that is not finite or has |x| >= DSB_WAV_LIMIT sets *err_flag (may be NULL). */
int dsb_wav_frames_f16(const float* wav, long long ld_wav, int B, int length, void* out_f16, int rows, int* err_flag, void* stream);
/* spec (B, T, ld_spec) fp32, bin k of frame t at columns (2k, 2k + 1) = (re, im) -> out (B, n_mels, T_out) fp32, T_out <= T:
 * mel[m, t] = sum_{i < fb_len[m]} fb_w[m * fb_ld + i] * |X[t, fb_start[m] + i]| (fp32, ascending i; |X| = sqrt(re^2 + im^2) in fp32), then
 * max(., 1e-5), log10, * 20, - 20, + 100, / 100, clip(0, 1), each step rounded in fp32 in the reference's order.  n_bins <= 383. */
int dsb_mel_log(const float* spec, long long ld_spec, long long spec_batch_stride, int B, int T, int T_out, int n_bins, const int* fb_start,
                const int* fb_len, const float* fb_w, int fb_ld, int n_mels, float* out, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Training (SURVEY.md section 8 row A13; reference sound_synthesis/modeling/transformers/diffusion_transformer.py:370-377, :408-476).
 * The reference obtains every gradient below from torch autograd; these entry points are the hand-written backward passes.
 * "dtype" selects the activation storage: DSB_DTYPE_TF32 (fp32 containers, tf32-rounded on store) or DSB_DTYPE_BF16.
 * ------------------------------------------------------------------------------------------------------------- */
/* q_sample (:370-377): x_t[b,l] = argmax_k(gumbel(uniform[b,k,l]) + q_pred(log_onehot(x0), t)[k]); uniform is (B, K+1, L). */
int dsb_q_sample(const int64_t* x0, const int64_t* t, const float* uniform, const float* sched, int64_t* x_t, int B, int K, int L, int T,
                 void* stream);
/* Fused _train_loss (:408-476) + the normalisation of forward() (:568-569), from the denoiser logits (B, L, K) on:
 *   fp64 log_softmax/clamp, q_posterior of the model and of the true x0, KL / decoder NLL / auxiliary KL, mask weights, 1/pt importance
 *   weights, and the analytic gradient d loss / d logits (dlogits, may be NULL for validation).
 * Outputs: log_model_prob (B, K+1, L) or NULL (exp() of it when prob_as_exp: forward()'s out['logits'], :573-574); col_loss (B, L, 2) per-column (main, aux) terms; hits (B, L, 2) int flags
 *   (argmax(log_x0_recon) == x0, argmax(log_model_prob) == x_t; :424-433) or NULL; kl_loss (B), vb_loss (B), loss (1).
 * lt_history / lt_count (T floats each, updated in place as :448-454 does) may be NULL; scratch_b is B floats.
 * aux_weight = 0 disables the auxiliary term (is_train=False or auxiliary_loss_weight=0).
 * K <= 4095: one warp per column up to K = 1055, one CTA of 256 threads per column above (block reductions in a fixed order). */
int dsb_train_loss(const float* logits, const int64_t* x0, const int64_t* x_t, const int64_t* t, const float* pt, const float* sched,
                   float* dlogits, float* log_model_prob, float* col_loss, int* hits, float* kl_loss, float* vb_loss, float* loss,
                   float* lt_history, float* lt_count, float* scratch_b, int B, int K, int L, int T, float aux_weight, int adaptive,
                   float mw0, float mw1, int prob_as_exp, void* stream);
/* out[b][c, r] = in[b][r, c] (2- or 4-byte elements): the K-major operand copies the weight-gradient GEMMs need. */
int dsb_transpose(const void* in, long long ld_in, long long in_batch_stride, void* out, long long ld_out, long long out_batch_stride,
                  int rows, int cols, int batch, int elem_bytes, void* stream);
/* token-major (B*Lx, ld) with head h in columns [64h, 64h+64)  <->  head-major (B*H, Lx, 64) */
int dsb_heads_split(const void* tok, long long ld, void* heads, int B, int H, int Lx, int elem_bytes, void* stream);
int dsb_heads_merge(const void* heads, void* tok, long long ld, int B, int H, int Lx, int elem_bytes, void* stream);
/* out = dtype(in * (scale ? *scale : 1)); scale is a device scalar (the upstream d loss of autograd / GradScaler) */
int dsb_cast_scale(const float* in, void* out, long long n, const float* scale, int dtype, void* stream);
/* out[n] = sum over rows of in[rows, N] (bias gradients); out is overwritten */
int dsb_colsum(const void* in, long long ld, float* out, long long rows, int N, int dtype, void* stream);
/* GELU2 (transformer_utils.py:111-115) as separate forward / backward passes (training keeps the pre-activation) */
int dsb_gelu2_fwd(const void* u, void* a, long long n, int dtype, void* stream);
int dsb_gelu2_bwd(const void* u, const void* da, void* du, long long n, int dtype, void* stream);
/* timestep-MLP pieces of AdaLayerNorm (transformer_utils.py:145-147) */
int dsb_silu_bwd(const float* x, const float* dy, float* dx, long long n, void* stream);
int dsb_gather_rows(const float* table, const int64_t* idx, float* out, int n, int D, void* stream);
int dsb_scatter_add_rows(float* table, const int64_t* idx, const float* src, int n, int D, void* stream);
/* LayerNorm backward: dx_io += dLN/dx (dx_io already holds the residual branch's gradient); dgamma / dbeta are ACCUMULATED.
 * dx_act (optional): also write the updated dx_io in the activation dtype (the dY operand of the next Linear backward). */
int dsb_layernorm_bwd(const float* x, const float* dy, float* dx_io, const float* gamma, float* dgamma, float* dbeta, long long rows, int D,
                      float eps, void* dx_act, int dtype, void* stream);
/* AdaLayerNorm backward: table (n, 2D) = (scale | shift) rows selected by idx[b]; dtable (same shape) is ACCUMULATED. */
int dsb_ada_layernorm_bwd(const float* x, const float* dy, float* dx_io, const float* table, const int64_t* idx, float* dtable, int B, int L,
                          int D, float eps, void* dx_act, int dtype, void* stream);
/* attention rows: P = softmax(S) and dS = alpha * P * (dP - sum(dP * P)) */
int dsb_softmax_fwd(const float* S, long long ld_s, void* P, long long ld_p, long long rows, int n, int dtype, void* stream);
int dsb_softmax_bwd(const void* P, long long ld_p, const float* dP, long long ld_dp, void* dS, long long ld_ds, long long rows, int n,
                    float alpha, int dtype, void* stream);
/* Fused attention for training (bf16, head_dim 64; FullAttention / CrossAttention, transformer_utils.py:43-58, :91-109): q/k/v/o/dout/dq/dk/dv
 * are token-major with row strides (head h = columns [64h, 64h+64); batch b starts at row b*Lq resp. b*Lk), so they alias the QKV and
 * gradient buffers of the surrounding GEMMs.  fwd also writes lse (B*H, Lq) = log2 sum_k exp(scale s_k); bwd rebuilds P from it and needs a
 * (B*H, Lq) fp32 scratch `delta`. */
int dsb_attention_train_fwd(const void* q, long long ldq, const void* k, long long ldk, const void* v, long long ldv, void* o, long long ldo,
                            float* lse, int B, int H, int Lq, int Lk, float scale, void* stream);
int dsb_attention_train_bwd(const void* q, long long ldq, const void* k, long long ldk, const void* v, long long ldv, const void* o, long long ldo,
                            const void* dout, long long lddo, const float* lse, float* delta, void* dq, long long lddq, void* dk, long long lddk,
                            void* dv, long long lddv, int B, int H, int Lq, int Lk, float scale, void* stream);
/* DalleMaskImageEmbedding backward (dalle_mask_image_embedding.py:36-58): demb / dheight / dwidth are ACCUMULATED. */
int dsb_embed_bwd(const int64_t* ids, const float* dx, float* demb, float* dheight, float* dwidth, int B, int L, int D, int H, int W,
                  int num_embed, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DIFFSOUND_B200_H */
