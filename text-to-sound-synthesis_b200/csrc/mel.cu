// SpecVQGAN's log-mel front end (reference Codebook/feature_extraction/extract_mel_spectrogram.py: MelSpectrogram :15-38, the transform
// classes :40-139, TRANSFORMS :141-151, get_spectrogram :166-187; librosa 0.8.0 stft / filters.mel).  Three launches per batch:
//   1. dsb_wav_frames_f16: the reflect-padded clip as rows of 256 samples, each row a split-fp16 pair [hi 256 | lo 256] of 2^13 * x;
//   2. dsb_gemm_ex (unchanged): the windowed DFT as a 4-tap conv over those rows (frame t = rows t .. t+3), split-fp16 3-pass form, fp32 out;
//   3. dsb_mel_log: |X|, the sparse Slaney filterbank, max(., 1e-5), log10, *20, -20, +100, /100, clip(0, 1), mel-major out.
#include "common.cuh"
#include "diffsound_b200.h"
#include <cuda_fp16.h>

namespace dsb {

constexpr int kHop = 256, kPad = 512;

// padded sample i of the clip, numpy.pad(mode='reflect') by kPad on each side, zero past the padded end
__device__ __forceinline__ float padded_sample(const float* __restrict__ x, int length, long long i) {
  long long j = i - kPad;
  if (j < 0) j = -j;
  else if (j >= length) j = 2LL * (length - 1) - j;
  return (i < (long long)length + 2 * kPad) ? __ldg(x + j) : 0.f;
}

// one thread per 8 consecutive samples of a row: uint4 of hi, uint4 of lo
__global__ void wav_frames_f16_kernel(const float* __restrict__ wav, long long ld_wav, int B, int length, __half* __restrict__ out, int rows,
                                      int* __restrict__ err_flag) {
  const long long per_clip = (long long)rows * (kHop / 8);
  const long long total = per_clip * B;
  for (long long g = blockIdx.x * (long long)blockDim.x + threadIdx.x; g < total; g += (long long)gridDim.x * blockDim.x) {
    const int b = (int)(g / per_clip);
    const long long rem = g % per_clip;
    const int r = (int)(rem / (kHop / 8)), c = (int)(rem % (kHop / 8)) * 8;
    const float* x = wav + (long long)b * ld_wav;
    const long long i0 = (long long)r * kHop + c;
    __align__(16) __half h[8], l[8];
    bool bad = false;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const float v = padded_sample(x, length, i0 + k);
      // every sample of the clip appears once in the unreflected middle; check it there (NaN fails the comparison)
      const long long j = i0 + k - kPad;
      if (j >= 0 && j < length && !(fabsf(v) < DSB_WAV_LIMIT)) bad = true;
      const float s = v * DSB_WAV_SCALE;  // exact: a power of two
      h[k] = __float2half_rn(s);
      l[k] = __float2half_rn(s - __half2float(h[k]));
    }
    if (bad && err_flag) atomicExch(err_flag, 1);
    __half* o = out + ((long long)b * rows + r) * (2 * kHop) + c;
    *reinterpret_cast<uint4*>(o) = *reinterpret_cast<const uint4*>(h);
    *reinterpret_cast<uint4*>(o + kHop) = *reinterpret_cast<const uint4*>(l);
  }
}

constexpr int kMelFrames = 32;  // frames per CTA
constexpr int kMelThreads = 256;

// One CTA per (32 frames, clip): the magnitudes of the 32 frames' n_bins DFT bins go to shared memory (row stride n_bins | 1, odd, so the
// 32 lanes of a warp, one frame each, read distinct banks), then each warp produces whole mel rows of 32 consecutive frames.
__global__ void __launch_bounds__(kMelThreads) mel_log_kernel(const float* __restrict__ spec, long long ld_spec, long long spec_bstride, int T_out,
                                                             int n_bins, const int* __restrict__ fb_start, const int* __restrict__ fb_len,
                                                             const float* __restrict__ fb_w, int fb_ld, int n_mels, float* __restrict__ out) {
  extern __shared__ float mag[];
  const int ms = n_bins | 1;
  const int b = blockIdx.y, t0 = blockIdx.x * kMelFrames;
  const int nf = min(kMelFrames, T_out - t0);
  const float* sp = spec + (long long)b * spec_bstride + (long long)t0 * ld_spec;
  for (int e = threadIdx.x; e < nf * n_bins; e += kMelThreads) {
    const int f = e / n_bins, k = e % n_bins;
    const float2 v = __ldg(reinterpret_cast<const float2*>(sp + (long long)f * ld_spec) + k);
    mag[f * ms + k] = __fsqrt_rn(__fmaf_rn(v.x, v.x, __fmul_rn(v.y, v.y)));
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane >= nf) return;
  for (int m = warp; m < n_mels; m += kMelThreads / 32) {
    const int s = __ldg(fb_start + m), n = __ldg(fb_len + m);
    const float* w = fb_w + (long long)m * fb_ld;
    const float* a = mag + lane * ms + s;
    float acc = 0.f;
    for (int i = 0; i < n; ++i) acc = __fmaf_rn(__ldg(w + i), a[i], acc);
    // LowerThresh(1e-5), Log10, Multiply(20), Subtract(20), Add(100), Divide(100), Clip(0, 1) -- the reference's order, each step rounded
    float y = log10f(fmaxf(acc, 1e-5f));
    y = __fmul_rn(y, 20.f);
    y = __fsub_rn(y, 20.f);
    y = __fadd_rn(y, 100.f);
    y = __fdiv_rn(y, 100.f);
    y = fminf(fmaxf(y, 0.f), 1.f);
    out[((long long)b * n_mels + m) * T_out + t0 + lane] = y;
  }
}

}  // namespace dsb
using namespace dsb;

extern "C" int dsb_wav_frames_f16(const float* wav, long long ld_wav, int B, int length, void* out_f16, int rows, int* err_flag, void* stream) {
  DSB_REQUIRE(B > 0 && length > kPad, "dsb_wav_frames_f16: need B >= 1 and length > %d (reflect padding), got B=%d length=%d", kPad, B, length);
  DSB_REQUIRE(ld_wav >= length, "dsb_wav_frames_f16: row stride %lld below length %d", ld_wav, length);
  const long long need = (long long)length / kHop + 4;  // frames 1 + length / 256, each 4 rows, hop 1 row
  DSB_REQUIRE(rows >= need, "dsb_wav_frames_f16: %d rows per clip, need at least %lld", rows, need);
  DSB_REQUIRE((reinterpret_cast<uintptr_t>(out_f16) & 15) == 0, "dsb_wav_frames_f16: output must be 16-byte aligned");
  const long long total = (long long)B * rows * (kHop / 8);
  long long grid = (total + 255) / 256;
  const long long cap = (long long)sm_count() * 16;
  if (grid > cap) grid = cap;
  wav_frames_f16_kernel<<<(unsigned)grid, 256, 0, (cudaStream_t)stream>>>(wav, ld_wav, B, length, (__half*)out_f16, rows, err_flag);
  DSB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dsb_mel_log(const float* spec, long long ld_spec, long long spec_batch_stride, int B, int T, int T_out, int n_bins, const int* fb_start,
                           const int* fb_len, const float* fb_w, int fb_ld, int n_mels, float* out, void* stream) {
  DSB_REQUIRE(B > 0 && T > 0 && T_out > 0 && T_out <= T && n_bins > 0 && n_mels > 0, "dsb_mel_log: bad shape B=%d T=%d T_out=%d n_bins=%d n_mels=%d",
              B, T, T_out, n_bins, n_mels);
  DSB_REQUIRE(B <= 65535, "dsb_mel_log: at most 65535 clips per launch, got %d", B);
  DSB_REQUIRE(ld_spec >= 2LL * n_bins && ld_spec % 2 == 0 && spec_batch_stride % 2 == 0 && (reinterpret_cast<uintptr_t>(spec) & 7) == 0,
              "dsb_mel_log: spectrum rows must hold 2 * n_bins floats at 8-byte alignment");
  const size_t smem = sizeof(float) * kMelFrames * (n_bins | 1);
  DSB_REQUIRE(smem <= 48 * 1024, "dsb_mel_log: %d bins exceed the shared-memory tile", n_bins);
  dim3 grid((T_out + kMelFrames - 1) / kMelFrames, B);
  mel_log_kernel<<<grid, kMelThreads, smem, (cudaStream_t)stream>>>(spec, ld_spec, spec_batch_stride, T_out, n_bins, fb_start, fb_len, fb_w, fb_ld,
                                                                    n_mels, out);
  DSB_CHECK_CUDA(cudaGetLastError());
  return 0;
}
