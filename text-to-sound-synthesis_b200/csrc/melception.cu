// Melception (the Inception-v3 feature extractor of the Diffsound evaluation, reference Codebook/evaluation/feature_extractors/melception.py)
// support kernels.  Activations are split-fp16 PAIR IMAGES: channels-last (B, Hp, Wp, ld) fp16 whose pixel rows hold hi = f16(v) at [0, C) and
// lo = f16(v - hi) at [lo_off, lo_off + C), on a zero-bordered grid; the valid pixels of a tensor are a WINDOW [y0, y0 + H) x [x0, x0 + W) of
// that grid and everything else is exactly zero.  Every convolution except the 1-channel stem runs on the wgmma GEMM (gemm_wgmma.cu) with row-shift
// taps; the kernels here are the stem, the stride-2 phase rearrangement, the two 3x3 pools and the channel means that produce the features.
#include "common.cuh"
#include "diffsound_b200.h"
#include <cuda_fp16.h>

namespace dsb {

__device__ __forceinline__ void pair_store4(__half* o, long long lo_off, float4 v) {
  const __half2 h0 = __floats2half2_rn(v.x, v.y), h1 = __floats2half2_rn(v.z, v.w);
  const __half2 l0 = __floats2half2_rn(v.x - __low2float(h0), v.y - __high2float(h0));
  const __half2 l1 = __floats2half2_rn(v.z - __low2float(h1), v.w - __high2float(h1));
  uint2 u, w;
  u.x = *reinterpret_cast<const uint32_t*>(&h0); u.y = *reinterpret_cast<const uint32_t*>(&h1);
  w.x = *reinterpret_cast<const uint32_t*>(&l0); w.y = *reinterpret_cast<const uint32_t*>(&l1);
  *reinterpret_cast<uint2*>(o) = u;
  *reinterpret_cast<uint2*>(o + lo_off) = w;
}

__device__ __forceinline__ float pair_value(const __half* p, long long lo_off) { return __half2float(p[0]) + __half2float(p[lo_off]); }

// One thread per grid pixel: Cout channels of relu(sum_{dy,dx} w[c, dy*3+dx] * xn(2i+dy, 2j+dx) + bias[c]) * scale,
// xn(f, t) = (x[b, f, t] - mean[f]) / std[f] (or x when mean == NULL).  Pixels outside the window are written as zeros.
__global__ void mel_stem_kernel(const float* __restrict__ x, const float* __restrict__ mean, const float* __restrict__ stdv, const float* __restrict__ w,
                                const float* __restrict__ bias, float scale, __half* __restrict__ out, int B, int F, int T, int Cout, int Hp, int Wp,
                                int y0, int x0, int Ho, int Wo) {
  const long long total = (long long)B * Hp * Wp;
  for (long long pix = blockIdx.x * (long long)blockDim.x + threadIdx.x; pix < total; pix += (long long)gridDim.x * blockDim.x) {
    const int b = pix / ((long long)Hp * Wp);
    const int pp = pix % ((long long)Hp * Wp);
    const int i = pp / Wp - y0, j = pp % Wp - x0;
    __half* o = out + pix * 2 * Cout;
    if (i < 0 || j < 0 || i >= Ho || j >= Wo) {
      for (int c = 0; c < 2 * Cout; c += 8) *reinterpret_cast<uint4*>(o + c) = make_uint4(0u, 0u, 0u, 0u);
      continue;
    }
    float xn[9];
#pragma unroll
    for (int dy = 0; dy < 3; ++dy) {
      const int f = 2 * i + dy;
      const float m = mean ? __ldg(mean + f) : 0.f, s = stdv ? __ldg(stdv + f) : 1.f;
#pragma unroll
      for (int dx = 0; dx < 3; ++dx) {
        const float v = __ldg(x + ((long long)b * F + f) * T + 2 * j + dx);
        xn[dy * 3 + dx] = mean ? (v - m) / s : v;
      }
    }
    for (int c = 0; c < Cout; c += 4) {
      float a[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        float acc = 0.f;
#pragma unroll
        for (int t = 0; t < 9; ++t) acc = fmaf(__ldg(w + (c + k) * 9 + t), xn[t], acc);
        acc += __ldg(bias + c + k);
        a[k] = (acc < 0.f ? 0.f : acc) * scale;
      }
      pair_store4(o + c, Cout, make_float4(a[0], a[1], a[2], a[3]));
    }
  }
}

// Stride-2 phases of a pair image: out pixel (oy0 + u, ox0 + v), phase ph = 2 py + px holds input window pixel (2u + py, 2v + px) -- hi at
// columns [ph C, ph C + C), lo at [4C + ph C, ...) -- or zeros where that pixel lies outside the window or (u, v) outside [0, ceil(H/2)) x [0, ceil(W/2)).
// A 3x3 stride-2 valid conv is then a 9-tap GEMM over `out` with row shifts (dy/2) Wpo + dx/2 and A column offsets (2 (dy%2) + dx%2) C.
__global__ void pair_space_to_depth_kernel(const __half* __restrict__ in, int Hpi, int Wpi, int y0, int x0, int H, int W, __half* __restrict__ out,
                                           int Hpo, int Wpo, int oy0, int ox0, int B, int C) {
  const int c8n = C / 8;
  const long long total = (long long)B * Hpo * Wpo * 4 * c8n;
  const int Hh = (H + 1) / 2, Wh = (W + 1) / 2;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int c8 = idx % c8n;
    const int ph = (idx / c8n) % 4;
    const long long orow = idx / (4 * c8n);
    const int b = orow / ((long long)Hpo * Wpo);
    const int pp = orow % ((long long)Hpo * Wpo);
    const int u = pp / Wpo - oy0, v = pp % Wpo - ox0;
    const int r = 2 * u + (ph >> 1), s = 2 * v + (ph & 1);
    uint4 hi = make_uint4(0u, 0u, 0u, 0u), lo = hi;
    if (u >= 0 && v >= 0 && u < Hh && v < Wh && r < H && s < W) {
      const __half* p = in + (((long long)b * Hpi + y0 + r) * Wpi + x0 + s) * 2 * C + c8 * 8;
      hi = *reinterpret_cast<const uint4*>(p);
      lo = *reinterpret_cast<const uint4*>(p + C);
    }
    __half* o = out + orow * 8 * C + ph * C + c8 * 8;
    *reinterpret_cast<uint4*>(o) = hi;
    *reinterpret_cast<uint4*>(o + 4 * C) = lo;
  }
}

// 3x3 stride-2 valid max pool: out window pixel (i, j) = the pair of the largest of the nine input pixels (2i + dy, 2j + dx) of the input window
// (compared by hi + lo in fp32; the first one in (dy, dx) order wins a tie, a NaN wins over any number), multiplied by the power of two `scale`.
// Input rows: [hi C | lo C]; output rows: hi at out[pixel * ldo + c], lo at + lo_off.  Pixels outside the output window get zeros.
__global__ void pair_maxpool3s2_kernel(const __half* __restrict__ in, int Hpi, int Wpi, int y0, int x0, __half* __restrict__ out, long long ldo,
                                       long long lo_off, int Hpo, int Wpo, int oy0, int ox0, int Ho, int Wo, int B, int C, float scale) {
  const long long total = (long long)B * Hpo * Wpo * C;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int c = idx % C;
    const long long orow = idx / C;
    const int b = orow / ((long long)Hpo * Wpo);
    const int pp = orow % ((long long)Hpo * Wpo);
    const int i = pp / Wpo - oy0, j = pp % Wpo - ox0;
    __half hv = __float2half_rn(0.f), lv = hv;
    if (i >= 0 && j >= 0 && i < Ho && j < Wo) {
      float best = -INFINITY;
      const __half* base = in + (((long long)b * Hpi + y0 + 2 * i) * Wpi + x0 + 2 * j) * 2 * C + c;
      const __half* win = base;
#pragma unroll
      for (int dy = 0; dy < 3; ++dy)
#pragma unroll
        for (int dx = 0; dx < 3; ++dx) {
          const __half* p = base + ((long long)dy * Wpi + dx) * 2 * C;
          const float v = pair_value(p, C);
          if ((v > best || isnan(v)) && !isnan(best)) { best = v; win = p; }
        }
      hv = __float2half_rn(__half2float(win[0]) * scale);
      lv = __float2half_rn(__half2float(win[C]) * scale);
    }
    out[orow * ldo + c] = hv;
    out[orow * ldo + lo_off + c] = lv;
  }
}

// 3x3 stride-1 average pool with zero padding 1 and divisor 9 (count_include_pad) over the window of a pair image; the grid around the window is
// zero, so the nine grid neighbours of a window pixel are summed (hi + lo in fp32, (dy, dx) order) and the sum / 9 is re-split.  Same grid in and out;
// pixels outside the window get zeros.  Input rows [hi C | lo C]; output rows hi at out[pixel * ldo + c], lo at + lo_off.
__global__ void pair_avgpool3_kernel(const __half* __restrict__ in, int Hp, int Wp, int y0, int x0, int H, int W, __half* __restrict__ out, long long ldo,
                                     long long lo_off, int B, int C) {
  const int c4n = C / 4;
  const long long total = (long long)B * Hp * Wp * c4n;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int c4 = idx % c4n;
    const long long row = idx / c4n;
    const int pp = row % ((long long)Hp * Wp);
    const int y = pp / Wp, x = pp % Wp;
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
    if (y >= y0 && y < y0 + H && x >= x0 && x < x0 + W) {
#pragma unroll
      for (int dy = -1; dy <= 1; ++dy)
#pragma unroll
        for (int dx = -1; dx <= 1; ++dx) {
          if (y + dy < 0 || y + dy >= Hp || x + dx < 0 || x + dx >= Wp) continue;
          const __half* p = in + (row + (long long)dy * Wp + dx) * 2 * C + c4 * 4;
          const uint2 h = *reinterpret_cast<const uint2*>(p), l = *reinterpret_cast<const uint2*>(p + C);
          const float2 h0 = __half22float2(*reinterpret_cast<const __half2*>(&h.x)), h1 = __half22float2(*reinterpret_cast<const __half2*>(&h.y));
          const float2 l0 = __half22float2(*reinterpret_cast<const __half2*>(&l.x)), l1 = __half22float2(*reinterpret_cast<const __half2*>(&l.y));
          s.x += h0.x + l0.x; s.y += h0.y + l0.y; s.z += h1.x + l1.x; s.w += h1.y + l1.y;
        }
      s = make_float4(s.x / 9.f, s.y / 9.f, s.z / 9.f, s.w / 9.f);
    }
    pair_store4(out + row * ldo + c4 * 4, lo_off, s);
  }
}

// out[b, c] = inv_scale * mean over the window of (hi + lo): 32 channels x 8 pixel lanes per block, fp64 partial sums over a fixed pixel stride,
// combined in a fixed order -- the result does not depend on scheduling.
__global__ void pair_channel_mean_kernel(const __half* __restrict__ in, long long ld, long long lo_off, int Hp, int Wp, int y0, int x0, int H, int W,
                                         int C, float inv_scale, float* __restrict__ out) {
  __shared__ double part[8][32];
  const int b = blockIdx.y, c = blockIdx.x * 32 + (threadIdx.x & 31), lane_p = threadIdx.x >> 5;
  double s = 0.0;
  if (c < C) {
    const __half* base = in + (long long)b * Hp * Wp * ld + c;
    for (int p = lane_p; p < H * W; p += 8) {
      const int y = y0 + p / W, x = x0 + p % W;
      s += (double)pair_value(base + ((long long)y * Wp + x) * ld, lo_off);
    }
  }
  part[lane_p][threadIdx.x & 31] = s;
  __syncthreads();
  if (lane_p == 0 && c < C) {
    double t = 0.0;
#pragma unroll
    for (int k = 0; k < 8; ++k) t += part[k][threadIdx.x];
    out[(long long)b * C + c] = (float)(t / ((double)H * W) * (double)inv_scale);
  }
}

}  // namespace dsb

using namespace dsb;

static int mel_grid(long long n) {
  long long g = (n + 255) / 256;
  const long long cap = (long long)sm_count() * 16;
  return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

static bool a16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

extern "C" int dsb_mel_stem(const float* x, const float* mean, const float* stdv, const float* w, const float* bias, float scale, void* out, int B, int F,
                            int T, int Cout, int Hp, int Wp, int y0, int x0, void* stream) {
  const int Ho = (F - 3) / 2 + 1, Wo = (T - 3) / 2 + 1;
  DSB_REQUIRE(B > 0 && F >= 3 && T >= 3 && Cout > 0 && Cout % 4 == 0 && (2 * Cout) % 8 == 0, "dsb_mel_stem: bad shape B=%d F=%d T=%d Cout=%d", B, F, T, Cout);
  DSB_REQUIRE((mean == nullptr) == (stdv == nullptr), "dsb_mel_stem: mean and std go together");
  DSB_REQUIRE(y0 >= 0 && x0 >= 0 && y0 + Ho <= Hp && x0 + Wo <= Wp, "dsb_mel_stem: the %dx%d output window does not fit the %dx%d grid at (%d, %d)", Ho, Wo,
              Hp, Wp, y0, x0);
  DSB_REQUIRE(a16(out), "dsb_mel_stem: out must be 16-byte aligned");
  mel_stem_kernel<<<mel_grid((long long)B * Hp * Wp), 256, 0, (cudaStream_t)stream>>>(x, mean, stdv, w, bias, scale, (__half*)out, B, F, T, Cout, Hp, Wp,
                                                                                        y0, x0, Ho, Wo);
  DSB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dsb_pair_space_to_depth(const void* in, int Hpi, int Wpi, int y0, int x0, int H, int W, void* out, int Hpo, int Wpo, int oy0, int ox0,
                                       int B, int C, void* stream) {
  DSB_REQUIRE(B > 0 && C > 0 && C % 8 == 0 && H > 0 && W > 0, "dsb_pair_space_to_depth: bad shape (C=%d must be a multiple of 8)", C);
  DSB_REQUIRE(y0 >= 0 && x0 >= 0 && y0 + H <= Hpi && x0 + W <= Wpi, "dsb_pair_space_to_depth: input window outside the grid");
  DSB_REQUIRE(oy0 >= 0 && ox0 >= 0 && oy0 + (H + 1) / 2 <= Hpo && ox0 + (W + 1) / 2 <= Wpo, "dsb_pair_space_to_depth: phase window outside the output grid");
  DSB_REQUIRE(a16(in) && a16(out), "dsb_pair_space_to_depth: pointers must be 16-byte aligned");
  pair_space_to_depth_kernel<<<mel_grid((long long)B * Hpo * Wpo * C / 2), 256, 0, (cudaStream_t)stream>>>((const __half*)in, Hpi, Wpi, y0, x0, H, W,
                                                                                                          (__half*)out, Hpo, Wpo, oy0, ox0, B, C);
  DSB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dsb_pair_maxpool3s2(const void* in, int Hpi, int Wpi, int y0, int x0, int H, int W, void* out, long long ldo, long long lo_off, int Hpo,
                                   int Wpo, int oy0, int ox0, int B, int C, float scale, void* stream) {
  const int Ho = (H - 3) / 2 + 1, Wo = (W - 3) / 2 + 1;
  DSB_REQUIRE(B > 0 && C > 0 && H >= 3 && W >= 3, "dsb_pair_maxpool3s2: bad shape");
  DSB_REQUIRE(y0 >= 0 && x0 >= 0 && y0 + H <= Hpi && x0 + W <= Wpi, "dsb_pair_maxpool3s2: input window outside the grid");
  DSB_REQUIRE(oy0 >= 0 && ox0 >= 0 && oy0 + Ho <= Hpo && ox0 + Wo <= Wpo, "dsb_pair_maxpool3s2: output window outside the grid");
  DSB_REQUIRE(ldo >= C && lo_off >= C, "dsb_pair_maxpool3s2: ldo / lo_off too small");
  pair_maxpool3s2_kernel<<<mel_grid((long long)B * Hpo * Wpo * C), 256, 0, (cudaStream_t)stream>>>((const __half*)in, Hpi, Wpi, y0, x0, (__half*)out, ldo,
                                                                                                 lo_off, Hpo, Wpo, oy0, ox0, Ho, Wo, B, C, scale);
  DSB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dsb_pair_avgpool3(const void* in, int Hp, int Wp, int y0, int x0, int H, int W, void* out, long long ldo, long long lo_off, int B, int C,
                                 void* stream) {
  DSB_REQUIRE(B > 0 && C > 0 && C % 4 == 0 && ldo % 4 == 0 && lo_off % 4 == 0, "dsb_pair_avgpool3: C, ldo and lo_off must be multiples of 4");
  DSB_REQUIRE(y0 >= 0 && x0 >= 0 && y0 + H <= Hp && x0 + W <= Wp, "dsb_pair_avgpool3: window outside the grid");
  DSB_REQUIRE((reinterpret_cast<uintptr_t>(in) & 7) == 0 && (reinterpret_cast<uintptr_t>(out) & 7) == 0, "dsb_pair_avgpool3: pointers must be 8-byte aligned");
  pair_avgpool3_kernel<<<mel_grid((long long)B * Hp * Wp * C / 4), 256, 0, (cudaStream_t)stream>>>((const __half*)in, Hp, Wp, y0, x0, H, W, (__half*)out, ldo,
                                                                                                 lo_off, B, C);
  DSB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dsb_pair_channel_mean(const void* in, long long ld, long long lo_off, int Hp, int Wp, int y0, int x0, int H, int W, int B, int C,
                                     float inv_scale, float* out, void* stream) {
  DSB_REQUIRE(B > 0 && C > 0 && H > 0 && W > 0 && ld >= C && lo_off >= C, "dsb_pair_channel_mean: bad shape");
  DSB_REQUIRE(y0 >= 0 && x0 >= 0 && y0 + H <= Hp && x0 + W <= Wp, "dsb_pair_channel_mean: window outside the grid");
  DSB_REQUIRE(B <= 65535, "dsb_pair_channel_mean: B=%d exceeds the grid's y extent", B);
  pair_channel_mean_kernel<<<dim3((C + 31) / 32, B), 256, 0, (cudaStream_t)stream>>>((const __half*)in, ld, lo_off, Hp, Wp, y0, x0, H, W, C, inv_scale, out);
  DSB_CHECK_CUDA(cudaGetLastError());
  return 0;
}
