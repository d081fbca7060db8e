// Tile schedule of the wgmma GEMM (gemm_wgmma.cu): which (tile, k-block range) pieces each CTA runs, and in which order.
//
// * data-parallel: CTA c runs whole tiles c, c + G, c + 2G, ... (G = gridDim.x).
// * ordered stream-K: all but the last G + num_tiles % G tiles run data-parallel.  The k-blocks of those last tiles, in tile-major /
//   k-block-minor order, are cut into G contiguous ranges, CTA c owning [floor(c U / G), floor((c + 1) U / G)) of the U units.  As more
//   than G tiles are cut, every range is at least num_kb long, so a tile
//   spans at most two CTAs and a CTA holds at most
//     - one HEAD: k-blocks [0, head_kb) of the tile its range ends in, finished by CTA c + 1, and
//     - one TAIL: k-blocks [tail_kb, num_kb) of the tile its range starts in, started by CTA c - 1.
//   A CTA runs its head FIRST (and publishes the fp32 accumulator), then its data-parallel and its stream-K whole tiles, then its tail
//   (which continues CTA c - 1's published accumulator).  So a CTA only ever waits at its end, and only on the CTA before it, which published before doing anything else.
//
// Shared by the kernel's producer and consumers (their smem ring stages must match piece for piece) and by the host-side unit test
// (tests/native/stream_k_host.cpp), hence plain C++ outside nvcc.
#pragma once

#ifdef __CUDACC__
#define DSB_SK __host__ __device__ __forceinline__
#else
#define DSB_SK inline
#endif

namespace dsb_sk {

struct Piece {
  int tile, kb0, kb1;  // k-blocks [kb0, kb1) of tile; kb0 > 0: a tail, kb1 < num_kb: a head
};

struct Work {
  int head_tile, head_kb;          // head_kb == 0: no head
  int dp0, dp_step, n_dp;          // data-parallel whole tiles dp0, dp0 + dp_step, ... (n_dp of them)
  int tile0, n_whole;              // stream-K whole tiles tile0, tile0 + 1, ... (n_whole of them)
  int tail_tile, tail_kb;          // tail_kb == 0: no tail
};

// Stream-K pays when the tiles leave a partial last wave that is a large share of the launch: with three waves or more (the denoiser's qkv
// and mlp1 GEMMs at batch 16) the idle share is at most 12 % and, measured on an H100, the split tiles cost more than they save.  The waits
// between neighbouring CTAs are deadlock-free only when every CTA of the grid is resident at once (grid <= SM count, 1 CTA per SM).
// The unit count must fit an int: the kernel's partition arithmetic is 32-bit (a 64-bit division is a call on the GPU).
DSB_SK bool stream_k_applies(int num_tiles, int num_kb, int grid, int sms) {
  return grid <= sms && num_tiles > grid && num_tiles < 3 * grid && num_tiles % grid != 0 && num_kb > 1 &&
         (long long)num_tiles * num_kb <= 0x7fffffff;
}

// With stream-K, only the last full wave and the partial one (grid + num_tiles % grid tiles) are cut into k-block ranges; the waves before
// them stay data-parallel, so that the CTAs run neighbouring tiles at the same time and share their operands in L2.
DSB_SK Work cta_work(int num_tiles, int num_kb, int grid, int c, bool stream_k) {
  Work w{};
  w.dp0 = c;
  w.dp_step = grid;
  if (!stream_k) {
    w.n_dp = c < num_tiles ? (num_tiles - c + grid - 1) / grid : 0;
    return w;
  }
  const int sk_tiles = grid + num_tiles % grid, dp_tiles = num_tiles - sk_tiles;
  w.n_dp = dp_tiles / grid;
  // CTA c owns units [u0, u1) of the sk_tiles x num_kb stream-K units; u0 = floor(units * c / grid) without overflow: units = q grid + r,
  // so u0 = q c + floor(r c / grid) with r c < grid^2.  Every range is longer than num_kb, as sk_tiles > grid.
  const int units = sk_tiles * num_kb, q = units / grid, r = units % grid;
  const int u0 = q * c + r * c / grid, u1 = q * (c + 1) + r * (c + 1) / grid;
  const int t0 = dp_tiles + u0 / num_kb, k0 = u0 % num_kb;
  const int t1 = dp_tiles + u1 / num_kb, k1 = u1 % num_kb;
  w.tail_tile = t0;
  w.tail_kb = k0;
  w.tile0 = k0 > 0 ? t0 + 1 : t0;
  w.n_whole = t1 - w.tile0;
  w.head_tile = t1;
  w.head_kb = k1;
  return w;
}

DSB_SK int num_pieces(const Work& w) { return (w.head_kb > 0) + w.n_dp + w.n_whole + (w.tail_kb > 0); }

// piece i of a CTA, in time order: head, data-parallel tiles, stream-K whole tiles, tail
DSB_SK Piece piece(const Work& w, int num_kb, int i) {
  if (w.head_kb > 0) {
    if (i == 0) return Piece{w.head_tile, 0, w.head_kb};
    --i;
  }
  if (i < w.n_dp) return Piece{w.dp0 + i * w.dp_step, 0, num_kb};
  i -= w.n_dp;
  if (i < w.n_whole) return Piece{w.tile0 + i, 0, num_kb};
  return Piece{w.tail_tile, w.tail_kb, num_kb};
}

}  // namespace dsb_sk
