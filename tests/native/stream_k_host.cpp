// Host build of csrc/stream_k.cuh (the wgmma GEMM's tile schedule) -- TEST INFRASTRUCTURE.  tests/test_cpu_stream_k.py compiles this with
// g++ and checks the partition: every k-block of every tile covered once, at most two CTAs per tile, at most one head and one tail per CTA.
#include "stream_k.cuh"

extern "C" int sk_applies(int num_tiles, int num_kb, int grid, int sms) { return dsb_sk::stream_k_applies(num_tiles, num_kb, grid, sms) ? 1 : 0; }

// CTA c's pieces in time order as (tile, kb0, kb1) triples; returns the piece count, or -1 when more than max_pieces
extern "C" int sk_pieces(int num_tiles, int num_kb, int grid, int c, int stream_k, int* out, int max_pieces) {
  const dsb_sk::Work w = dsb_sk::cta_work(num_tiles, num_kb, grid, c, stream_k != 0);
  const int n = dsb_sk::num_pieces(w);
  if (n > max_pieces) return -1;
  for (int i = 0; i < n; ++i) {
    const dsb_sk::Piece p = dsb_sk::piece(w, num_kb, i);
    out[3 * i] = p.tile;
    out[3 * i + 1] = p.kb0;
    out[3 * i + 2] = p.kb1;
  }
  return n;
}
