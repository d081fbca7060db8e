// Split-fp16 ("f16x3") attention core at head_dim 64 -- the parity-grade twin of attention_tc.cu
// (reference transformer_utils.py:48-54 FullAttention, :99-105 CrossAttention: softmax(Q K^T / sqrt(64)) V, 16 heads x 64).
// The kernel is attention_split.cuh's, instantiated for 64-column heads: 128-byte (SWIZZLE_128B) head rows, S as 12 wgmma m64n64k16 (SS)
// and P V as 12 wgmma m64n64k16 (RS) per 64-key chunk.  fp32-class accuracy: measured against an fp64 reference in tests/test_gpu_split.py
// and tests/test_gpu_attention_wgmma.py.
#include "attention_split.cuh"

extern "C" int dsb_attention_tc_split(const void* q, long long ldq, long long q_lo_off, const void* k, long long ldk, long long k_lo_off, const void* v,
                                      long long ldv, long long v_lo_off, void* o, long long ldo, long long o_lo_off, int B, int H, int Lq, int Lk,
                                      float scale, void* stream) {
  return dsb::attention_tc_split_launch<64>("dsb_attention_tc_split", q, ldq, q_lo_off, k, ldk, k_lo_off, v, ldv, v_lo_off, o, ldo, o_lo_off, B, H, Lq,
                                            Lk, scale, stream);
}
