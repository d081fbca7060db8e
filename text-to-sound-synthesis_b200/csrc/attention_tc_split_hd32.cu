// Split-fp16 ("f16x3") attention core at head_dim 32 (Diffsound caps_small_transformer.yaml: n_embd 512, 16 heads; reference
// transformer_utils.py:48-54 FullAttention, :99-105 CrossAttention: softmax(Q K^T / sqrt(32)) V).
// The kernel is attention_split.cuh's, instantiated for 32-column heads: 64-byte (SWIZZLE_64B) head rows, S as 6 wgmma m64n64k16 (SS) and
// P V as 12 wgmma m64n32k16 (RS) per 64-key chunk.  It has its own translation unit so that
// attention_tc_split.cu holds the head_dim-64 kernel alone.
#include "attention_split.cuh"

extern "C" int dsb_attention_tc_split_hd32(const void* q, long long ldq, long long q_lo_off, const void* k, long long ldk, long long k_lo_off,
                                           const void* v, long long ldv, long long v_lo_off, void* o, long long ldo, long long o_lo_off, int B, int H,
                                           int Lq, int Lk, float scale, void* stream) {
  return dsb::attention_tc_split_launch<32>("dsb_attention_tc_split_hd32", q, ldq, q_lo_off, k, ldk, k_lo_off, v, ldv, v_lo_off, o, ldo, o_lo_off, B,
                                            H, Lq, Lk, scale, stream);
}
