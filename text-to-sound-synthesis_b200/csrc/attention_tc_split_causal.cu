// Causal split-fp16 ("f16x3") attention core, head_dim 64 and 32: the autoregressive SpecVQGAN transformer's full-sequence forward
// (reference mingpt.py:53-94 CausalSelfAttention with n_unmasked = 0: key j of query row i is masked when j > i, condition rows included).
// The kernel is attention_split.cuh's with CAUSAL set: a 64-row query tile t multiplies K / V chunks 0 ... t only, the element mask runs on
// the diagonal chunk alone, the producer streams a pair's chunks up to the odd tile's diagonal, and units run heaviest pair first.  Its own
// translation unit, so attention_tc_split.cu and attention_tc_split_hd32.cu keep their non-causal kernels alone.
#include "attention_split.cuh"

extern "C" int dsb_attention_tc_split_causal(const void* q, long long ldq, long long q_lo_off, const void* k, long long ldk, long long k_lo_off,
                                             const void* v, long long ldv, long long v_lo_off, void* o, long long ldo, long long o_lo_off, int B, int H,
                                             int Lq, int Lk, float scale, int head_dim, void* stream) {
  const char* name = "dsb_attention_tc_split_causal";
  if (head_dim == 64)
    return dsb::attention_tc_split_launch<64, true>(name, q, ldq, q_lo_off, k, ldk, k_lo_off, v, ldv, v_lo_off, o, ldo, o_lo_off, B, H, Lq, Lk, scale,
                                                    stream);
  DSB_REQUIRE(head_dim == 32, "%s: head_dim=%d unsupported (64 or 32)", name, head_dim);
  return dsb::attention_tc_split_launch<32, true>(name, q, ldq, q_lo_off, k, ldk, k_lo_off, v, ldv, v_lo_off, o, ldo, o_lo_off, B, H, Lq, Lk, scale,
                                                  stream);
}
