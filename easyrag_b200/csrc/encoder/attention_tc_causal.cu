// The causal instances of the wgmma attention kernel (attention_tc.cuh), in a translation unit of their own: compiled
// in the same module as the bidirectional instances, they changed the code nvcc generated for those, and the
// bidirectional kernels are kept instruction-for-instruction as they were (DESIGN.md 4.5).
#include "attention_tc.cuh"

namespace ezr {

int attn_tc_causal_launch(int head_dim, const CUtensorMap& map_q, const CUtensorMap& map_kv, const int32_t* cu,
                          int n_seq, int max_len, int n_heads, int n_kv_heads, float scale_log2, __nv_bfloat16* out,
                          int64_t ldo, cudaStream_t st) {
    return head_dim == 64 ? attn_tc_launch<64, true>(map_q, map_kv, cu, n_seq, max_len, n_heads, n_kv_heads, scale_log2,
                                                     out, ldo, st)
                          : attn_tc_launch<128, true>(map_q, map_kv, cu, n_seq, max_len, n_heads, n_kv_heads, scale_log2,
                                                      out, ldo, st);
}

}  // namespace ezr
