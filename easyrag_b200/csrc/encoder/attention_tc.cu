// Entry points of the wgmma attention kernel (attention_tc.cuh): argument checks, tensor maps and the bidirectional
// instances.  ezr_attn_set_kernel(1) routes ezr_attn_bidir to the warp-level mma.sync kernel
// (attention.cu) instead.
#include "attention_tc.cuh"

namespace ezr {

int attn_bidir_legacy(const void* qkv, int64_t ld, const int32_t* cu_seqlens, int32_t n_seq, int32_t max_len,
                      int32_t n_heads, int32_t n_kv_heads, int32_t head_dim, float softmax_scale, void* out, int64_t ldo,
                      cudaStream_t st);

static int g_attn_kernel = 0;     // ezr_attn_set_kernel: 0 = wgmma (default), 1 = legacy mma.sync kernel (cross-checks,
                                  // bidirectional only)
static thread_local const char* g_attn_last = "none";

// the entry points' shared argument checks and dispatch
static int attn_run(bool causal, const void* qkv, int64_t n_tokens, int64_t ld, const int32_t* cu_seqlens, int32_t n_seq,
                    int32_t max_len, int32_t n_heads, int32_t n_kv_heads, int32_t head_dim, float softmax_scale,
                    void* out, int64_t ldo, void* stream) {
    EZR_CHECK_ARG(head_dim == 64 || head_dim == 128, "attn: head_dim must be 64 or 128 (got %d)", head_dim);
    EZR_CHECK_ARG(n_kv_heads >= 1 && n_heads % n_kv_heads == 0, "attn: n_heads must be a multiple of n_kv_heads");
    EZR_CHECK_ARG(ld % 8 == 0 && ldo % 8 == 0, "attn: row strides must be multiples of 8 elements");
    EZR_CHECK_ARG(ld >= (int64_t)(n_heads + 2 * n_kv_heads) * head_dim, "attn: qkv rows narrower than (H + 2 KV) * head_dim");
    EZR_CHECK_ARG(((reinterpret_cast<uintptr_t>(qkv) | reinterpret_cast<uintptr_t>(out)) & 15) == 0,
                  "attn: qkv / out must be 16-byte aligned");
    EZR_CHECK_ARG(softmax_scale > 0.f, "attn: softmax_scale must be positive");
    EZR_CHECK_ARG(!(causal && g_attn_kernel == 1),
                  "attn_causal: the legacy mma.sync kernel (ezr_attn_set_kernel(1)) is bidirectional only");
    if (n_seq == 0 || max_len == 0 || n_tokens == 0) return EZR_OK;
    EZR_CHECK_ARG(n_seq <= 65535 && n_heads <= 65535, "attn: grid too large");
    cudaStream_t st = (cudaStream_t)stream;
    if (g_attn_kernel == 1) {
        g_attn_last = "mma.sync";
        return attn_bidir_legacy(qkv, ld, cu_seqlens, n_seq, max_len, n_heads, n_kv_heads, head_dim, softmax_scale, out,
                                 ldo, st);
    }
    g_attn_last = causal ? "wgmma-causal" : "wgmma";
    CUtensorMap map_q, map_kv;
    const uint64_t width = (uint64_t)(n_heads + 2 * n_kv_heads) * head_dim;
    int rc = encode_tmap_2d_bf16(&map_q, qkv, width, (uint64_t)n_tokens, (uint64_t)ld, 64, AT_M);
    if (rc) return rc;
    rc = encode_tmap_2d_bf16(&map_kv, qkv, width, (uint64_t)n_tokens, (uint64_t)ld, 64, AT_N);
    if (rc) return rc;
    const float scale_log2 = softmax_scale * 1.4426950408889634f;
    __nv_bfloat16* o = (__nv_bfloat16*)out;
    if (causal)
        return attn_tc_causal_launch(head_dim, map_q, map_kv, cu_seqlens, n_seq, max_len, n_heads, n_kv_heads,
                                     scale_log2, o, ldo, st);
    return head_dim == 64 ? attn_tc_launch<64, false>(map_q, map_kv, cu_seqlens, n_seq, max_len, n_heads, n_kv_heads,
                                                      scale_log2, o, ldo, st)
                          : attn_tc_launch<128, false>(map_q, map_kv, cu_seqlens, n_seq, max_len, n_heads, n_kv_heads,
                                                       scale_log2, o, ldo, st);
}

}  // namespace ezr

extern "C" int ezr_attn_set_kernel(int32_t which) {
    EZR_CHECK_ARG(which == 0 || which == 1, "attn_set_kernel: 0 = wgmma, 1 = legacy mma.sync");
    ezr::g_attn_kernel = which;
    return EZR_OK;
}

extern "C" const char* ezr_attn_last_kernel(void) { return ezr::g_attn_last; }

extern "C" int ezr_attn_bidir(const void* qkv, int64_t n_tokens, int64_t ld, const int32_t* cu_seqlens, int32_t n_seq,
                              int32_t max_len, int32_t n_heads, int32_t n_kv_heads, int32_t head_dim, float softmax_scale,
                              void* out, int64_t ldo, void* stream) {
    return ezr::attn_run(false, qkv, n_tokens, ld, cu_seqlens, n_seq, max_len, n_heads, n_kv_heads, head_dim,
                         softmax_scale, out, ldo, stream);
}

extern "C" int ezr_attn_causal(const void* qkv, int64_t n_tokens, int64_t ld, const int32_t* cu_seqlens, int32_t n_seq,
                               int32_t max_len, int32_t n_heads, int32_t n_kv_heads, int32_t head_dim, float softmax_scale,
                               void* out, int64_t ldo, void* stream) {
    return ezr::attn_run(true, qkv, n_tokens, ld, cu_seqlens, n_seq, max_len, n_heads, n_kv_heads, head_dim,
                         softmax_scale, out, ldo, stream);
}
