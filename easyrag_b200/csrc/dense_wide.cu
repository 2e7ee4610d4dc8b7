// Dense cosine top-k for any dim % 64 == 0 and any k <= 1024 on the Hopper tensor cores: the encoder's bf16 GEMM kernel
// (encoder/gemm_tc.cu, through gemm_scores_f32) writes a block of fp32 score rows, and the generic row select
// (ezr_select_rows) takes the top-k from it, in the block loop of dense.cu (score_rows_topk).
//
// The forms of dense_tc.cu keep the query block resident in shared memory and the top-k in registers, which limits
// them to dim <= 1024 and k <= 16.  The GEMM holds nothing resident: both operands stream through one TMA ring, so the
// width is unbounded (gte-Qwen2-7B: 3584), and the scores go to HBM so that k is only bounded by the select (the
// pipeline's f_topk_1 = 288).
//
// One CTA computes one 128-query x 256-row tile of the block's score rows, with the queries as A and the corpus rows
// as W.  Each score is one accumulator chain over the k16 steps in increasing k order, no split-K: the fp32 sum of the
// same k16 products in the same order as forms 2-4, so the scores are bit-identical to theirs.
//
// Tile order: query tiles fastest.  The CTAs in flight then cover all query tiles of a few corpus tiles: a corpus
// tile is read from HBM about once per block, and the query block (a few MB) stays in the 50 MB L2.
#include <algorithm>

#include "ezr_common.cuh"
#include "dense_tc.h"
#include "../../include/easyrag_b200.h"

namespace ezr {

constexpr int WQ = 128, WN = 256, WK = 64;    // the GEMM's tile: queries, corpus rows and dims of one k-chunk
// queries per block: the select launches one CTA row per query (grid.y <= 65535)
constexpr int W_MAX_BLOCK = 65535;

bool dense_wide_supported(const __nv_bfloat16* corpus, int64_t n_rows, int dim, int64_t ldc,
                          const __nv_bfloat16* queries, int64_t ldq) {
    if (dim <= 0 || dim % WK != 0) return false;
    if (ldc % 8 != 0 || ldq % 8 != 0) return false;
    if ((reinterpret_cast<uintptr_t>(corpus) & 15) || (reinterpret_cast<uintptr_t>(queries) & 15)) return false;
    return n_rows >= 1;
}

size_t dense_wide_workspace(int64_t n_rows, int n_queries, int k, int block_queries) {
    return score_rows_workspace(n_rows, n_queries, k, std::min(block_queries, W_MAX_BLOCK));
}

// The largest query block whose work fits ws_bytes (0: not even one query).
static int wide_block_queries(int64_t n_rows, int n_queries, int k, size_t ws_bytes) {
    const int64_t tiles_r = (n_rows + WN - 1) / WN;
    int64_t qb = (int64_t)(ws_bytes / ((size_t)n_rows * 4));
    qb = std::min(qb, (int64_t)std::min(n_queries, W_MAX_BLOCK));
    qb = std::min(qb, ((int64_t)INT32_MAX / tiles_r) * WQ);       // one CTA per tile: the grid stays below 2^31
    while (qb > 0 && dense_wide_workspace(n_rows, n_queries, k, (int)qb) > ws_bytes) --qb;
    return (int)qb;
}

static int wide_scores(const __nv_bfloat16* corpus, int64_t n_rows, int dim, int64_t ldc,
                       const __nv_bfloat16* queries, int nq, int64_t ldq, float* out, cudaStream_t st) {
    return gemm_scores_f32(queries, nq, dim, ldq, corpus, (int)n_rows, ldc, out, n_rows, EZR_PROF_DENSE_WIDE, st);
}

int dense_wide_topk(const __nv_bfloat16* corpus, int64_t n_rows, int dim, int64_t ldc, const __nv_bfloat16* queries,
                    int n_queries, int64_t ldq, int k, const int32_t* doc_group, const int32_t* q_group, int id_base,
                    float* out_scores, int32_t* out_ids, int32_t* out_counts, void* ws, size_t ws_bytes,
                    cudaStream_t st) {
    const int qb = ws ? wide_block_queries(n_rows, n_queries, k, ws_bytes) : 0;
    if (qb < 1) {
        set_error("dense_topk(wgmma-scores): workspace %zu < %zu (one query per block)", ws ? ws_bytes : (size_t)0,
                  dense_wide_workspace(n_rows, n_queries, k, 1));
        return EZR_ERR_WORKSPACE;
    }
    return score_rows_topk(wide_scores, qb, corpus, n_rows, dim, ldc, queries, n_queries, ldq, k, doc_group, q_group,
                           id_base, out_scores, out_ids, out_counts, ws, ws_bytes, st);
}

}  // namespace ezr

extern "C" size_t ezr_dense_wide_workspace(int64_t n_rows, int32_t n_queries, int32_t k, int32_t block_queries) {
    return ezr::dense_wide_workspace(n_rows, n_queries, k, block_queries);
}
