// wgmma dense cosine top-k (dense_tc.cu): host-side entry points.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stddef.h>

namespace ezr {

bool dense_tc_supported(const __nv_bfloat16* corpus, int64_t n_rows, int dim, int64_t ldc, const __nv_bfloat16* queries,
                        int n_queries, int64_t ldq, int k);
size_t dense_tc_workspace(int64_t n_rows, int dim, int n_queries, int k);
int dense_tc_topk(const __nv_bfloat16* corpus, int64_t n_rows, int dim, int64_t ldc, const __nv_bfloat16* queries,
                  int n_queries, int64_t ldq, int k, const int32_t* doc_group, const int32_t* q_group, int id_base,
                  float* out_scores, int32_t* out_ids, int32_t* out_counts, void* ws, size_t ws_bytes,
                  cudaStream_t st, int form);   // form 0: 128-query blocks (dim <= 768), 1: 64-query blocks,
                                                // 2: 64-query blocks and 128-row corpus tiles, 3: 2 in cluster pairs
const char* dense_tc_form_name(int form);
int dense_tc_max_qw(int dim);   // 2 while the 128-query block fits shared memory beside the ring (dim <= 768), else 1
// corpus splits of the persistent work units (cost model in dense_tc.cu) and the rows of one split
int ts_choose_splits(int qblocks, int64_t n_rows, int dim, int sms, int tn);
int tc_rows_per_slice(int64_t n_rows, int slices, int tn);

// Score rows + ezr_select_rows (dense.cu): the loop of form 1 / the SIMT fallback, dense_exact_topk and form 6.  For
// each block of block_queries queries, `score` writes the block's fp32 score rows out[q][r] = queries[q] . corpus[r]
// (row stride n_rows) at the front of the workspace, and the select's workspace follows the block's own rows.
// score_rows_workspace = the bytes for blocks of block_queries: the larger of a full block and the smaller last one.
typedef int (*score_rows_fn)(const __nv_bfloat16* corpus, int64_t n_rows, int dim, int64_t ldc,
                             const __nv_bfloat16* queries, int nq, int64_t ldq, float* out, cudaStream_t st);
size_t score_rows_workspace(int64_t n_rows, int n_queries, int k, int block_queries);
int score_rows_topk(score_rows_fn score, int block_queries, const __nv_bfloat16* corpus, int64_t n_rows, int dim,
                    int64_t ldc, const __nv_bfloat16* queries, int n_queries, int64_t ldq, int k,
                    const int32_t* doc_group, const int32_t* q_group, int id_base, float* out_scores, int32_t* out_ids,
                    int32_t* out_counts, void* ws, size_t ws_bytes, cudaStream_t st);

// Full scan with the rescore arithmetic of dense_s8.cu (fp32, increasing coordinate order, no FMA contraction):
// score rows + ezr_select_rows (dense.cu).
size_t dense_exact_workspace(int64_t n_rows, int n_queries, int k);
int dense_exact_topk(const __nv_bfloat16* corpus, int64_t n_rows, int dim, int64_t ldc, const __nv_bfloat16* queries,
                     int n_queries, int64_t ldq, int k, const int32_t* doc_group, const int32_t* q_group, int id_base,
                     float* out_scores, int32_t* out_ids, int32_t* out_counts, void* ws, size_t ws_bytes,
                     cudaStream_t st);

// Form 6 (dense_wide.cu): wgmma score rows for any dim % 64 == 0, then ezr_select_rows (k <= 1024).  The query block is
// the largest whose rows and select workspace fit ws_bytes; dense_wide_workspace = the bytes for blocks of
// block_queries queries.  The score rows come from the encoder's bf16 GEMM kernel (encoder/gemm_tc.cu):
// out[m][n] = A[m] . W[n] in fp32 (-0.0 stored as +0.0), M tiles fastest, timed in profiling slot prof_slot.
bool dense_wide_supported(const __nv_bfloat16* corpus, int64_t n_rows, int dim, int64_t ldc,
                          const __nv_bfloat16* queries, int64_t ldq);
size_t dense_wide_workspace(int64_t n_rows, int n_queries, int k, int block_queries);
int dense_wide_topk(const __nv_bfloat16* corpus, int64_t n_rows, int dim, int64_t ldc, const __nv_bfloat16* queries,
                    int n_queries, int64_t ldq, int k, const int32_t* doc_group, const int32_t* q_group, int id_base,
                    float* out_scores, int32_t* out_ids, int32_t* out_counts, void* ws, size_t ws_bytes,
                    cudaStream_t st);
int gemm_scores_f32(const __nv_bfloat16* A, int M, int K, int64_t lda, const __nv_bfloat16* W, int N, int64_t ldw,
                    float* out, int64_t ldo, int prof_slot, cudaStream_t st);

extern int g_dense_probe;       // see ezr_dense_set_probe
extern int g_dense_stage_cap;   // see ezr_dense_set_stage_cap

}  // namespace ezr
