// Cross-encoder head + per-query re-ordering (SentenceTransformerRerank._postprocess_nodes, rerankers.py:57-99).
//
// The head of BertForSequenceClassification / (XLM)RobertaForSequenceClassification with num_labels == 1 is
//     CLS row -> Linear(d, d) + bias -> tanh -> Linear(d, 1) + bias -> sigmoid      (CrossEncoder.predict)
// The CLS gather and the first Linear run as ezr_pool_normalize + ezr_gemm_bf16; this file is the rest, one CTA per
// query: tanh, the d-wide dot with the output row, bias and sigmoid in fp32 for each of the query's pairs, then the
// order of sorted(nodes, key=lambda x: -x.score if x.score else 0): score descending, ties in coarse-rank order
// (a sigmoid is never negative, so a score of exactly 0 simply sorts last).  The order is taken on the fp32 sigmoid,
// not on the logit: a trained reranker saturates many candidates to 1.0f, and the reference keeps their coarse order.
// The same head also runs in two launches (ezr_cross_pair_scores, then ezr_cross_order_topk) with a [P] fp32 score
// vector between them; both forms share the per-pair and per-query device functions, so their outputs are identical.
#include "ezr_common.cuh"
#include "rerank_common.cuh"
#include "../../include/easyrag_b200.h"

namespace ezr {

__device__ __forceinline__ float cross_warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// sigmoid(tanh(row) . w_out + b_out) of one pair, computed by one whole warp (every lane returns it).  The lane-strided
// partial sums and the shuffle tree fix the summation order, so every path that scores a pair gets the same bits.
__device__ __forceinline__ float cross_pair_sigmoid(const __nv_bfloat16* __restrict__ row,
                                                    const float* __restrict__ w_out, float b_out, int dim, int lane) {
    float acc = 0.f;
    for (int i = lane; i < dim; i += 32) acc = fmaf(tanhf(__bfloat162float(row[i])), w_out[i], acc);
    acc = cross_warp_sum(acc);
    return 1.f / (1.f + expf(-(acc + b_out)));
}

__global__ void __launch_bounds__(kCrossThreads)
cross_score_topk_kernel(const __nv_bfloat16* __restrict__ dense, int64_t ldd, const int32_t* __restrict__ pair_off,
                        int k, const int32_t* __restrict__ cand_ids, int k_stride, const float* __restrict__ w_out,
                        float b_out, int dim, int top_n, float* __restrict__ out_all, float* __restrict__ out_scores,
                        int32_t* __restrict__ out_ids, int32_t* __restrict__ out_counts) {
    __shared__ float s_sc[kCrossMaxK];
    const int q = blockIdx.x;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int p0 = pair_off[q];
    const int n = min(pair_off[q + 1] - p0, k);
    for (int r = warp; r < n; r += kCrossThreads / 32) {
        const float s = cross_pair_sigmoid(dense + (int64_t)(p0 + r) * ldd, w_out, b_out, dim, lane);
        if (lane == 0) s_sc[r] = s;
    }
    __syncthreads();
    cross_order_write(s_sc, q, n, k, cand_ids, k_stride, top_n, out_all, out_scores, out_ids, out_counts);
}

// The two halves of cross_score_topk_kernel, for callers that score the pairs in one place and order them in another
// (several GPUs each scoring a run of the pairs, then exchanging 4 bytes per pair).  One warp per pair:
__global__ void __launch_bounds__(kCrossThreads)
cross_pair_scores_kernel(const __nv_bfloat16* __restrict__ dense, int dim, int n_pairs,
                         const float* __restrict__ w_out, float b_out, float* __restrict__ out_sig) {
    const int lane = threadIdx.x & 31;
    const int p = blockIdx.x * (kCrossThreads / 32) + (threadIdx.x >> 5);
    if (p >= n_pairs) return;
    const float s = cross_pair_sigmoid(dense + (int64_t)p * dim, w_out, b_out, dim, lane);
    if (lane == 0) out_sig[p] = s;
}

// ... and one CTA per query over the scores of all pairs.
__global__ void __launch_bounds__(kCrossThreads)
cross_order_topk_kernel(const float* __restrict__ sig, const int32_t* __restrict__ pair_off, int k,
                        const int32_t* __restrict__ cand_ids, int k_stride, int top_n, float* __restrict__ out_all,
                        float* __restrict__ out_scores, int32_t* __restrict__ out_ids,
                        int32_t* __restrict__ out_counts) {
    __shared__ float s_sc[kCrossMaxK];
    const int q = blockIdx.x;
    const int p0 = pair_off[q];
    const int n = min(pair_off[q + 1] - p0, k);
    for (int r = threadIdx.x; r < n; r += kCrossThreads) s_sc[r] = sig[p0 + r];
    __syncthreads();
    cross_order_write(s_sc, q, n, k, cand_ids, k_stride, top_n, out_all, out_scores, out_ids, out_counts);
}

}  // namespace ezr

using namespace ezr;

extern "C" {

int ezr_cross_score_topk(const void* dense, int64_t ldd, const int32_t* pair_off, int32_t n_queries, int32_t k,
                         const int32_t* cand_ids, int32_t k_stride, const float* w_out, float b_out, int32_t dim,
                         int32_t top_n, float* out_all, float* out_scores, int32_t* out_ids, int32_t* out_counts,
                         void* stream) {
    EZR_CHECK_ARG(n_queries >= 0 && k >= 1 && k <= kCrossMaxK && k_stride >= k,
                  "cross_score_topk: k=%d out of [1, %d] (or k_stride < k)", k, kCrossMaxK);
    EZR_CHECK_ARG(dim >= 1 && top_n >= 1, "cross_score_topk: dim and top_n must be >= 1");
    EZR_CHECK_ARG(pair_off && cand_ids && w_out && out_all && out_scores && out_ids && out_counts,
                  "cross_score_topk: NULL argument");
    if (n_queries == 0) return EZR_OK;
    cross_score_topk_kernel<<<n_queries, kCrossThreads, 0, (cudaStream_t)stream>>>(
        (const __nv_bfloat16*)dense, ldd, pair_off, k, cand_ids, k_stride, w_out, b_out, dim, top_n, out_all,
        out_scores, out_ids, out_counts);
    EZR_LAUNCH_CHECK();
    return EZR_OK;
}

int ezr_cross_pair_scores(const void* dense, int32_t dim, int32_t n_pairs, const float* w_out, float b_out,
                          float* out_sig, void* stream) {
    EZR_CHECK_ARG(dim >= 1 && n_pairs >= 0, "cross_pair_scores: dim=%d must be >= 1 and n_pairs=%d >= 0", dim,
                  n_pairs);
    if (n_pairs == 0) return EZR_OK;
    EZR_CHECK_ARG(dense && w_out && out_sig, "cross_pair_scores: NULL argument");
    cross_pair_scores_kernel<<<ceil_div(n_pairs, kCrossThreads / 32), kCrossThreads, 0, (cudaStream_t)stream>>>(
        (const __nv_bfloat16*)dense, dim, n_pairs, w_out, b_out, out_sig);
    EZR_LAUNCH_CHECK();
    return EZR_OK;
}

int ezr_cross_order_topk(const float* sig, const int32_t* pair_off, int32_t n_queries, int32_t k,
                         const int32_t* cand_ids, int32_t k_stride, int32_t top_n, float* out_all, float* out_scores,
                         int32_t* out_ids, int32_t* out_counts, void* stream) {
    EZR_CHECK_ARG(n_queries >= 0 && k >= 1 && k <= kCrossMaxK && k_stride >= k,
                  "cross_order_topk: k=%d out of [1, %d] (or k_stride < k)", k, kCrossMaxK);
    EZR_CHECK_ARG(top_n >= 1, "cross_order_topk: top_n must be >= 1");
    EZR_CHECK_ARG(pair_off && cand_ids && out_all && out_scores && out_ids && out_counts,
                  "cross_order_topk: NULL argument");
    if (n_queries == 0) return EZR_OK;
    cross_order_topk_kernel<<<n_queries, kCrossThreads, 0, (cudaStream_t)stream>>>(
        sig, pair_off, k, cand_ids, k_stride, top_n, out_all, out_scores, out_ids, out_counts);
    EZR_LAUNCH_CHECK();
    return EZR_OK;
}

}  // extern "C"
