// Merge of sorted per-shard top-k lists (k <= 1024), read in place from the all-gathered records of
// easyrag_b200/dist.py.
//
// Every part of a row is already in canonical order (ezr_common.cuh better(): score desc, id desc) up to its first
// id < 0, and ids are distinct across parts (disjoint shards).  So the output rank of an element is its index in its
// own list plus, for every other part, how many of that part's elements are better than it -- one binary search per
// other part.  An element whose rank is < k writes its output slot directly: no sort of the G*k candidates, no pack
// or transpose of the gathered buffer, O(G * k * G * log k) comparisons per row.
#include "ezr_common.cuh"
#include "../../include/easyrag_b200.h"

namespace ezr {

constexpr int kMergeThreads = 256;
constexpr int kMergeMaxK = 1024;          // k and n_cand
constexpr int kMergeMaxTotal = 8192;      // n_parts * n_cand

template <typename S>
static size_t merge_sorted_smem(int n_parts, int n_cand) {
    return (size_t)n_parts * n_cand * (sizeof(S) + 4) + (size_t)n_parts * 4;
}

// One CTA per row.  Shared memory: the row's n_parts lists (scores, then ids, part-major), then the per-part counts.
template <typename S>
__global__ void __launch_bounds__(kMergeThreads)
merge_sorted_kernel(const S* __restrict__ cs, const int32_t* __restrict__ cid, int n_cand, int64_t stride, int n_parts,
                    int64_t part_bytes, int k, S* __restrict__ out_s, int32_t* __restrict__ out_id,
                    int32_t* __restrict__ out_cnt, int64_t out_stride) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int total = n_parts * n_cand;
    S* s_s = reinterpret_cast<S*>(smem_raw);
    int32_t* s_id = reinterpret_cast<int32_t*>(s_s + total);
    int32_t* s_cnt = s_id + total;
    __shared__ int s_valid;
    const int row = blockIdx.x;
    if (threadIdx.x == 0) s_valid = 0;
    for (int e = threadIdx.x; e < total; e += blockDim.x) {
        const int p = e / n_cand, j = e - p * n_cand;
        const int64_t off = p * part_bytes;
        const int64_t at = (int64_t)row * stride + j;
        s_id[e] = reinterpret_cast<const int32_t*>(reinterpret_cast<const char*>(cid) + off)[at];
        s_s[e] = reinterpret_cast<const S*>(reinterpret_cast<const char*>(cs) + off)[at];
    }
    __syncthreads();
    // a part's count: its first slot with id < 0 (ids >= 0 form a prefix)
    for (int p = threadIdx.x; p < n_parts; p += blockDim.x) {
        const int32_t* ids = s_id + p * n_cand;
        int lo = 0, hi = n_cand;
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if (ids[mid] >= 0) lo = mid + 1; else hi = mid;
        }
        s_cnt[p] = lo;
        atomicAdd(&s_valid, lo);
    }
    __syncthreads();
    const int64_t o = (int64_t)row * out_stride;
    for (int e = threadIdx.x; e < total; e += blockDim.x) {
        const int p = e / n_cand, j = e - p * n_cand;
        if (j >= s_cnt[p] || j >= k) continue;               // rank >= j: past k already
        const S x = s_s[e];
        const int xi = s_id[e];
        int rank = j;
        for (int q = 0; q < n_parts && rank < k; ++q) {
            if (q == p) continue;
            const S* qs = s_s + q * n_cand;
            const int32_t* qi = s_id + q * n_cand;
            int lo = 0, hi = s_cnt[q];                        // elements of q better than x form a prefix
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                if (better<S>(qs[mid], qi[mid], x, xi)) lo = mid + 1; else hi = mid;
            }
            rank += lo;
        }
        if (rank < k) {
            out_s[o + rank] = x;
            out_id[o + rank] = xi;
        }
    }
    const int count = min(s_valid, k);
    for (int64_t i = count + threadIdx.x; i < out_stride; i += blockDim.x) {
        out_s[o + i] = ScoreTraits<S>::lowest();
        out_id[o + i] = -1;
    }
    if (threadIdx.x == 0) out_cnt[row] = count;
}

template <typename S>
static int merge_sorted_impl(const S* cs, const int32_t* cid, int n_rows, int n_cand, int64_t stride, int n_parts,
                             int64_t part_bytes, int k, S* out_s, int32_t* out_id, int32_t* out_cnt,
                             int64_t out_stride, cudaStream_t st) {
    if (n_rows == 0) return EZR_OK;
    const size_t smem = merge_sorted_smem<S>(n_parts, n_cand);
    static bool attr_done = false;
    if (!attr_done) {
        EZR_CUDA(cudaFuncSetAttribute(merge_sorted_kernel<S>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      (int)merge_sorted_smem<S>(kMergeMaxTotal, 1)));
        attr_done = true;
    }
    ProfScope prof(EZR_PROF_MERGE, st);
    merge_sorted_kernel<S><<<n_rows, kMergeThreads, smem, st>>>(cs, cid, n_cand, stride, n_parts, part_bytes, k, out_s,
                                                                out_id, out_cnt, out_stride);
    EZR_LAUNCH_CHECK();
    return EZR_OK;
}

}  // namespace ezr

using namespace ezr;

extern "C" {

int ezr_merge_sorted_parts(const void* cand_scores, const int32_t* cand_ids, int32_t score_type, int32_t n_rows,
                           int32_t n_cand, int64_t cand_stride, int32_t n_parts, int64_t part_stride_bytes, int32_t k,
                           void* out_scores, int32_t* out_ids, int32_t* out_counts, int64_t out_stride, void* stream) {
    EZR_CHECK_ARG(k >= 1 && k <= kMergeMaxK, "merge_sorted_parts: k=%d out of [1,%d]", k, kMergeMaxK);
    EZR_CHECK_ARG(score_type == EZR_F64 || score_type == EZR_F32, "merge_sorted_parts: bad score_type");
    EZR_CHECK_ARG(n_rows >= 0, "merge_sorted_parts: n_rows=%d < 0", n_rows);
    EZR_CHECK_ARG(n_cand >= 0 && n_cand <= kMergeMaxK && cand_stride >= n_cand,
                  "merge_sorted_parts: n_cand=%d / cand_stride=%lld (n_cand in [0,%d], stride >= n_cand)", n_cand,
                  (long long)cand_stride, kMergeMaxK);
    EZR_CHECK_ARG(n_parts >= 1 && part_stride_bytes >= 0 && part_stride_bytes % 8 == 0,
                  "merge_sorted_parts: bad n_parts/part_stride_bytes (%d, %lld)", n_parts, (long long)part_stride_bytes);
    EZR_CHECK_ARG((int64_t)n_parts * n_cand <= kMergeMaxTotal, "merge_sorted_parts: n_parts * n_cand = %lld > %d",
                  (long long)n_parts * n_cand, kMergeMaxTotal);
    EZR_CHECK_ARG(out_stride >= k, "merge_sorted_parts: out_stride=%lld < k=%d", (long long)out_stride, k);
    EZR_CHECK_ARG(n_rows == 0 || (out_scores && out_ids && out_counts && (n_cand == 0 || (cand_scores && cand_ids))),
                  "merge_sorted_parts: NULL pointer");
    cudaStream_t st = (cudaStream_t)stream;
    return score_type == EZR_F64
               ? merge_sorted_impl<double>((const double*)cand_scores, cand_ids, n_rows, n_cand, cand_stride, n_parts,
                                           part_stride_bytes, k, (double*)out_scores, out_ids, out_counts, out_stride,
                                           st)
               : merge_sorted_impl<float>((const float*)cand_scores, cand_ids, n_rows, n_cand, cand_stride, n_parts,
                                          part_stride_bytes, k, (float*)out_scores, out_ids, out_counts, out_stride,
                                          st);
}

}  // extern "C"
