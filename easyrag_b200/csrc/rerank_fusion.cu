// Rerank fusion (generation_with_rerank_fusion, pipeline.py:393-452): the dense and the sparse coarse list of a query
// are reranked separately and the two reranked lists fused with reciprocal_rank_fusion.  A document in both lists
// makes the same (query, passage) pair twice, and a pair's score does not depend on the encoder pass it is in, so the
// pairs of both lists are encoded once, as their union, and each list is ordered from the union's scores:
//   pair_union:         one CTA per query: the distinct ids of list a then list b, and each list slot's union index.
//   order_topk_mapped:  one CTA per query: ezr_cross_order_topk on one list, reading its scores through that map.
#include "ezr_common.cuh"
#include "bm25_common.cuh"
#include "rerank_common.cuh"
#include "../../include/easyrag_b200.h"

namespace ezr {

constexpr int kUnionThreads = kCrossMaxK;      // one thread per slot of the two lists
static_assert(kUnionThreads % 32 == 0 && kUnionThreads <= 1024, "one CTA holds every slot");

// Slots s < na are list a's [0, na), slots na + r are list b's r.  The (id, slot) keys are sorted in shared memory, so
// equal ids sit together with the smallest slot -- the first appearance in slot order -- first.  A slot is a union
// entry iff it is that first appearance; the union index of an entry is the number of entries before it in slot
// order (a ballot scan), which makes the union order "a's new ids, then b's new ids", independent of scheduling.
// Every slot then takes the union index of its id's first appearance.  Finding a run's start walks back over the
// equal keys: at most one step when each list holds distinct ids, quadratic in the run length otherwise.
__global__ void __launch_bounds__(kUnionThreads)
pair_union_kernel(const int32_t* __restrict__ ids_a, const int32_t* __restrict__ cnt_a, int k_a, int stride_a,
                  const int32_t* __restrict__ ids_b, const int32_t* __restrict__ cnt_b, int k_b, int stride_b,
                  int32_t* __restrict__ out_ids, int32_t* __restrict__ out_counts, int32_t* __restrict__ out_map_a,
                  int32_t* __restrict__ out_map_b) {
    __shared__ unsigned long long s_key[kUnionThreads];
    __shared__ int s_first[kUnionThreads];     // slot -> slot of its id's first appearance
    __shared__ int s_index[kUnionThreads];     // entry slot -> union index
    __shared__ int s_warp[kUnionThreads / 32];
    const int q = blockIdx.x, t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const int na = min(max(cnt_a[q], 0), k_a), nb = min(max(cnt_b[q], 0), k_b);
    const int n = na + nb, k_u = k_a + k_b;
    int n_pow2 = 1;
    while (n_pow2 < n) n_pow2 <<= 1;
    int32_t id = -1;
    if (t < n) id = t < na ? ids_a[(int64_t)q * stride_a + t] : ids_b[(int64_t)q * stride_b + (t - na)];
    if (t < n_pow2) s_key[t] = t < n ? ((unsigned long long)(uint32_t)id << 32) | (uint32_t)t : ~0ull;
    __syncthreads();
    bitonic_sort_u64(s_key, n_pow2, t, kUnionThreads);
    if (t < n) {
        const unsigned long long key = s_key[t];
        int h = t;
        while (h > 0 && (s_key[h - 1] >> 32) == (key >> 32)) --h;
        s_first[(uint32_t)key] = (int)(uint32_t)s_key[h];
    }
    __syncthreads();
    const bool entry = t < n && s_first[t] == t;
    const unsigned m = __ballot_sync(0xffffffffu, entry);
    if (lane == 0) s_warp[warp] = __popc(m);
    __syncthreads();
    int base = 0, total = 0;
    for (int w = 0; w < kUnionThreads / 32; ++w) {
        const int c = s_warp[w];
        base += w < warp ? c : 0;
        total += c;
    }
    const int u = base + __popc(m & ((1u << lane) - 1u));
    if (entry) {
        s_index[t] = u;
        out_ids[(int64_t)q * k_u + u] = id;
    }
    __syncthreads();
    if (t < na) out_map_a[(int64_t)q * k_a + t] = s_index[s_first[t]];
    else if (t < n) out_map_b[(int64_t)q * k_b + (t - na)] = s_index[s_first[t]];
    for (int j = total + t; j < k_u; j += kUnionThreads) out_ids[(int64_t)q * k_u + j] = -1;
    for (int r = na + t; r < k_a; r += kUnionThreads) out_map_a[(int64_t)q * k_a + r] = -1;
    for (int r = nb + t; r < k_b; r += kUnionThreads) out_map_b[(int64_t)q * k_b + r] = -1;
    if (t == 0) out_counts[q] = total;
}

// cross_order_topk_kernel for one list whose pairs are packed as the union's: list slot r is pair
// pair_off[q] + slot_map[q, r].  The list's count is the length of the map's leading run of entries inside the query's
// pairs (pair_union_kernel writes -1 past the count), so the order, its ties and the padding are those of
// ezr_cross_order_topk on the list alone.
__global__ void __launch_bounds__(kCrossThreads)
cross_order_topk_mapped_kernel(const float* __restrict__ sig, const int32_t* __restrict__ pair_off, int k,
                               const int32_t* __restrict__ slot_map, int map_stride,
                               const int32_t* __restrict__ cand_ids, int k_stride, int top_n,
                               float* __restrict__ out_all, float* __restrict__ out_scores,
                               int32_t* __restrict__ out_ids, int32_t* __restrict__ out_counts) {
    __shared__ float s_sc[kCrossMaxK];
    __shared__ int s_n;
    const int q = blockIdx.x;
    const int p0 = pair_off[q];
    const int n_u = pair_off[q + 1] - p0;
    if (threadIdx.x == 0) s_n = k;
    __syncthreads();
    for (int r = threadIdx.x; r < k; r += kCrossThreads) {
        const int u = slot_map[(int64_t)q * map_stride + r];
        if (u >= 0 && u < n_u) s_sc[r] = sig[p0 + u];
        else atomicMin(&s_n, r);
    }
    __syncthreads();
    cross_order_write(s_sc, q, s_n, k, cand_ids, k_stride, top_n, out_all, out_scores, out_ids, out_counts);
}

}  // namespace ezr

using namespace ezr;

extern "C" {

int ezr_pair_union(const int32_t* ids_a, const int32_t* cnt_a, int32_t k_a, int32_t stride_a, const int32_t* ids_b,
                   const int32_t* cnt_b, int32_t k_b, int32_t stride_b, int32_t n_queries, int32_t* out_ids,
                   int32_t* out_counts, int32_t* out_map_a, int32_t* out_map_b, void* stream) {
    EZR_CHECK_ARG(n_queries >= 0 && k_a >= 1 && k_b >= 1 && stride_a >= k_a && stride_b >= k_b,
                  "pair_union: k_a=%d / k_b=%d must be >= 1 (and each stride >= its k)", k_a, k_b);
    EZR_CHECK_ARG(k_a + k_b <= kCrossMaxK, "pair_union: k_a + k_b = %d exceeds %d", k_a + k_b, kCrossMaxK);
    EZR_CHECK_ARG(ids_a && cnt_a && ids_b && cnt_b && out_ids && out_counts && out_map_a && out_map_b,
                  "pair_union: NULL argument");
    if (n_queries == 0) return EZR_OK;
    pair_union_kernel<<<n_queries, kUnionThreads, 0, (cudaStream_t)stream>>>(
        ids_a, cnt_a, k_a, stride_a, ids_b, cnt_b, k_b, stride_b, out_ids, out_counts, out_map_a, out_map_b);
    EZR_LAUNCH_CHECK();
    return EZR_OK;
}

int ezr_cross_order_topk_mapped(const float* sig, const int32_t* pair_off, int32_t n_queries, int32_t k,
                                const int32_t* slot_map, int32_t map_stride, const int32_t* cand_ids, int32_t k_stride,
                                int32_t top_n, float* out_all, float* out_scores, int32_t* out_ids,
                                int32_t* out_counts, void* stream) {
    EZR_CHECK_ARG(n_queries >= 0 && k >= 1 && k <= kCrossMaxK && k_stride >= k && map_stride >= k,
                  "cross_order_topk_mapped: k=%d out of [1, %d] (or k_stride / map_stride < k)", k, kCrossMaxK);
    EZR_CHECK_ARG(top_n >= 1, "cross_order_topk_mapped: top_n must be >= 1");
    EZR_CHECK_ARG(pair_off && slot_map && cand_ids && out_all && out_scores && out_ids && out_counts,
                  "cross_order_topk_mapped: NULL argument");
    if (n_queries == 0) return EZR_OK;
    cross_order_topk_mapped_kernel<<<n_queries, kCrossThreads, 0, (cudaStream_t)stream>>>(
        sig, pair_off, k, slot_map, map_stride, cand_ids, k_stride, top_n, out_all, out_scores, out_ids, out_counts);
    EZR_LAUNCH_CHECK();
    return EZR_OK;
}

}  // extern "C"
