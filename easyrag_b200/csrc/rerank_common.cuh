// The cross-encoder head's per-query order, shared by csrc/rerank.cu (one coarse list per query) and
// csrc/rerank_fusion.cu (two coarse lists per query scored through their union).
#pragma once
#include "ezr_common.cuh"

namespace ezr {

constexpr int kCrossThreads = 256;
constexpr int kCrossMaxK = 1024;

// Query q's order, by the whole CTA, from its n scores in s_sc (n <= k): every score to out_all (-inf past n), the
// top_n by counting -- score descending, then coarse rank ascending -- to out_scores / out_ids (-inf / -1 padded).
__device__ __forceinline__ void cross_order_write(const float* s_sc, int q, int n, int k,
                                                  const int32_t* __restrict__ cand_ids, int k_stride, int top_n,
                                                  float* __restrict__ out_all, float* __restrict__ out_scores,
                                                  int32_t* __restrict__ out_ids, int32_t* __restrict__ out_counts) {
    for (int r = threadIdx.x; r < k; r += kCrossThreads) out_all[(int64_t)q * k + r] = r < n ? s_sc[r] : -INFINITY;
    for (int r = threadIdx.x; r < n; r += kCrossThreads) {
        const float sr = s_sc[r];
        int pos = 0;
        for (int j = 0; j < n; ++j) {
            const float sj = s_sc[j];
            pos += (sj > sr || (sj == sr && j < r)) ? 1 : 0;       // stable descending
        }
        if (pos < top_n) {
            out_scores[(int64_t)q * top_n + pos] = sr;
            out_ids[(int64_t)q * top_n + pos] = cand_ids[(int64_t)q * k_stride + r];
        }
    }
    const int c = min(n, top_n);
    for (int i = c + threadIdx.x; i < top_n; i += kCrossThreads) {
        out_scores[(int64_t)q * top_n + i] = -INFINITY;
        out_ids[(int64_t)q * top_n + i] = -1;
    }
    if (threadIdx.x == 0) out_counts[q] = c;
}

}  // namespace ezr
