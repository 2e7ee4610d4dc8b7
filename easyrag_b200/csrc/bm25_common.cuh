// Device pieces shared by the BM25 index build (bm25_build.cu, bm25.cu) and the per-context BM25-Extract kernel
// (bm25_extract.cu): the shared-memory key sort and the round-to-nearest, FMA-free arithmetic of rank_bm25's
// denominator and per-posting contribution (operation order: oracle/bm25.py, OkapiCSR docstring).
#pragma once
#include <cuda_runtime.h>

namespace ezr {

// ascending sort of n_pow2 64-bit keys in shared (or global) memory by the whole CTA; ends on a barrier
__device__ __forceinline__ void bitonic_sort_u64(unsigned long long* key, int n_pow2, int tid, int nthreads) {
    for (int k = 2; k <= n_pow2; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = tid; i < n_pow2; i += nthreads) {
                const int ixj = i ^ j;
                if (ixj > i) {
                    const unsigned long long a = key[i], b = key[ixj];
                    const bool up = (i & k) == 0;
                    if ((a > b) == up) { key[i] = b; key[ixj] = a; }
                }
            }
            __syncthreads();
        }
    }
}

// K_d = k1 * (one_minus_b + (b*dl) / avgdl)
__device__ __forceinline__ double bm25_doc_norm(double dl, double k1, double b, double one_minus_b, double avgdl) {
    const double t1 = __dmul_rn(b, dl);
    const double t2 = __ddiv_rn(t1, avgdl);
    const double t3 = __dadd_rn(one_minus_b, t2);
    return __dmul_rn(k1, t3);
}

// idf * ((tf*num_scale) / (tf + K_d)); num_scale = k1+1 (rank_bm25) or 1 (bm25s, which stores the float32 of it)
__device__ __forceinline__ double bm25_contribution(double idf, double tf, double kd, double num_scale) {
    const double num = __dmul_rn(tf, num_scale);
    const double den = __dadd_rn(tf, kd);
    const double r = __ddiv_rn(num, den);
    return __dmul_rn(idf, r);
}

}  // namespace ezr
