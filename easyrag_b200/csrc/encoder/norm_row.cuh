// Warp reductions and the row body of the warp-per-row RMSNorm / LayerNorm kernels: norm_warp_kernel (ops.cu) and
// norm_fp8_kernel (quant_fp8.cu) both run norm_row_warp, so the bf16 row the e4m3 norms quantise is the bf16 norms'
// row bit for bit.
#pragma once
#include "../ezr_common.cuh"

namespace ezr {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// One warp normalises row r of x (dim % 8 == 0, dim <= 256 * MAXC); nothing is done when r >= n_rows.
// MODE 0: Qwen2RMSNorm (gamma), MODE 1: LayerNorm (gamma, beta).  The row lives in registers: the lane owns the
// 16-byte chunks lane + 32 c, c < MAXC, held in v[c]; statistics by warp shuffles only; same rounding points as
// norm_kernel.  On return v[c] holds the lane's chunks of the bf16 result (as floats), which are also stored to row r
// of out when `store` is set; the return value is their largest magnitude (the e4m3 norms' absmax; the bf16 kernel
// ignores it and nvcc drops its computation).
template <int MODE, int MAXC>
__device__ __forceinline__ float norm_row_warp(const __nv_bfloat16* __restrict__ x, int64_t ldx,
                                              const __nv_bfloat16* __restrict__ gamma,
                                              const __nv_bfloat16* __restrict__ beta, float eps, int dim, int r,
                                              int n_rows, bool store, __nv_bfloat16* __restrict__ out, int64_t ldo,
                                              float (&v)[MAXC][8]) {
    const int lane = threadIdx.x & 31;
    if (r >= n_rows) return 0.f;
    const int n_chunks = dim >> 3;
    const uint4* xr = reinterpret_cast<const uint4*>(x + (int64_t)r * ldx);
    float s = 0.f, q = 0.f;
#pragma unroll
    for (int c = 0; c < MAXC; ++c) {
        const int ci = lane + c * 32;
        if (ci < n_chunks) {
            const uint4 u = __ldg(xr + ci);
            const __nv_bfloat16* h = reinterpret_cast<const __nv_bfloat16*>(&u);
#pragma unroll
            for (int j = 0; j < 8; ++j) { v[c][j] = __bfloat162float(h[j]); s += v[c][j]; q += v[c][j] * v[c][j]; }
        }
    }
    float mean = 0.f, rstd;
    if (MODE == 0) {
        rstd = rsqrtf(warp_sum(q) / dim + eps);
    } else {
        mean = warp_sum(s) / dim;
        float q2 = 0.f;
#pragma unroll
        for (int c = 0; c < MAXC; ++c) {
            if (lane + c * 32 < n_chunks) {
#pragma unroll
                for (int j = 0; j < 8; ++j) { const float d = v[c][j] - mean; q2 += d * d; }
            }
        }
        rstd = rsqrtf(warp_sum(q2) / dim + eps);
    }
    float amax = 0.f;
#pragma unroll
    for (int c = 0; c < MAXC; ++c) {
        const int ci = lane + c * 32;
        if (ci < n_chunks) {
            const uint4 g4 = __ldg(reinterpret_cast<const uint4*>(gamma) + ci);
            const __nv_bfloat16* gh = reinterpret_cast<const __nv_bfloat16*>(&g4);
            uint4 b4 = make_uint4(0u, 0u, 0u, 0u);
            if (MODE == 1) b4 = __ldg(reinterpret_cast<const uint4*>(beta) + ci);
            const __nv_bfloat16* bh = reinterpret_cast<const __nv_bfloat16*>(&b4);
            uint4 o4;
            __nv_bfloat16* oh = reinterpret_cast<__nv_bfloat16*>(&o4);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                if (MODE == 0) {
                    const float y = __bfloat162float(__float2bfloat16(v[c][j] * rstd));      // .to(input_dtype)
                    oh[j] = __float2bfloat16(__bfloat162float(gh[j]) * y);
                } else {
                    oh[j] = __float2bfloat16((v[c][j] - mean) * rstd * __bfloat162float(gh[j]) + __bfloat162float(bh[j]));
                }
                v[c][j] = __bfloat162float(oh[j]);
                amax = fmaxf(amax, fabsf(v[c][j]));
            }
            if (store) reinterpret_cast<uint4*>(out + (int64_t)r * ldo)[ci] = o4;
        }
    }
    return amax;
}

}  // namespace ezr
