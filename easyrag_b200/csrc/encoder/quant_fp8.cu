// Row-wise e4m3 quantisation for the FP8 encoder path (gemm_fp8.cu), alone or fused into RMSNorm / LayerNorm.
//
// Every row gets one power-of-two scale s = 2^ceil(log2(amax / 448)) (448 is e4m3's largest finite value; an all-zero
// row gets s = 1), and q = e4m3_rn(x / s).  With amax = f 2^E, f in [0.5, 1): s = 2^(E - 9) if f <= 0.875 else
// 2^(E - 8), taken from the exponent bits, so no log2 rounding can pick a scale one octave too small.  x / s is exact
// in fp32 (a power-of-two rescaling of a bf16 value, applied as one or two exact multiplies), |x / s| <= 448, and
// the conversion (cvt.rn.satfinite.e4m3x2.f32) rounds to nearest-even without ever saturating; the result equals
// torch's (x.float() / s).to(torch.float8_e4m3fn) bit for bit.
//
// The fused norms run the row body of ops.cu's warp-per-row norm kernels (norm_row.cuh), so their bf16 row is that
// kernel's row bit for bit; they optionally store it and quantise it from registers: the GEMM that follows a norm
// reads e4m3 without a bf16 round trip through memory.
#include <cuda_fp8.h>
#include "norm_row.cuh"

namespace ezr {

// The row's scale exponent e (s = 2^e) and two factors whose product is 2^-e, each a normal fp32 power of two, so
// (x * m1) * m2 is exact: e ranges over [-141, 119] (bf16 amax from 2^-133 to below 2^128).
struct Pow2Scale {
    int e;
    float m1, m2;
};
__device__ __forceinline__ Pow2Scale pow2_scale(float amax) {
    Pow2Scale r;
    r.e = 0;
    if (amax > 0.f) {
        int E;
        const float f = frexpf(amax, &E);
        r.e = f <= 0.875f ? E - 9 : E - 8;
    }
    const int ne = -r.e;                                   // in [-119, 141]
    const int n1 = ne > 126 ? 126 : ne;
    r.m1 = __int_as_float((127 + n1) << 23);
    r.m2 = __int_as_float((127 + ne - n1) << 23);
    return r;
}

// 8 scaled values -> 8 e4m3 bytes (element 0 in the lowest byte)
__device__ __forceinline__ uint2 to_e4m3x8(const float (&v)[8], float m1, float m2) {
    uint32_t w[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const float2 f = make_float2(v[2 * i] * m1 * m2, v[2 * i + 1] * m1 * m2);
        w[i] = (uint32_t)__nv_cvt_float2_to_fp8x2(f, __NV_SATFINITE, __NV_E4M3);
    }
    return make_uint2(w[0] | (w[1] << 16), w[2] | (w[3] << 16));
}

// one warp per row, 8 rows per 256-thread CTA; two passes over the row (absmax, then quantise)
__global__ void __launch_bounds__(256)
quant_rows_fp8_kernel(const __nv_bfloat16* __restrict__ x, int64_t ldx, int rows, int cols, uint8_t* __restrict__ out,
                      int64_t ldo, float* __restrict__ scale) {
    const int lane = threadIdx.x & 31;
    const int r = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (r >= rows) return;
    const uint4* xr = reinterpret_cast<const uint4*>(x + (int64_t)r * ldx);
    uint2* orow = reinterpret_cast<uint2*>(out + (int64_t)r * ldo);
    const int n8 = cols >> 3;
    float amax = 0.f;
    for (int i = lane; i < n8; i += 32) {
        const uint4 u = __ldg(xr + i);
        const __nv_bfloat16* h = reinterpret_cast<const __nv_bfloat16*>(&u);
#pragma unroll
        for (int j = 0; j < 8; ++j) amax = fmaxf(amax, fabsf(__bfloat162float(h[j])));
    }
    const Pow2Scale s = pow2_scale(warp_max(amax));
    for (int i = lane; i < n8; i += 32) {
        const uint4 u = __ldg(xr + i);
        const __nv_bfloat16* h = reinterpret_cast<const __nv_bfloat16*>(&u);
        float v[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = __bfloat162float(h[j]);
        orow[i] = to_e4m3x8(v, s.m1, s.m2);
    }
    if (lane == 0) scale[r] = ldexpf(1.f, s.e);
}

// MODE 0: Qwen2RMSNorm, MODE 1: LayerNorm -- norm_warp_kernel's row (norm_row_warp), stored to out unless it is
// null, then quantised from registers with the absmax norm_row_warp returns.
template <int MODE, int MAXC>
__global__ void __launch_bounds__(256)
norm_fp8_kernel(const __nv_bfloat16* __restrict__ x, int64_t ldx, const __nv_bfloat16* __restrict__ gamma,
                const __nv_bfloat16* __restrict__ beta, float eps, int dim, __nv_bfloat16* __restrict__ out, int64_t ldo,
                uint8_t* __restrict__ out8, int64_t ldq, float* __restrict__ scale, int n_rows) {
    const int lane = threadIdx.x & 31;
    const int r = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (r >= n_rows) return;
    float v[MAXC][8];
    const float amax = norm_row_warp<MODE, MAXC>(x, ldx, gamma, beta, eps, dim, r, n_rows, out != nullptr, out, ldo, v);
    const int n_chunks = dim >> 3;
    const Pow2Scale sc = pow2_scale(warp_max(amax));
    uint2* qrow = reinterpret_cast<uint2*>(out8 + (int64_t)r * ldq);
#pragma unroll
    for (int c = 0; c < MAXC; ++c) {
        const int ci = lane + c * 32;
        if (ci < n_chunks) qrow[ci] = to_e4m3x8(v[c], sc.m1, sc.m2);
    }
    if (lane == 0) scale[r] = ldexpf(1.f, sc.e);
}

static int quant_rows_launch(const void* x, int64_t ldx, int32_t rows, int32_t cols, void* out, int64_t ldo,
                             float* scale, cudaStream_t st) {
    EZR_CHECK_ARG(rows >= 0 && cols >= 8 && cols % 8 == 0, "quant_fp8: need cols %% 8 == 0 (rows=%d cols=%d)", rows, cols);
    EZR_CHECK_ARG(ldx % 8 == 0 && ldo % 8 == 0 && ldx >= cols && ldo >= cols,
                  "quant_fp8: row strides must be multiples of 8 and >= cols");
    EZR_CHECK_ARG((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 7) == 0,
                  "quant_fp8: x must be 16-byte and out 8-byte aligned");
    EZR_CHECK_ARG(scale != nullptr, "quant_fp8: scale output is required");
    if (rows == 0) return EZR_OK;
    ProfScope prof(EZR_PROF_ENC_OTHER, st);
    quant_rows_fp8_kernel<<<(rows + 7) / 8, 256, 0, st>>>((const __nv_bfloat16*)x, ldx, rows, cols, (uint8_t*)out, ldo,
                                                          scale);
    EZR_LAUNCH_CHECK();
    return EZR_OK;
}

template <int MODE>
static int norm_fp8_launch(const void* x, int64_t ldx, const void* gamma, const void* beta, float eps, int32_t n_rows,
                           int32_t dim, void* out, int64_t ldo, void* out8, int64_t ldq, float* scale,
                           cudaStream_t st) {
    EZR_CHECK_ARG(dim >= 8 && dim % 8 == 0 && dim <= 4096, "norm_fp8: need dim %% 8 == 0 and dim <= 4096 (dim=%d)", dim);
    EZR_CHECK_ARG(ldx % 8 == 0 && ldq % 8 == 0 && ldx >= dim && ldq >= dim && (!out || (ldo % 8 == 0 && ldo >= dim)),
                  "norm_fp8: row strides must be multiples of 8 and >= dim");
    EZR_CHECK_ARG(((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(out) |
                    reinterpret_cast<uintptr_t>(gamma) | reinterpret_cast<uintptr_t>(beta)) & 15) == 0 &&
                      (reinterpret_cast<uintptr_t>(out8) & 7) == 0,
                  "norm_fp8: x, out, gamma and beta must be 16-byte aligned, out8 8-byte aligned");
    EZR_CHECK_ARG(gamma && out8 && scale && (MODE == 0 || beta), "norm_fp8: missing gamma / beta / out8 / scale");
    if (n_rows == 0) return EZR_OK;
    ProfScope prof(EZR_PROF_ENC_OTHER, st);
    const int grid = (n_rows + 7) / 8;
    if (dim <= 1024)
        norm_fp8_kernel<MODE, 4><<<grid, 256, 0, st>>>((const __nv_bfloat16*)x, ldx, (const __nv_bfloat16*)gamma,
                                                       (const __nv_bfloat16*)beta, eps, dim, (__nv_bfloat16*)out, ldo,
                                                       (uint8_t*)out8, ldq, scale, n_rows);
    else
        norm_fp8_kernel<MODE, 16><<<grid, 256, 0, st>>>((const __nv_bfloat16*)x, ldx, (const __nv_bfloat16*)gamma,
                                                        (const __nv_bfloat16*)beta, eps, dim, (__nv_bfloat16*)out, ldo,
                                                        (uint8_t*)out8, ldq, scale, n_rows);
    EZR_LAUNCH_CHECK();
    return EZR_OK;
}

}  // namespace ezr

using namespace ezr;

extern "C" {

int ezr_quant_rows_fp8(const void* x, int64_t ldx, int32_t rows, int32_t cols, void* out_e4m3, int64_t ldo,
                       float* out_scale, void* stream) {
    return quant_rows_launch(x, ldx, rows, cols, out_e4m3, ldo, out_scale, (cudaStream_t)stream);
}

int ezr_quant_weight_fp8(const void* w, int64_t ldw, int32_t n, int32_t k, void* out_e4m3, int64_t ldo,
                         float* out_scale, void* stream) {
    return quant_rows_launch(w, ldw, n, k, out_e4m3, ldo, out_scale, (cudaStream_t)stream);
}

int ezr_rmsnorm_fp8(const void* x, int64_t ldx, const void* gamma, float eps, int32_t n_rows, int32_t dim, void* out,
                    int64_t ldo, void* out_e4m3, int64_t ldq, float* out_scale, void* stream) {
    return norm_fp8_launch<0>(x, ldx, gamma, nullptr, eps, n_rows, dim, out, ldo, out_e4m3, ldq, out_scale,
                              (cudaStream_t)stream);
}

int ezr_layernorm_fp8(const void* x, int64_t ldx, const void* gamma, const void* beta, float eps, int32_t n_rows,
                      int32_t dim, void* out, int64_t ldo, void* out_e4m3, int64_t ldq, float* out_scale,
                      void* stream) {
    return norm_fp8_launch<1>(x, ldx, gamma, beta, eps, n_rows, dim, out, ldo, out_e4m3, ldq, out_scale,
                              (cudaStream_t)stream);
}

}  // extern "C"
