// Epilogue shared by the encoder GEMMs (gemm_tc.cu: bf16 wgmma, gemm_fp8.cu: e4m3 wgmma).  Both kernels hand it one
// pair of adjacent output columns of one row, in fp32, after their own accumulation; it adds the bias, applies GELU or
// SwiGLU, adds the residual and stores bf16.  EPI_SCORES (gemm_tc.cu only) stores the fp32 dot products themselves:
// the score rows of dense top-k form 6 (dense_wide.cu).
#pragma once
#include <cuda_bf16.h>
#include <stdint.h>

namespace ezr {

enum { EPI_NONE = 0, EPI_GELU = 1, EPI_SWIGLU = 2, EPI_SCORES = 3 };

// erf GELU (HF "gelu"): gelu(x) = 0.5 x (1 + erf(x / sqrt 2)).  erfc(|z|) = t (a1 + t (a2 + t (a3 + t (a4 + t a5)))) exp(-z^2),
// t = 1 / (1 + p |z|) (Abramowitz & Stegun 7.1.26, |error| <= 1.5e-7), evaluated through erfc on BOTH sides so the
// negative tail keeps its relative accuracy: x <= 0: 0.5 x erfc(|z|);  x > 0: x - 0.5 x erfc(z).  Against the float64
// definition the fp32 evaluation is within 4.7e-7 absolute over [-12, 12] and 2.3e-4 relative wherever |gelu| > 1e-3 (the bf16 output rounds to 3.9e-3 relative).
// 15 instructions with two MUFU ops (rcp, ex2); libdevice erff is ~26 FMA-pipe instructions per element.
__device__ __forceinline__ float gelu_erf(float x) {
    const float z = fabsf(x) * 0.70710678118654752f;
    float t, e;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.3275911f, z, 1.0f)));
    float poly = fmaf(1.061405429f, t, -1.453152027f);
    poly = fmaf(poly, t, 1.421413741f);
    poly = fmaf(poly, t, -0.284496736f);
    poly = fmaf(poly, t, 0.254829592f);
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(z * z * -1.4426950408889634f));
    const float h = 0.5f * x * (poly * t * e);                      // 0.5 x erfc(|z|)
    return x > 0.f ? x - h : h;
}
__device__ __forceinline__ float silu(float x) { return x / (1.0f + __expf(-x)); }

// out[row, col], col and col + 1 (when inside the output): bf16 pair stores where the address allows, else scalar
__device__ __forceinline__ void store_pair(__nv_bfloat16* o, bool pair_ok, bool second, float x0, float x1) {
    if (pair_ok && second) {
        *reinterpret_cast<__nv_bfloat162*>(o) = __floats2bfloat162_rn(x0, x1);
    } else {
        o[0] = __float2bfloat16(x0);
        if (second) o[1] = __float2bfloat16(x1);
    }
}
__device__ __forceinline__ void store_pair(float* o, bool pair_ok, bool second, float x0, float x1) {
    if (pair_ok && second) {
        *reinterpret_cast<float2*>(o) = make_float2(x0, x1);
    } else {
        o[0] = x0;
        if (second) o[1] = x1;
    }
}

// One pair of outputs: x0 / x1 are accumulator columns col, col + 1 (the gate columns for SwiGLU, whose "up" columns
// col + UP, col + UP + 1 arrive as u0 / u1; UP is half the kernel's tile width).  ocol is the output column, `second`
// says whether ocol + 1 is inside the output, rrow is the residual row or null.  OUT: __nv_bfloat16, float for EPI_SCORES.
template <int EPI, int UP, typename OUT>
__device__ __forceinline__ void epilogue_pair(float x0, float x1, float u0, float u1, const __nv_bfloat16* bias, int col,
                                              const __nv_bfloat16* rrow, bool res_pair, OUT* orow,
                                              bool out_pair, int ocol, bool second) {
    if constexpr (EPI == EPI_SCORES) {         // no bias, no residual; -0.0 -> +0.0 as in every dense form
        store_pair(orow + ocol, out_pair, second, x0 + 0.0f, x1 + 0.0f);
        return;
    }
    if (EPI == EPI_SWIGLU) {
        if (bias) {
            x0 += __bfloat162float(bias[col]);
            x1 += __bfloat162float(bias[col + 1]);
            u0 += __bfloat162float(bias[col + UP]);
            u1 += __bfloat162float(bias[col + UP + 1]);
        }
        x0 = silu(x0) * u0;
        x1 = silu(x1) * u1;
    } else {
        if (bias) {
            x0 += __bfloat162float(bias[col]);
            if (second) x1 += __bfloat162float(bias[col + 1]);
        }
        if (EPI == EPI_GELU) { x0 = gelu_erf(x0); x1 = gelu_erf(x1); }
    }
    if (rrow) {
        if (res_pair && second) {
            const float2 r2 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(rrow + ocol));
            x0 += r2.x;
            x1 += r2.y;
        } else {
            x0 += __bfloat162float(rrow[ocol]);
            if (second) x1 += __bfloat162float(rrow[ocol + 1]);
        }
    }
    store_pair(orow + ocol, out_pair, second, x0, x1);
}

}  // namespace ezr
