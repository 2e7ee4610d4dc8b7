// bf16 GEMM on wgmma (Hopper warpgroup MMA) with fused epilogues, for the chunk-embedding forward pass.
//
//   out[M, N'] = epilogue( A[M, K] . W[N, K]^T + bias[N] ) (+ residual[M, N'])
//
// A = activations (tokens x features, row-major), W = an nn.Linear weight ([out, in], row-major), so both
// operands are K-major and load straight into 128B-swizzled shared-memory tiles by TMA.  Replaces the
// cuBLAS calls behind the reference's projections: Qwen2 q/k/v/o and SwiGLU MLP (modeling_qwen.py:261-263,
// 319,186) and the BERT-shaped encoder's dense layers behind SentenceTransformer.encode (hf_embeddings.py:118-123).
//
// One CTA computes one 128 x 256 output tile with the mainloop of gemm_tc.cuh (a 4-stage TMA ring feeding
// wgmma.m64n256k16 into 128 fp32 accumulator registers per consumer thread).  The epilogue runs on the accumulator
// registers: bias / GELU / SwiGLU / residual in fp32, bf16 pairs stored straight to global memory.  SwiGLU needs no exchange: the gate
// column c and its "up" column c + 128 of a 256-column tile sit in the same thread.
//
// Tile order: N tiles fastest.  The activations of a 147k-token batch (226 MB at K = 768, 905 MB at K = 3072) do not fit
// the 50 MB L2, the weights (a few MB) do: with N fastest the CTAs in flight cover a few M tiles x all N tiles, so an A
// tile is fetched from HBM about once.
//
// Dense top-k form 6 (dense_wide.cu) runs the same kernel on A = a block of queries, W = the corpus rows, with the
// EPI_SCORES epilogue (fp32 score rows, gemm_scores_f32) and M tiles fastest: there the query block (a few MB) fits L2
// and the corpus does not, so the CTAs in flight cover all query tiles of a few corpus tiles.  The dense candidate pass
// (dense_cand.cu) runs the same mainloop in the same tile order with an epilogue that keeps only the scores that can
// still reach each query's top-k.
#include <type_traits>

#include "../ezr_common.cuh"
#include "../ptx.cuh"
#include "../dense_tc.h"
#include "gemm_epi.cuh"
#include "gemm_tc.cuh"

namespace ezr {

template <int EPI, bool M_FAST>
__global__ void __launch_bounds__(G_THREADS, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_w, const GemmParams p) {
    // N tiles fastest, M tiles for the score rows: see the header
    const int tn = M_FAST ? blockIdx.x / p.tiles_m : blockIdx.x % p.tiles_n;
    const int tm = M_FAST ? blockIdx.x % p.tiles_m : blockIdx.x / p.tiles_n;
    float acc[128];
    GemmThread t;
    if (!gemm_tile_mainloop(&map_a, &map_w, tm, tn, p.K / GK, acc, t)) return;
    const int cw = t.cw, lane = t.lane, wq = t.wq;

    // ---------------- epilogue on the accumulator registers
    typedef typename std::conditional<EPI == EPI_SCORES, float, __nv_bfloat16>::type out_t;
    const int n_out = (EPI == EPI_SWIGLU) ? p.N / 2 : p.N;
    const bool out_pair = (p.ldo % 2 == 0) && ((reinterpret_cast<uintptr_t>(p.out) & (2 * sizeof(out_t) - 1)) == 0);
    const bool res_pair = p.residual && (p.ldr % 2 == 0) && ((reinterpret_cast<uintptr_t>(p.residual) & 3) == 0);
    const int cq = (lane & 3) * 2;
    constexpr int NJ = (EPI == EPI_SWIGLU) ? GN / 16 : GN / 8;       // 8-column groups of output per thread row
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int row = tm * GM + cw * 64 + wq * 16 + (lane >> 2) + 8 * h;
        if (row >= p.M) continue;
        out_t* orow = static_cast<out_t*>(p.out) + (int64_t)row * p.ldo;
        const __nv_bfloat16* rrow = p.residual ? p.residual + (int64_t)row * p.ldr : nullptr;
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
            const int col = tn * GN + j * 8 + cq;                       // accumulator column (gate column for SwiGLU)
            const int ocol = (EPI == EPI_SWIGLU) ? tn * (GN / 2) + j * 8 + cq : col;
            if (ocol >= n_out) continue;
            const bool second = ocol + 1 < n_out;
            float u0 = 0.f, u1 = 0.f;
            if constexpr (EPI == EPI_SWIGLU) { u0 = acc[4 * (j + NJ) + 2 * h]; u1 = acc[4 * (j + NJ) + 2 * h + 1]; }
            epilogue_pair<EPI, GN / 2>(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1], u0, u1, p.bias, col, rrow, res_pair,
                                       orow, out_pair, ocol, second);
        }
    }
}

static int gemm_launch(const __nv_bfloat16* A, int M, int K, int64_t lda, const __nv_bfloat16* W, int N, int64_t ldw,
                       const __nv_bfloat16* bias, const __nv_bfloat16* residual, int64_t ldr, void* out,
                       int64_t ldo, int epi, int prof_slot, cudaStream_t st) {
    EZR_CHECK_ARG(M >= 0 && N >= 1 && K >= GK && K % GK == 0, "gemm: need K %% 64 == 0 (M=%d N=%d K=%d)", M, N, K);
    EZR_CHECK_ARG(lda % 8 == 0 && ldw % 8 == 0 && lda >= K && ldw >= K, "gemm: row strides must be multiples of 8 and >= K");
    EZR_CHECK_ARG(((reinterpret_cast<uintptr_t>(A) | reinterpret_cast<uintptr_t>(W)) & 15) == 0, "gemm: A/W must be 16-byte aligned");
    EZR_CHECK_ARG(epi != EPI_SWIGLU || N % GN == 0, "gemm: SwiGLU epilogue needs N %% 256 == 0 (gate/up interleaved in blocks of 128 rows)");
    if (M == 0) return EZR_OK;
    GemmParams p;
    p.M = M; p.N = N; p.K = K;
    p.tiles_m = (M + GM - 1) / GM;
    p.tiles_n = (N + GN - 1) / GN;
    p.bias = bias; p.residual = residual; p.ldr = ldr; p.out = out; p.ldo = ldo;
    CUtensorMap map_a, map_w;
    int rc = encode_tmap_2d_bf16(&map_a, A, (uint64_t)K, (uint64_t)M, (uint64_t)lda, GK, GM);
    if (rc) return rc;
    rc = encode_tmap_2d_bf16(&map_w, W, (uint64_t)K, (uint64_t)N, (uint64_t)ldw, GK, GN);
    if (rc) return rc;
    const size_t smem = G_SMEM_BYTES;
    typedef void (*kern_t)(const CUtensorMap, const CUtensorMap, const GemmParams);
    static const kern_t table[4] = {gemm_wgmma_kernel<EPI_NONE, false>, gemm_wgmma_kernel<EPI_GELU, false>,
                                    gemm_wgmma_kernel<EPI_SWIGLU, false>, gemm_wgmma_kernel<EPI_SCORES, true>};
    static bool attr_done[4] = {false, false, false, false};
    if (!attr_done[epi]) {
        EZR_CUDA(cudaFuncSetAttribute(table[epi], cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr_done[epi] = true;
    }
    const long long tiles = (long long)p.tiles_m * p.tiles_n;
    EZR_CHECK_ARG(tiles < (1ll << 31), "gemm: too many tiles");
    {
        ProfScope prof(prof_slot, st);
        table[epi]<<<(unsigned)tiles, G_THREADS, smem, st>>>(map_a, map_w, p);
    }
    EZR_LAUNCH_CHECK();
    return EZR_OK;
}

int gemm_scores_f32(const __nv_bfloat16* A, int M, int K, int64_t lda, const __nv_bfloat16* W, int N, int64_t ldw,
                    float* out, int64_t ldo, int prof_slot, cudaStream_t st) {
    return gemm_launch(A, M, K, lda, W, N, ldw, nullptr, nullptr, 0, out, ldo, EPI_SCORES, prof_slot, st);
}

}  // namespace ezr

extern "C" int ezr_gemm_bf16(const void* a, int32_t m, int32_t k, int64_t lda, const void* w, int32_t n, int64_t ldw,
                             const void* bias, const void* residual, int64_t ldr, void* out, int64_t ldo,
                             int32_t epilogue, void* stream) {
    using namespace ezr;
    EZR_CHECK_ARG(epilogue >= EPI_NONE && epilogue <= EPI_SWIGLU, "gemm: bad epilogue %d", epilogue);
    return gemm_launch((const __nv_bfloat16*)a, m, k, lda, (const __nv_bfloat16*)w, n, ldw, (const __nv_bfloat16*)bias,
                       (const __nv_bfloat16*)residual, ldr, out, ldo, epilogue, EZR_PROF_ENC_GEMM, (cudaStream_t)stream);
}
