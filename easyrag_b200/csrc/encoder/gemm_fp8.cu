// e4m3 GEMM on wgmma with per-row activation scales, per-channel weight scales and the bf16 kernel's fused epilogues:
//
//   out[M, N'] = epilogue( diag(sa) . A8[M, K] . W8[N, K]^T . diag(sw) + bias[N] ) (+ residual[M, N'])
//
// A8 holds activations quantised per row (quant_fp8.cu), W8 an nn.Linear weight quantised per output channel; both are
// e4m3, K-major, and every scale is a power of two, so sa[row] * sw[col] rescales the fp32 accumulator exactly
// (outside fp32 under- and overflow).  The opt-in FP8 path of the encoders (encoder.py, precision="fp8").
//
// One CTA computes one 128 x 128 output tile.  Warpgroup 0 is the TMA producer (one thread; a 6-stage ring of 128 x 128
// A tiles and 128 x 128 W tiles, 32 KB a stage: a 128-byte swizzled box row is 128 e4m3 values, so a stage is one
// K-chunk of 128); warpgroups 1 and 2 each own 64 rows of the tile and issue wgmma.m64n128k32.f32.e4m3.e4m3.
//
// Promotion interval: 128 (one K-chunk, 4 MMAs).  Hopper's fp8 MMA does not accumulate in full fp32 (DeepSeek-V3
// report, section 3.3.2: about 14 bits are kept), so each chunk's MMA chain starts from zero into `part` (64 fp32
// registers), and once it completes `part` is added into the fp32 register accumulator `acc` (64 more) with ordinary
// FADDs.  The error bound of the path (tests/_bounds_fp8.py, fp8_gemm_bound) allows the in-MMA error once per chunk of
// 128 products and full fp32 rounding for the K / 128 promotions.  acc + part is 128 registers; with n256 it would be
// 256, over the 232-register cap of a consumer warpgroup, hence the 128-wide tile.
//
// The consumer waits for its own chunk before promoting it (wgmma.wait_group 0), then releases the stage; the other
// consumer warpgroup's MMAs run on the tensor cores meanwhile.  Tile order: N tiles fastest, as in gemm_tc.cu.
//
// SwiGLU: the W8 rows are interleaved in blocks of 64 (64 gate rows, then the matching 64 up rows), so gate column c
// and up column c + 64 of a tile sit in the same thread (the bf16 weights keep their 128-row blocks).
#include "../ezr_common.cuh"
#include "../ptx.cuh"
#include "gemm_epi.cuh"

namespace ezr {

constexpr int F8_GM = 128, F8_GN = 128, F8_GK = 128;   // F8_GK: e4m3 values per K-chunk = the promotion interval
constexpr int F8_STAGES = 6;
constexpr int F8_THREADS = 384;                        // producer warpgroup + two consumer warpgroups
constexpr int F8_A_BYTES = F8_GM * F8_GK;              // 16 KB
constexpr int F8_B_BYTES = F8_GN * F8_GK;              // 16 KB

struct Fp8GemmParams {
    int M, N, K;
    int tiles_m, tiles_n;
    const float* sa;                 // [M] activation row scales
    const float* sw;                 // [N] weight channel scales
    const __nv_bfloat16* bias;       // [N] or null
    const __nv_bfloat16* residual;   // [M, ldr] or null
    int64_t ldr;
    __nv_bfloat16* out;              // [M, ldo]
    int64_t ldo;
};

struct Fp8GemmBarriers {
    uint64_t full[F8_STAGES];
    uint64_t empty[F8_STAGES];
};

// D[64 x 128] (+)= A[64 x 32] . B[128 x 32]^T, e4m3 from shared-memory descriptors (both K-major), fp32 accumulator
__device__ __forceinline__ void wgmma_e4m3_n128(float (&d)[64], uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k32.f32.e4m3.e4m3 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
        "}, %64, %65, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
          "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
          "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]),
          "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),
          "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]),
          "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]),
          "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db), "r"(acc));
}

template <int EPI>
__global__ void __launch_bounds__(F8_THREADS, 1)
gemm_fp8_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_w,
                const Fp8GemmParams p) {
    extern __shared__ __align__(1024) unsigned char smem_dyn[];
    unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~(uintptr_t)1023);
    unsigned char* smem_a = smem;
    unsigned char* smem_b = smem + (size_t)F8_STAGES * F8_A_BYTES;
    Fp8GemmBarriers* bars = reinterpret_cast<Fp8GemmBarriers*>(smem_b + (size_t)F8_STAGES * F8_B_BYTES);
    const int tn = blockIdx.x % p.tiles_n, tm = blockIdx.x / p.tiles_n;
    const int kchunks = p.K / F8_GK;
    const int wg = threadIdx.x >> 7;

    if (threadIdx.x == 0) {
        ptx::prefetch_tensormap(&map_a);
        ptx::prefetch_tensormap(&map_w);
        for (int i = 0; i < F8_STAGES; ++i) { ptx::mbar_init(&bars->full[i], 1); ptx::mbar_init(&bars->empty[i], 2); }
        ptx::fence_barrier_init();
    }
    __syncthreads();

    if (wg == 0) {
        ptx::regs_dealloc<40>();
        if (threadIdx.x == 0) {
            // the maps describe the byte matrices as bf16 pairs: column coordinates count pairs
            for (int kc = 0; kc < kchunks; ++kc) {
                const int s = kc % F8_STAGES;
                ptx::mbar_wait(&bars->empty[s], ((uint32_t)(kc / F8_STAGES) & 1u) ^ 1u);
                ptx::mbar_expect_tx(&bars->full[s], (uint32_t)(F8_A_BYTES + F8_B_BYTES));
                ptx::tma_load_2d(smem_a + (size_t)s * F8_A_BYTES, &map_a, &bars->full[s], kc * (F8_GK / 2), tm * F8_GM);
                ptx::tma_load_2d(smem_b + (size_t)s * F8_B_BYTES, &map_w, &bars->full[s], kc * (F8_GK / 2), tn * F8_GN);
            }
        }
        return;
    }
    ptx::regs_alloc<232>();
    const int cw = wg - 1;                                   // this warpgroup's 64 rows of the tile
    const int lane = threadIdx.x & 31, wq = (threadIdx.x >> 5) & 3;
    float acc[64], part[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) { acc[i] = 0.f; part[i] = 0.f; }
    const uint32_t a0 = ptx::smem_u32(smem_a) + (uint32_t)(cw * 64 * 128);
    const uint32_t b0 = ptx::smem_u32(smem_b);
    for (int kc = 0; kc < kchunks; ++kc) {
        const int s = kc % F8_STAGES;
        ptx::mbar_wait(&bars->full[s], (uint32_t)(kc / F8_STAGES) & 1u);
        ptx::wgmma_fence();
#pragma unroll
        for (int k4 = 0; k4 < F8_GK / 32; ++k4)              // a k32 slice is 32 bytes of a 128-byte swizzled row
            wgmma_e4m3_n128(part, ptx::make_desc_sw128(a0 + (uint32_t)(s * F8_A_BYTES + k4 * 32)),
                            ptx::make_desc_sw128(b0 + (uint32_t)(s * F8_B_BYTES + k4 * 32)), (uint32_t)(k4 != 0));
        ptx::wgmma_commit();
        ptx::wgmma_wait<0>();
        ptx::fence_regs(part);
        if ((threadIdx.x & 127) == 0) ptx::mbar_arrive(&bars->empty[s]);
#pragma unroll
        for (int i = 0; i < 64; ++i) acc[i] += part[i];     // the promotion: full fp32 adds, once per 128-K chunk
    }

    // ---------------- epilogue on the accumulator registers: rescale, then the bf16 kernel's epilogue
    const int n_out = (EPI == EPI_SWIGLU) ? p.N / 2 : p.N;
    const bool out_pair = (p.ldo % 2 == 0) && ((reinterpret_cast<uintptr_t>(p.out) & 3) == 0);
    const bool res_pair = p.residual && (p.ldr % 2 == 0) && ((reinterpret_cast<uintptr_t>(p.residual) & 3) == 0);
    const int cq = (lane & 3) * 2;
    constexpr int NJ = (EPI == EPI_SWIGLU) ? F8_GN / 16 : F8_GN / 8;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int row = tm * F8_GM + cw * 64 + wq * 16 + (lane >> 2) + 8 * h;
        if (row >= p.M) continue;
        const float sa = p.sa[row];
        __nv_bfloat16* orow = p.out + (int64_t)row * p.ldo;
        const __nv_bfloat16* rrow = p.residual ? p.residual + (int64_t)row * p.ldr : nullptr;
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
            const int col = tn * F8_GN + j * 8 + cq;                    // accumulator column (gate column for SwiGLU)
            const int ocol = (EPI == EPI_SWIGLU) ? tn * (F8_GN / 2) + j * 8 + cq : col;
            if (ocol >= n_out) continue;
            const bool second = ocol + 1 < n_out;
            const float x0 = acc[4 * j + 2 * h] * sa * p.sw[col];
            const float x1 = second || EPI == EPI_SWIGLU ? acc[4 * j + 2 * h + 1] * sa * p.sw[col + 1] : 0.f;
            float u0 = 0.f, u1 = 0.f;
            if constexpr (EPI == EPI_SWIGLU) {
                u0 = acc[4 * (j + NJ) + 2 * h] * sa * p.sw[col + F8_GN / 2];
                u1 = acc[4 * (j + NJ) + 2 * h + 1] * sa * p.sw[col + F8_GN / 2 + 1];
            }
            epilogue_pair<EPI, F8_GN / 2>(x0, x1, u0, u1, p.bias, col, rrow, res_pair, orow, out_pair, ocol, second);
        }
    }
}

static int gemm_fp8_launch(const uint8_t* A, const float* sa, int M, int K, int64_t lda, const uint8_t* W,
                           const float* sw, int N, int64_t ldw, const __nv_bfloat16* bias,
                           const __nv_bfloat16* residual, int64_t ldr, __nv_bfloat16* out, int64_t ldo, int epi,
                           cudaStream_t st) {
    EZR_CHECK_ARG(M >= 0 && N >= 1 && K >= F8_GK && K % F8_GK == 0, "gemm_fp8: need K %% 128 == 0 (M=%d N=%d K=%d)", M,
                  N, K);
    EZR_CHECK_ARG(lda % 16 == 0 && ldw % 16 == 0 && lda >= K && ldw >= K,
                  "gemm_fp8: row strides must be multiples of 16 bytes and >= K");
    EZR_CHECK_ARG(((reinterpret_cast<uintptr_t>(A) | reinterpret_cast<uintptr_t>(W)) & 15) == 0,
                  "gemm_fp8: A8/W8 must be 16-byte aligned");
    EZR_CHECK_ARG(sa != nullptr && sw != nullptr && out != nullptr, "gemm_fp8: scales and output are required");
    EZR_CHECK_ARG(epi >= EPI_NONE && epi <= EPI_SWIGLU, "gemm_fp8: bad epilogue %d", epi);
    EZR_CHECK_ARG(epi != EPI_SWIGLU || N % F8_GN == 0,
                  "gemm_fp8: SwiGLU epilogue needs N %% 128 == 0 (gate/up interleaved in blocks of 64 rows)");
    if (M == 0) return EZR_OK;
    Fp8GemmParams p;
    p.M = M; p.N = N; p.K = K;
    p.tiles_m = (M + F8_GM - 1) / F8_GM;
    p.tiles_n = (N + F8_GN - 1) / F8_GN;
    p.sa = sa; p.sw = sw;
    p.bias = bias; p.residual = residual; p.ldr = ldr; p.out = out; p.ldo = ldo;
    CUtensorMap map_a, map_w;
    int rc = encode_tmap_2d_bf16(&map_a, A, (uint64_t)K / 2, (uint64_t)M, (uint64_t)lda / 2, F8_GK / 2, F8_GM);
    if (rc) return rc;
    rc = encode_tmap_2d_bf16(&map_w, W, (uint64_t)K / 2, (uint64_t)N, (uint64_t)ldw / 2, F8_GK / 2, F8_GN);
    if (rc) return rc;
    const size_t smem = 1024 + (size_t)F8_STAGES * (F8_A_BYTES + F8_B_BYTES) + sizeof(Fp8GemmBarriers);
    typedef void (*kern_t)(const CUtensorMap, const CUtensorMap, const Fp8GemmParams);
    static const kern_t table[3] = {gemm_fp8_kernel<EPI_NONE>, gemm_fp8_kernel<EPI_GELU>, gemm_fp8_kernel<EPI_SWIGLU>};
    static bool attr_done[3] = {false, false, false};
    if (!attr_done[epi]) {
        EZR_CUDA(cudaFuncSetAttribute(table[epi], cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr_done[epi] = true;
    }
    const long long tiles = (long long)p.tiles_m * p.tiles_n;
    EZR_CHECK_ARG(tiles < (1ll << 31), "gemm_fp8: too many tiles");
    {
        ProfScope prof(EZR_PROF_ENC_GEMM, st);
        table[epi]<<<(unsigned)tiles, F8_THREADS, smem, st>>>(map_a, map_w, p);
    }
    EZR_LAUNCH_CHECK();
    return EZR_OK;
}

}  // namespace ezr

extern "C" int ezr_gemm_fp8(const void* a8, const float* sa, int32_t m, int32_t k, int64_t lda, const void* w8,
                            const float* sw, int32_t n, int64_t ldw, const void* bias, const void* residual, int64_t ldr,
                            void* out, int64_t ldo, int32_t epilogue, void* stream) {
    using namespace ezr;
    return gemm_fp8_launch((const uint8_t*)a8, sa, m, k, lda, (const uint8_t*)w8, sw, n, ldw,
                           (const __nv_bfloat16*)bias, (const __nv_bfloat16*)residual, ldr, (__nv_bfloat16*)out, ldo,
                           epilogue, (cudaStream_t)stream);
}
