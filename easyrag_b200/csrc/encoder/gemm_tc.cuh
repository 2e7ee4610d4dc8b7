// The mainloop of the bf16 wgmma GEMM (gemm_tc.cu), shared with the kernels that run other epilogues on its
// accumulators: the encoder GEMM's instances (gemm_tc.cu) and the dense candidate pass (dense_cand.cu).
//
// One CTA computes one GM x GN = 128 x 256 tile.  Warpgroup 0 is the TMA producer (one thread; a 4-stage ring of
// 128 x 64 A tiles and 256 x 64 W tiles, 48 KB a stage); warpgroups 1 and 2 each own 64 rows of the tile and issue
// wgmma.m64n256k16 from the ring into 128 fp32 accumulator registers per thread, keeping one k-chunk of MMAs in flight
// while the previous stage is handed back to the producer.  Each accumulator is one chain over the k16 steps in
// increasing k order (no split-K).
//
// Accumulator layout (wgmma m64n256 D fragment): thread (wq = warp in the warpgroup, lane) holds, for h in {0, 1} and
// j in [0, 32), columns j * 8 + (lane & 3) * 2 and + 1 of tile row cw * 64 + wq * 16 + (lane >> 2) + 8 * h in
// acc[4 * j + 2 * h] and acc[4 * j + 2 * h + 1].
#pragma once
#include "../ezr_common.cuh"
#include "../ptx.cuh"

namespace ezr {

constexpr int GM = 128, GN = 256, GK = 64;
constexpr int G_STAGES = 4;
constexpr int G_THREADS = 384;                 // producer warpgroup + two consumer warpgroups
constexpr int G_A_BYTES = GM * GK * 2;         // 16 KB
constexpr int G_B_BYTES = GN * GK * 2;         // 32 KB

struct GemmParams {
    int M, N, K;
    int tiles_m, tiles_n;
    const __nv_bfloat16* bias;       // [N] or null
    const __nv_bfloat16* residual;   // [M, ldr] or null
    int64_t ldr;
    void* out;                       // [M, ldo] bf16; fp32 for EPI_SCORES
    int64_t ldo;
};

struct GemmBarriers {
    uint64_t full[G_STAGES];
    uint64_t empty[G_STAGES];
};

// dynamic shared memory of a kernel running gemm_tile_mainloop
constexpr size_t G_SMEM_BYTES = 1024 + (size_t)G_STAGES * (G_A_BYTES + G_B_BYTES) + sizeof(GemmBarriers);

// Where a consumer thread's accumulators sit in the tile (layout: see the header)
struct GemmThread {
    int cw;     // consumer warpgroup: tile rows cw * 64 ..
    int lane;
    int wq;     // warp in the warpgroup
};

// The tile whose A rows start at tile row tm (of GM) and whose W rows start at tile row tn (of GN), over kchunks
// k-chunks of GK.  All 384 threads call it.  The producer warpgroup returns false once its loads are issued and must
// leave the kernel; the two consumer warpgroups return true with their accumulators in acc and their place in t.
__device__ __forceinline__ bool gemm_tile_mainloop(const CUtensorMap* map_a, const CUtensorMap* map_w, int tm, int tn,
                                                   int kchunks, float (&acc)[128], GemmThread& t) {
    extern __shared__ __align__(1024) unsigned char smem_dyn[];
    unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~(uintptr_t)1023);
    unsigned char* smem_a = smem;
    unsigned char* smem_b = smem + (size_t)G_STAGES * G_A_BYTES;
    GemmBarriers* bars = reinterpret_cast<GemmBarriers*>(smem_b + (size_t)G_STAGES * G_B_BYTES);
    const int wg = threadIdx.x >> 7;

    if (threadIdx.x == 0) {
        ptx::prefetch_tensormap(map_a);
        ptx::prefetch_tensormap(map_w);
        for (int i = 0; i < G_STAGES; ++i) { ptx::mbar_init(&bars->full[i], 1); ptx::mbar_init(&bars->empty[i], 2); }
        ptx::fence_barrier_init();
    }
    __syncthreads();

    if (wg == 0) {
        ptx::regs_dealloc<40>();
        if (threadIdx.x == 0) {
            for (int kc = 0; kc < kchunks; ++kc) {
                const int s = kc % G_STAGES;
                ptx::mbar_wait(&bars->empty[s], ((uint32_t)(kc / G_STAGES) & 1u) ^ 1u);
                ptx::mbar_expect_tx(&bars->full[s], (uint32_t)(G_A_BYTES + G_B_BYTES));
                ptx::tma_load_2d(smem_a + (size_t)s * G_A_BYTES, map_a, &bars->full[s], kc * GK, tm * GM);
                ptx::tma_load_2d(smem_b + (size_t)s * G_B_BYTES, map_w, &bars->full[s], kc * GK, tn * GN);
            }
        }
        return false;
    }
    ptx::regs_alloc<232>();
    const int cw = wg - 1;                                   // this warpgroup's 64 rows of the tile
    t.cw = cw;
    t.lane = threadIdx.x & 31;
    t.wq = (threadIdx.x >> 5) & 3;
#pragma unroll
    for (int i = 0; i < 128; ++i) acc[i] = 0.f;
    const uint32_t a0 = ptx::smem_u32(smem_a) + (uint32_t)(cw * 64 * 128);
    const uint32_t b0 = ptx::smem_u32(smem_b);
    for (int kc = 0; kc < kchunks; ++kc) {
        const int s = kc % G_STAGES;
        ptx::mbar_wait(&bars->full[s], (uint32_t)(kc / G_STAGES) & 1u);
        ptx::wgmma_fence();
#pragma unroll
        for (int k4 = 0; k4 < GK / 16; ++k4)
            ptx::wgmma_ss_n256(acc, ptx::make_desc_sw128(a0 + (uint32_t)(s * G_A_BYTES + k4 * 32)),
                               ptx::make_desc_sw128(b0 + (uint32_t)(s * G_B_BYTES + k4 * 32)), (uint32_t)((kc | k4) != 0));
        ptx::wgmma_commit();
        if (kc > 0) {                                        // the previous chunk's MMAs are done: hand its stage back
            ptx::wgmma_wait<1>();
            if ((threadIdx.x & 127) == 0) ptx::mbar_arrive(&bars->empty[(kc - 1) % G_STAGES]);
        }
    }
    ptx::wgmma_wait<0>();
    ptx::fence_regs(acc);
    // (the last stage is never handed back: no later load of this CTA needs it)
    return true;
}

}  // namespace ezr
