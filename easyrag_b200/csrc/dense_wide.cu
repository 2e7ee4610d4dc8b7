// Dense cosine top-k for any dim % 64 == 0 and any k <= 1024 on the Hopper tensor cores: a wgmma kernel writes a
// block of fp32 score rows, and the generic row select (ezr_select_rows) takes the top-k from it.
//
// The forms of dense_tc.cu keep the query block resident in shared memory and the top-k in registers, which limits
// them to dim <= 1024 and k <= 16.  This kernel holds nothing resident: both operands stream through one TMA ring, as
// in encoder/gemm_tc.cu, so the width is unbounded (gte-Qwen2-7B: 3584), and the scores go to HBM so that k is only
// bounded by the select (the pipeline's f_topk_1 = 288).
//
// One CTA computes one 128-query x 256-row tile of the block's score rows.  Warpgroup 0 is the TMA producer (one
// thread; a 4-stage ring of 128 x 64 query tiles and 256 x 64 corpus tiles, 48 KB a stage, both K-major with the
// 128-byte swizzle); warpgroups 1 and 2 each own 64 queries of the tile (the A operand, as in the other forms) and
// issue wgmma.m64n256k16 with the corpus rows as B, keeping one k-chunk of MMAs in flight while the previous stage is
// handed back.  Each score is one accumulator chain over the k16 steps in increasing k order, no split-K: the fp32
// sum of the same k16 products in the same order as forms 2-4, so the scores are bit-identical to theirs.
//
// Tile order: query tiles fastest.  The CTAs in flight then cover all query tiles of a few corpus tiles: a corpus
// tile is read from HBM about once per block, and the query block (a few MB) stays in the 50 MB L2.
#include <algorithm>

#include "ezr_common.cuh"
#include "ptx.cuh"
#include "dense_tc.h"
#include "../../include/easyrag_b200.h"

namespace ezr {

constexpr int WQ = 128, WN = 256, WK = 64;    // queries, corpus rows and dims of one tile / k-chunk
constexpr int W_STAGES = 4;
constexpr int W_THREADS = 384;                // producer warpgroup + two consumer warpgroups
constexpr int W_A_BYTES = WQ * WK * 2;        // 16 KB
constexpr int W_B_BYTES = WN * WK * 2;        // 32 KB
// queries per block: the select launches one CTA row per query (grid.y <= 65535)
constexpr int W_MAX_BLOCK = 65535;

struct WideParams {
    int kchunks;         // dim / 64
    int tiles_q;         // query tiles of the block
    int q0;              // the block's first query (row coordinate in the query tensor map)
    int nq;              // queries in the block
    int64_t n_rows;
    float* out;          // [nq][ldo] score rows
    int64_t ldo;
};

struct WideBarriers {
    uint64_t full[W_STAGES];
    uint64_t empty[W_STAGES];
};

__global__ void __launch_bounds__(W_THREADS, 1)
dense_scores_wgmma_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_c,
                          const WideParams p) {
    extern __shared__ __align__(1024) unsigned char smem_dyn[];
    unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~(uintptr_t)1023);
    unsigned char* smem_a = smem;
    unsigned char* smem_b = smem + (size_t)W_STAGES * W_A_BYTES;
    WideBarriers* bars = reinterpret_cast<WideBarriers*>(smem_b + (size_t)W_STAGES * W_B_BYTES);
    const int tq = (int)(blockIdx.x % (unsigned)p.tiles_q);          // query tiles fastest: see the header
    const int64_t tr = blockIdx.x / (unsigned)p.tiles_q;
    const int wg = threadIdx.x >> 7;

    if (threadIdx.x == 0) {
        ptx::prefetch_tensormap(&map_q);
        ptx::prefetch_tensormap(&map_c);
        for (int i = 0; i < W_STAGES; ++i) { ptx::mbar_init(&bars->full[i], 1); ptx::mbar_init(&bars->empty[i], 2); }
        ptx::fence_barrier_init();
    }
    __syncthreads();

    if (wg == 0) {
        ptx::regs_dealloc<40>();
        if (threadIdx.x == 0) {
            for (int kc = 0; kc < p.kchunks; ++kc) {
                const int s = kc % W_STAGES;
                ptx::mbar_wait(&bars->empty[s], ((uint32_t)(kc / W_STAGES) & 1u) ^ 1u);
                ptx::mbar_expect_tx(&bars->full[s], (uint32_t)(W_A_BYTES + W_B_BYTES));
                ptx::tma_load_2d(smem_a + (size_t)s * W_A_BYTES, &map_q, &bars->full[s], kc * WK, p.q0 + tq * WQ);
                ptx::tma_load_2d(smem_b + (size_t)s * W_B_BYTES, &map_c, &bars->full[s], kc * WK, (int)(tr * WN));
            }
        }
        return;
    }
    ptx::regs_alloc<232>();
    const int cw = wg - 1;                                   // this warpgroup's 64 queries of the tile
    const int lane = threadIdx.x & 31, wq = (threadIdx.x >> 5) & 3;
    float acc[128];
#pragma unroll
    for (int i = 0; i < 128; ++i) acc[i] = 0.f;
    const uint32_t a0 = ptx::smem_u32(smem_a) + (uint32_t)(cw * 64 * 128);
    const uint32_t b0 = ptx::smem_u32(smem_b);
    for (int kc = 0; kc < p.kchunks; ++kc) {
        const int s = kc % W_STAGES;
        ptx::mbar_wait(&bars->full[s], (uint32_t)(kc / W_STAGES) & 1u);
        ptx::wgmma_fence();
#pragma unroll
        for (int k4 = 0; k4 < WK / 16; ++k4)
            ptx::wgmma_ss_n256(acc, ptx::make_desc_sw128(a0 + (uint32_t)(s * W_A_BYTES + k4 * 32)),
                               ptx::make_desc_sw128(b0 + (uint32_t)(s * W_B_BYTES + k4 * 32)), (uint32_t)((kc | k4) != 0));
        ptx::wgmma_commit();
        if (kc > 0) {                                        // the previous chunk's MMAs are done: hand its stage back
            ptx::wgmma_wait<1>();
            if ((threadIdx.x & 127) == 0) ptx::mbar_arrive(&bars->empty[(kc - 1) % W_STAGES]);
        }
    }
    ptx::wgmma_wait<0>();
    ptx::fence_regs(acc);
    // (the last stage is never handed back: no later load of this CTA needs it)

    // ---------------- epilogue: thread column pair (2 (lane % 4), + 1) of each 8-column group = two adjacent rows
    const bool pair_ok = (p.ldo & 1) == 0 && (reinterpret_cast<uintptr_t>(p.out) & 7) == 0;   // rows start 8-byte aligned
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int ql = tq * WQ + cw * 64 + wq * 16 + (lane >> 2) + 8 * h;
        if (ql >= p.nq) continue;
        float* orow = p.out + (int64_t)ql * p.ldo;
#pragma unroll
        for (int j = 0; j < WN / 8; ++j) {
            const int64_t row = tr * WN + j * 8 + (lane & 3) * 2;
            const float s0 = acc[4 * j + 2 * h] + 0.0f, s1 = acc[4 * j + 2 * h + 1] + 0.0f;   // -0.0 -> +0.0
            if (pair_ok && row + 1 < p.n_rows) {
                *reinterpret_cast<float2*>(orow + row) = make_float2(s0, s1);
            } else {
                if (row < p.n_rows) orow[row] = s0;
                if (row + 1 < p.n_rows) orow[row + 1] = s1;
            }
        }
    }
}

bool dense_wide_supported(const __nv_bfloat16* corpus, int64_t n_rows, int dim, int64_t ldc,
                          const __nv_bfloat16* queries, int64_t ldq) {
    if (dim <= 0 || dim % WK != 0) return false;
    if (ldc % 8 != 0 || ldq % 8 != 0) return false;
    if ((reinterpret_cast<uintptr_t>(corpus) & 15) || (reinterpret_cast<uintptr_t>(queries) & 15)) return false;
    return n_rows >= 1;
}

// Score rows of a block of m queries, then the select workspace behind them.  The last block of a call may be smaller
// than the others and its select may need more (it splits each row into more parts); its rows take less room.
static size_t wide_block_bytes(int64_t n_rows, int m, int k) {
    return align_up((size_t)m * n_rows * 4, 256) + ezr_select_rows_workspace(m, n_rows, k, EZR_F32);
}

size_t dense_wide_workspace(int64_t n_rows, int n_queries, int k, int block_queries) {
    if (n_rows <= 0 || n_queries <= 0 || k <= 0 || block_queries <= 0) return 0;
    const int qb = std::min(block_queries, std::min(n_queries, W_MAX_BLOCK));
    size_t need = wide_block_bytes(n_rows, qb, k);
    const int last = n_queries % qb;
    if (last) {
        const size_t l = wide_block_bytes(n_rows, last, k);
        if (l > need) need = l;
    }
    return need;
}

// The largest query block whose work fits ws_bytes (0: not even one query).
static int wide_block_queries(int64_t n_rows, int n_queries, int k, size_t ws_bytes) {
    const int64_t tiles_r = (n_rows + WN - 1) / WN;
    int64_t qb = (int64_t)(ws_bytes / ((size_t)n_rows * 4));
    qb = std::min(qb, (int64_t)std::min(n_queries, W_MAX_BLOCK));
    qb = std::min(qb, ((int64_t)INT32_MAX / tiles_r) * WQ);       // one CTA per tile: the grid stays below 2^31
    while (qb > 0 && dense_wide_workspace(n_rows, n_queries, k, (int)qb) > ws_bytes) --qb;
    return (int)qb;
}

int dense_wide_topk(const __nv_bfloat16* corpus, int64_t n_rows, int dim, int64_t ldc, const __nv_bfloat16* queries,
                    int n_queries, int64_t ldq, int k, const int32_t* doc_group, const int32_t* q_group, int id_base,
                    float* out_scores, int32_t* out_ids, int32_t* out_counts, void* ws, size_t ws_bytes,
                    cudaStream_t st) {
    const int qb = ws ? wide_block_queries(n_rows, n_queries, k, ws_bytes) : 0;
    if (qb < 1) {
        set_error("dense_topk(wgmma-scores): workspace %zu < %zu (one query per block)", ws ? ws_bytes : (size_t)0,
                  dense_wide_workspace(n_rows, n_queries, k, 1));
        return EZR_ERR_WORKSPACE;
    }
    CUtensorMap map_q, map_c;
    int rc = encode_tmap_2d_bf16(&map_q, queries, (uint64_t)dim, (uint64_t)n_queries, (uint64_t)ldq, WK, WQ);
    if (rc) return rc;
    rc = encode_tmap_2d_bf16(&map_c, corpus, (uint64_t)dim, (uint64_t)n_rows, (uint64_t)ldc, WK, WN);
    if (rc) return rc;
    const size_t smem = 1024 + (size_t)W_STAGES * (W_A_BYTES + W_B_BYTES) + sizeof(WideBarriers);
    static bool attr_done = false;
    if (!attr_done) {
        EZR_CUDA(cudaFuncSetAttribute(dense_scores_wgmma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr_done = true;
    }
    const int64_t tiles_r = (n_rows + WN - 1) / WN;
    float* rows = reinterpret_cast<float*>(ws);
    WideParams p;
    p.kchunks = dim / WK;
    p.n_rows = n_rows;
    p.out = rows;
    p.ldo = n_rows;
    for (int q0 = 0; q0 < n_queries; q0 += qb) {
        const int nq = n_queries - q0 < qb ? n_queries - q0 : qb;
        p.q0 = q0;
        p.nq = nq;
        p.tiles_q = (nq + WQ - 1) / WQ;
        {
            ProfScope prof(EZR_PROF_DENSE_WIDE, st);
            dense_scores_wgmma_kernel<<<(unsigned)(p.tiles_q * tiles_r), W_THREADS, smem, st>>>(map_q, map_c, p);
        }
        EZR_LAUNCH_CHECK();
        // this block's select workspace sits right behind its own rows (see wide_block_bytes)
        const size_t rows_bytes = align_up((size_t)nq * n_rows * 4, 256);
        rc = ezr_select_rows(rows, EZR_F32, nq, n_rows, n_rows, k, 0, doc_group, q_group ? q_group + q0 : nullptr,
                             id_base, out_scores + (int64_t)q0 * k, out_ids + (int64_t)q0 * k,
                             out_counts ? out_counts + q0 : nullptr, (char*)ws + rows_bytes, ws_bytes - rows_bytes, st);
        if (rc) return rc;
    }
    return EZR_OK;
}

}  // namespace ezr

extern "C" size_t ezr_dense_wide_workspace(int64_t n_rows, int32_t n_queries, int32_t k, int32_t block_queries) {
    return ezr::dense_wide_workspace(n_rows, n_queries, k, block_queries);
}
