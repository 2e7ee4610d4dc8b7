// Dense cosine top-k on the Hopper tensor cores: TMA -> shared memory -> wgmma -> registers, with the top-k taken
// in the epilogue straight from the accumulators.
//
// Replaces the vector search behind QdrantRetriever._aretrieve (retrievers.py:37-52;
// Distance.COSINE, ingestion.py:180-182).  Work decomposition (DESIGN.md "Dense"):
//   persistent CTAs walk work units (corpus split s, query block b), ordered split-major: a CTA keeps ONE query block
//   for a long run of corpus rows (n_rows / n_splits), so the per-thread top-k lists warm up once per unit and almost
//   nothing passes the threshold afterwards, and the query blocks resident at the same time stream the SAME corpus
//   split, so a corpus tile is fetched from HBM once and served to the other CTAs from the L2.
//   A query block (QW x 64 queries, QW = 2 consumer warpgroups for dim <= 768, 1 above) stays resident for the whole
//   unit (A operand; in shared memory as K-major, 128B-swizzled 64 x 64 TMA boxes, with the 128-query form holding
//   its first k-chunks in registers instead); the corpus rows stream through a ring of TMA stages (B operand: TN rows
//   x 64 bf16).  Each consumer warpgroup issues wgmma.m64nTNk16 into TN / 2 fp32 registers per thread and scans its
//   scores with a per-thread register-resident sorted list of k <= 16 per query row.  Scores never reach HBM: per
//   (query, split) the four threads that share a query row write k (score, id) pairs each, and a warp-per-query merge
//   produces the final list.
#include "ezr_common.cuh"
#include "ptx.cuh"
#include "dense_tc.h"
#include "../../include/easyrag_b200.h"

namespace ezr {

int g_dense_probe = 0;       // ezr_dense_set_probe
int g_dense_stage_cap = 0;   // 0: use all shared memory for the TMA ring (ezr_dense_set_stage_cap)

constexpr int TC_TN = 64;       // the narrower corpus tile (rows): bounds the number of corpus splits
constexpr int TC_KC = 64;       // bf16 per k-chunk = one 128-byte swizzle row
constexpr int TC_MAXD = 1024;
constexpr int TC_LISTS = 4;     // lists per (query, split): the four threads of a query row
constexpr int TC_MAX_STAGES = 32;
constexpr int TC_KMAX = 16;
constexpr int TC_A_BOX_BYTES = 64 * TC_KC * 2;       // 8192: 64 queries x one k-chunk
constexpr int TC_B_STAGE_BYTES = TC_TN * TC_KC * 2;  // 8192
constexpr int TC_SMEM_LIMIT = 232448;                 // 227 KB opt-in maximum per CTA

struct TcParams {
    int dim;
    int64_t n_rows;
    int rows_per_slice;   // multiple of the corpus tile rows
    int n_queries;
    int kchunks;          // dim / 64
    int n_stages;
    int k;
    int id_base;
    const int32_t* doc_group;
    const int32_t* q_group;
    float* part_s;        // [n_queries][n_slices][TC_LISTS][k]
    int32_t* part_id;
    int32_t* bound;       // [n_queries] float bits (0 = none) of a proven lower bound of each query's final k-th best
                          // score, raised by every finished unit; later units of the query start from it
    int n_slices;
    int n_qblocks;        // units = n_slices x n_qblocks, walked by persistent CTAs
    int probe;            // measurement probes (ezr_dense_set_probe): 1 = no TMA loads, 2 = no MMAs, 4 = no epilogue scan; results are garbage
    const __nv_bfloat16* queries;   // read directly (register-held query chunks of dense_wgmma_rq_kernel)
    int64_t ldq;
};

// Query k-chunks the 128-query kernel holds in registers as wgmma A fragments (16 registers per thread each): the
// most that fit beside 64 accumulators and the two top-k lists without spilling under the 232-register budget (lists of
// 12 take 56 registers, of 16 take 72).
__host__ __device__ constexpr int tc_reg_chunks(int kt) { return kt <= 8 ? 4 : kt == 12 ? 2 : 0; }

struct TcBarriers {
    uint64_t a_full;       // the unit's query block has landed
    uint64_t a_empty;      // ... and every MMA of the previous unit that read it has retired (one arrival per consumer)
    uint64_t b_full[TC_MAX_STAGES];
    uint64_t b_empty[TC_MAX_STAGES];
};

// candidates arrive in increasing id order per list, so on equal score the newcomer (higher id) ranks first under the
// canonical order: ">=" everywhere
template <int KT>
__device__ __forceinline__ void list_insert(float (&ts)[KT], int (&ti)[KT], float cv, int ci) {
#pragma unroll
    for (int s = 0; s < KT; ++s) {
        const bool b = cv >= ts[s];
        const float fs = ts[s];
        const int is = ti[s];
        ts[s] = b ? cv : fs;
        ti[s] = b ? ci : is;
        cv = b ? fs : cv;
        ci = b ? is : ci;
    }
}

// The top-k list of one query row of a thread (accumulator fragment row r + 8 H).
template <int KT>
struct RowList {
    float ts[KT];
    int ti[KT];
    float seed, thr;
    int qg, want;
    bool active;
};

// this thread's TN / 4 scores of row H of a TN-row corpus tile (columns 8 j + 2 (lane % 4) + e, in increasing
// document order)
template <bool FILTER, int KT, int H, int TN>
__device__ __forceinline__ void scan_row(const float (&acc)[TN / 2], RowList<KT>& L, int64_t doc0, int64_t left,
                                         const TcParams& p) {
    constexpr int NJ = TN / 8;
    float mx = -INFINITY;
#pragma unroll
    for (int j = 0; j < NJ; ++j) mx = fmaxf(mx, fmaxf(acc[4 * j + 2 * H], acc[4 * j + 2 * H + 1]));
    if (p.probe & 4) mx = -INFINITY;
    if (!(L.active && mx >= L.thr)) return;
    // slow path: which of them reach the threshold (bit 2 j + e), then ONE copy of the insertion code over the set
    // bits, in increasing document order
    uint32_t mask = 0;
    float vals[2 * NJ];
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const float v = acc[4 * j + 2 * H + e];
            vals[2 * j + e] = v;
            mask |= ((8 * j + e < left && v >= L.thr) ? 1u : 0u) << (2 * j + e);
        }
    }
    while (mask) {
        const int b = __ffs(mask) - 1;
        mask &= mask - 1;
        const float v = vals[b] + 0.0f;                           // -0.0 -> +0.0
        const int64_t doc = doc0 + 8 * (b >> 1) + (b & 1);
        bool ok = v >= L.thr;                                     // thr may have risen inside this batch
        if (FILTER) {
            if (ok && L.want != -1) ok = (__ldg(p.doc_group + doc) == L.want);
        }
        if (ok) {
            list_insert<KT>(L.ts, L.ti, v, (int)doc + p.id_base);
            L.thr = fmaxf(L.ts[KT - 1], L.seed);
        }
    }
}

template <int KT>
__device__ __forceinline__ void row_start(RowList<KT>& L, int qg, const TcParams& p, bool filter) {
    L.qg = qg;
    L.active = qg < p.n_queries;
    L.want = (filter && L.active) ? p.q_group[qg] : -1;
#pragma unroll
    for (int j = 0; j < KT; ++j) { L.ts[j] = -INFINITY; L.ti[j] = -1; }
    // Seed: k documents with a score >= seed are already known for this query (published by units that finished
    // earlier, possibly on other SMs), so nothing below it can reach the final top-k; equal scores stay in (ties are
    // decided by id in the merge).
    L.seed = -INFINITY;
    if (L.active) {
        const int b = *reinterpret_cast<const volatile int32_t*>(p.bound + qg);
        if (b > 0) L.seed = __int_as_float(b);
    }
    L.thr = L.seed;
}

template <int KT>
__device__ __forceinline__ void row_finish(const RowList<KT>& L, int slice, int list, const TcParams& p) {
    if (!L.active) return;
    const int k = p.k;
    if (L.ti[k - 1] >= 0 && L.ts[k - 1] > 0.f)
        atomicMax(p.bound + L.qg, __float_as_int(L.ts[k - 1]));   // positive floats order like their bit patterns
    const int64_t o = (((int64_t)L.qg * p.n_slices + slice) * TC_LISTS + list) * k;
#pragma unroll
    for (int s = 0; s < KT; ++s) {
        if (s < k) {
            p.part_s[o + s] = L.ts[s];
            p.part_id[o + s] = L.ti[s];
        }
    }
}

// Warpgroup 0 = TMA producer (one thread), then QW consumer warpgroups (64 query rows each; a warpgroup issuing wgmma
// must start at a warp index that is a multiple of 4).  KT = compile-time list length (smallest of 4/8/12/16 >= k) so
// the per-thread lists stay in registers; TN = corpus rows per tile (wgmma N, 64 or 128).
// CL = 2: CTAs run in cluster pairs on the same corpus split with two neighbouring query blocks; each CTA loads HALF of
// every corpus tile and TMA-multicasts it into both CTAs' rings, so a pair pulls each tile from L2 once instead of
// twice.  A ring stage is then free only when the consumers of BOTH CTAs have released it (the peer's multicast writes
// into it), so consumers arrive on the stage's empty barrier in both CTAs.
template <bool FILTER, int KT, int QW, int TN, int CL>
__global__ void __launch_bounds__(128 + 128 * QW, 1)
dense_wgmma_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_c,
                   const TcParams p) {
    constexpr int B_STAGE_BYTES = TN * TC_KC * 2;
    extern __shared__ unsigned char smem_dyn[];
    unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~(uintptr_t)1023);
    unsigned char* smem_a = smem;                                             // [QW][kchunks] boxes of 8 KB
    unsigned char* smem_b = smem + (size_t)QW * p.kchunks * TC_A_BOX_BYTES;
    TcBarriers* bars = reinterpret_cast<TcBarriers*>(smem_b + (size_t)p.n_stages * B_STAGE_BYTES);

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    // work unit = (corpus split, group of CL neighbouring query blocks); this CTA owns query block group * CL + rank
    const int rank = CL > 1 ? (int)ptx::cluster_ctarank() : 0;
    const int worker = blockIdx.x / CL, n_workers = gridDim.x / CL;
    const int qb_groups = (p.n_qblocks + CL - 1) / CL;
    const int n_units = p.n_slices * qb_groups;

    if (threadIdx.x == 0) {
        ptx::prefetch_tensormap(&map_c);
        ptx::prefetch_tensormap(&map_q);
        ptx::mbar_init(&bars->a_full, 1);
        ptx::mbar_init(&bars->a_empty, QW);
        for (int i = 0; i < p.n_stages; ++i) {
            ptx::mbar_init(&bars->b_full[i], 1);
            ptx::mbar_init(&bars->b_empty[i], QW * CL);
        }
        ptx::fence_barrier_init();
    }
    __syncthreads();
    if (CL > 1) ptx::cluster_sync();     // the peer's barriers exist before anything is multicast into this CTA

    if (warp < 4) {
        ptx::regs_dealloc<40>();
        if (threadIdx.x == 0) {
            // ---------------- TMA producer: query block + corpus tiles of every unit of this CTA, back to back
            int stage = 0;
            uint32_t phase = 0;
            int ui = 0;
            for (int u = worker; u < n_units; u += n_workers, ++ui) {
                const int slice = u / qb_groups;
                const int q0 = ((u % qb_groups) * CL + rank) * (64 * QW);
                const int64_t row_begin = (int64_t)slice * p.rows_per_slice;
                const int64_t row_end = min(p.n_rows, row_begin + p.rows_per_slice);
                const int n_tiles = (int)((row_end - row_begin + TN - 1) / TN);
                ptx::mbar_wait(&bars->a_empty, ((uint32_t)ui & 1u) ^ 1u);    // the previous unit's MMAs are done
                ptx::mbar_expect_tx(&bars->a_full, (uint32_t)(QW * p.kchunks * TC_A_BOX_BYTES));
                for (int w = 0; w < QW; ++w)
                    for (int kc = 0; kc < p.kchunks; ++kc)
                        ptx::tma_load_2d_hint(smem_a + (size_t)(w * p.kchunks + kc) * TC_A_BOX_BYTES, &map_q, &bars->a_full,
                                              kc * TC_KC, q0 + w * 64, ptx::kEvictLast);
                for (int t = 0; t < n_tiles; ++t) {
                    const int row0 = (int)(row_begin + (int64_t)t * TN);
                    for (int kc = 0; kc < p.kchunks; ++kc) {
                        ptx::mbar_wait(&bars->b_empty[stage], phase ^ 1);
                        unsigned char* dst = smem_b + (size_t)stage * B_STAGE_BYTES;
                        if (p.probe & 1) {                       // probe: pipeline without the loads
                            ptx::mbar_arrive(&bars->b_full[stage]);
                        } else if (CL == 1) {
                            ptx::mbar_expect_tx(&bars->b_full[stage], B_STAGE_BYTES);
                            // no evict_first hint: the CTAs on the same split find this tile in L2 (measured faster)
                            ptx::tma_load_2d(dst, &map_c, &bars->b_full[stage], kc * TC_KC, row0);
                        } else {
                            // the whole tile lands here (both halves); this CTA's half goes to both CTAs
                            ptx::mbar_expect_tx(&bars->b_full[stage], B_STAGE_BYTES);
                            ptx::tma_load_2d_mcast(dst + (size_t)rank * (B_STAGE_BYTES / CL), &map_c, &bars->b_full[stage],
                                                   kc * TC_KC, row0 + rank * (TN / CL), (uint16_t)((1u << CL) - 1u));
                        }
                        if (++stage == p.n_stages) { stage = 0; phase ^= 1; }
                    }
                }
            }
        }
    } else {
        // ---------------- consumers: warpgroup cw owns query rows [64 cw, 64 cw + 64) of the block
        ptx::regs_alloc<QW == 2 ? 232 : 240>();
        const int cw = (threadIdx.x >> 7) - 1;
        const int wq = warp & 3;                            // warp within the warpgroup
        const bool leader = (threadIdx.x & 127) == 0;
        const uint32_t a_base = ptx::smem_u32(smem_a) + (uint32_t)(cw * p.kchunks * TC_A_BOX_BYTES);
        const uint32_t b_base = ptx::smem_u32(smem_b);
        // hand a ring stage back: to this CTA's producer, and with CL = 2 to the peer's (whose multicast fills it too)
        auto release = [&](int s) {
            if (CL == 1) ptx::mbar_arrive(&bars->b_empty[s]);
            else
                for (int c = 0; c < CL; ++c) ptx::mbar_arrive_cluster(&bars->b_empty[s], (uint32_t)c);
        };
        int stage = 0;
        uint32_t phase = 0;
        int ui = 0;
        for (int u = worker; u < n_units; u += n_workers, ++ui) {
            const int slice = u / qb_groups;
            const int q0 = ((u % qb_groups) * CL + rank) * (64 * QW) + cw * 64;
            const int64_t row_begin = (int64_t)slice * p.rows_per_slice;
            const int64_t row_end = min(p.n_rows, row_begin + p.rows_per_slice);
            const int n_tiles = (int)((row_end - row_begin + TN - 1) / TN);
            // this thread's two query rows (accumulator fragment rows r and r + 8)
            RowList<KT> L0, L1;
            row_start<KT>(L0, q0 + wq * 16 + (lane >> 2), p, FILTER);
            row_start<KT>(L1, q0 + wq * 16 + (lane >> 2) + 8, p, FILTER);
            ptx::mbar_wait(&bars->a_full, (uint32_t)ui & 1u);

            for (int t = 0; t < n_tiles; ++t) {
                float acc[TN / 2];
#pragma unroll
                for (int i = 0; i < TN / 2; ++i) acc[i] = 0.f;
                int prev = -1;
                for (int kc = 0; kc < p.kchunks; ++kc) {
                    ptx::mbar_wait(&bars->b_full[stage], phase);
                    if (!(p.probe & 2) || kc == 0) {
                        ptx::wgmma_fence();
#pragma unroll
                        for (int k4 = 0; k4 < TC_KC / 16; ++k4) {
                            const uint64_t da = ptx::make_desc_sw128(a_base + (uint32_t)(kc * TC_A_BOX_BYTES + k4 * 32));
                            const uint64_t db = ptx::make_desc_sw128(b_base + (uint32_t)(stage * B_STAGE_BYTES + k4 * 32));
                            if constexpr (TN == 64) ptx::wgmma_ss_n64(acc, da, db, (uint32_t)((kc | k4) != 0));
                            else ptx::wgmma_ss_n128(acc, da, db, (uint32_t)((kc | k4) != 0));
                        }
                        ptx::wgmma_commit();
                    }
                    // the previous chunk's MMAs are done: hand its stage back to the producer(s)
                    ptx::wgmma_wait<1>();
                    if (prev >= 0 && leader) release(prev);
                    prev = stage;
                    if (++stage == p.n_stages) { stage = 0; phase ^= 1; }
                }
                ptx::wgmma_wait<0>();
                ptx::fence_regs(acc);
                if (leader) {
                    release(prev);
                    if (t == n_tiles - 1) ptx::mbar_arrive(&bars->a_empty);    // the unit's last read of the query block
                }
                // ---- epilogue: this thread's TN / 4 scores of each of its two rows
                const int64_t doc0 = row_begin + (int64_t)t * TN + (lane & 3) * 2;
                scan_row<FILTER, KT, 0, TN>(acc, L0, doc0, row_end - doc0, p);
                scan_row<FILTER, KT, 1, TN>(acc, L1, doc0, row_end - doc0, p);
            }
            row_finish<KT>(L0, slice, lane & 3, p);
            row_finish<KT>(L1, slice, lane & 3, p);
        }
    }
    // no CTA leaves while its peer may still multicast into it or arrive on its barriers
    if (CL > 1) ptx::cluster_sync();
}

// The 128-query form.  Warpgroup 0 = TMA producer (one thread, register budget lowered to 40), then two consumer
// warpgroups (64 query rows each, raised to 232 registers).  A 9-warp CTA with a producer warp would not have more:
// warps are spread over the SM's four register files, and the one holding three warps caps every thread at 168.
// Each consumer keeps the first nreg = min(RQ, kchunks) k-chunks of its 64 query rows in registers as wgmma A
// fragments, loaded once per unit from global memory (the query matrix stays in L2), and only the remaining chunks
// sit in shared memory.  The freed space holds a deeper ring of 128-row corpus stages (16 KB).  Chunks below nreg
// issue the register-A form (m64n128k16, B K-major), the others the shared-memory form; every score is still the
// fp32 sum of the same k16 products in increasing k order.
template <bool FILTER, int KT>
__global__ void __launch_bounds__(384, 1)
dense_wgmma_rq_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_c,
                      const TcParams p) {
    constexpr int RQ = tc_reg_chunks(KT);
    constexpr int TN = 128;
    constexpr int B_STAGE_BYTES = TN * TC_KC * 2;
    extern __shared__ unsigned char smem_dyn[];
    unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~(uintptr_t)1023);
    const int nreg = min(RQ, p.kchunks);
    const int nsm = p.kchunks - nreg;                                         // query chunks in shared memory
    unsigned char* smem_a = smem;                                             // [2][nsm] boxes of 8 KB
    unsigned char* smem_b = smem + (size_t)2 * nsm * TC_A_BOX_BYTES;
    TcBarriers* bars = reinterpret_cast<TcBarriers*>(smem_b + (size_t)p.n_stages * B_STAGE_BYTES);

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int n_units = p.n_slices * p.n_qblocks;

    if (threadIdx.x == 0) {
        ptx::prefetch_tensormap(&map_c);
        ptx::prefetch_tensormap(&map_q);
        ptx::mbar_init(&bars->a_full, 1);
        ptx::mbar_init(&bars->a_empty, 2);
        for (int i = 0; i < p.n_stages; ++i) {
            ptx::mbar_init(&bars->b_full[i], 1);
            ptx::mbar_init(&bars->b_empty[i], 2);
        }
        ptx::fence_barrier_init();
    }
    __syncthreads();

    if (warp < 4) {
        ptx::regs_dealloc<40>();
        if (threadIdx.x == 0) {
            // ---------------- TMA producer: shared-memory query chunks + corpus tiles of every unit, back to back
            int stage = 0;
            uint32_t phase = 0;
            int ui = 0;
            for (int u = blockIdx.x; u < n_units; u += gridDim.x, ++ui) {
                const int slice = u / p.n_qblocks;
                const int q0 = (u % p.n_qblocks) * 128;
                const int64_t row_begin = (int64_t)slice * p.rows_per_slice;
                const int64_t row_end = min(p.n_rows, row_begin + p.rows_per_slice);
                const int n_tiles = (int)((row_end - row_begin + TN - 1) / TN);
                ptx::mbar_wait(&bars->a_empty, ((uint32_t)ui & 1u) ^ 1u);    // the previous unit's MMAs are done
                if (nsm == 0) {
                    ptx::mbar_arrive(&bars->a_full);
                } else {
                    ptx::mbar_expect_tx(&bars->a_full, (uint32_t)(2 * nsm * TC_A_BOX_BYTES));
                    for (int w = 0; w < 2; ++w)
                        for (int kc = nreg; kc < p.kchunks; ++kc)
                            ptx::tma_load_2d_hint(smem_a + (size_t)(w * nsm + kc - nreg) * TC_A_BOX_BYTES, &map_q,
                                                  &bars->a_full, kc * TC_KC, q0 + w * 64, ptx::kEvictLast);
                }
                for (int t = 0; t < n_tiles; ++t) {
                    const int row0 = (int)(row_begin + (int64_t)t * TN);
                    for (int kc = 0; kc < p.kchunks; ++kc) {
                        ptx::mbar_wait(&bars->b_empty[stage], phase ^ 1);
                        if (p.probe & 1) {
                            ptx::mbar_arrive(&bars->b_full[stage]);
                        } else {
                            ptx::mbar_expect_tx(&bars->b_full[stage], B_STAGE_BYTES);
                            ptx::tma_load_2d(smem_b + (size_t)stage * B_STAGE_BYTES, &map_c, &bars->b_full[stage],
                                             kc * TC_KC, row0);
                        }
                        if (++stage == p.n_stages) { stage = 0; phase ^= 1; }
                    }
                }
            }
        }
    } else {
        // ---------------- consumers: warpgroup cw owns query rows [64 cw, 64 cw + 64) of the block
        ptx::regs_alloc<232>();
        const int cw = (threadIdx.x >> 7) - 1;
        const int wq = warp & 3;
        const bool leader = (threadIdx.x & 127) == 0;
        const uint32_t a_base = ptx::smem_u32(smem_a) + (uint32_t)(cw * nsm * TC_A_BOX_BYTES);
        const uint32_t b_base = ptx::smem_u32(smem_b);
        int stage = 0;
        uint32_t phase = 0;
        int ui = 0;
        for (int u = blockIdx.x; u < n_units; u += gridDim.x, ++ui) {
            const int slice = u / p.n_qblocks;
            const int q0 = (u % p.n_qblocks) * 128 + cw * 64;
            const int64_t row_begin = (int64_t)slice * p.rows_per_slice;
            const int64_t row_end = min(p.n_rows, row_begin + p.rows_per_slice);
            const int n_tiles = (int)((row_end - row_begin + TN - 1) / TN);
            const int qr = q0 + wq * 16 + (lane >> 2);        // accumulator fragment rows qr and qr + 8
            RowList<KT> L0, L1;
            row_start<KT>(L0, qr, p, FILTER);
            row_start<KT>(L1, qr + 8, p, FILTER);
            // A fragments of the register chunks (ptx.cuh, wgmma fragment layout); rows past n_queries are zero
            uint32_t qa[RQ > 0 ? RQ : 1][4][4];
            {
                const unsigned int* r0 = reinterpret_cast<const unsigned int*>(p.queries + (int64_t)qr * p.ldq);
                const unsigned int* r1 = reinterpret_cast<const unsigned int*>(p.queries + (int64_t)(qr + 8) * p.ldq);
                const bool ok0 = qr < p.n_queries, ok1 = qr + 8 < p.n_queries;
#pragma unroll
                for (int kc = 0; kc < RQ; ++kc) {
#pragma unroll
                    for (int k4 = 0; k4 < 4; ++k4) {
                        const int c = (kc * TC_KC + k4 * 16 + 2 * (lane & 3)) >> 1;     // bf16 pair index
                        const bool in = kc < nreg;
                        qa[kc][k4][0] = (in && ok0) ? __ldg(r0 + c) : 0u;
                        qa[kc][k4][1] = (in && ok1) ? __ldg(r1 + c) : 0u;
                        qa[kc][k4][2] = (in && ok0) ? __ldg(r0 + c + 4) : 0u;
                        qa[kc][k4][3] = (in && ok1) ? __ldg(r1 + c + 4) : 0u;
                    }
                }
            }
            ptx::mbar_wait(&bars->a_full, (uint32_t)ui & 1u);

            for (int t = 0; t < n_tiles; ++t) {
                float acc[TN / 2];
#pragma unroll
                for (int i = 0; i < TN / 2; ++i) acc[i] = 0.f;
                int prev = -1;
                // the previous chunk's MMAs are done: hand its stage back to the producer
                auto next_stage = [&]() {
                    ptx::wgmma_wait<1>();
                    if (prev >= 0 && leader) ptx::mbar_arrive(&bars->b_empty[prev]);
                    prev = stage;
                    if (++stage == p.n_stages) { stage = 0; phase ^= 1; }
                };
#pragma unroll
                for (int kc = 0; kc < RQ; ++kc) {
                    if (kc < nreg) {
                        ptx::mbar_wait(&bars->b_full[stage], phase);
                        if (!(p.probe & 2) || kc == 0) {
                            ptx::wgmma_fence();
#pragma unroll
                            for (int k4 = 0; k4 < TC_KC / 16; ++k4) {
                                const uint64_t db = ptx::make_desc_sw128(b_base + (uint32_t)(stage * B_STAGE_BYTES + k4 * 32));
                                ptx::wgmma_rs_n128(acc, qa[kc][k4], db, (uint32_t)((kc | k4) != 0));
                            }
                            ptx::wgmma_commit();
                        }
                        next_stage();
                    }
                }
                for (int kc = nreg; kc < p.kchunks; ++kc) {
                    ptx::mbar_wait(&bars->b_full[stage], phase);
                    if (!(p.probe & 2)) {
                        ptx::wgmma_fence();
#pragma unroll
                        for (int k4 = 0; k4 < TC_KC / 16; ++k4) {
                            const uint64_t da = ptx::make_desc_sw128(a_base + (uint32_t)((kc - nreg) * TC_A_BOX_BYTES + k4 * 32));
                            const uint64_t db = ptx::make_desc_sw128(b_base + (uint32_t)(stage * B_STAGE_BYTES + k4 * 32));
                            ptx::wgmma_ss_n128(acc, da, db, 1u);
                        }
                        ptx::wgmma_commit();
                    }
                    next_stage();
                }
                ptx::wgmma_wait<0>();
                ptx::fence_regs(acc);
                if (leader) {
                    ptx::mbar_arrive(&bars->b_empty[prev]);
                    if (t == n_tiles - 1) ptx::mbar_arrive(&bars->a_empty);    // the unit's last read of the query block
                }
                // ---- epilogue: this thread's 32 scores of each of its two rows
                const int64_t doc0 = row_begin + (int64_t)t * TN + (lane & 3) * 2;
                scan_row<FILTER, KT, 0, TN>(acc, L0, doc0, row_end - doc0, p);
                scan_row<FILTER, KT, 1, TN>(acc, L1, doc0, row_end - doc0, p);
            }
            row_finish<KT>(L0, slice, lane & 3, p);
            row_finish<KT>(L1, slice, lane & 3, p);
        }
    }
}

// ------------------------------------------------------------------ host ----
int tc_rows_per_slice(int64_t n_rows, int slices, int tn) {
    const int64_t tiles = (n_rows + tn - 1) / tn;
    return (int)((tiles + slices - 1) / slices) * tn;
}

// Number of corpus splits.  Units = splits x query blocks are walked by `sms` persistent CTAs.
// Cost model: makespan = waves x (unit length + re-warm time of the per-thread top-k lists), in units of the time
// one CTA needs to stream the whole corpus (~45 GB/s per SM); re-warming costs ~20 us per unit.
int ts_choose_splits(int qblocks, int64_t n_rows, int dim, int sms, int tn) {
    const int64_t tiles = (n_rows + tn - 1) / tn;
    int64_t max_s = tiles / 4;                 // at least 4 tiles per unit
    if (max_s > sms) max_s = sms;
    if (max_s < 1) max_s = 1;
    const double t_corpus = (double)n_rows * dim * 2 / 45e9;
    const double eps = 20e-6 / (t_corpus > 1e-9 ? t_corpus : 1e-9);
    int best = 1;
    double best_cost = 1e30;
    for (int s = 1; s <= (int)max_s; ++s) {
        const int64_t units = (int64_t)qblocks * s;
        const int64_t waves = (units + sms - 1) / sms;
        const double cost = (double)waves * (1.0 / s + eps);
        if (cost < best_cost * (1 - 1e-9)) { best_cost = cost; best = s; }
    }
    return best;
}

bool dense_tc_supported(const __nv_bfloat16* corpus, int64_t n_rows, int dim, int64_t ldc, const __nv_bfloat16* queries,
                        int n_queries, int64_t ldq, int k) {
    if (dim % TC_KC != 0 || dim > TC_MAXD || dim <= 0) return false;
    if (k < 1 || k > TC_KMAX) return false;
    if (ldc % 8 != 0 || ldq % 8 != 0) return false;
    if ((reinterpret_cast<uintptr_t>(corpus) & 15) || (reinterpret_cast<uintptr_t>(queries) & 15)) return false;
    if (n_rows < 1 || n_queries < 1) return false;
    return true;
}

size_t dense_tc_workspace(int64_t n_rows, int dim, int n_queries, int k) {
    if (dim % TC_KC != 0 || dim > TC_MAXD || k > TC_KMAX || n_rows < 1) return 0;
    const int64_t tiles = (n_rows + TC_TN - 1) / TC_TN;
    const int slices = (int)(tiles < sm_count() ? tiles : sm_count());     // upper bound of ts_choose_splits
    const size_t n = (size_t)n_queries * slices * k * TC_LISTS;
    return align_up(n * 4, 256) * 2 + align_up((size_t)n_queries * 4, 256);      // + the per-query score bounds
}

int dense_tc_max_qw(int dim) { return dim <= 768 ? 2 : 1; }

// kernel forms: (query blocks of 64 * QW rows, corpus tiles of TN rows, CTAs per cluster)
struct TcForm { int qw, tn, cl; const char* name; };
static const TcForm kForms[4] = {{2, 128, 1, "wgmma"}, {1, 64, 1, "wgmma-q64"}, {1, 128, 1, "wgmma-q64-n128"},
                                 {1, 128, 2, "wgmma-q64-n128-mc2"}};

const char* dense_tc_form_name(int form) { return kForms[form].name; }

int dense_tc_topk(const __nv_bfloat16* corpus, int64_t n_rows, int dim, int64_t ldc, const __nv_bfloat16* queries,
                  int n_queries, int64_t ldq, int k, const int32_t* doc_group, const int32_t* q_group, int id_base,
                  float* out_scores, int32_t* out_ids, int32_t* out_counts, void* ws, size_t ws_bytes,
                  cudaStream_t st, int form) {
    const size_t need = dense_tc_workspace(n_rows, dim, n_queries, k);
    if (ws_bytes < need || !ws) {
        set_error("dense_topk(wgmma): workspace %zu < %zu", ws_bytes, need);
        return EZR_ERR_WORKSPACE;
    }
    if (form < 0 || form > 3) {
        set_error("dense_topk(wgmma): bad kernel form %d", form);
        return EZR_ERR_INVALID;
    }
    const TcForm f = kForms[form];
    if (f.qw > dense_tc_max_qw(dim)) {
        set_error("dense_topk(wgmma): %d-query blocks need dim <= 768 (got %d)", 64 * f.qw, dim);
        return EZR_ERR_UNSUPPORTED;
    }
    TcParams p;
    p.dim = dim;
    p.n_rows = n_rows;
    p.n_qblocks = (n_queries + 64 * f.qw - 1) / (64 * f.qw);
    const int sms = sm_count();
    const int qb_groups = (p.n_qblocks + f.cl - 1) / f.cl;     // work units per corpus split
    p.n_slices = ts_choose_splits(qb_groups, n_rows, dim, sms / f.cl, f.tn);
    p.rows_per_slice = tc_rows_per_slice(n_rows, p.n_slices, f.tn);
    // with the rounded-up slice size the last slices may be empty: shrink to the non-empty ones
    p.n_slices = (int)((n_rows + p.rows_per_slice - 1) / p.rows_per_slice);
    p.n_queries = n_queries;
    p.kchunks = dim / TC_KC;
    p.k = k;
    p.id_base = id_base;
    p.doc_group = doc_group;
    p.q_group = q_group;
    p.probe = g_dense_probe;
    p.queries = queries;
    p.ldq = ldq;
    const int kt = (k + 3) / 4 - 1;
    // form 0 (dense_wgmma_rq_kernel) holds the first query chunks in registers; the rest sit in shared memory
    const int reg_chunks = form == 0 ? min(tc_reg_chunks(4 * (kt + 1)), p.kchunks) : 0;
    const size_t a_bytes = (size_t)f.qw * (p.kchunks - reg_chunks) * TC_A_BOX_BYTES;
    const size_t b_stage = (size_t)f.tn * TC_KC * 2;
    const size_t fixed = 1024 /*alignment slack*/ + sizeof(TcBarriers);
    int stages = (int)((TC_SMEM_LIMIT - fixed - a_bytes) / b_stage);
    if (stages > TC_MAX_STAGES) stages = TC_MAX_STAGES;
    // leave shared memory to kernels of another stream (the BM25 route) when the caller overlaps the two routes
    if (g_dense_stage_cap > 0 && stages > g_dense_stage_cap) stages = g_dense_stage_cap;
    if (stages < 2) {
        set_error("dense_topk(wgmma): dim=%d leaves no room for a TMA ring", dim);
        return EZR_ERR_UNSUPPORTED;
    }
    p.n_stages = stages;
    const size_t smem = fixed + a_bytes + (size_t)stages * b_stage;
    const size_t n_part = (size_t)n_queries * p.n_slices * k * TC_LISTS;
    p.part_s = reinterpret_cast<float*>(ws);
    p.part_id = reinterpret_cast<int32_t*>((char*)ws + align_up(n_part * 4, 256));
    p.bound = reinterpret_cast<int32_t*>((char*)ws + need - align_up((size_t)n_queries * 4, 256));
    EZR_CUDA(cudaMemsetAsync(p.bound, 0, (size_t)n_queries * 4, st));

    CUtensorMap map_q, map_c;
    int rc = encode_tmap_2d_bf16(&map_q, queries, (uint64_t)dim, (uint64_t)n_queries, (uint64_t)ldq, TC_KC, 64);
    if (rc) return rc;
    rc = encode_tmap_2d_bf16(&map_c, corpus, (uint64_t)dim, (uint64_t)n_rows, (uint64_t)ldc, TC_KC,
                             (uint32_t)(f.tn / f.cl));
    if (rc) return rc;

    const int fi = (q_group != nullptr) ? 1 : 0;
    typedef void (*kern_t)(const CUtensorMap, const CUtensorMap, const TcParams);
#define EZR_DENSE_FORM(QW, TN, CL)                                                                                  \
    {{dense_wgmma_kernel<false, 4, QW, TN, CL>, dense_wgmma_kernel<false, 8, QW, TN, CL>,                           \
      dense_wgmma_kernel<false, 12, QW, TN, CL>, dense_wgmma_kernel<false, 16, QW, TN, CL>},                        \
     {dense_wgmma_kernel<true, 4, QW, TN, CL>, dense_wgmma_kernel<true, 8, QW, TN, CL>,                             \
      dense_wgmma_kernel<true, 12, QW, TN, CL>, dense_wgmma_kernel<true, 16, QW, TN, CL>}}
    static const kern_t table[4][2][4] = {
        {{dense_wgmma_rq_kernel<false, 4>, dense_wgmma_rq_kernel<false, 8>, dense_wgmma_rq_kernel<false, 12>,
          dense_wgmma_rq_kernel<false, 16>},
         {dense_wgmma_rq_kernel<true, 4>, dense_wgmma_rq_kernel<true, 8>, dense_wgmma_rq_kernel<true, 12>,
          dense_wgmma_rq_kernel<true, 16>}},
        EZR_DENSE_FORM(1, 64, 1), EZR_DENSE_FORM(1, 128, 1), EZR_DENSE_FORM(1, 128, 2)};
#undef EZR_DENSE_FORM
    kern_t kern = table[form][fi][kt];
    static bool attr_done[4][2][4] = {};
    if (!attr_done[form][fi][kt]) {
        EZR_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM_LIMIT));
        // always configure the SM for the largest shared-memory carveout: with a capped ring the rest of the
        // shared memory is then available to co-resident CTAs of other streams
        EZR_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
        attr_done[form][fi][kt] = true;
    }
    const int units = p.n_slices * qb_groups;
    const int workers = units < sms / f.cl ? units : sms / f.cl;
    {
        ProfScope prof(EZR_PROF_DENSE_TC, st);
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3((unsigned)(workers * f.cl));
        cfg.blockDim = dim3((unsigned)(128 + 128 * f.qw));
        cfg.dynamicSmemBytes = smem;
        cfg.stream = st;
        cudaLaunchAttribute attr[1];
        attr[0].id = cudaLaunchAttributeClusterDimension;
        attr[0].val.clusterDim.x = (unsigned)f.cl;
        attr[0].val.clusterDim.y = 1;
        attr[0].val.clusterDim.z = 1;
        cfg.attrs = attr;
        cfg.numAttrs = 1;
        EZR_CUDA(cudaLaunchKernelEx(&cfg, kern, map_q, map_c, p));
    }
    EZR_LAUNCH_CHECK();
    const int n_cand = p.n_slices * k * TC_LISTS;
    return ezr_merge_topk(p.part_s, p.part_id, EZR_F32, n_queries, n_cand, n_cand, k, out_scores, out_ids, out_counts,
                          nullptr, 0, st);
}

}  // namespace ezr
