// Dense cosine top-k for any dim % 64 == 0 and any k <= 1024 without score rows: "the candidate form"
// (ezr_dense_cand_topk).  The result is the canonical top-k under form 6's scores, bit for bit (DESIGN §4.3b).
//
// Form 6 (dense_wide.cu) writes every score to HBM, 4 MB per query per 1M rows, so its query blocks are small and each
// block rereads the corpus.  Here the encoder GEMM's mainloop (encoder/gemm_tc.cuh) runs over the corpus in chunks of
// rows, and its epilogue keeps only the scores that can still enter their query's top-k:
//
//   1. Query blocks: as many queries as fit CAND_BLOCK_BYTES of bf16 rows (one block of 10 000 queries at dim 768),
//      so the block stays in L2 while the corpus streams past it once.
//   2. Chunks: the first chunk is roundup(k, 256) rows, each later one CAND_GROWTH times the one before.  For each chunk
//      dense_cand_kernel runs the GEMM on A = the query block, W = the chunk (a tensor map based at the chunk's first
//      row, so rows past it load as zeros), M tiles fastest as form 6.  Its epilogue normalises each score as
//      EPI_SCORES does (x + 0.0f), and appends (score, id) to the query's candidate buffer when score >= T_q and the
//      row passes the filter: an atomicAdd on the query's count, stored while the slot is below the capacity.
//   3. Bound step (dense_cand_bound_kernel, one CTA per query): the canonical top-k of the buffer (the kept list and
//      the chunk's candidates) goes back, sorted, to the front of the buffer; T_q becomes its k-th score (-inf while
//      fewer than k are kept).  A buffer whose count passed the capacity marks the query overflowed: T_q = +inf, it
//      emits nothing more.  After the last chunk the same kernel writes the outputs.
//   4. Overflowed queries are listed on the device; the host reads their number (one 4-byte copy and one stream
//      synchronisation), and form 6 answers them from the workspace the candidate buffers used.
//
// Why a row is never lost: after a bound step the kept list is the canonical top-k of the filtered rows seen so far,
// and a later row has a higher id than every row seen, so it can only enter that top-k with score >= T_q -- which is
// exactly what the epilogue emits.  The scores come from the same accumulator chain as form 6's, so the capacity, the
// chunk schedule and the query block change the work done, never the result.
#include <algorithm>

#include "ezr_common.cuh"
#include "ptx.cuh"
#include "select.cuh"
#include "dense_tc.h"
#include "encoder/gemm_tc.cuh"
#include "../../include/easyrag_b200.h"

namespace ezr {

constexpr size_t CAND_BLOCK_BYTES = (size_t)16 << 20;   // bf16 query rows of one query block (L2 is 50 MB)
#ifndef EZR_CAND_GROWTH
#define EZR_CAND_GROWTH 2
#endif
// chunk c + 1 holds CAND_GROWTH times the rows of chunk c.  Measured on an H100 80GB HBM3 at 700 W (1M x 768, 10 000
// queries, k 288): 38.2 / 38.5 / 40.6 ms for 2 / 3 / 4 on random rows, and 64 / 147 / 227 ms on the clustered corpus of
// scripts/bench_dense_cand.py, where larger chunks overflow more buffers (687 / 3869 / 6984 queries) into form 6.
constexpr int CAND_GROWTH = EZR_CAND_GROWTH;
constexpr int CAND_BOUND_THREADS = 256;
constexpr int CAND_MAX_CAP = 1 << 20;
static thread_local int g_cand_cap = 0;                 // ezr_dense_cand_set_capacity; 0: cand_default_cap(k)

static int cand_default_cap(int k) { return 4 * k + 1024; }
static int cand_cap(int k) { return g_cand_cap ? g_cand_cap : cand_default_cap(k); }

struct CandParams {
    int M;                       // queries of the block
    int N;                       // rows of the chunk
    int K;                       // dim
    int tiles_m;
    int row0;                    // the chunk's first row
    int id_base;
    int cap;                     // candidate slots per query
    const float* thr;            // [M] T_q
    int32_t* cnt;                // [M] candidates in the buffer (> cap: overflowed)
    float* cand_s;               // [M][cap]
    int32_t* cand_i;             // [M][cap]
    const int32_t* doc_group;    // [n_rows] (FILTER)
    const int32_t* q_group;      // [M] (FILTER)
};

template <bool FILTER>
__global__ void __launch_bounds__(G_THREADS, 1)
dense_cand_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_c, const CandParams p) {
    // query tiles fastest, as form 6: the CTAs in flight cover every query tile of a few corpus tiles
    const int tn = blockIdx.x / p.tiles_m;
    const int tm = blockIdx.x % p.tiles_m;
    float acc[128];
    GemmThread t;
    if (!gemm_tile_mainloop(&map_q, &map_c, tm, tn, p.K / GK, acc, t)) return;

    // ---------------- epilogue: append the scores that can still reach their query's top-k
    const int cq = (t.lane & 3) * 2;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int q = tm * GM + t.cw * 64 + t.wq * 16 + (t.lane >> 2) + 8 * h;
        if (q >= p.M) continue;
        const float T = p.thr[q];
        const int g = FILTER ? p.q_group[q] : -1;
        float* cs = p.cand_s + (int64_t)q * p.cap;
        int32_t* ci = p.cand_i + (int64_t)q * p.cap;
#pragma unroll
        for (int j = 0; j < GN / 8; ++j) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const float s = acc[4 * j + 2 * h + e] + 0.0f;           // -0.0 -> +0.0, as EPI_SCORES
                const int col = tn * GN + j * 8 + cq + e;
                if (s >= T && col < p.N) {                               // >=: a later row wins a tie on its id
                    const int row = p.row0 + col;
                    if (FILTER && g != -1 && __ldg(p.doc_group + row) != g) continue;
                    const int slot = atomicAdd(p.cnt + q, 1);
                    if (slot < p.cap) {
                        cs[slot] = s;
                        ci[slot] = p.id_base + row;
                    }
                }
            }
        }
    }
}

__global__ void dense_cand_init_kernel(int n_q, float* __restrict__ thr, int32_t* __restrict__ cnt,
                                       int32_t* __restrict__ kept, int32_t* __restrict__ emitted) {
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= n_q) return;
    thr[q] = -INFINITY;
    cnt[q] = 0;
    kept[q] = 0;
    emitted[q] = 0;
}

// One CTA per query of the block (global query q0 + blockIdx.x).  Not last: the canonical top-k of the buffer goes
// back to its front, sorted, and T_q is raised.  Last: the outputs are written instead.  An overflowed query gets
// T_q = +inf and, at the last chunk, a place in the overflow list.
__global__ void __launch_bounds__(CAND_BOUND_THREADS)
dense_cand_bound_kernel(int k, int cap, int last, int q0, float* __restrict__ thr, int32_t* __restrict__ cnt,
                        int32_t* __restrict__ kept, int32_t* __restrict__ emitted, float* __restrict__ cand_s,
                        int32_t* __restrict__ cand_i, float* __restrict__ out_scores, int32_t* __restrict__ out_ids,
                        int32_t* __restrict__ out_counts, int32_t* __restrict__ out_cand,
                        int32_t* __restrict__ over_list, int32_t* __restrict__ over_n) {
    extern __shared__ unsigned char smem_dyn[];
    const int q = blockIdx.x;
    const int64_t gq = (int64_t)q0 + q;
    const int n = cnt[q];
    if (n > cap) {                                   // overflowed, at this chunk or an earlier one
        if (threadIdx.x == 0) {
            thr[q] = INFINITY;
            if (last) {
                if (out_cand) out_cand[gq] = -1;
                over_list[atomicAdd(over_n, 1)] = (int32_t)gq;
            }
        }
        return;
    }
    const int prev = kept[q];
    if (!last && n == prev) return;                  // nothing new: the kept list and T_q stand
    SelSmem<float> m = sel_carve<float>(smem_dyn);
    sel_init<float>(m);
    float* cs = cand_s + (int64_t)q * cap;
    int32_t* ci = cand_i + (int64_t)q * cap;
    for (int base = 0; base < n; base += CAND_BOUND_THREADS) {
        const int i = base + threadIdx.x;
        if (i < n) sel_push<float>(m, cs[i], ci[i]);
        sel_maybe_flush<float>(m, k);
    }
    sel_compact<float>(m, k);
    const int got = *m.cnt;
    if (last) {
        for (int i = threadIdx.x; i < k; i += blockDim.x) {
            out_scores[gq * k + i] = i < got ? m.ks[i] : -INFINITY;
            out_ids[gq * k + i] = i < got ? m.kid[i] : -1;
        }
        if (threadIdx.x == 0) {
            if (out_counts) out_counts[gq] = got;
            if (out_cand) out_cand[gq] = emitted[q] + (n - prev);
        }
        return;
    }
    for (int i = threadIdx.x; i < got; i += blockDim.x) {
        cs[i] = m.ks[i];
        ci[i] = m.kid[i];
    }
    if (threadIdx.x == 0) {
        cnt[q] = got;
        kept[q] = got;
        emitted[q] += n - prev;
        thr[q] = got >= k ? m.ks[k - 1] : -INFINITY;
    }
}

// the overflowed queries' rows (and filter classes), packed for form 6
__global__ void dense_cand_gather_kernel(const __nv_bfloat16* __restrict__ q, int64_t ldq, int dim,
                                         const int32_t* __restrict__ q_group, const int32_t* __restrict__ over_list,
                                         __nv_bfloat16* __restrict__ out, int32_t* __restrict__ out_group) {
    const int i = blockIdx.x;
    const int src = over_list[i];
    for (int c = threadIdx.x; c < dim; c += blockDim.x) out[(int64_t)i * dim + c] = q[(int64_t)src * ldq + c];
    if (threadIdx.x == 0 && q_group) out_group[i] = q_group[src];
}

// form 6's answers for the overflowed queries, into the caller's rows
__global__ void dense_cand_scatter_kernel(int k, const int32_t* __restrict__ over_list, const float* __restrict__ fb_s,
                                          const int32_t* __restrict__ fb_i, const int32_t* __restrict__ fb_c,
                                          float* __restrict__ out_scores, int32_t* __restrict__ out_ids,
                                          int32_t* __restrict__ out_counts) {
    const int i = blockIdx.x;
    const int64_t dst = over_list[i];
    const int got = fb_c[i];
    for (int j = threadIdx.x; j < k; j += blockDim.x) {
        out_scores[dst * k + j] = j < got ? fb_s[(int64_t)i * k + j] : -INFINITY;
        out_ids[dst * k + j] = j < got ? fb_i[(int64_t)i * k + j] : -1;
    }
    if (threadIdx.x == 0 && out_counts) out_counts[dst] = got;
}

// ------------------------------------------------------------------ host ----
// over_list / over_n live through the call; the candidate state and the fallback's buffers share one region (the
// candidate buffers are dead once the outputs are written).
struct CandLayout {
    size_t over_list, over_n, region;
    size_t thr, cnt, kept, emitted, cand_s, cand_i;         // candidate pass (offsets from region)
    size_t g_q, g_group, fb_s, fb_i, fb_c, wide;            // fallback (offsets from region)
    size_t total;
};

static CandLayout cand_layout(int64_t n_rows, int dim, int n_q, int k, int cap) {
    CandLayout l;
    size_t o = 0;
    auto take = [&](size_t bytes) { const size_t at = o; o += align_up(bytes, 256); return at; };
    l.over_list = take((size_t)n_q * 4);
    l.over_n = take(4);
    l.region = o;
    o = 0;
    l.thr = take((size_t)n_q * 4);
    l.cnt = take((size_t)n_q * 4);
    l.kept = take((size_t)n_q * 4);
    l.emitted = take((size_t)n_q * 4);
    l.cand_s = take((size_t)n_q * cap * 4);
    l.cand_i = take((size_t)n_q * cap * 4);
    const size_t cand_end = o;
    o = 0;
    l.g_q = take((size_t)n_q * dim * 2);
    l.g_group = take((size_t)n_q * 4);
    l.fb_s = take((size_t)n_q * k * 4);
    l.fb_i = take((size_t)n_q * k * 4);
    l.fb_c = take((size_t)n_q * 4);
    l.wide = o;
    // form 6 runs the largest query block the rest of the region holds: at least one query
    const size_t fb_end = o + dense_wide_workspace(n_rows, n_q, k, 1);
    l.total = l.region + std::max(cand_end, fb_end);
    return l;
}

// queries per block: the bf16 rows stay within CAND_BLOCK_BYTES, in whole 128-query tiles
static int cand_block_queries(int dim, int n_queries) {
    int64_t qb = (int64_t)(CAND_BLOCK_BYTES / ((size_t)dim * 2)) / GM * GM;
    qb = std::max<int64_t>(qb, GM);
    return (int)std::min<int64_t>(qb, n_queries);
}

static int cand_launch_chunk(const CUtensorMap& map_q, const __nv_bfloat16* corpus, int64_t ldc, int dim,
                             int64_t row0, int rows, CandParams p, bool filter, cudaStream_t st) {
    CUtensorMap map_c;
    const int rc = encode_tmap_2d_bf16(&map_c, corpus + row0 * ldc, (uint64_t)dim, (uint64_t)rows, (uint64_t)ldc, GK,
                                       GN);
    if (rc) return rc;
    p.N = rows;
    p.row0 = (int)row0;
    typedef void (*kern_t)(const CUtensorMap, const CUtensorMap, const CandParams);
    static const kern_t table[2] = {dense_cand_kernel<false>, dense_cand_kernel<true>};
    static bool attr_done[2] = {false, false};
    const int fi = filter ? 1 : 0;
    if (!attr_done[fi]) {
        EZR_CUDA(cudaFuncSetAttribute(table[fi], cudaFuncAttributeMaxDynamicSharedMemorySize, (int)G_SMEM_BYTES));
        attr_done[fi] = true;
    }
    const int64_t tiles = (int64_t)p.tiles_m * ((rows + GN - 1) / GN);
    {
        ProfScope prof(EZR_PROF_DENSE_CAND_GEMM, st);
        table[fi]<<<(unsigned)tiles, G_THREADS, G_SMEM_BYTES, st>>>(map_q, map_c, p);
    }
    EZR_LAUNCH_CHECK();
    return EZR_OK;
}

}  // namespace ezr

using namespace ezr;

extern "C" {

int ezr_dense_cand_set_capacity(int32_t cap) {
    EZR_CHECK_ARG(cap >= 0 && cap <= CAND_MAX_CAP,
                  "dense_cand_set_capacity: 0 (default, 4k + 1024) or 1..2^20 candidates per query");
    g_cand_cap = cap;
    return EZR_OK;
}

size_t ezr_dense_cand_topk_workspace(int64_t n_rows, int32_t dim, int32_t n_queries, int32_t k) {
    if (n_rows <= 0 || n_queries <= 0 || k <= 0 || dim <= 0) return 0;
    return cand_layout(n_rows, dim, n_queries, k, cand_cap(k)).total;
}

int ezr_dense_cand_topk(const void* corpus_bf16, int64_t n_rows, int32_t dim, int64_t ld_corpus,
                        const void* queries_bf16, int32_t n_queries, int64_t ld_queries, int32_t k,
                        const int32_t* doc_group, const int32_t* q_group, int32_t id_base, float* out_scores,
                        int32_t* out_ids, int32_t* out_counts, int32_t* out_cand_counts, void* workspace,
                        size_t workspace_bytes, void* stream) {
    EZR_CHECK_ARG(k >= 1 && k <= 1024, "dense_cand_topk: k=%d out of [1,1024]", k);
    EZR_CHECK_ARG(dim >= 1, "dense_cand_topk: dim must be >= 1");
    EZR_CHECK_ARG(n_rows >= 0 && n_rows < ((int64_t)1 << 31), "dense_cand_topk: n_rows out of range");
    EZR_CHECK_ARG(n_queries >= 0, "dense_cand_topk: n_queries < 0");
    EZR_CHECK_ARG(ld_corpus >= dim && ld_queries >= dim, "dense_cand_topk: row stride smaller than dim");
    // an empty shard's doc_group is empty, and an empty tensor has no address: nothing is filtered, so no check
    EZR_CHECK_ARG(q_group == nullptr || doc_group != nullptr || n_rows == 0,
                  "dense_cand_topk: q_group without doc_group");
    cudaStream_t st = (cudaStream_t)stream;
    if (n_queries == 0) return EZR_OK;
    if (n_rows == 0) {
        if (out_counts) EZR_CUDA(cudaMemsetAsync(out_counts, 0, (size_t)n_queries * 4, st));
        if (out_cand_counts) EZR_CUDA(cudaMemsetAsync(out_cand_counts, 0, (size_t)n_queries * 4, st));
        EZR_CUDA(cudaMemsetAsync(out_ids, 0xff, (size_t)n_queries * k * 4, st));
        return EZR_OK;
    }
    const __nv_bfloat16* c = reinterpret_cast<const __nv_bfloat16*>(corpus_bf16);
    const __nv_bfloat16* qv = reinterpret_cast<const __nv_bfloat16*>(queries_bf16);
    if (!dense_wide_supported(c, n_rows, dim, ld_corpus, qv, ld_queries)) {
        set_error("dense_cand_topk: shape unsupported (needs dim %% 64 == 0, row strides %% 8 == 0, 16-byte aligned "
                  "rows; dim=%d ld=%lld/%lld)", dim, (long long)ld_corpus, (long long)ld_queries);
        return EZR_ERR_UNSUPPORTED;
    }
    const int cap = cand_cap(k);
    const CandLayout l = cand_layout(n_rows, dim, n_queries, k, cap);
    if (!workspace || workspace_bytes < l.total) {
        set_error("dense_cand_topk: workspace %zu < %zu", workspace ? workspace_bytes : (size_t)0, l.total);
        return EZR_ERR_WORKSPACE;
    }
    char* ws = reinterpret_cast<char*>(workspace);
    char* reg = ws + l.region;
    int32_t* over_list = reinterpret_cast<int32_t*>(ws + l.over_list);
    int32_t* over_n = reinterpret_cast<int32_t*>(ws + l.over_n);
    float* thr = reinterpret_cast<float*>(reg + l.thr);
    int32_t* cnt = reinterpret_cast<int32_t*>(reg + l.cnt);
    int32_t* kept = reinterpret_cast<int32_t*>(reg + l.kept);
    int32_t* emitted = reinterpret_cast<int32_t*>(reg + l.emitted);
    float* cand_s = reinterpret_cast<float*>(reg + l.cand_s);
    int32_t* cand_i = reinterpret_cast<int32_t*>(reg + l.cand_i);
    const bool filter = q_group != nullptr;

    static bool bound_attr = false;
    if (!bound_attr) {
        EZR_CUDA(cudaFuncSetAttribute(dense_cand_bound_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      (int)sel_smem_bytes<float>()));
        bound_attr = true;
    }
    EZR_CUDA(cudaMemsetAsync(over_n, 0, 4, st));
    {
        ProfScope prof(EZR_PROF_DENSE_CAND_BOUND, st);
        dense_cand_init_kernel<<<(unsigned)((n_queries + 255) / 256), 256, 0, st>>>(n_queries, thr, cnt, kept, emitted);
    }
    EZR_LAUNCH_CHECK();

    const int qb = cand_block_queries(dim, n_queries);
    const int64_t first = ((int64_t)k + GN - 1) / GN * GN;
    for (int q0 = 0; q0 < n_queries; q0 += qb) {
        const int nb = std::min(qb, n_queries - q0);
        CUtensorMap map_q;
        int rc = encode_tmap_2d_bf16(&map_q, qv + (int64_t)q0 * ld_queries, (uint64_t)dim, (uint64_t)nb,
                                     (uint64_t)ld_queries, GK, GM);
        if (rc) return rc;
        CandParams p;
        p.M = nb;
        p.K = dim;
        p.tiles_m = (nb + GM - 1) / GM;
        p.id_base = id_base;
        p.cap = cap;
        p.thr = thr + q0;
        p.cnt = cnt + q0;
        p.cand_s = cand_s + (int64_t)q0 * cap;
        p.cand_i = cand_i + (int64_t)q0 * cap;
        p.doc_group = doc_group;
        p.q_group = filter ? q_group + q0 : nullptr;
        int64_t rows = first;
        for (int64_t row0 = 0; row0 < n_rows; row0 += rows, rows *= CAND_GROWTH) {
            const int n_chunk = (int)std::min(rows, n_rows - row0);
            rc = cand_launch_chunk(map_q, c, ld_corpus, dim, row0, n_chunk, p, filter, st);
            if (rc) return rc;
            const int last = row0 + n_chunk >= n_rows ? 1 : 0;
            {
                ProfScope prof(EZR_PROF_DENSE_CAND_BOUND, st);
                dense_cand_bound_kernel<<<nb, CAND_BOUND_THREADS, sel_smem_bytes<float>(), st>>>(
                    k, cap, last, q0, thr + q0, cnt + q0, kept + q0, emitted + q0, p.cand_s, p.cand_i, out_scores,
                    out_ids, out_counts, out_cand_counts, over_list, over_n);
            }
            EZR_LAUNCH_CHECK();
        }
    }

    // the host learns how many queries overflowed (one small copy + stream sync) to size form 6's run
    int32_t n_over = 0;
    EZR_CUDA(cudaMemcpyAsync(&n_over, over_n, 4, cudaMemcpyDeviceToHost, st));
    EZR_CUDA(cudaStreamSynchronize(st));
    if (n_over == 0) return EZR_OK;
    __nv_bfloat16* g_q = reinterpret_cast<__nv_bfloat16*>(reg + l.g_q);
    int32_t* g_group = reinterpret_cast<int32_t*>(reg + l.g_group);
    float* fb_s = reinterpret_cast<float*>(reg + l.fb_s);
    int32_t* fb_i = reinterpret_cast<int32_t*>(reg + l.fb_i);
    int32_t* fb_c = reinterpret_cast<int32_t*>(reg + l.fb_c);
    {
        ProfScope prof(EZR_PROF_DENSE_WIDE, st);
        dense_cand_gather_kernel<<<n_over, 256, 0, st>>>(qv, ld_queries, dim, q_group, over_list, g_q, g_group);
    }
    EZR_LAUNCH_CHECK();
    const int rc = dense_wide_topk(c, n_rows, dim, ld_corpus, g_q, n_over, dim, k, doc_group,
                                   filter ? g_group : nullptr, id_base, fb_s, fb_i, fb_c, reg + l.wide,
                                   workspace_bytes - l.region - l.wide, st);
    if (rc) return rc;
    {
        ProfScope prof(EZR_PROF_DENSE_WIDE, st);
        dense_cand_scatter_kernel<<<n_over, 256, 0, st>>>(k, over_list, fb_s, fb_i, fb_c, out_scores, out_ids,
                                                          out_counts);
    }
    EZR_LAUNCH_CHECK();
    return EZR_OK;
}

}  // extern "C"
