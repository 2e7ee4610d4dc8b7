// Dense cosine top-k: dispatch + the generic SIMT kernel.
//
// Replaces QdrantRetriever._aretrieve's vector search (retrievers.py:37-52 ->
// QdrantVectorStore.aquery on a Distance.COSINE collection, ingestion.py:180-182).
// The fast path is the wgmma kernel in dense_tc.cu (bf16, dim % 64 == 0, dim <= 1024,
// k <= 16); everything else (odd dims, k up to 1024 as used by the drop-in
// retrievers with f_topk_1 = 288) goes through the kernel below: a plain tiled
// fp32-FMA score kernel writing a block of score rows, followed by the generic
// row top-k.  Same canonical order, same filter semantics.  Form 6 (dense_wide.cu,
// opt-in through ezr_dense_set_kernel(6)) writes the score rows with the encoder's
// wgmma GEMM instead, for any dim % 64 == 0; both go through score_rows_topk below.
#include "ezr_common.cuh"
#include "dense_tc.h"
#include "../../include/easyrag_b200.h"

namespace ezr {

constexpr int kSimtTile = 64;
constexpr int kSimtK = 32;

// SEP: separate __fmul_rn / __fadd_rn (the rescore arithmetic of dense_s8.cu) instead of fmaf
template <bool SEP>
__global__ void __launch_bounds__(256)
dense_scores_simt_kernel(const __nv_bfloat16* __restrict__ corpus, int64_t n_rows, int dim, int64_t ldc,
                         const __nv_bfloat16* __restrict__ queries, int n_q, int64_t ldq, float* __restrict__ out,
                         int64_t ldo) {
    __shared__ float sC[kSimtTile][kSimtK + 1];
    __shared__ float sQ[kSimtTile][kSimtK + 1];
    const int64_t r0 = (int64_t)blockIdx.x * kSimtTile;
    const int q0 = blockIdx.y * kSimtTile;
    const int tid = threadIdx.x;
    const int tx = tid & 15, ty = tid >> 4;
    float acc[4][4];
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int i = 0; i < 4; ++i) acc[j][i] = 0.f;

    for (int k0 = 0; k0 < dim; k0 += kSimtK) {
        for (int e = tid; e < kSimtTile * kSimtK; e += 256) {
            const int rr = e / kSimtK, kk = e % kSimtK;
            const int64_t row = r0 + rr;
            const int col = k0 + kk;
            sC[rr][kk] = (row < n_rows && col < dim) ? __bfloat162float(corpus[row * ldc + col]) : 0.f;
            const int qq = q0 + rr;
            sQ[rr][kk] = (qq < n_q && col < dim) ? __bfloat162float(queries[(int64_t)qq * ldq + col]) : 0.f;
        }
        __syncthreads();
#pragma unroll 8
        for (int kk = 0; kk < kSimtK; ++kk) {
            float a[4], b[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) a[i] = sC[tx * 4 + i][kk];
#pragma unroll
            for (int j = 0; j < 4; ++j) b[j] = sQ[ty * 4 + j][kk];
#pragma unroll
            for (int j = 0; j < 4; ++j)
#pragma unroll
                for (int i = 0; i < 4; ++i) acc[j][i] = SEP ? __fadd_rn(acc[j][i], __fmul_rn(b[j], a[i])) : fmaf(a[i], b[j], acc[j][i]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int qq = q0 + ty * 4 + j;
        if (qq >= n_q) continue;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int64_t row = r0 + tx * 4 + i;
            if (row < n_rows) out[(int64_t)qq * ldo + row] = acc[j][i] + 0.0f;   // -0.0 -> +0.0
        }
    }
}

static int simt_block_queries(int64_t n_rows, int n_queries) {
    // score rows of one query block stay under 256 MB
    int64_t qb = ((int64_t)256 << 20) / (n_rows > 0 ? n_rows * 4 : 4);
    if (qb < 1) qb = 1;
    if (qb > 1024) qb = 1024;
    if (qb > n_queries) qb = n_queries;
    return (int)qb;
}

template <bool SEP>
static int simt_scores(const __nv_bfloat16* corpus, int64_t n_rows, int dim, int64_t ldc,
                       const __nv_bfloat16* queries, int nq, int64_t ldq, float* out, cudaStream_t st) {
    dim3 grid(ceil_div(n_rows, kSimtTile), ceil_div(nq, kSimtTile));
    {
        ProfScope prof(EZR_PROF_DENSE_SIMT, st);
        dense_scores_simt_kernel<SEP><<<grid, 256, 0, st>>>(corpus, n_rows, dim, ldc, queries, nq, ldq, out, n_rows);
    }
    EZR_LAUNCH_CHECK();
    return EZR_OK;
}

// A block of m queries: its score rows, then the select workspace behind them.  The last block of a call may be
// smaller than the others and its select may need more (it splits each row into more parts); its rows take less room.
static size_t score_block_bytes(int64_t n_rows, int m, int k) {
    return align_up((size_t)m * n_rows * 4, 256) + ezr_select_rows_workspace(m, n_rows, k, EZR_F32);
}

size_t score_rows_workspace(int64_t n_rows, int n_queries, int k, int block_queries) {
    if (n_rows <= 0 || n_queries <= 0 || k <= 0 || block_queries <= 0) return 0;
    const int qb = block_queries < n_queries ? block_queries : n_queries;
    size_t need = score_block_bytes(n_rows, qb, k);
    const int last = n_queries % qb;
    if (last) {
        const size_t l = score_block_bytes(n_rows, last, k);
        if (l > need) need = l;
    }
    return need;
}

int score_rows_topk(score_rows_fn score, int block_queries, const __nv_bfloat16* corpus, int64_t n_rows, int dim,
                    int64_t ldc, const __nv_bfloat16* queries, int n_queries, int64_t ldq, int k,
                    const int32_t* doc_group, const int32_t* q_group, int id_base, float* out_scores, int32_t* out_ids,
                    int32_t* out_counts, void* ws, size_t ws_bytes, cudaStream_t st) {
    const size_t need = score_rows_workspace(n_rows, n_queries, k, block_queries);
    if (ws_bytes < need || !ws) {
        set_error("dense_topk: workspace %zu < %zu (score rows of %d-query blocks)", ws_bytes, need, block_queries);
        return EZR_ERR_WORKSPACE;
    }
    float* rows = reinterpret_cast<float*>(ws);
    for (int q0 = 0; q0 < n_queries; q0 += block_queries) {
        const int nq = n_queries - q0 < block_queries ? n_queries - q0 : block_queries;
        int rc = score(corpus, n_rows, dim, ldc, queries + (int64_t)q0 * ldq, nq, ldq, rows, st);
        if (rc) return rc;
        // this block's select workspace sits right behind its own rows (see score_block_bytes)
        const size_t rows_bytes = align_up((size_t)nq * n_rows * 4, 256);
        rc = ezr_select_rows(rows, EZR_F32, nq, n_rows, n_rows, k, 0, doc_group, q_group ? q_group + q0 : nullptr,
                             id_base, out_scores + (int64_t)q0 * k, out_ids + (int64_t)q0 * k,
                             out_counts ? out_counts + q0 : nullptr, (char*)ws + rows_bytes, ws_bytes - rows_bytes, st);
        if (rc) return rc;
    }
    return EZR_OK;
}

// Covers every call with at most n_queries queries, including a last query block smaller than the others (the
// select workspace of fewer rows can be larger: it splits each row into more parts).
size_t dense_exact_workspace(int64_t n_rows, int n_queries, int k) {
    const int qb = simt_block_queries(n_rows, n_queries);
    size_t sel = 0;
    for (int m = 1; m <= qb; ++m) {
        const size_t s = ezr_select_rows_workspace(m, n_rows, k, EZR_F32);
        if (s > sel) sel = s;
    }
    return align_up((size_t)qb * n_rows * 4, 256) + sel;
}

int dense_exact_topk(const __nv_bfloat16* corpus, int64_t n_rows, int dim, int64_t ldc, const __nv_bfloat16* queries,
                     int n_queries, int64_t ldq, int k, const int32_t* doc_group, const int32_t* q_group, int id_base,
                     float* out_scores, int32_t* out_ids, int32_t* out_counts, void* ws, size_t ws_bytes,
                     cudaStream_t st) {
    return score_rows_topk(simt_scores<true>, simt_block_queries(n_rows, n_queries), corpus, n_rows, dim, ldc, queries,
                           n_queries, ldq, k, doc_group, q_group, id_base, out_scores, out_ids, out_counts, ws, ws_bytes,
                           st);
}

static thread_local int g_force_kernel = 0;
static thread_local const char* g_last_kernel = "none";

}  // namespace ezr

namespace ezr {
// Insert path of the vector store (a Distance.COSINE collection normalises at insert, ingestion.py:180-182):
// out[r] = bf16( x[r] / max(||x[r]||_2, 1e-12) ), fp32 math, one warp per row.  SRC = float or __nv_bfloat16.
template <typename SRC>
__global__ void normalize_rows_kernel(const SRC* __restrict__ x, int64_t ldx, int64_t n_rows, int dim,
                                      __nv_bfloat16* __restrict__ out, int64_t ldo) {
    const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= n_rows) return;
    const SRC* xr = x + row * ldx;
    float q = 0.f;
    for (int i = lane; i < dim; i += 32) {
        const float v = (float)xr[i];
        q = fmaf(v, v, q);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
    const float inv = 1.0f / fmaxf(sqrtf(q), 1e-12f);
    for (int i = lane; i < dim; i += 32) out[row * ldo + i] = __float2bfloat16((float)xr[i] * inv);
}
}  // namespace ezr

using namespace ezr;

extern "C" {

int ezr_dense_set_kernel(int32_t which) {
    EZR_CHECK_ARG(which >= 0 && which <= 6,
                  "dense_set_kernel: 0 auto, 1 simt, 2 wgmma (128-query blocks, dim <= 768), 3 wgmma (64-query blocks), "
                  "4 wgmma (64-query blocks, 128-row corpus tiles), 5 = 4 in cluster pairs (multicast corpus tiles), "
                  "6 wgmma score rows + select (any dim %% 64 == 0, k <= 1024)");
    g_force_kernel = which;
    return EZR_OK;
}

const char* ezr_dense_last_kernel(void) { return g_last_kernel; }

int ezr_dense_set_probe(int32_t probe) {
    EZR_CHECK_ARG(probe >= 0 && probe <= 7, "dense_set_probe: bit mask 0..7");
    g_dense_probe = probe;
    return EZR_OK;
}

int ezr_dense_set_stage_cap(int32_t stages) {
    EZR_CHECK_ARG(stages == 0 || stages >= 2, "dense_set_stage_cap: 0 (no cap) or >= 2 TMA stages");
    g_dense_stage_cap = stages;
    return EZR_OK;
}

size_t ezr_dense_topk_workspace(int64_t n_rows, int32_t dim, int32_t n_queries, int32_t k) {
    if (n_rows <= 0 || n_queries <= 0 || k <= 0) return 0;
    size_t a = score_rows_workspace(n_rows, n_queries, k, simt_block_queries(n_rows, n_queries));
    size_t b = dense_tc_workspace(n_rows, dim, n_queries, k);
    return a > b ? a : b;
}

int ezr_dense_topk(const void* corpus_bf16, int64_t n_rows, int32_t dim, int64_t ld_corpus,
                   const void* queries_bf16, int32_t n_queries, int64_t ld_queries, int32_t k,
                   const int32_t* doc_group, const int32_t* q_group, int32_t id_base, float* out_scores,
                   int32_t* out_ids, int32_t* out_counts, void* workspace, size_t workspace_bytes, void* stream) {
    EZR_CHECK_ARG(k >= 1 && k <= 1024, "dense_topk: k=%d out of [1,1024]", k);
    EZR_CHECK_ARG(dim >= 1, "dense_topk: dim must be >= 1");
    EZR_CHECK_ARG(n_rows >= 0 && n_rows < ((int64_t)1 << 31), "dense_topk: n_rows out of range");
    EZR_CHECK_ARG(ld_corpus >= dim && ld_queries >= dim, "dense_topk: row stride smaller than dim");
    // an empty shard's doc_group is empty, and an empty tensor has no address: nothing is filtered, so no check
    EZR_CHECK_ARG(q_group == nullptr || doc_group != nullptr || n_rows == 0, "dense_topk: q_group without doc_group");
    cudaStream_t st = (cudaStream_t)stream;
    if (n_queries == 0) return EZR_OK;
    if (n_rows == 0) {
        if (out_counts) EZR_CUDA(cudaMemsetAsync(out_counts, 0, (size_t)n_queries * 4, st));
        EZR_CUDA(cudaMemsetAsync(out_ids, 0xff, (size_t)n_queries * k * 4, st));
        return EZR_OK;
    }
    const __nv_bfloat16* c = reinterpret_cast<const __nv_bfloat16*>(corpus_bf16);
    const __nv_bfloat16* q = reinterpret_cast<const __nv_bfloat16*>(queries_bf16);
    if (g_force_kernel == 6) {
        if (!dense_wide_supported(c, n_rows, dim, ld_corpus, q, ld_queries)) {
            set_error("dense_topk: wgmma-scores kernel forced but shape unsupported (needs dim %% 64 == 0, row strides "
                      "%% 8 == 0, 16-byte aligned rows; dim=%d ld=%lld/%lld)", dim, (long long)ld_corpus,
                      (long long)ld_queries);
            return EZR_ERR_UNSUPPORTED;
        }
        g_last_kernel = "wgmma-scores";
        return dense_wide_topk(c, n_rows, dim, ld_corpus, q, n_queries, ld_queries, k, doc_group, q_group, id_base,
                               out_scores, out_ids, out_counts, workspace, workspace_bytes, st);
    }
    const bool tc_ok = dense_tc_supported(c, n_rows, dim, ld_corpus, q, n_queries, ld_queries, k);
    if (g_force_kernel >= 2 && !tc_ok) {
        set_error("dense_topk: wgmma kernel forced but shape unsupported (dim=%d k=%d ld=%lld)", dim, k,
                  (long long)ld_corpus);
        return EZR_ERR_UNSUPPORTED;
    }
    if (tc_ok && g_force_kernel != 1) {
        // auto (measured on one H100, 1M rows): 128-query blocks while they fit (dim <= 768) and the batch fills them
        // (23.7 ms with query chunks in registers and 128-row tiles vs 34.9 ms for 64-query blocks, 10k queries at
        // dim 768; 0.87 ms at 256 queries); otherwise 64-query blocks with 128-row corpus tiles
        // (dim 1024, 10k queries: 43.6 vs 60.4 ms for 64-row tiles; 64 queries at dim 768: 0.59 vs 0.68 ms)
        const bool wide_block = dense_tc_max_qw(dim) == 2 && n_queries > 64;
        const int form = g_force_kernel >= 2 ? g_force_kernel - 2 : (wide_block ? 0 : 2);
        g_last_kernel = dense_tc_form_name(form);
        return dense_tc_topk(c, n_rows, dim, ld_corpus, q, n_queries, ld_queries, k, doc_group, q_group, id_base,
                             out_scores, out_ids, out_counts, workspace, workspace_bytes, st, form);
    }
    g_last_kernel = "simt";
    return score_rows_topk(simt_scores<false>, simt_block_queries(n_rows, n_queries), c, n_rows, dim, ld_corpus, q,
                           n_queries, ld_queries, k, doc_group, q_group, id_base, out_scores, out_ids, out_counts,
                           workspace, workspace_bytes, st);
}

int ezr_normalize_rows(const void* x, int32_t x_is_f32, int64_t ldx, int64_t n_rows, int32_t dim, void* out_bf16,
                       int64_t ldo, void* stream) {
    EZR_CHECK_ARG(dim >= 1 && ldx >= dim && ldo >= dim, "normalize_rows: bad dim / strides");
    if (n_rows <= 0) return EZR_OK;
    cudaStream_t st = (cudaStream_t)stream;
    const int wpb = 8;
    const unsigned grid = (unsigned)((n_rows + wpb - 1) / wpb);
    if (x_is_f32)
        normalize_rows_kernel<float><<<grid, wpb * 32, 0, st>>>((const float*)x, ldx, n_rows, dim, (__nv_bfloat16*)out_bf16, ldo);
    else
        normalize_rows_kernel<__nv_bfloat16><<<grid, wpb * 32, 0, st>>>((const __nv_bfloat16*)x, ldx, n_rows, dim,
                                                                     (__nv_bfloat16*)out_bf16, ldo);
    EZR_LAUNCH_CHECK();
    return EZR_OK;
}

}  // extern "C"
