// BM25 index construction on the GPU: tokenised corpus -> term-major postings (CSC) with term frequencies.
//
// Replaces the Python dict building of BM25Retriever.__init__ (retrievers.py:98-118 -> rank_bm25.BM25Okapi.__init__:
// per-document frequency dicts, nd[word] += 1, doc_len) and the first-seen term order that rank_bm25's sequential
// idf sum depends on.  Everything that has to be bit-identical to CPython (math.log, the float64 sum) stays on the
// host (easyrag_b200/index.py); these kernels only count, sort and place integers:
//
//   1. bm25_doc_unique_kernel   one CTA per document: (term, position) keys sorted in shared memory (bitonic), runs of
//                               equal terms -> (term, tf) pairs in a doc-major scratch list; per term: document
//                               frequency per 8192-document block (atomicAdd on a [vocab][blocks+1] table) and the
//                               position of its first occurrence in the corpus (atomicMin).
//   2. bm25_block_scan_kernel   per term: exclusive scan of its per-block counts -> block offsets, df.
//      bm25_indptr_scan_kernel  exclusive scan of df over the vocabulary -> indptr (int64).
//   3. bm25_place_kernel        one CTA per document block walks its documents IN ORDER; every (term, tf) pair of a
//                               document takes the next free slot of its (term, block) segment.  Only this CTA touches
//                               the segment, so no atomics are needed and postings come out sorted by document id
//                               without a sort: (block offsets are ascending, slots inside a block are handed out in
//                               document order).
//   4. bm25_shard_*             a row shard's postings are a contiguous sub-segment of every term's list: two binary
//                               searches per term, a scan, one copy (global idf / avgdl stay global, SURVEY.md 8(e)).
#include "ezr_common.cuh"
#include "bm25_common.cuh"
#include "../../include/easyrag_b200.h"

namespace ezr {

constexpr int kBuildThreads = 256;
constexpr int kBuildCap = 8192;          // tokens of a document sorted in shared memory (64 KB of 64-bit keys)
constexpr int kBuildBlock = 8192;        // documents per placement block (independent of the query-time range)

// status[0] != 0: a token id outside [0, vocab) was seen (its document index + 1)
// LONG = false: documents of at most kBuildCap tokens, keys in shared memory; longer ones are skipped.
// LONG = true : blockIdx.x indexes long_docs[], keys live in the global scratch long_keys at long_off[i].
template <bool LONG>
__global__ void __launch_bounds__(kBuildThreads)
bm25_doc_unique_kernel(const int32_t* __restrict__ tokens, const int64_t* __restrict__ doc_ptr, int64_t n_docs, int32_t vocab,
                       int32_t n_blocks, int32_t* __restrict__ u_term, int32_t* __restrict__ u_tf,
                       int32_t* __restrict__ u_cnt, uint32_t* __restrict__ blk_cnt,
                       unsigned long long* __restrict__ first_pos, int32_t* __restrict__ status,
                       const int32_t* __restrict__ long_docs, const int64_t* __restrict__ long_off,
                       unsigned long long* __restrict__ long_keys) {
    extern __shared__ __align__(16) unsigned char build_smem[];
    __shared__ int s_n;
    const int64_t d = LONG ? long_docs[blockIdx.x] : (int64_t)blockIdx.x;
    const int64_t beg = doc_ptr[d];
    const int64_t len64 = doc_ptr[d + 1] - beg;
    if (!LONG && len64 > kBuildCap) return;                          // handled by the LONG launch
    const int len = (int)len64;
    const int tid = threadIdx.x;
    if (len == 0) {
        if (tid == 0) u_cnt[d] = 0;
        return;
    }
    int n2 = 1;
    while (n2 < len) n2 <<= 1;
    unsigned long long* key = LONG ? long_keys + long_off[blockIdx.x] : reinterpret_cast<unsigned long long*>(build_smem);
    for (int i = tid; i < n2; i += kBuildThreads) {
        unsigned long long k = ~0ull;                                // padding sorts last
        if (i < len) {
            const int t = tokens[beg + i];
            if (t < 0 || t >= vocab) atomicMax(status, (int)min((long long)d + 1, 2147483647ll));
            k = ((unsigned long long)(unsigned)t << 32) | (unsigned)i;
        }
        key[i] = k;
    }
    if (tid == 0) s_n = 0;
    __syncthreads();
    bitonic_sort_u64(key, n2, tid, kBuildThreads);
    // heads of runs of equal terms; their rank among the heads = slot in the document's unique list (sorted by term)
    for (int base = 0; base < len; base += kBuildThreads) {
        const int i = base + tid;
        bool head = false;
        int term = 0;
        if (i < len) {
            term = (int)(key[i] >> 32);
            head = (i == 0) || ((int)(key[i - 1] >> 32) != term);
        }
        // block-wide exclusive count of heads in this sweep (ballot per warp + shared partials)
        __shared__ int s_w[kBuildThreads / 32];
        const unsigned m = __ballot_sync(0xffffffffu, head);
        const int lane = tid & 31, warp = tid >> 5;
        if (lane == 0) s_w[warp] = __popc(m);
        __syncthreads();
        int before = s_n;
        for (int w = 0; w < warp; ++w) before += s_w[w];
        const int slot = before + __popc(m & ((1u << lane) - 1u));
        if (head) {
            int e = i + 1;                                           // run length = term frequency in this document
            while (e < len && (int)(key[e] >> 32) == term) ++e;
            u_term[beg + slot] = term;
            u_tf[beg + slot] = e - i;
            const int blk = (int)(d / kBuildBlock);
            atomicAdd(blk_cnt + (int64_t)term * (n_blocks + 1) + blk, 1u);
            atomicMin(first_pos + term, (unsigned long long)(beg + (long long)(key[i] & 0xffffffffull)));
        }
        __syncthreads();
        if (tid == 0) {
            int tot = 0;
            for (int w = 0; w < kBuildThreads / 32; ++w) tot += s_w[w];
            s_n += tot;
        }
        __syncthreads();
    }
    if (tid == 0) u_cnt[d] = s_n;
}

// per term: counts per block -> exclusive offsets in place; blk[t][n_blocks] = df[t]
__global__ void bm25_block_scan_kernel(uint32_t* __restrict__ blk_cnt, int32_t vocab, int32_t n_blocks,
                                       int64_t* __restrict__ df) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= vocab) return;
    uint32_t* row = blk_cnt + (int64_t)t * (n_blocks + 1);
    uint32_t run = 0;
    for (int b = 0; b < n_blocks; ++b) {
        const uint32_t c = row[b];
        row[b] = run;
        run += c;
    }
    row[n_blocks] = run;
    df[t] = (int64_t)run;
}

// indptr[0] = 0, indptr[t + 1] = sum_{u <= t} df[u]: one CTA, chunks of 1024 with a running carry
__global__ void __launch_bounds__(1024)
bm25_indptr_scan_kernel(const int64_t* __restrict__ df, int32_t vocab, int64_t* __restrict__ indptr) {
    __shared__ long long s_warp[32];
    __shared__ long long s_carry;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) { s_carry = 0; indptr[0] = 0; }
    __syncthreads();
    for (int base = 0; base < vocab; base += 1024) {
        const int i = base + tid;
        long long v = i < vocab ? (long long)df[i] : 0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const long long u = __shfl_up_sync(0xffffffffu, v, o);
            if (lane >= o) v += u;
        }
        if (lane == 31) s_warp[warp] = v;
        __syncthreads();
        if (warp == 0) {
            long long w = s_warp[lane];
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const long long u = __shfl_up_sync(0xffffffffu, w, o);
                if (lane >= o) w += u;
            }
            s_warp[lane] = w;
        }
        __syncthreads();
        const long long incl = v + (warp > 0 ? s_warp[warp - 1] : 0) + s_carry;
        if (i < vocab) indptr[i + 1] = incl;
        __syncthreads();
        if (tid == 1023) s_carry = incl;
        __syncthreads();
    }
}

// one CTA per block of kBuildBlock documents, documents strictly in order (see the header comment)
__global__ void __launch_bounds__(kBuildThreads)
bm25_place_kernel(const int64_t* __restrict__ doc_ptr, int64_t n_docs, int32_t n_blocks, const int32_t* __restrict__ u_term,
                  const int32_t* __restrict__ u_tf, const int32_t* __restrict__ u_cnt,
                  const uint32_t* __restrict__ blk_off, uint32_t* __restrict__ cursor, const int64_t* __restrict__ indptr,
                  int32_t* __restrict__ post_doc, int32_t* __restrict__ post_tf) {
    const int blk = blockIdx.x;
    const int64_t d0 = (int64_t)blk * kBuildBlock;
    const int64_t d1 = min(n_docs, d0 + kBuildBlock);
    for (int64_t d = d0; d < d1; ++d) {
        const int64_t beg = doc_ptr[d];
        const int n = u_cnt[d];
        for (int i = threadIdx.x; i < n; i += kBuildThreads) {
            const int t = u_term[beg + i];                            // distinct terms inside one document
            const int64_t cell = (int64_t)t * (n_blocks + 1) + blk;
            const uint32_t c = cursor[cell];
            cursor[cell] = c + 1;
            const int64_t pos = indptr[t] + blk_off[cell] + c;
            post_doc[pos] = (int32_t)d;
            post_tf[pos] = u_tf[beg + i];
        }
        __syncthreads();                                             // the next document sees this one's cursors
    }
}

// ---- row shards: postings of documents [doc_lo, doc_hi) ----
__global__ void bm25_shard_bounds_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ post_doc,
                                         int32_t vocab, int32_t doc_lo, int32_t doc_hi, int64_t* __restrict__ first,
                                         int64_t* __restrict__ df_local) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= vocab) return;
    const int64_t s = indptr[t], e = indptr[t + 1];
    int64_t lo = s, hi = e;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (post_doc[mid] < doc_lo) lo = mid + 1; else hi = mid;
    }
    const int64_t a = lo;
    hi = e;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (post_doc[mid] < doc_hi) lo = mid + 1; else hi = mid;
    }
    first[t] = a;
    df_local[t] = lo - a;
}

__global__ void bm25_shard_copy_kernel(const int64_t* __restrict__ first, const int64_t* __restrict__ indptr_local,
                                       const int32_t* __restrict__ post_doc, const int32_t* __restrict__ post_tf,
                                       int32_t vocab, int32_t doc_lo, int32_t* __restrict__ out_doc,
                                       int32_t* __restrict__ out_tf) {
    const int t = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (t >= vocab) return;
    const int64_t src = first[t], dst = indptr_local[t];
    const int64_t n = indptr_local[t + 1] - dst;
    for (int64_t i = lane; i < n; i += 32) {
        out_doc[dst + i] = post_doc[src + i] - doc_lo;
        out_tf[dst + i] = post_tf[src + i];
    }
}

}  // namespace ezr

using namespace ezr;

extern "C" {

int ezr_bm25_build_block(void) { return kBuildBlock; }

size_t ezr_bm25_build_workspace(int64_t n_docs, int64_t n_tokens, int32_t vocab) {
    if (n_docs <= 0 || vocab <= 0) return 0;
    const int64_t n_blocks = (n_docs + kBuildBlock - 1) / kBuildBlock;
    size_t b = 0;
    b += align_up((size_t)n_tokens * 4, 256) * 2;                       // u_term, u_tf
    b += align_up((size_t)n_docs * 4, 256);                             // u_cnt
    b += align_up((size_t)vocab * (n_blocks + 1) * 4, 256) * 2;         // block counts / offsets, cursors
    b += align_up(16, 256);                                             // status
    return b;
}

/* Phase A: count.  Fills df[vocab] (int64), indptr[vocab+1] (int64), first_pos[vocab] (uint64; ~0 = term absent) and the
 * workspace that phase B consumes.  long_* describe the documents longer than the shared-memory sort (may be NULL when
 * n_long == 0): long_docs[n_long] (device), long_off[n_long] (device, offsets into long_keys in keys),
 * long_keys: device scratch of sum(next_pow2(len)) uint64.  *status_host: 0 ok, else 1 + index of a document
 * holding a token id outside [0, vocab).  Synchronises the stream (index-build time). */
int ezr_bm25_build_count(const int32_t* tokens, const int64_t* doc_ptr, int64_t n_docs, int64_t n_tokens, int32_t vocab,
                         int32_t max_doc_len, int64_t* out_df, int64_t* out_indptr, uint64_t* out_first_pos, const int32_t* long_docs,
                         const int64_t* long_off, uint64_t* long_keys, int32_t n_long, void* workspace,
                         size_t workspace_bytes, int32_t* status_host, void* stream) {
    EZR_CHECK_ARG(n_docs >= 1 && n_docs < ((int64_t)1 << 31) && vocab >= 1, "bm25_build: bad n_docs / vocab");
    EZR_CHECK_ARG(tokens || n_tokens == 0, "bm25_build: tokens is NULL");
    EZR_CHECK_ARG(doc_ptr && out_df && out_indptr && out_first_pos && status_host, "bm25_build: NULL argument");
    const size_t need = ezr_bm25_build_workspace(n_docs, n_tokens, vocab);
    if (workspace_bytes < need || !workspace) {
        set_error("bm25_build: workspace %zu < %zu", workspace_bytes, need);
        return EZR_ERR_WORKSPACE;
    }
    cudaStream_t st = (cudaStream_t)stream;
    const int n_blocks = (int)((n_docs + kBuildBlock - 1) / kBuildBlock);
    char* w = reinterpret_cast<char*>(workspace);
    int32_t* u_term = reinterpret_cast<int32_t*>(w); w += align_up((size_t)n_tokens * 4, 256);
    int32_t* u_tf = reinterpret_cast<int32_t*>(w); w += align_up((size_t)n_tokens * 4, 256);
    int32_t* u_cnt = reinterpret_cast<int32_t*>(w); w += align_up((size_t)n_docs * 4, 256);
    uint32_t* blk = reinterpret_cast<uint32_t*>(w); w += align_up((size_t)vocab * (n_blocks + 1) * 4, 256);
    uint32_t* cursor = reinterpret_cast<uint32_t*>(w); w += align_up((size_t)vocab * (n_blocks + 1) * 4, 256);
    int32_t* status = reinterpret_cast<int32_t*>(w);
    EZR_CUDA(cudaMemsetAsync(blk, 0, (size_t)vocab * (n_blocks + 1) * 4, st));
    EZR_CUDA(cudaMemsetAsync(cursor, 0, (size_t)vocab * (n_blocks + 1) * 4, st));
    EZR_CUDA(cudaMemsetAsync(status, 0, 16, st));
    EZR_CUDA(cudaMemsetAsync(out_first_pos, 0xff, (size_t)vocab * 8, st));
    static bool attr_done = false;
    if (!attr_done) {
        EZR_CUDA(cudaFuncSetAttribute(bm25_doc_unique_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      kBuildCap * 8));
        attr_done = true;
    }
    // shared memory for the longest document this launch sorts (more CTAs per SM for short-chunk corpora)
    int keys = 32;
    while (keys < kBuildCap && keys < max_doc_len) keys <<= 1;
    bm25_doc_unique_kernel<false><<<(unsigned)n_docs, kBuildThreads, (size_t)keys * 8, st>>>(
        tokens, doc_ptr, n_docs, vocab, n_blocks, u_term, u_tf, u_cnt, blk,
        reinterpret_cast<unsigned long long*>(out_first_pos), status, nullptr, nullptr, nullptr);
    EZR_LAUNCH_CHECK();
    if (n_long > 0) {
        EZR_CHECK_ARG(long_docs && long_off && long_keys, "bm25_build: long-document scratch missing");
        bm25_doc_unique_kernel<true><<<(unsigned)n_long, kBuildThreads, 0, st>>>(
            tokens, doc_ptr, n_docs, vocab, n_blocks, u_term, u_tf, u_cnt, blk,
            reinterpret_cast<unsigned long long*>(out_first_pos), status, long_docs, long_off,
            reinterpret_cast<unsigned long long*>(long_keys));
        EZR_LAUNCH_CHECK();
    }
    bm25_block_scan_kernel<<<ceil_div(vocab, 256), 256, 0, st>>>(blk, vocab, n_blocks, out_df);
    EZR_LAUNCH_CHECK();
    bm25_indptr_scan_kernel<<<1, 1024, 0, st>>>(out_df, vocab, out_indptr);
    EZR_LAUNCH_CHECK();
    EZR_CUDA(cudaMemcpyAsync(status_host, status, 4, cudaMemcpyDeviceToHost, st));
    EZR_CUDA(cudaStreamSynchronize(st));
    return EZR_OK;
}

/* Phase B: place.  out_post_doc / out_post_tf hold indptr[vocab] entries; needs the workspace of phase A untouched. */
int ezr_bm25_build_fill(const int64_t* doc_ptr, int64_t n_docs, int64_t n_tokens, int32_t vocab, const int64_t* indptr,
                        int32_t* out_post_doc, int32_t* out_post_tf, void* workspace, size_t workspace_bytes,
                        void* stream) {
    EZR_CHECK_ARG(n_docs >= 1 && vocab >= 1 && doc_ptr && indptr, "bm25_build_fill: bad arguments");
    const size_t need = ezr_bm25_build_workspace(n_docs, n_tokens, vocab);
    if (workspace_bytes < need || !workspace) {
        set_error("bm25_build_fill: workspace %zu < %zu", workspace_bytes, need);
        return EZR_ERR_WORKSPACE;
    }
    cudaStream_t st = (cudaStream_t)stream;
    const int n_blocks = (int)((n_docs + kBuildBlock - 1) / kBuildBlock);
    char* w = reinterpret_cast<char*>(workspace);
    const int32_t* u_term = reinterpret_cast<int32_t*>(w); w += align_up((size_t)n_tokens * 4, 256);
    const int32_t* u_tf = reinterpret_cast<int32_t*>(w); w += align_up((size_t)n_tokens * 4, 256);
    const int32_t* u_cnt = reinterpret_cast<int32_t*>(w); w += align_up((size_t)n_docs * 4, 256);
    const uint32_t* blk = reinterpret_cast<uint32_t*>(w); w += align_up((size_t)vocab * (n_blocks + 1) * 4, 256);
    uint32_t* cursor = reinterpret_cast<uint32_t*>(w);
    bm25_place_kernel<<<n_blocks, kBuildThreads, 0, st>>>(doc_ptr, n_docs, n_blocks, u_term, u_tf, u_cnt, blk, cursor,
                                                         indptr, out_post_doc, out_post_tf);
    EZR_LAUNCH_CHECK();
    return EZR_OK;
}

/* Row shard, step 1: first[t] = position of term t's first posting with doc >= doc_lo, df_local[t] = postings with
 * doc in [doc_lo, doc_hi); out_indptr_local[vocab+1] = their exclusive scan. */
int ezr_bm25_shard_count(const int64_t* indptr, const int32_t* post_doc, int32_t vocab, int32_t doc_lo, int32_t doc_hi,
                         int64_t* out_first, int64_t* out_df_local, int64_t* out_indptr_local, void* stream) {
    EZR_CHECK_ARG(indptr && post_doc && out_first && out_df_local && out_indptr_local && vocab >= 1 && doc_lo <= doc_hi,
                  "bm25_shard_count: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    bm25_shard_bounds_kernel<<<ceil_div(vocab, 256), 256, 0, st>>>(indptr, post_doc, vocab, doc_lo, doc_hi, out_first,
                                                                  out_df_local);
    EZR_LAUNCH_CHECK();
    bm25_indptr_scan_kernel<<<1, 1024, 0, st>>>(out_df_local, vocab, out_indptr_local);
    EZR_LAUNCH_CHECK();
    return EZR_OK;
}

/* Row shard, step 2: copy the sub-segments, document ids rebased to doc_lo. */
int ezr_bm25_shard_copy(const int64_t* first, const int64_t* indptr_local, const int32_t* post_doc,
                        const int32_t* post_tf, int32_t vocab, int32_t doc_lo, int32_t* out_post_doc,
                        int32_t* out_post_tf, void* stream) {
    EZR_CHECK_ARG(first && indptr_local && post_doc && post_tf && vocab >= 1, "bm25_shard_copy: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    bm25_shard_copy_kernel<<<ceil_div(vocab, 8), 256, 0, st>>>(first, indptr_local, post_doc, post_tf, vocab, doc_lo,
                                                              out_post_doc, out_post_tf);
    EZR_LAUNCH_CHECK();
    return EZR_OK;
}

}  // extern "C"
