// BM25 for the coarse-ranking path: index-side weight precompute, batched
// scoring with shared-memory accumulators, fused top-k.
//
// Reference behaviour being replaced: retrievers.py:128-151 (get_scores ->
// rank_bm25.BM25Okapi.get_scores / bm25s.get_scores) and retrievers.py:191-210
// (filter).  Arithmetic order: oracle/bm25.py (OkapiCSR docstring).
//
// Design (DESIGN.md "BM25"): the per-posting contribution is query independent,
// so it is computed once at index build with explicit round-to-nearest
// intrinsics (no FMA contraction) and stored next to the doc id (12 B/posting).
// Two query-time paths share this index:
//  * bm25_score_kernel (this file, "ordered"): a CTA owns (query, range of 8192
//    documents); float64 accumulators live in shared memory, query terms are
//    applied strictly in token order (one barrier per term keeps the float64
//    sum order of the reference), top-k by threshold -> compact -> rank.  Used
//    for indices without packed postings (float32 by default, negative idf),
//    score rows (k > 32) and as the hand-over target of the path below.
//  * bm25_cand_kernel + bm25_bound_kernel + bm25_rescore_kernel (bm25_pk.cuh,
//    "two-phase", the default for the fused top-k of float64 indices, opt-in
//    for float32 ones): integer upper-bound scores from 4-byte packed postings
//    with shared-memory atomics, then the exact ordered score (float64 or
//    float32) of the surviving candidates only.
// Score vectors never touch HBM on the fused paths.
#include "ezr_common.cuh"
#include "bm25_common.cuh"
#include "select.cuh"
#include "../../include/easyrag_b200.h"

namespace ezr {

// ------------------------------------------------------------ index build --
__global__ void bm25_doc_norm_kernel(const int32_t* __restrict__ doc_len, int64_t n, double k1, double b,
                                     double one_minus_b, double avgdl, double* __restrict__ kd) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    kd[i] = bm25_doc_norm((double)doc_len[i], k1, b, one_minus_b, avgdl);
}

template <typename S>
__global__ void bm25_weights_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ post_doc,
                                    const int32_t* __restrict__ post_tf, int32_t vocab, int64_t n_post,
                                    const double* __restrict__ idf, const double* __restrict__ kd,
                                    double num_scale, S* __restrict__ out_w) {
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n_post) return;
    // term of posting p: largest t with indptr[t] <= p
    int lo = 0, hi = vocab;   // invariant: indptr[lo] <= p < indptr[hi]
    while (hi - lo > 1) {
        const int mid = lo + ((hi - lo) >> 1);
        if (indptr[mid] <= p) lo = mid; else hi = mid;
    }
    out_w[p] = (S)bm25_contribution(idf[lo], (double)post_tf[p], kd[post_doc[p]], num_scale);
}

__global__ void bm25_range_index_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ post_doc,
                                        int32_t vocab, int32_t range_size, int32_t n_ranges,
                                        uint32_t* __restrict__ range_off) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t total = (int64_t)vocab * (n_ranges + 1);
    if (i >= total) return;
    const int t = (int)(i / (n_ranges + 1));
    const int r = (int)(i % (n_ranges + 1));
    const int64_t s = indptr[t], e = indptr[t + 1];
    const int64_t want = (int64_t)r * range_size;    // first doc id of range r
    int64_t lo = s, hi = e;                           // lower_bound(post_doc[s:e], want)
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (post_doc[mid] < want) lo = mid + 1; else hi = mid;
    }
    range_off[i] = (uint32_t)(lo - s);
}

// ---------------------------------------------------------------- scoring --
// Launch shapes.  Since the two-phase path (bm25_pk.cuh) took over the fused top-k, the range is chosen for ITS
// candidate pass, which is issue bound and wants fewer, larger CTAs (8192 documents, 256 threads, 6 CTAs/SM).  These
// shapes were chosen on an earlier GPU generation and have not been re-swept on the H100.
#ifndef EZR_BM25_RANGE
#define EZR_BM25_RANGE 8192
#endif
#ifndef EZR_BM25_THREADS
#define EZR_BM25_THREADS 512
#endif
#ifndef EZR_BM25_MINB
#define EZR_BM25_MINB 3
#endif
constexpr int kBmRange = EZR_BM25_RANGE;     // documents per CTA (8192 -> 64 KB of float64 accumulators)
constexpr int kBmThreads = EZR_BM25_THREADS;
constexpr int kBmGroup = kBmThreads / 32;    // lanes per group: 32 group maxima bound the k-th score (k <= 32)
static_assert(kBmGroup == 8 || kBmGroup == 16 || kBmGroup == 32, "BM25 CTA must have 256, 512 or 1024 threads");
constexpr int kBmMaxT = 12;      // query terms preloaded per round (queries are 4-12 terms; longer ones loop)
constexpr int kBmRpc = 1;        // document ranges per CTA

struct Bm25Params {
    const int64_t* indptr;
    const int32_t* post_doc;
    const void* post_w;
    const uint32_t* range_off;
    const int32_t* doc_group;
    const int32_t* q_ptr;
    const int32_t* q_terms;
    const int32_t* q_group;
    int64_t n_docs;
    int32_t vocab;
    int32_t n_ranges;
    int32_t k;
    int32_t id_base;
    void* out_scores;   // fused: partial [Q][n_ranges][k]; rows: [Q][n_docs]
    int32_t* out_ids;   // fused: partial ids
    int32_t monotone;   // every posting weight is >= 0 (no negative idf): partial sums only grow
    int32_t* thr_key;   // fused: [Q] running lower bound (integer key) of each query's k-th best score, zeroed per call
    const int32_t* q_list;   // optional indirection: CTA column i works on query q_list[i] ...
    const int32_t* q_count;  // ... for i < *q_count (the two-phase path hands its overflowed queries over this way)
};

// Integer sort key of a non-negative score: IEEE-754 ordering of non-negative floats equals the ordering of their
// bit patterns, so the high word of a float64 (all of a float32) is a monotone, slightly coarse key.
template <typename S> struct KeyOf;
template <> struct KeyOf<double> {
    static __device__ __forceinline__ int load(const double* acc, int i) { return reinterpret_cast<const int*>(acc)[2 * i + 1]; }
};
template <> struct KeyOf<float> {
    static __device__ __forceinline__ int load(const float* acc, int i) { return reinterpret_cast<const int*>(acc)[i]; }
};

template <typename S> __device__ __forceinline__ int score_key(S v);
template <> __device__ __forceinline__ int score_key<double>(double v) { return __double2hiint(v); }
template <> __device__ __forceinline__ int score_key<float>(float v) { return __float_as_int(v); }

// MODE 0: fused top-k (k<=32) -> per-(query,range) partial lists.  MODE 1: write the score row.
// A CTA owns one query and kBmRpc consecutive document ranges.  Range i+1's first postings are issued right after
// range i's accumulation, so their latency hides behind range i's selection phases; term ids / indptr / range
// offsets are fetched once per CTA.
template <typename S, int MODE>
__device__ __forceinline__ void bm25_score_body(const Bm25Params& p, const int q) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    S* acc = reinterpret_cast<S*>(smem_raw);
    __shared__ int s_off[kBmRpc + 1][kBmMaxT];      // first-chunk terms: absolute posting offset at each range boundary
    __shared__ int s_lo[kBmMaxT], s_len2[kBmMaxT];  // later chunks of long queries (> kBmMaxT terms), per range
    __shared__ S s_ws[kBmThreads];
    __shared__ int s_wi[kBmThreads];
    __shared__ int s_thr;
    __shared__ int s_cnt;

    const int r0 = blockIdx.y * kBmRpc;
    const int n_r = min(kBmRpc, p.n_ranges - r0);
    const int tid = threadIdx.x;
    const int lane = tid & 31, warp = tid >> 5;
    const int qs = p.q_ptr[q];
    const int m = p.q_ptr[q + 1] - qs;
    const int m0 = min(m, kBmMaxT);
    const S* __restrict__ post_w = reinterpret_cast<const S*>(p.post_w);
    const int32_t* __restrict__ post_doc = p.post_doc;
    constexpr int kVec = 16 / sizeof(S);                        // scores per 128-bit shared-memory access
    constexpr int kPer = kBmRange / kBmThreads;                 // documents scanned per thread
    const int want = (MODE == 0 && p.q_group) ? p.q_group[q] : -1;
    // Lower bound of this query's k-th best score established by CTAs of earlier document ranges (range-major grid:
    // they finished long ago).  Anything below it cannot reach the final top-k, so it may be dropped here already.
    // ONE thread reads it (other CTAs raise it concurrently; the branch below must be block-uniform).
    __shared__ int s_gthr;
    if (MODE == 0 && tid == kBmThreads - 1) {
        s_gthr = *reinterpret_cast<const volatile int32_t*>(p.thr_key + q);
        s_cnt = 0;
    }

    int longest = 0;
    if (tid < m0) {
        const int t = p.q_terms[qs + tid];
        if (t >= 0 && t < p.vocab) {
            const int base = (int)p.indptr[t];                  // n_postings < 2^31 (checked on the host)
            const uint32_t* ro = p.range_off + (int64_t)t * (p.n_ranges + 1) + r0;
#pragma unroll
            for (int i = 0; i <= kBmRpc; ++i) {
                s_off[i][tid] = base + (int)ro[min(i, n_r)];
                if (i > 0) longest = max(longest, s_off[i][tid] - s_off[i - 1][tid]);
            }
        } else {
#pragma unroll
            for (int i = 0; i <= kBmRpc; ++i) s_off[i][tid] = 0;
        }
    }
    // barrier + vote: is some (term, range) segment longer than the CTA?  Only then do the residual loops run.
    const bool any_long = __syncthreads_or(longest > kBmThreads) != 0;

    const int shared_thr = (MODE == 0) ? s_gthr : 0;
    // With a bound from earlier ranges and non-negative weights, a document qualifies exactly once: when its
    // partial sum crosses the bound.  It is appended to the candidate list right there, and the selection scan over
    // all 8192 accumulators is not needed at all for this (query, range).
    const bool track = (MODE == 0) && shared_thr > 0 && p.monotone != 0;
    auto rmw = [&](int doc, S wv, int rbase_) {
        S* a = acc + (doc - rbase_);
        const S old = *a;
        const S nw = old + wv;
        *a = nw;
        if (track && score_key<S>(nw) >= shared_thr && score_key<S>(old) < shared_thr) {
            if (want == -1 || p.doc_group[doc] == want) {
                const int idx = atomicAdd(&s_cnt, 1);
                if (idx < kBmThreads) s_wi[idx] = doc;
            }
        }
    };
    int d[kBmMaxT];
    S w[kBmMaxT];
    // first posting of every (first-chunk) term of range 0: all loads in flight together
#pragma unroll
    for (int j = 0; j < kBmMaxT; ++j) {
        d[j] = -1;
        w[j] = (S)0;
        if (j < m0) {
            const int beg = s_off[0][j];
            if (tid < s_off[1][j] - beg) { d[j] = __ldg(post_doc + beg + tid); w[j] = __ldg(post_w + beg + tid); }
        }
    }
    {
        uint4* a4 = reinterpret_cast<uint4*>(acc);
#pragma unroll
        for (int i = 0; i < kBmRange / kVec / kBmThreads; ++i) a4[tid + i * kBmThreads] = make_uint4(0u, 0u, 0u, 0u);
    }
    __syncthreads();

    for (int ri = 0; ri < n_r; ++ri) {
        const int r = r0 + ri;
        const int rbase = r * kBmRange;
        const int rn = (int)min((int64_t)kBmRange, p.n_docs - rbase);

        // ---- accumulate: terms strictly in token order, one barrier per term (float sum order of the reference)
#pragma unroll
        for (int j = 0; j < kBmMaxT; ++j) {
            if (j < m0) {   // block-uniform
                if (d[j] >= 0) rmw(d[j], w[j], rbase);
                if (any_long) {                                  // rare: a segment longer than the CTA
                    const int beg = s_off[ri][j];
                    const int len = s_off[ri + 1][j] - beg;
                    for (int o = tid + kBmThreads; o < len; o += kBmThreads)
                        rmw(__ldg(post_doc + beg + o), __ldg(post_w + beg + o), rbase);
                }
                __syncthreads();
            }
        }
        for (int tb = kBmMaxT; tb < m; tb += kBmMaxT) {          // queries longer than kBmMaxT terms (rare)
            const int mt = min(kBmMaxT, m - tb);
            if (tid < mt) {
                const int t = p.q_terms[qs + tb + tid];
                int beg = 0, len = 0;
                if (t >= 0 && t < p.vocab) {
                    const uint32_t* ro = p.range_off + (int64_t)t * (p.n_ranges + 1) + r;
                    const uint32_t o0 = ro[0], o1 = ro[1];
                    beg = (int)p.indptr[t] + (int)o0;
                    len = (int)(o1 - o0);
                }
                s_lo[tid] = beg;
                s_len2[tid] = len;
            }
            __syncthreads();
            for (int j = 0; j < mt; ++j) {
                const int beg = s_lo[j], len = s_len2[j];
                for (int o = tid; o < len; o += kBmThreads)
                    rmw(__ldg(post_doc + beg + o), __ldg(post_w + beg + o), rbase);
                __syncthreads();
            }
        }

        // ---- prefetch the next range's first postings: they land while this range is being selected from
        const bool more = ri + 1 < n_r;
        if (more) {
#pragma unroll
            for (int j = 0; j < kBmMaxT; ++j) {
                d[j] = -1;
                if (j < m0) {
                    const int beg = s_off[ri + 1][j];
                    if (tid < s_off[ri + 2][j] - beg) { d[j] = __ldg(post_doc + beg + tid); w[j] = __ldg(post_w + beg + tid); }
                }
            }
        }

        if (MODE == 1) {
            S* out = reinterpret_cast<S*>(p.out_scores) + (int64_t)q * p.n_docs + rbase;
            for (int i = tid; i < rn; i += kBmThreads) out[i] = acc[i];
        } else {
            // ---- fused top-k from shared memory: threshold -> compact -> rank ----
            // 1. every half-warp finds the best key among the documents it scans; the k-th largest of those 32 group
            //    maxima is a lower bound of the range's k-th best score (32 distinct documents), and a tight one: on
            //    average only ~k/2 extra documents pass it.  Keys = high words of the scores (KeyOf).
            // 2. documents whose key reaches the bound are appended to a small candidate list (smem atomics).
            // 3. each candidate counts how many candidates rank before it under the canonical order and writes
            //    itself to that output slot.  No sort, no serial insertion chain.
            // Exact ties at the bound (or fewer than k non-empty groups) can overflow the list; then the robust
            // warp-shuffle selection takes over.  Rows >= rn of the last range hold zeros and never qualify.
            constexpr int kCand = kBmThreads;                   // candidate capacity (s_ws / s_wi are reused)
            if (track) {
                // candidates were collected while accumulating (the last term's barrier made them visible): fetch
                // their final scores
                const int nc = min(s_cnt, kCand);
                if (tid < nc) s_ws[tid] = acc[s_wi[tid] - rbase];
            } else {
                int tmax = 0x7fffffff;                              // "this thread must re-scan" when phase 1 is skipped
                if (shared_thr > 0) {
                    if (tid == 0) s_thr = shared_thr;               // single pass: the shared bound replaces phase 1
                } else {
                    tmax = 0;
                    if (want == -1) {
#pragma unroll
                        for (int i = 0; i < kPer; ++i) tmax = max(tmax, KeyOf<S>::load(acc, tid + i * kBmThreads));
                    } else {
#pragma unroll 4
                        for (int i = 0; i < kPer; ++i) {
                            const int doc = tid + i * kBmThreads;
                            const int key = KeyOf<S>::load(acc, doc);
                            if (key > tmax && p.doc_group[rbase + doc] == want) tmax = key;
                        }
                    }
                    int gmax = tmax;
#pragma unroll
                    for (int o = kBmGroup / 2; o > 0; o >>= 1) gmax = max(gmax, __shfl_xor_sync(0xffffffffu, gmax, o));
                    if ((lane & (kBmGroup - 1)) == 0) s_wi[tid / kBmGroup] = gmax;   // 32 group maxima (0: none positive)
                    __syncthreads();
                    if (warp == 0) {
                        const int mine = s_wi[lane];
                        int rank = 0;
#pragma unroll
                        for (int j = 0; j < 32; ++j) {
                            const int o = s_wi[j];
                            rank += (o > mine || (o == mine && j < lane)) ? 1 : 0;
                        }
                        if (rank == p.k - 1) s_thr = mine;          // ranks are a permutation: exactly one lane writes
                    }
                }
                __syncthreads();
                const int thr = s_thr;                              // 0 when fewer than k groups saw a positive score
                __syncthreads();                                    // s_thr / s_wi read by everyone: reuse them
                if (tmax >= thr) {                                  // only threads owning a qualifying document re-scan
#pragma unroll 4
                    for (int i = 0; i < kPer; ++i) {
                        const int doc = tid + i * kBmThreads;
                        if (KeyOf<S>::load(acc, doc) >= thr) {
                            const S s = acc[doc];
                            if (s > (S)0 && (want == -1 || p.doc_group[rbase + doc] == want)) {
                                const int idx = atomicAdd(&s_cnt, 1);
                                if (idx < kCand) { s_ws[idx] = s; s_wi[idx] = rbase + doc; }
                            }
                        }
                    }
                }
            }
            __syncthreads();
            const int n = s_cnt;
            const int64_t obase = ((int64_t)q * p.n_ranges + r) * p.k;
            S* out_s = reinterpret_cast<S*>(p.out_scores);
            if (n <= kCand) {
                if (tid < n) {
                    const S ms = s_ws[tid];
                    const int mi = s_wi[tid];
                    int rank = 0;
                    for (int j = 0; j < n; ++j) rank += better<S>(s_ws[j], s_wi[j], ms, mi) ? 1 : 0;
                    if (rank < p.k) { out_s[obase + rank] = ms; p.out_ids[obase + rank] = mi; }
                    if (rank == p.k - 1) {                      // this range alone has k documents at or above ms
                        const int key = KeyOf<S>::load(s_ws, tid);
                        if (key > shared_thr) atomicMax(p.thr_key + q, key);
                    }
                }
                if (tid >= n && tid < p.k) { out_s[obase + tid] = ScoreTraits<S>::lowest(); p.out_ids[obase + tid] = -1; }
            } else {
                // ---- overflow fallback: per-warp shuffle lists, then warp 0 merges them ----
                __syncthreads();
                WarpTopK<S> tk;
                tk.init(p.k);
                for (int i0 = warp * 32; i0 < rn; i0 += kBmThreads) {
                    const int i = i0 + lane;
                    S s = (S)0;
                    bool ok = false;
                    if (i < rn) {
                        s = acc[i];
                        ok = s > (S)0 && better<S>(s, rbase + i, tk.kth_s, tk.kth_id);
                        if (ok && want != -1) ok = (p.doc_group[rbase + i] == want);
                    }
                    tk.offer(s, rbase + i, ok);
                }
                __syncthreads();
                s_ws[warp * 32 + lane] = tk.s;
                s_wi[warp * 32 + lane] = tk.id;
                __syncthreads();
                if (warp == 0) {
                    WarpTopK<S> fin;
                    fin.init(p.k);
                    for (int w2 = 0; w2 < kBmThreads / 32; ++w2) {
                        const S s = s_ws[w2 * 32 + lane];
                        const int id = s_wi[w2 * 32 + lane];
                        fin.offer(s, id, lane < p.k && id >= 0);
                    }
                    if (lane < p.k) {
                        out_s[obase + lane] = fin.s;
                        p.out_ids[obase + lane] = fin.id;      // local id, -1 = empty
                    }
                }
            }
        }
        if (more) {
            __syncthreads();                                    // everyone is done with acc / s_ws / s_wi of this range
            if (tid == 0) s_cnt = 0;
            uint4* a4 = reinterpret_cast<uint4*>(acc);
#pragma unroll
            for (int i = 0; i < kBmRange / kVec / kBmThreads; ++i) a4[tid + i * kBmThreads] = make_uint4(0u, 0u, 0u, 0u);
            __syncthreads();
        }
    }
}

template <typename S, int MODE>
__global__ void __launch_bounds__(kBmThreads, EZR_BM25_MINB)
bm25_score_kernel(const Bm25Params p) {
    if (p.q_list == nullptr) {
        bm25_score_body<S, MODE>(p, blockIdx.x);
        return;
    }
    const int nq = *p.q_count;
    for (int qi = blockIdx.x; qi < nq; qi += gridDim.x) {
        bm25_score_body<S, MODE>(p, p.q_list[qi]);
        __syncthreads();                                        // shared state is re-initialised per query
    }
}

}  // namespace ezr
#include "bm25_pk.cuh"
namespace ezr {

// One warp per row: merge n_cand candidates (id<0 = empty) into the final top-k (k<=32).
// row_list / row_count (optional): warp i handles row row_list[i] for i < *row_count.
// n_parts > 1: the row's candidates are n_parts segments of n_cand entries, segment p at byte offset
// p * part_bytes from the row's first segment (the all-gathered per-shard records of easyrag_b200/dist.py).
template <typename S>
__global__ void merge_warp_kernel(const S* __restrict__ cs, const int32_t* __restrict__ cid, int n_rows, int n_cand,
                                  int64_t stride, int k, int id_add, S* __restrict__ out_s,
                                  int32_t* __restrict__ out_id, int32_t* __restrict__ out_cnt,
                                  const int32_t* __restrict__ row_list, const int32_t* __restrict__ row_count,
                                  int n_parts, int64_t part_bytes) {
    int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= n_rows) return;
    if (row_list) {
        if (row >= *row_count) return;
        row = row_list[row];
    }
    WarpTopK<S> tk;
    tk.init(k);
    for (int part = 0; part < n_parts; ++part) {
        const S* rs = reinterpret_cast<const S*>(reinterpret_cast<const char*>(cs) + part * part_bytes) +
                      (int64_t)row * stride;
        const int32_t* ri = reinterpret_cast<const int32_t*>(reinterpret_cast<const char*>(cid) + part * part_bytes) +
                            (int64_t)row * stride;
        for (int i0 = 0; i0 < n_cand; i0 += 32) {
            const int i = i0 + lane;
            S s = (S)0;
            int id = -1;
            if (i < n_cand) { s = rs[i]; id = ri[i]; }
            tk.offer(s, id, id >= 0);
        }
    }
    if (lane < k) {
        out_s[(int64_t)row * k + lane] = tk.id >= 0 ? tk.s : ScoreTraits<S>::lowest();
        out_id[(int64_t)row * k + lane] = tk.id >= 0 ? tk.id + id_add : -1;
    }
    const unsigned have = __ballot_sync(0xffffffffu, lane < k && tk.id >= 0);
    if (lane == 0 && out_cnt) out_cnt[row] = __popc(have);
}

// ------------------------------------------------------------ generic select
// grid (parts, rows).  Each CTA reduces a slice of one row to its sorted top-k.
// ids == nullptr: candidate id = column index.  Output slot (row*parts+part)*k.
template <typename S>
__global__ void __launch_bounds__(256)
select_kernel(const S* __restrict__ scores, const int32_t* __restrict__ ids, int64_t n_cols, int64_t row_stride,
              int parts, int k, int positive_only, const int32_t* __restrict__ doc_group,
              const int32_t* __restrict__ q_group, int id_add, S* __restrict__ out_s, int32_t* __restrict__ out_id,
              int32_t* __restrict__ out_cnt) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    SelSmem<S> sm = sel_carve<S>(smem_raw);
    sel_init<S>(sm);
    const int part = blockIdx.x, row = blockIdx.y;
    const int64_t chunk = (n_cols + parts - 1) / parts;
    const int64_t c0 = part * chunk;
    const int64_t c1 = min(n_cols, c0 + chunk);
    const S* rs = scores + (int64_t)row * row_stride;
    const int32_t* ri = ids ? ids + (int64_t)row * row_stride : nullptr;
    const int want = q_group ? q_group[row] : -1;
    constexpr int kItems = kSelReserve / 256;
    for (int64_t base = c0; base < c1; base += kSelReserve) {
#pragma unroll
        for (int it = 0; it < kItems; ++it) {
            const int64_t c = base + it * 256 + threadIdx.x;
            if (c < c1) {
                const S s = rs[c];
                const int id = ri ? ri[c] : (int)c;
                bool ok = id >= 0 && (!positive_only || s > (S)0) && s > ScoreTraits<S>::lowest();
                if (ok && better<S>(s, id, *sm.thr_s, *sm.thr_id)) {
                    if (want != -1) ok = (doc_group[id] == want);
                    if (ok) sel_push<S>(sm, s, id);
                }
            }
        }
        sel_maybe_flush<S>(sm, k);
    }
    sel_compact<S>(sm, k);
    const int n = *sm.cnt;
    const int64_t o = ((int64_t)row * parts + part) * k;
    for (int i = threadIdx.x; i < k; i += blockDim.x) {
        out_s[o + i] = i < n ? sm.ks[i] : ScoreTraits<S>::lowest();
        out_id[o + i] = i < n ? sm.kid[i] + id_add : -1;
    }
    if (threadIdx.x == 0 && out_cnt) out_cnt[row] = n;
}

template <typename S>
static int launch_select(const S* scores, const int32_t* ids, int n_rows, int64_t n_cols, int64_t row_stride,
                         int parts, int k, int positive_only, const int32_t* doc_group, const int32_t* q_group,
                         int id_add, S* out_s, int32_t* out_id, int32_t* out_cnt, cudaStream_t st) {
    const size_t smem = sel_smem_bytes<S>();
    static bool attr_done[2] = {false, false};
    const int which = sizeof(S) == 8 ? 0 : 1;
    if (!attr_done[which]) {
        EZR_CUDA(cudaFuncSetAttribute(select_kernel<S>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr_done[which] = true;
    }
    dim3 grid(parts, n_rows);
    ProfScope prof(EZR_PROF_MERGE, st);
    select_kernel<S><<<grid, 256, smem, st>>>(scores, ids, n_cols, row_stride, parts, k, positive_only, doc_group,
                                              q_group, id_add, out_s, out_id, out_cnt);
    EZR_LAUNCH_CHECK();
    return EZR_OK;
}

static int select_parts(int n_rows, int64_t n_cols) {
    // enough CTAs to fill the machine, at least 4096 columns each
    int64_t want = (int64_t)4 * sm_count() / (n_rows > 0 ? n_rows : 1);
    int64_t maxp = (n_cols + 4095) / 4096;
    int64_t parts = want < 1 ? 1 : want;
    if (parts > maxp) parts = maxp;
    if (parts < 1) parts = 1;
    return (int)parts;
}

template <typename S>
static size_t select_rows_ws(int n_rows, int64_t n_cols, int k) {
    const int parts = select_parts(n_rows, n_cols);
    if (parts == 1) return 0;
    return align_up((size_t)n_rows * parts * k * sizeof(S), 256) + align_up((size_t)n_rows * parts * k * 4, 256);
}

template <typename S>
static int select_rows_impl(const S* scores, int n_rows, int64_t n_cols, int64_t row_stride, int k,
                            int positive_only, const int32_t* doc_group, const int32_t* q_group, int id_base,
                            S* out_s, int32_t* out_id, int32_t* out_cnt, void* ws, size_t ws_bytes,
                            cudaStream_t st) {
    const int parts = select_parts(n_rows, n_cols);
    if (parts == 1)
        return launch_select<S>(scores, nullptr, n_rows, n_cols, row_stride, 1, k, positive_only, doc_group,
                                q_group, id_base, out_s, out_id, out_cnt, st);
    const size_t need = select_rows_ws<S>(n_rows, n_cols, k);
    if (ws_bytes < need || !ws) {
        set_error("select_rows: workspace %zu < %zu", ws_bytes, need);
        return EZR_ERR_WORKSPACE;
    }
    S* ps = reinterpret_cast<S*>(ws);
    int32_t* pi = reinterpret_cast<int32_t*>((char*)ws + align_up((size_t)n_rows * parts * k * sizeof(S), 256));
    int rc = launch_select<S>(scores, nullptr, n_rows, n_cols, row_stride, parts, k, positive_only, doc_group,
                              q_group, 0, ps, pi, nullptr, st);
    if (rc) return rc;
    return launch_select<S>(ps, pi, n_rows, (int64_t)parts * k, (int64_t)parts * k, 1, k, 0, nullptr, nullptr,
                            id_base, out_s, out_id, out_cnt, st);
}

template <typename S>
static int merge_impl(const S* cs, const int32_t* cid, int n_rows, int n_cand, int64_t stride, int k, int id_add,
                      S* out_s, int32_t* out_id, int32_t* out_cnt, cudaStream_t st,
                      const int32_t* row_list = nullptr, const int32_t* row_count = nullptr, int n_parts = 1,
                      int64_t part_bytes = 0) {
    if (n_rows == 0) return EZR_OK;
    if (k <= 32) {
        const int wpb = 8;
        ProfScope prof(EZR_PROF_MERGE, st);
        merge_warp_kernel<S><<<ceil_div(n_rows, wpb), wpb * 32, 0, st>>>(cs, cid, n_rows, n_cand, stride, k, id_add,
                                                                        out_s, out_id, out_cnt, row_list, row_count,
                                                                        n_parts, part_bytes);
        EZR_LAUNCH_CHECK();
        return EZR_OK;
    }
    if (n_parts != 1) {
        set_error("merge_topk_parts: k=%d > 32 needs contiguous candidates", k);
        return EZR_ERR_UNSUPPORTED;
    }
    return launch_select<S>(cs, cid, n_rows, n_cand, stride, 1, k, 0, nullptr, nullptr, id_add, out_s, out_id,
                            out_cnt, st);
}

template <typename S>
static int bm25_launch(const ezr_bm25_index* ix, const int32_t* q_ptr, const int32_t* q_terms, int n_queries,
                       int k, const int32_t* q_group, int id_base, int mode, void* out_scores, int32_t* out_ids,
                       int32_t* thr_key, cudaStream_t st, const int32_t* q_list = nullptr,
                       const int32_t* q_count = nullptr) {
    Bm25Params p;
    p.q_list = q_list; p.q_count = q_count;
    p.indptr = ix->indptr; p.post_doc = ix->post_doc; p.post_w = ix->post_w; p.range_off = ix->range_off;
    p.doc_group = ix->doc_group; p.q_ptr = q_ptr; p.q_terms = q_terms; p.q_group = q_group;
    p.n_docs = ix->n_docs; p.vocab = ix->vocab; p.n_ranges = ix->n_ranges; p.k = k; p.id_base = id_base;
    p.out_scores = out_scores; p.out_ids = out_ids; p.thr_key = thr_key; p.monotone = ix->monotone;
    const size_t smem = (size_t)kBmRange * sizeof(S);
    static bool attr_done[4] = {false, false, false, false};
    const int which = (sizeof(S) == 8 ? 0 : 2) + mode;
    auto kern = mode == 0 ? bm25_score_kernel<S, 0> : bm25_score_kernel<S, 1>;
    if (!attr_done[which]) {
        EZR_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr_done[which] = true;
    }
    // with a query list the CTA columns loop over it (it is normally empty: keep the grid small)
    dim3 grid(q_list ? (n_queries < 16 ? n_queries : 16) : n_queries, (ix->n_ranges + kBmRpc - 1) / kBmRpc);
    ProfScope prof(EZR_PROF_BM25_SCORE, st);
    kern<<<grid, kBmThreads, smem, st>>>(p);
    EZR_LAUNCH_CHECK();
    return EZR_OK;
}


// ---- two-phase path (bm25_pk.cuh) ----
// ezr_bm25_set_skipping.  OFF by default: the candidate pass reads fewer postings but the rescoring grows, because
// candidates then only carry partial lower bounds and the running bound tightens more slowly (not re-measured on
// the H100).  Kept (and parity-tested) as the starting point for a
// version that refines the bounds between chunks.
static int g_bm25_skip = 0;
static int g_bm25_span = 4;     // ezr_bm25_set_span: ranges in the first candidate launch (then the same again, then doubling)
static int g_bm25_plan = 1;     // ezr_bm25_set_plan: 1 = per-launch plan table (default), 0 = resolve segments inside the CTAs

// Packed postings (float64 weights from ezr_bm25_pack, float32 ones from ezr_bm25_pack_f32) on a monotone index
static bool pk_usable(const ezr_bm25_index* ix, int k) {
    return kPkEnabled && ix->post_pk != nullptr && ix->monotone && k <= 32;
}

// the deep form of the two-phase path (bm25_pk.cuh): the same index types, 32 < k <= kSelMaxK
static bool pk_deep_usable(const ezr_bm25_index* ix, int k) {
    return kPkEnabled && ix->post_pk != nullptr && ix->monotone && k > 32 && k <= kSelMaxK;
}

struct PkWorkspace {
    int32_t *thr_key, *thr_q, *cand_cnt, *ovf, *ne_sum, *ovf_n, *ovf_list, *cand_ids, *cand_q, *cand_u;
    uint32_t* ne_mask;
    int2* plan;
    void* rows;     // deep form: [Q][list_cap] exact scores (the index's score type) beside cand_ids
    size_t zero_bytes, total;
};

// list_cap: candidates per query (kPkListCap, or pk_deep_list_cap(k) with deep, which adds the score rows of
// score_bytes each)
static PkWorkspace pk_carve(void* base, int n_queries, int list_cap = kPkListCap, bool deep = false,
                            size_t score_bytes = 8) {
    PkWorkspace w;
    const size_t q = (size_t)n_queries;
    char* b = reinterpret_cast<char*>(base);
    w.thr_key = reinterpret_cast<int32_t*>(b);
    w.thr_q = w.thr_key + q;
    w.cand_cnt = w.thr_q + q;
    w.ovf = w.cand_cnt + q;
    w.ne_mask = reinterpret_cast<uint32_t*>(w.ovf + q);
    w.ne_sum = w.ovf + 2 * q;
    w.ovf_n = w.ovf + 3 * q;
    w.zero_bytes = (6 * q + 1) * 4;                     // everything up to here is zeroed per call
    size_t off = align_up(w.zero_bytes, 256);
    w.ovf_list = reinterpret_cast<int32_t*>(b + off);
    off += align_up(q * 4, 256);
    const size_t lc = (size_t)list_cap;
    w.cand_ids = reinterpret_cast<int32_t*>(b + off);
    off += align_up(q * lc * 4, 256);
    w.cand_q = reinterpret_cast<int32_t*>(b + off);
    off += align_up(q * lc * 4, 256);
    w.cand_u = reinterpret_cast<int32_t*>(b + off);
    off += align_up(q * lc * 4, 256);
    w.plan = reinterpret_cast<int2*>(b + off);
    off += align_up(q * kPkMaxChunk * kPkPlanTok * sizeof(int2), 256);
    w.rows = deep ? reinterpret_cast<void*>(b + off) : nullptr;
    if (deep) off += align_up(q * lc * score_bytes, 256);
    w.total = off;
    return w;
}

// deep: the deep form's kernels; rescoring then fills w.rows instead of the outputs (the caller selects the top-k).
// S: the index's score type (the kernel instances and their attributes are per type).
template <typename S>
static int pk_launch(const ezr_bm25_index* ix, const int32_t* q_ptr, const int32_t* q_terms, int n_queries, int k,
                     const int32_t* q_group, int id_base, const PkWorkspace& w, S* out_scores,
                     int32_t* out_ids, int32_t* out_counts, cudaStream_t st, bool deep = false) {
    Bm25Params p;
    p.indptr = ix->indptr; p.post_doc = ix->post_doc; p.post_w = ix->post_w; p.range_off = ix->range_off;
    p.doc_group = ix->doc_group; p.q_ptr = q_ptr; p.q_terms = q_terms; p.q_group = q_group;
    p.n_docs = ix->n_docs; p.vocab = ix->vocab; p.n_ranges = ix->n_ranges; p.k = k; p.id_base = id_base;
    p.out_scores = nullptr; p.out_ids = nullptr; p.thr_key = nullptr; p.monotone = ix->monotone;
    p.q_list = nullptr; p.q_count = nullptr;
    PkParams c;
    c.post_pk = ix->post_pk; c.thr_q = w.thr_q; c.cand_cnt = w.cand_cnt; c.cand_ids = w.cand_ids; c.cand_q = w.cand_q; c.cand_u = w.cand_u; c.ovf = w.ovf;
    c.term_max = g_bm25_skip ? ix->term_max : nullptr; c.ne_mask = w.ne_mask; c.ne_sum = w.ne_sum;
    c.ovf_n = w.ovf_n; c.ovf_list = w.ovf_list; c.plan = g_bm25_plan ? w.plan : nullptr;
    const size_t smem = deep ? pk_deep_cand_smem(k) : (size_t)(kBmRange + 32) * 4;
    const size_t bd_smem = deep ? pk_deep_bound_smem(k) : 0;
    static bool attr_done = false, deep_attr_done = false;
    if (!deep && !attr_done) {
        EZR_CUDA(cudaFuncSetAttribute(bm25_cand_kernel<false, S>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        EZR_CUDA(cudaFuncSetAttribute(bm25_cand_kernel<false, S>, cudaFuncAttributePreferredSharedMemoryCarveout,
                                      cudaSharedmemCarveoutMaxShared));
        attr_done = true;
    }
    if (deep && !deep_attr_done) {                      // sized for the largest k
        EZR_CUDA(cudaFuncSetAttribute(bm25_cand_kernel<true, S>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      (int)pk_deep_cand_smem(kSelMaxK)));
        EZR_CUDA(cudaFuncSetAttribute(bm25_cand_kernel<true, S>, cudaFuncAttributePreferredSharedMemoryCarveout,
                                      cudaSharedmemCarveoutMaxShared));
        EZR_CUDA(cudaFuncSetAttribute(bm25_bound_deep_kernel<S>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      (int)pk_deep_bound_smem(kSelMaxK)));
        deep_attr_done = true;
    }
    // Document ranges go in chunks of doubling size (4, 4, 8, 16, ...); between chunks every query's bound is
    // raised to the k-th best of all candidates so far, so the expected number of candidates a chunk adds stays
    // around k however many ranges it spans.
    {
        ProfScope prof(EZR_PROF_BM25_CAND, st);
        int r0 = 0, span = g_bm25_span;
        const int first = span;
        while (r0 < ix->n_ranges) {
            int len = ix->n_ranges - r0 < span ? ix->n_ranges - r0 : span;
            if (span < kPkMaxChunk && ix->n_ranges - (r0 + len) < span / 2) len = ix->n_ranges - r0;   // no tiny last chunk
            if (len > kPkMaxChunk) len = kPkMaxChunk;                                 // the plan table holds this many
            const int64_t n_plan = (int64_t)n_queries * len * kPkPlanTok;
            if (g_bm25_plan) {
                bm25_plan_kernel<<<(unsigned)((n_plan + 255) / 256), 256, 0, st>>>(p, r0, len, n_queries, w.plan);
                EZR_LAUNCH_CHECK();
            }
            if (deep) bm25_cand_kernel<true, S><<<dim3(n_queries, len), kPkThreads, smem, st>>>(p, c, r0);
            else bm25_cand_kernel<false, S><<<dim3(n_queries, len), kPkThreads, smem, st>>>(p, c, r0);
            EZR_LAUNCH_CHECK();
            r0 += len;
            if (r0 < ix->n_ranges) {
                ProfScope prof_bd(EZR_PROF_BM25_BOUND, st);   // inside the candidate span
                if (deep) bm25_bound_deep_kernel<S><<<n_queries, kBdThreads, bd_smem, st>>>(p, c);
                else bm25_bound_kernel<S><<<n_queries, kBdThreads, 0, st>>>(p, c);
                EZR_LAUNCH_CHECK();
            }
            if (r0 > first && span < kPkMaxChunk) span *= 2;
        }
    }
    {
        ProfScope prof(EZR_PROF_BM25_RESCORE, st);
        if (deep) bm25_rescore_deep_kernel<S><<<n_queries, kRsThreads, 0, st>>>(p, c, (S*)w.rows);
        else bm25_rescore_kernel<S><<<n_queries, kRsThreads, 0, st>>>(p, c, out_scores, out_ids, out_counts);
        EZR_LAUNCH_CHECK();
    }
    return EZR_OK;
}

static int check_index(const ezr_bm25_index* ix) {
    EZR_CHECK_ARG(ix != nullptr, "bm25: index is NULL");
    EZR_CHECK_ARG(ix->range_size == kBmRange, "bm25: range_size must be %d (got %d)", kBmRange, ix->range_size);
    EZR_CHECK_ARG(ix->n_docs >= 0 && ix->n_docs < ((int64_t)1 << 31), "bm25: n_docs out of range");
    EZR_CHECK_ARG(ix->n_ranges == ceil_div(ix->n_docs, kBmRange), "bm25: n_ranges != ceil(n_docs/range_size)");
    EZR_CHECK_ARG(ix->n_ranges <= 65535 * kBmRpc, "bm25: too many ranges (%d) for one shard", ix->n_ranges);
    EZR_CHECK_ARG(ix->score_type == EZR_F64 || ix->score_type == EZR_F32, "bm25: bad score_type");
    EZR_CHECK_ARG(ix->n_postings >= 0 && ix->n_postings < ((int64_t)1 << 31),
                  "bm25: %lld postings in one index; shard the corpus (limit 2^31-1 per shard)", (long long)ix->n_postings);
    return EZR_OK;
}

// ---- score rows in query blocks: k > 32 without the deep form, and the deep form's overflowed queries ----
// The rows of one block take at most kRowsBudget bytes, so the workspace does not grow with Q * n_docs.  A block's
// queries (a run of the batch, or entries of a query list) are gathered into a table with two q_ptr entries per
// query: block query i is table query 2i, which the ordered kernel reaches through its query list, with its terms
// read from the caller's q_terms, and whose row lands at 2i * n_docs (the odd rows are never written or read).
constexpr size_t kRowsBudget = (size_t)1 << 30;

__global__ void bm25_rows_gather_kernel(const int32_t* __restrict__ q_ptr, const int32_t* __restrict__ q_group,
                                        const int32_t* __restrict__ list, int j0, int nb, int32_t* __restrict__ qp,
                                        int32_t* __restrict__ ql, int32_t* __restrict__ qg, int32_t* __restrict__ cnt) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0) *cnt = nb;
    if (i >= nb) return;
    const int q = list ? list[j0 + i] : j0 + i;
    qp[2 * i] = q_ptr[q];
    qp[2 * i + 1] = q_ptr[q + 1];
    ql[i] = 2 * i;
    if (q_group) qg[i] = q_group[q];
}

template <typename S>
__global__ void bm25_rows_scatter_kernel(const S* __restrict__ bs, const int32_t* __restrict__ bi,
                                         const int32_t* __restrict__ bc, const int32_t* __restrict__ list, int j0,
                                         int k, S* __restrict__ out_s, int32_t* __restrict__ out_i,
                                         int32_t* __restrict__ out_c) {
    const int i = blockIdx.x;
    const int64_t q = list ? list[j0 + i] : j0 + i;
    for (int t = threadIdx.x; t < k; t += blockDim.x) {
        out_s[q * k + t] = bs[(int64_t)i * k + t];
        out_i[q * k + t] = bi[(int64_t)i * k + t];
    }
    if (threadIdx.x == 0) out_c[q] = bc[i];
}

struct RowsWorkspace {
    void* rows;
    void* sel;
    size_t sel_bytes;
    void* blk_s;
    int32_t *blk_i, *blk_c, *qp, *ql, *qg, *cnt;
    int block;
    size_t total;
};

static RowsWorkspace rows_carve(void* base, const ezr_bm25_index* ix, int n_queries, int k) {
    RowsWorkspace w;
    const bool f64 = ix->score_type == EZR_F64;
    const size_t ss = f64 ? 8 : 4, nd = (size_t)ix->n_docs;
    const size_t per = 2 * nd * ss;
    size_t b = per ? kRowsBudget / per : (size_t)n_queries;
    b = b < 1 ? 1 : (b > (size_t)n_queries ? (size_t)n_queries : b);
    w.block = (int)b;
    w.sel_bytes = 0;                                    // a smaller last block can need more (more parts per row)
    for (int m = 1; m <= w.block; ++m) {
        const size_t sb = f64 ? select_rows_ws<double>(m, ix->n_docs, k) : select_rows_ws<float>(m, ix->n_docs, k);
        if (sb > w.sel_bytes) w.sel_bytes = sb;
    }
    char* p = reinterpret_cast<char*>(base);
    size_t off = 0;
    w.rows = p + off;   off += align_up((2 * b - 1) * nd * ss, 256);
    w.sel = p + off;    off += align_up(w.sel_bytes, 256);
    w.blk_s = p + off;  off += align_up(b * k * ss, 256);
    w.blk_i = reinterpret_cast<int32_t*>(p + off);  off += align_up(b * k * 4, 256);
    w.blk_c = reinterpret_cast<int32_t*>(p + off);  off += align_up(b * 4, 256);
    w.qp = reinterpret_cast<int32_t*>(p + off);     off += align_up(2 * b * 4, 256);
    w.ql = reinterpret_cast<int32_t*>(p + off);     off += align_up(b * 4, 256);
    w.qg = reinterpret_cast<int32_t*>(p + off);     off += align_up(b * 4, 256);
    w.cnt = reinterpret_cast<int32_t*>(p + off);    off += 256;
    w.total = off;
    return w;
}

// top-k of queries list[0 .. n) (list == NULL: queries 0 .. n) from their score rows, block by block
template <typename S>
static int rows_topk(const ezr_bm25_index* ix, const int32_t* q_ptr, const int32_t* q_terms, int k,
                     const int32_t* q_group, int id_base, const int32_t* list, int n, S* out_s, int32_t* out_ids,
                     int32_t* out_counts, const RowsWorkspace& w, cudaStream_t st) {
    for (int j0 = 0; j0 < n; j0 += w.block) {
        const int nb = n - j0 < w.block ? n - j0 : w.block;
        bm25_rows_gather_kernel<<<ceil_div(nb, 256), 256, 0, st>>>(q_ptr, q_group, list, j0, nb, w.qp, w.ql, w.qg,
                                                                   w.cnt);
        EZR_LAUNCH_CHECK();
        int rc = bm25_launch<S>(ix, w.qp, q_terms, nb, k, nullptr, 0, 1, w.rows, nullptr, nullptr, st, w.ql, w.cnt);
        if (rc) return rc;
        rc = select_rows_impl<S>((const S*)w.rows, nb, ix->n_docs, 2 * ix->n_docs, k, 1, ix->doc_group,
                                 q_group ? w.qg : nullptr, id_base, (S*)w.blk_s, w.blk_i, w.blk_c, w.sel, w.sel_bytes,
                                 st);
        if (rc) return rc;
        bm25_rows_scatter_kernel<S><<<nb, 256, 0, st>>>((const S*)w.blk_s, w.blk_i, w.blk_c, list, j0, k, out_s,
                                                        out_ids, out_counts);
        EZR_LAUNCH_CHECK();
    }
    return EZR_OK;
}

// two-phase top-k, k <= 32: candidates from packed postings -> exact rescoring; overflowed queries (normally none)
// go through the ordered kernel, restricted to ovf_list.  lists: the ordered kernel's [Q][ranges][k] partial lists
// (scores, then ids at ids_off), followed by the two-phase workspace.
template <typename S>
static int pk_topk(const ezr_bm25_index* ix, const int32_t* q_ptr, const int32_t* q_terms, int n_queries, int k,
                   const int32_t* q_group, int id_base, void* lists, size_t ids_off, int32_t* thr, S* out_scores,
                   int32_t* out_ids, int32_t* out_counts, cudaStream_t st) {
    int32_t* pi = reinterpret_cast<int32_t*>((char*)lists + ids_off);
    const PkWorkspace w = pk_carve(thr, n_queries);
    EZR_CUDA(cudaMemsetAsync(thr, 0, w.zero_bytes, st));
    int rc = pk_launch<S>(ix, q_ptr, q_terms, n_queries, k, q_group, id_base, w, out_scores, out_ids, out_counts, st);
    if (rc) return rc;
    rc = bm25_launch<S>(ix, q_ptr, q_terms, n_queries, k, q_group, id_base, 0, lists, pi, w.thr_key, st, w.ovf_list,
                        w.ovf_n);
    if (rc) return rc;
    const int n_cand = ix->n_ranges * k;
    return merge_impl<S>((const S*)lists, pi, n_queries, n_cand, n_cand, k, id_base, out_scores, out_ids, out_counts,
                         st, w.ovf_list, w.ovf_n);
}

// deep form, 32 < k <= kSelMaxK: candidates from packed postings -> exact scores in [Q][cap] rows -> the select
// takes each top-k; overflowed queries (normally none) are then answered from their score rows
template <typename S>
static int pk_topk_deep(const ezr_bm25_index* ix, const int32_t* q_ptr, const int32_t* q_terms, int n_queries, int k,
                        const int32_t* q_group, int id_base, void* workspace, S* out_scores, int32_t* out_ids,
                        int32_t* out_counts, cudaStream_t st) {
    const int cap = pk_deep_list_cap(k);
    const PkWorkspace w = pk_carve(workspace, n_queries, cap, true, sizeof(S));
    const RowsWorkspace rw = rows_carve((char*)workspace + w.total, ix, n_queries, k);
    EZR_CUDA(cudaMemsetAsync(workspace, 0, w.zero_bytes, st));
    int rc = pk_launch<S>(ix, q_ptr, q_terms, n_queries, k, q_group, id_base, w, nullptr, nullptr, nullptr, st, true);
    if (rc) return rc;
    rc = launch_select<S>((const S*)w.rows, w.cand_ids, n_queries, cap, cap, 1, k, 1, nullptr, nullptr, id_base,
                          out_scores, out_ids, out_counts, st);
    if (rc) return rc;
    // the host learns how many queries overflowed (one small copy + stream sync) to size the score-row pass
    int32_t n_ovf = 0;
    EZR_CUDA(cudaMemcpyAsync(&n_ovf, w.ovf_n, 4, cudaMemcpyDeviceToHost, st));
    EZR_CUDA(cudaStreamSynchronize(st));
    if (n_ovf == 0) return EZR_OK;
    return rows_topk<S>(ix, q_ptr, q_terms, k, q_group, id_base, w.ovf_list, n_ovf, out_scores, out_ids, out_counts,
                        rw, st);
}

// ezr_bm25_pack / ezr_bm25_pack_f32: W = the stored weight type, widened to double exactly
template <typename W>
static int bm25_pack_impl(const int32_t* post_doc, const W* post_w, int64_t n_postings, int32_t range_size,
                          uint32_t* out_pk, int32_t* out_scale_log2, void* scratch16, cudaStream_t st) {
    EZR_CHECK_ARG(kPkEnabled, "bm25_pack: this build's range size %d is not a power of two", kBmRange);
    EZR_CHECK_ARG(range_size == kBmRange, "bm25_pack: range_size must be %d (got %d)", kBmRange, range_size);
    EZR_CHECK_ARG(out_scale_log2 != nullptr && scratch16 != nullptr, "bm25_pack: NULL argument");
    EZR_CHECK_ARG(n_postings >= 0 && n_postings < ((int64_t)1 << 31), "bm25_pack: n_postings out of range");
    *out_scale_log2 = 0;
    if (n_postings == 0) return EZR_OK;
    unsigned long long* d = reinterpret_cast<unsigned long long*>(scratch16);
    EZR_CUDA(cudaMemsetAsync(d, 0, 16, st));
    bm25_wmax_kernel<W><<<sm_count() * 8, 256, 0, st>>>(post_w, n_postings, d);
    EZR_LAUNCH_CHECK();
    unsigned long long h[2];
    EZR_CUDA(cudaMemcpyAsync(h, d, 16, cudaMemcpyDeviceToHost, st));
    EZR_CUDA(cudaStreamSynchronize(st));
    if (h[1] != 0ull) {
        set_error("bm25_pack: negative or non-finite contribution; the two-phase path needs non-negative weights");
        return EZR_ERR_INVALID;
    }
    double wmax;
    memcpy(&wmax, &h[0], 8);
    int e = 0;
    if (wmax > 0.0) {
        int ex;
        frexp(wmax, &ex);                       // wmax < 2^ex
        e = kPkWBits - 1 - ex;                  // wmax * 2^e < 2^(WBits-1): ceil() fits, sums of 2^(31-WBits) terms too
    }
    const double scale = ldexp(1.0, e);
    bm25_pack_kernel<W><<<(unsigned)((n_postings + 255) / 256), 256, 0, st>>>(post_doc, post_w, n_postings, scale,
                                                                             out_pk);
    EZR_LAUNCH_CHECK();
    *out_scale_log2 = e;
    return EZR_OK;
}

}  // namespace ezr

using namespace ezr;

extern "C" {

int ezr_bm25_range_size(void) { return kBmRange; }

int ezr_bm25_doc_norm(const int32_t* doc_len, int64_t n_docs, double k1, double b, double one_minus_b,
                      double avgdl, double* out_kd, void* stream) {
    if (n_docs == 0) return EZR_OK;
    bm25_doc_norm_kernel<<<ceil_div(n_docs, 256), 256, 0, (cudaStream_t)stream>>>(doc_len, n_docs, k1, b,
                                                                                  one_minus_b, avgdl, out_kd);
    EZR_LAUNCH_CHECK();
    return EZR_OK;
}

int ezr_bm25_weights(const int64_t* indptr, const int32_t* post_doc, const int32_t* post_tf, int32_t vocab,
                     int64_t n_postings, const double* idf, const double* kd, double num_scale,
                     int32_t score_type, void* out_w, void* stream) {
    if (n_postings == 0) return EZR_OK;
    EZR_CHECK_ARG(score_type == EZR_F64 || score_type == EZR_F32, "bm25_weights: bad score_type");
    const int64_t blocks = (n_postings + 255) / 256;
    EZR_CHECK_ARG(blocks < ((int64_t)1 << 31), "bm25_weights: too many postings");
    if (score_type == EZR_F64)
        bm25_weights_kernel<double><<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(
            indptr, post_doc, post_tf, vocab, n_postings, idf, kd, num_scale, (double*)out_w);
    else
        bm25_weights_kernel<float><<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(
            indptr, post_doc, post_tf, vocab, n_postings, idf, kd, num_scale, (float*)out_w);
    EZR_LAUNCH_CHECK();
    return EZR_OK;
}

int ezr_bm25_range_index(const int64_t* indptr, const int32_t* post_doc, int32_t vocab, int32_t range_size,
                         int32_t n_ranges, uint32_t* out_range_off, void* stream) {
    const int64_t total = (int64_t)vocab * (n_ranges + 1);
    if (total == 0) return EZR_OK;
    const int64_t blocks = (total + 255) / 256;
    EZR_CHECK_ARG(blocks < ((int64_t)1 << 31), "bm25_range_index: table too large");
    bm25_range_index_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(indptr, post_doc, vocab, range_size,
                                                                               n_ranges, out_range_off);
    EZR_LAUNCH_CHECK();
    return EZR_OK;
}

int ezr_bm25_pack(const int32_t* post_doc, const double* post_w, int64_t n_postings, int32_t range_size,
                  uint32_t* out_pk, int32_t* out_scale_log2, void* scratch16, void* stream) {
    return bm25_pack_impl<double>(post_doc, post_w, n_postings, range_size, out_pk, out_scale_log2, scratch16,
                                  (cudaStream_t)stream);
}

int ezr_bm25_pack_f32(const int32_t* post_doc, const float* post_w, int64_t n_postings, int32_t range_size,
                      uint32_t* out_pk, int32_t* out_scale_log2, void* scratch16, void* stream) {
    return bm25_pack_impl<float>(post_doc, post_w, n_postings, range_size, out_pk, out_scale_log2, scratch16,
                                 (cudaStream_t)stream);
}

int ezr_bm25_term_max(const int64_t* indptr, const uint32_t* post_pk, int32_t vocab, uint32_t* out_term_max,
                      void* stream) {
    EZR_CHECK_ARG(kPkEnabled, "bm25_term_max: this build has no packed postings");
    if (vocab <= 0) return EZR_OK;
    const int wpb = 8;
    bm25_term_max_kernel<<<ceil_div(vocab, wpb), wpb * 32, 0, (cudaStream_t)stream>>>(indptr, post_pk, vocab,
                                                                                      out_term_max);
    EZR_LAUNCH_CHECK();
    return EZR_OK;
}

int ezr_bm25_set_skipping(int32_t on) {
    g_bm25_skip = on != 0;
    return EZR_OK;
}

int ezr_bm25_set_span(int32_t first_ranges) {
    EZR_CHECK_ARG(first_ranges >= 1 && first_ranges <= kPkMaxChunk, "bm25_set_span: %d out of [1,%d]", first_ranges, kPkMaxChunk);
    g_bm25_span = first_ranges;
    return EZR_OK;
}

int ezr_bm25_set_plan(int32_t on) {
    g_bm25_plan = on != 0;
    return EZR_OK;
}

int ezr_bm25_cand_capacity(void) { return kPkEnabled ? kPkListCap : 0; }

size_t ezr_bm25_topk_workspace(const ezr_bm25_index* ix, int32_t n_queries, int32_t k) {
    if (!ix || n_queries <= 0 || k <= 0) return 0;
    const size_t ss = ix->score_type == EZR_F64 ? 8 : 4;
    if (k <= 32) {
        const size_t n = (size_t)n_queries * ix->n_ranges * k;
        const size_t lists = align_up(n * ss, 256) + align_up(n * 4, 256);
        if (pk_usable(ix, k)) return lists + pk_carve(nullptr, n_queries).total;
        return lists + align_up((size_t)n_queries * 4, 256);
    }
    // deep form: candidate lists and their score rows (Q * pk_deep_list_cap(k)), plus one block of score rows for
    // the queries that overflow them; otherwise blocks of score rows only
    const size_t rows = rows_carve(nullptr, ix, n_queries, k).total;
    if (pk_deep_usable(ix, k)) return pk_carve(nullptr, n_queries, pk_deep_list_cap(k), true, ss).total + rows;
    return rows;
}

int ezr_bm25_topk(const ezr_bm25_index* ix, const int32_t* q_ptr, const int32_t* q_terms, int32_t n_queries,
                  int32_t k, const int32_t* q_group, int32_t id_base, void* out_scores, int32_t* out_ids,
                  int32_t* out_counts, void* workspace, size_t workspace_bytes, void* stream) {
    int rc = check_index(ix);
    if (rc) return rc;
    EZR_CHECK_ARG(k >= 1 && k <= kSelMaxK, "bm25_topk: k=%d out of [1,%d]", k, kSelMaxK);
    // an empty shard's doc_group is empty, and an empty tensor has no address: nothing is filtered, so no check
    EZR_CHECK_ARG(q_group == nullptr || ix->doc_group != nullptr || ix->n_docs == 0,
                  "bm25_topk: q_group given but index has no doc_group");
    if (n_queries == 0) return EZR_OK;
    cudaStream_t st = (cudaStream_t)stream;
    const size_t need = ezr_bm25_topk_workspace(ix, n_queries, k);
    if (workspace_bytes < need || (need && !workspace)) {
        set_error("bm25_topk: workspace %zu < %zu", workspace_bytes, need);
        return EZR_ERR_WORKSPACE;
    }
    if (ix->n_docs == 0) {
        EZR_CUDA(cudaMemsetAsync(out_counts, 0, (size_t)n_queries * 4, st));
        EZR_CUDA(cudaMemsetAsync(out_ids, 0xff, (size_t)n_queries * k * 4, st));
        return EZR_OK;
    }
    const bool f64 = ix->score_type == EZR_F64;
    const size_t ss = f64 ? 8 : 4;
    if (k <= 32) {
        const size_t n = (size_t)n_queries * ix->n_ranges * k;
        void* ps = workspace;
        int32_t* pi = reinterpret_cast<int32_t*>((char*)workspace + align_up(n * ss, 256));
        int32_t* thr = reinterpret_cast<int32_t*>((char*)workspace + align_up(n * ss, 256) + align_up(n * 4, 256));
        if (pk_usable(ix, k)) {
            const size_t ids_off = align_up(n * ss, 256);
            return f64 ? pk_topk<double>(ix, q_ptr, q_terms, n_queries, k, q_group, id_base, ps, ids_off, thr,
                                         (double*)out_scores, out_ids, out_counts, st)
                       : pk_topk<float>(ix, q_ptr, q_terms, n_queries, k, q_group, id_base, ps, ids_off, thr,
                                        (float*)out_scores, out_ids, out_counts, st);
        }
        EZR_CUDA(cudaMemsetAsync(thr, 0, (size_t)n_queries * 4, st));
        rc = f64 ? bm25_launch<double>(ix, q_ptr, q_terms, n_queries, k, q_group, id_base, 0, ps, pi, thr, st)
                 : bm25_launch<float>(ix, q_ptr, q_terms, n_queries, k, q_group, id_base, 0, ps, pi, thr, st);
        if (rc) return rc;
        const int n_cand = ix->n_ranges * k;
        return f64 ? merge_impl<double>((const double*)ps, pi, n_queries, n_cand, n_cand, k, id_base,
                                        (double*)out_scores, out_ids, out_counts, st)
                   : merge_impl<float>((const float*)ps, pi, n_queries, n_cand, n_cand, k, id_base,
                                       (float*)out_scores, out_ids, out_counts, st);
    }
    if (pk_deep_usable(ix, k))
        return f64 ? pk_topk_deep<double>(ix, q_ptr, q_terms, n_queries, k, q_group, id_base, workspace,
                                          (double*)out_scores, out_ids, out_counts, st)
                   : pk_topk_deep<float>(ix, q_ptr, q_terms, n_queries, k, q_group, id_base, workspace,
                                         (float*)out_scores, out_ids, out_counts, st);
    const RowsWorkspace rw = rows_carve(workspace, ix, n_queries, k);
    return f64 ? rows_topk<double>(ix, q_ptr, q_terms, k, q_group, id_base, nullptr, n_queries, (double*)out_scores,
                                   out_ids, out_counts, rw, st)
               : rows_topk<float>(ix, q_ptr, q_terms, k, q_group, id_base, nullptr, n_queries, (float*)out_scores,
                                  out_ids, out_counts, rw, st);
}

int ezr_bm25_scores(const ezr_bm25_index* ix, const int32_t* q_ptr, const int32_t* q_terms, int32_t n_queries,
                    void* out_scores, void* stream) {
    int rc = check_index(ix);
    if (rc) return rc;
    if (n_queries == 0 || ix->n_docs == 0) return EZR_OK;
    return ix->score_type == EZR_F64
               ? bm25_launch<double>(ix, q_ptr, q_terms, n_queries, 1, nullptr, 0, 1, out_scores, nullptr, nullptr,
                                     (cudaStream_t)stream)
               : bm25_launch<float>(ix, q_ptr, q_terms, n_queries, 1, nullptr, 0, 1, out_scores, nullptr, nullptr,
                                    (cudaStream_t)stream);
}

size_t ezr_select_rows_workspace(int32_t n_rows, int64_t n_cols, int32_t k, int32_t score_type) {
    if (n_rows <= 0 || n_cols <= 0 || k <= 0) return 0;
    return score_type == EZR_F64 ? select_rows_ws<double>(n_rows, n_cols, k) : select_rows_ws<float>(n_rows, n_cols, k);
}

int ezr_select_rows(const void* scores, int32_t score_type, int32_t n_rows, int64_t n_cols, int64_t row_stride,
                    int32_t k, int32_t positive_only, const int32_t* doc_group, const int32_t* q_group,
                    int32_t id_base, void* out_scores, int32_t* out_ids, int32_t* out_counts, void* workspace,
                    size_t workspace_bytes, void* stream) {
    EZR_CHECK_ARG(k >= 1 && k <= kSelMaxK, "select_rows: k=%d out of [1,%d]", k, kSelMaxK);
    EZR_CHECK_ARG(score_type == EZR_F64 || score_type == EZR_F32, "select_rows: bad score_type");
    EZR_CHECK_ARG(n_cols < ((int64_t)1 << 31), "select_rows: n_cols too large");
    EZR_CHECK_ARG(q_group == nullptr || doc_group != nullptr, "select_rows: q_group without doc_group");
    if (n_rows == 0) return EZR_OK;
    cudaStream_t st = (cudaStream_t)stream;
    if (n_cols == 0) {
        if (out_counts) EZR_CUDA(cudaMemsetAsync(out_counts, 0, (size_t)n_rows * 4, st));
        EZR_CUDA(cudaMemsetAsync(out_ids, 0xff, (size_t)n_rows * k * 4, st));
        return EZR_OK;
    }
    return score_type == EZR_F64
               ? select_rows_impl<double>((const double*)scores, n_rows, n_cols, row_stride, k, positive_only,
                                          doc_group, q_group, id_base, (double*)out_scores, out_ids, out_counts,
                                          workspace, workspace_bytes, st)
               : select_rows_impl<float>((const float*)scores, n_rows, n_cols, row_stride, k, positive_only,
                                         doc_group, q_group, id_base, (float*)out_scores, out_ids, out_counts,
                                         workspace, workspace_bytes, st);
}

size_t ezr_merge_topk_workspace(int32_t, int32_t, int32_t, int32_t) { return 0; }

int ezr_merge_topk(const void* cand_scores, const int32_t* cand_ids, int32_t score_type, int32_t n_rows,
                   int32_t n_cand, int64_t cand_stride, int32_t k, void* out_scores, int32_t* out_ids,
                   int32_t* out_counts, void*, size_t, void* stream) {
    EZR_CHECK_ARG(k >= 1 && k <= kSelMaxK, "merge_topk: k=%d out of [1,%d]", k, kSelMaxK);
    EZR_CHECK_ARG(score_type == EZR_F64 || score_type == EZR_F32, "merge_topk: bad score_type");
    EZR_CHECK_ARG(n_cand >= 0 && cand_stride >= n_cand, "merge_topk: bad n_cand/stride");
    cudaStream_t st = (cudaStream_t)stream;
    return score_type == EZR_F64
               ? merge_impl<double>((const double*)cand_scores, cand_ids, n_rows, n_cand, cand_stride, k, 0,
                                    (double*)out_scores, out_ids, out_counts, st)
               : merge_impl<float>((const float*)cand_scores, cand_ids, n_rows, n_cand, cand_stride, k, 0,
                                   (float*)out_scores, out_ids, out_counts, st);
}

int ezr_merge_topk_parts(const void* cand_scores, const int32_t* cand_ids, int32_t score_type, int32_t n_rows,
                         int32_t n_cand, int64_t cand_stride, int32_t n_parts, int64_t part_stride_bytes, int32_t k,
                         void* out_scores, int32_t* out_ids, int32_t* out_counts, void* stream) {
    EZR_CHECK_ARG(k >= 1 && k <= 32, "merge_topk_parts: k=%d out of [1,32]", k);
    EZR_CHECK_ARG(score_type == EZR_F64 || score_type == EZR_F32, "merge_topk_parts: bad score_type");
    EZR_CHECK_ARG(n_cand >= 0 && cand_stride >= n_cand, "merge_topk_parts: bad n_cand/stride");
    EZR_CHECK_ARG(n_parts >= 1 && part_stride_bytes >= 0 && part_stride_bytes % 8 == 0,
                  "merge_topk_parts: bad n_parts/part_stride_bytes");
    cudaStream_t st = (cudaStream_t)stream;
    return score_type == EZR_F64
               ? merge_impl<double>((const double*)cand_scores, cand_ids, n_rows, n_cand, cand_stride, k, 0,
                                    (double*)out_scores, out_ids, out_counts, st, nullptr, nullptr, n_parts,
                                    part_stride_bytes)
               : merge_impl<float>((const float*)cand_scores, cand_ids, n_rows, n_cand, cand_stride, k, 0,
                                   (float*)out_scores, out_ids, out_counts, st, nullptr, nullptr, n_parts,
                                   part_stride_bytes);
}

}  // extern "C"
