// Two-phase BM25 top-k (float64 Okapi and float32 bm25s indices with non-negative weights): included by bm25.cu.
//
// The ordered float64 accumulation of bm25_score_kernel pays one block barrier per query term to reproduce the
// reference's sum order (retrievers.py:128-151 -> rank_bm25 get_scores adds term by term) for EVERY document,
// although only the few documents near the top-k boundary need their exact score.  Here:
//
//   phase 1  bm25_cand_kernel      integer upper-bound scores from 4-byte packed postings
//                                  (doc-in-range | ceil(w * 2^e)), shared-memory integer atomics, NO ordering and
//                                  no per-term barrier; documents that may reach the top-k are appended to a
//                                  per-query candidate list.
//   phase 2  bm25_rescore_kernel   every candidate's exact score (float64 or float32), terms added strictly in token order
//                                  (binary search of the candidate in each term's posting segment), then the
//                                  canonical top-k of the candidates.
//
// Why the candidate set is a superset of the exact top-k.  For a document d and a query of m tokens let
//   s(d)  = the reference's float64 score (sequentially rounded sum of the stored contributions w_j),
//   Q(d)  = sum_j ceil(w_j * S) (S = 2^e, the multiplication is exact), the integer phase 1 accumulates.
// The real sum R = sum w_j satisfies S*R <= Q <= S*R + m, and |s - R| <= m * 2^-53 * R, far below 1/S.  Hence
//   Q(d) - m - 1  <=  S*s(d)  <=  Q(d) + 1.
// If k distinct documents have Q >= G then the final k-th best score s* has S*s* >= B := G - m - 1, and a
// document with Q(d) + 1 < B cannot reach the top-k.  Phase 1 keeps every document with Q(d) >= B - 1 where B is
// the running bound of the query (raised with atomicMax as document ranges complete), phase 2 decides exactly.
// Queries whose candidate list overflows (mass ties) are handed to bm25_score_kernel, so results never depend on
// the capacity constants.
//
// Skipping the long posting lists (MaxScore).  Let gm_j be the largest packed weight of token j's term.  Once a
// bound B exists, bm25_bound_kernel marks as NON-ESSENTIAL the tokens with the smallest gm whose sum NE stays
// below kPkNeNum/kPkNeDen of B - 1.  The candidate pass does not read their postings at all: with
// Q = Q_ess + Q_ne and Q_ne <= NE, a document with Q >= B - 1 has Q_ess >= B - 1 - NE, so that becomes the
// crossing threshold.  The high-df terms have the smallest weights and the longest lists.  Pushing those relaxed
// crossers as candidates with partial bounds (L = Q_ess, U = L + NE) made the candidate pass faster, but candidates
// multiplied and the rescoring ate the gain.  So the kernel COMPLETES the relaxed crossers
// inside the candidate kernel (binary search of each skipped token's postings for just those documents) and then
// applies the exact test, so the candidate set and the bounds are those of a full pass (L = U = Q).
//
// Float32 scores (bm25s, Lucene idf log(1 + (N - df + 0.5)/(df + 0.5)) > 0, so every such index is monotone).  bm25s
// adds a query's contributions with np.add.at token by token, so s(d) is a float32 sum rounded after every add
// (u = 2^-24).  For m non-negative addends the sequential sum satisfies |s - R| <= gamma_{m-1} * R with
// gamma_n = n*u / (1 - n*u).  The weights are widened to double (exactly) and packed with the same scale rule, so
// S*w < 2^(kPkWBits-1) = 2^18 for every posting and S*R < m * 2^18.  Hence, with
//   e(m) = ceil(gamma_{m-1} * m * 2^18) = ceil((m-1) * m * 2^18 / (2^24 - (m-1)))      (0 at m = 1, 14 at m = 30,
//                                                                                      2^18 at kPkMaxTerms)
//   Q(d) - m - e(m)  <=  S*s(d)  <=  Q(d) + e(m).
// The float64 bracket above is the same statement with u = 2^-53: there gamma_{m-1} * m * 2^18 < 1 for every
// m <= kPkMaxTerms, so e = 1.  Everything else carries over with e in place of that 1: B := G - m - e, a document
// is kept when Q(d) >= B - e (S*s(d) >= B is then possible), the bound steps subtract m + e, and with skipped
// tokens the relaxed crossing threshold is B - e - NE.  PkSlack<S>::e is that constant; the candidate and bound
// kernels are instantiated per score type (the float64 instances compile to the code they had with the literal 1),
// and phase 2 adds float32 contributions with __fadd_rn in token order from +0.0f (absent tokens add +0.0f, exact).
// All integer quantities stay below 2^31: Q <= kPkMaxTerms * 2^18 = 2^30 and e(m) <= 2^18.
#pragma once
#include <type_traits>

namespace ezr {

constexpr int ilog2_c(int v) { return v <= 1 ? 0 : 1 + ilog2_c(v >> 1); }
constexpr bool kPkEnabled = (kBmRange & (kBmRange - 1)) == 0;
constexpr int kPkDocBits = ilog2_c(kBmRange);
constexpr int kPkWBits = 32 - kPkDocBits;                 // 19 bits of weight for 8192-document ranges
constexpr uint32_t kPkWMask = (1u << kPkWBits) - 1u;
constexpr int kPkMaxTerms = 1 << (31 - kPkWBits);         // packed weights are < 2^(WBits-1): sums stay below 2^30
constexpr int kPkLocalCap = 512;                          // candidates one (query, range) CTA can hold
constexpr int kPkPlanTok = 16;                            // tokens per query resolved by the plan kernel (the rest in-kernel)
constexpr int kPkMaxChunk = 32;                           // document ranges per candidate launch (size of the plan table)
#ifndef EZR_BM25_CAND_CAP
#define EZR_BM25_CAND_CAP 1024
#endif
constexpr int kPkListCap = EZR_BM25_CAND_CAP;             // candidates per query (per shard)
#ifndef EZR_BM25_PK_MINB
#define EZR_BM25_PK_MINB 6
#endif
#ifndef EZR_BM25_PK_THREADS
#define EZR_BM25_PK_THREADS 256
#endif
#ifndef EZR_BM25_PK_NE_NUM
#define EZR_BM25_PK_NE_NUM 3
#endif
constexpr int kPkNeNum = EZR_BM25_PK_NE_NUM;             // tokens worth up to NUM/10 of the bound may be skipped (0: off)
constexpr int kPkNeDen = 10;
#ifndef EZR_BM25_PK_VOTE_EACH
#define EZR_BM25_PK_VOTE_EACH 0
#endif
#ifndef EZR_BM25_PK_BRANCHY
#define EZR_BM25_PK_BRANCHY 0
#endif
#ifndef EZR_BM25_PK_UNROLL
#define EZR_BM25_PK_UNROLL 8
#endif
constexpr int kPkThreads = EZR_BM25_PK_THREADS;           // candidate-pass CTA (independent of the ordered kernel's)
// Deep form (32 < k <= 1024): the capacities grow with k.  A (query, range) CTA without a bound keeps the documents
// within the slack of its exact k-th best sum (k plus ties); with a bound, those crossing it.  Between range chunks
// the bound kernel cuts every list back to about k, and the next chunk adds about k more (its ranges are compared
// against the k-th best of all ranges before it).  The first chunk's ranges may all run before any bound exists
// (small batches): four ranges of k each.  Hence 2k + 512 per (query, range) and 4k + 1024 per query; a query that
// overflows either is answered from its score row, so results never depend on these numbers.
__host__ __device__ constexpr int pk_deep_local_cap(int k) { return 2 * k + 512; }
__host__ __device__ constexpr int pk_deep_list_cap(int k) { return 4 * k + 1024; }
constexpr int kPkHist = 256 + 4;                          // radix-select bins + broadcast slots (block_kth_largest)
constexpr int kPkGroup = kPkThreads / 32;                 // lanes per group: 32 disjoint group maxima
static_assert(kPkThreads % 32 == 0 && kPkThreads >= 64 && (kPkGroup & (kPkGroup - 1)) == 0, "bad EZR_BM25_PK_THREADS");
static_assert(kBmRange % (4 * kPkThreads) == 0, "range must be a multiple of 4 * EZR_BM25_PK_THREADS");

// e(m) of the bracket  Q - m - e <= S*s <= Q + e  for a query of m tokens (header): the rounding error of the
// sequential sum in the score type, in units of 1/S.
template <typename S> struct PkSlack;
template <> struct PkSlack<double> {
    static __host__ __device__ constexpr int e(int) { return 1; }
};
template <> struct PkSlack<float> {
    static __host__ __device__ constexpr int e(int m) {
        const int64_t n = m > 1 ? m - 1 : 0;              // gamma_{m-1} = n*2^-24 / (1 - n*2^-24), exactly in integers
        const int64_t num = n * m * ((int64_t)1 << (kPkWBits - 1)), den = ((int64_t)1 << 24) - n;
        return (int)((num + den - 1) / den);
    }
};
static_assert(kPkWBits != 19 || (PkSlack<float>::e(1) == 0 && PkSlack<float>::e(2) == 1 &&
                                 PkSlack<float>::e(30) == 14 && PkSlack<float>::e(kPkMaxTerms) == 262144),
              "float32 slack e(m)");

struct PkParams {
    const uint32_t* post_pk;   // [n_postings]
    int32_t* thr_q;            // [Q] running bound B (integer domain), zeroed per call
    int32_t* cand_cnt;         // [Q] zeroed per call
    int32_t* cand_ids;         // [Q][kPkListCap] shard-local document ids
    int32_t* cand_q;           // [Q][kPkListCap] lower bounds L(d) of their integer scores (skipped tokens left out)
    int32_t* cand_u;           // [Q][kPkListCap] upper bounds U(d) = L(d) + NE at the time of the push
    const uint32_t* term_max;  // [vocab] largest packed weight of each term in this shard, or NULL (no skipping)
    uint32_t* ne_mask;         // [Q] zeroed per call: tokens (of the first 32) the candidate pass may skip
    int32_t* ne_sum;           // [Q] zeroed per call: NE = sum of term_max over those tokens
    int32_t* ovf;              // [Q] zeroed per call: 1 = hand the query to the ordered kernel
    int32_t* ovf_n;            // [1] zeroed per call
    int32_t* ovf_list;         // [Q]
    int2* plan;                // [Q][ranges of the chunk][kPkPlanTok] (first posting, postings) of token j in that range
};

// ---- index build: largest weight (as bits; non-negative doubles order like their bit patterns) + validity ----
// W: the stored weight type; float32 weights are widened to double, which is exact.
template <typename W>
__global__ void bm25_wmax_kernel(const W* __restrict__ w, int64_t n, unsigned long long* __restrict__ out) {
    unsigned long long mx = 0ull;
    int bad = 0;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const double v = (double)w[i];
        if (!(v >= 0.0) || isinf(v)) bad = 1;
        else mx = max(mx, (unsigned long long)__double_as_longlong(v));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        bad |= __shfl_xor_sync(0xffffffffu, bad, o);
    }
    if ((threadIdx.x & 31) == 0) {
        atomicMax(out, mx);
        if (bad) atomicMax(out + 1, 1ull);
    }
}

template <typename W>
__global__ void bm25_pack_kernel(const int32_t* __restrict__ post_doc, const W* __restrict__ w, int64_t n,
                                 double scale, uint32_t* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double x = ceil(__dmul_rn((double)w[i], scale));   // exact product (power of two), exact ceil
    out[i] = ((uint32_t)(post_doc[i] & (kBmRange - 1)) << kPkWBits) | (uint32_t)x;
}

// largest packed weight of every term (one warp per term, index-build time)
__global__ void bm25_term_max_kernel(const int64_t* __restrict__ indptr, const uint32_t* __restrict__ pk, int vocab,
                                     uint32_t* __restrict__ out) {
    const int t = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (t >= vocab) return;
    uint32_t mx = 0u;
    for (int64_t i = indptr[t] + lane; i < indptr[t + 1]; i += 32) mx = max(mx, pk[i] & kPkWMask);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if (lane == 0) out[t] = mx;
}

// ---- per (query, range, token): where the token's postings of that range start and how many there are ----
// Resolved ONCE per candidate launch by fully parallel threads (token -> term -> range table -> offsets is a chain of
// three dependent loads); bm25_cand_kernel then starts from one coalesced 8-byte load per lane instead of walking that
// chain inside every (query, range) CTA while seven of its eight warps wait at a barrier.
__global__ void bm25_plan_kernel(const Bm25Params p, int r_begin, int n_r, int n_queries, int2* __restrict__ plan) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (int64_t)n_queries * n_r * kPkPlanTok) return;
    const int tk = (int)(i % kPkPlanTok);
    const int rr = (int)((i / kPkPlanTok) % n_r);
    const int q = (int)(i / ((int64_t)kPkPlanTok * n_r));
    const int qs = p.q_ptr[q];
    const int m = p.q_ptr[q + 1] - qs;
    int2 e = make_int2(0, 0);
    if (tk < m) {
        const int t = p.q_terms[qs + tk];
        if (t >= 0 && t < p.vocab) {
            const uint32_t* ro = p.range_off + (int64_t)t * (p.n_ranges + 1) + (r_begin + rr);
            const uint32_t o0 = __ldg(ro), o1 = __ldg(ro + 1);
            e.x = (int)__ldg(p.indptr + t) + (int)o0;
            e.y = (int)(o1 - o0);
        }
    }
    plan[i] = e;
}

// k-th largest POSITIVE value among val(0) .. val(n-1), equal values counted separately; 0 when fewer than k are
// positive.  Radix select in shared memory: 8-bit digits from the highest set bit of the largest value down, each
// pass histograms the values that agree with the digits fixed so far.  sh: kPkHist ints.  Every one of the NT
// threads calls it (it synchronises); n and k are block-uniform.
template <int NT, typename F>
__device__ uint32_t block_kth_largest(F val, const int n, const int k, int* sh) {
    const int tid = threadIdx.x, lane = tid & 31;
    if (tid == 0) sh[256] = 0;
    __syncthreads();
    uint32_t vmax = 0u;
    for (int i = tid; i < n; i += NT) vmax = max(vmax, val(i));
    vmax = __reduce_max_sync(0xffffffffu, vmax);
    if (lane == 0) atomicMax(reinterpret_cast<unsigned*>(sh + 256), vmax);
    __syncthreads();
    const uint32_t top = (uint32_t)sh[256];
    uint32_t prefix = 0u, mask = 0u;
    int kk = k;                                          // rank still to find among the values that match prefix
    int s = max(32 - __clz(top) - 8, 0);
    for (;;) {
        for (int i = tid; i < 256; i += NT) sh[i] = 0;
        __syncthreads();
        for (int i = tid; i < n; i += NT) {
            const uint32_t v = val(i);
            if (v != 0u && (v & mask) == prefix) atomicAdd(&sh[(v >> s) & 255u], 1);
        }
        __syncthreads();
        if (tid < 32) {                                  // lane l holds bins 255-8l .. 248-8l (descending)
            int c[8], sum = 0;
#pragma unroll
            for (int j = 0; j < 8; ++j) { c[j] = sh[255 - 8 * lane - j]; sum += c[j]; }
            int inc = sum;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int v = __shfl_up_sync(0xffffffffu, inc, o);
                if (lane >= o) inc += v;
            }
            int above = inc - sum;
            if (above < kk && kk <= inc) {               // exactly one lane: the digit of the k-th value is here
                int d = -1, a = 0;
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    if (d < 0 && above + c[j] >= kk) { d = 255 - 8 * lane - j; a = above; }
                    above += c[j];
                }
                sh[257] = d;
                sh[258] = a;
            }
            if (lane == 31 && inc < kk) sh[257] = -1;    // fewer than k positive values (first pass only)
        }
        __syncthreads();
        const int d = sh[257], above = sh[258];
        __syncthreads();                                 // the bins and slots are rewritten by the next pass
        if (d < 0) return 0u;
        prefix = (prefix & ~(255u << s)) | ((uint32_t)d << s);
        mask |= 255u << s;
        kk -= above;
        if (s == 0) return prefix;
        s = max(s - 8, 0);                               // the last pass may overlap fixed bits: they match prefix
    }
}

// ---- phase 1 ----
// One CTA per (query, document range).  Work is dealt to warps in pieces of kPkPiece postings (256 by default) over
// ALL terms of the query (a warp's lanes each hold one term's segment; ballot + shuffles map a piece number to its
// term), so a warp only executes code for pieces that exist: no per-term pass over empty segments, no ordering, one barrier before the
// atomics and one after.
constexpr int kPkWarps = kPkThreads / 32;
constexpr int kPkUnroll = EZR_BM25_PK_UNROLL;                             // loads a lane keeps in flight
constexpr int kPkPiece = 32 * kPkUnroll;                 // postings per work item

// DEEP (32 < k <= 1024): the first bound of a range is its exact k-th best sum (block_kth_largest over the
// accumulators), the candidate list lives in dynamic shared memory behind the accumulators, the capacities are
// pk_deep_local_cap / pk_deep_list_cap, and the in-range raise is a select over the range's candidates.  (A kernel
// template, not a body inlined into two kernels: inlining changes the k <= 32 instance's register allocation.)
// S: the index's score type, which fixes the slack e(m) of the bracket (PkSlack).
template <bool DEEP, typename S>
__global__ void __launch_bounds__(kPkThreads, DEEP ? 4 : EZR_BM25_PK_MINB)
bm25_cand_kernel(const Bm25Params p, const PkParams c, const int r_begin) {
    extern __shared__ __align__(16) unsigned char pk_smem_raw[];
    uint32_t* acc = reinterpret_cast<uint32_t*>(pk_smem_raw);   // [kBmRange + 32] integer upper-bound scores + spare
    __shared__ int s_wi_fixed[DEEP ? 1 : kPkLocalCap];
    __shared__ int s_cnt, s_b, s_thr;
    // DEEP: [kBmRange + 32] accumulators | [kPkHist] select scratch | [pk_deep_local_cap(k)] candidate list
    int* s_hist = reinterpret_cast<int*>(acc + kBmRange + 32);
    int* s_wi = DEEP ? s_hist + kPkHist : s_wi_fixed;
    const int local_cap = DEEP ? pk_deep_local_cap(p.k) : kPkLocalCap;
    const int list_cap = DEEP ? pk_deep_list_cap(p.k) : kPkListCap;

    const int q = blockIdx.x, r = r_begin + blockIdx.y;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int qs = p.q_ptr[q];
    const int m = p.q_ptr[q + 1] - qs;
    if (m > kPkMaxTerms) {                               // block-uniform: the integer sums could wrap
        if (tid == 0) c.ovf[q] = 1;
        return;
    }
    const int es = PkSlack<S>::e(m);                     // e(m): keep Q >= B - e, bounds step down by m + e
    const int rbase = r * kBmRange;
    const uint32_t* __restrict__ pk = c.post_pk;
    const int want = p.q_group ? p.q_group[q] : -1;
    // lane j of every warp: posting segment of token tb + j in this range
    auto load_seg = [&](int tb, int& beg, int& len) {
        beg = 0; len = 0;
        if (tb + lane < m) {
            const int t = p.q_terms[qs + tb + lane];
            if (t >= 0 && t < p.vocab) {
                const uint32_t* ro = p.range_off + (int64_t)t * (p.n_ranges + 1) + r;
                const uint32_t o0 = __ldg(ro), o1 = __ldg(ro + 1);
                beg = (int)__ldg(p.indptr + t) + (int)o0;
                len = (int)(o1 - o0);
            }
        }
    };
    // Set-up of the (query, range): the first kPkPlanTok token segments come from the plan table (one coalesced
    // 8-byte load per lane, no dependent chain), later tokens (queries longer than kPkPlanTok) are resolved here.
    __shared__ int s_ne, s_nm;
    int beg = 0, len = 0;
    if (c.plan != nullptr && lane < kPkPlanTok) {
        const int2 e = __ldg(c.plan + ((int64_t)q * gridDim.y + blockIdx.y) * kPkPlanTok + lane);
        beg = e.x; len = e.y;
    } else if (lane < m) {
        load_seg(0, beg, len);                           // tokens past the plan table (or no plan: A/B switch)
    }
    if (tid == kPkThreads - 1) {
        const int b0 = *reinterpret_cast<const volatile int32_t*>(c.thr_q + q);
        // tokens bm25_bound_kernel declared non-essential for this query (valid for every later, higher bound): their
        // postings are not read, their largest possible contribution NE is taken off the crossing threshold instead
        const uint32_t nm = (b0 > 0 && c.term_max) ? __ldg(c.ne_mask + q) : 0u;
        s_b = b0;
        s_cnt = 0;
        s_ne = nm ? __ldg(c.ne_sum + q) : 0;
        s_nm = (int)nm;
    }
    {
        uint4* a4 = reinterpret_cast<uint4*>(acc);
#pragma unroll
        for (int i = 0; i < kBmRange / 4 / kPkThreads; ++i) a4[tid + i * kPkThreads] = make_uint4(0u, 0u, 0u, 0u);
        if (tid < 32) acc[kBmRange + tid] = 0u;         // spare slots of apply()
    }
    __syncthreads();

    if (((uint32_t)s_nm >> lane) & 1u) len = 0;           // skipped tokens: first token batch only (the mask covers 0..31)
    const int bound = s_b;                               // B: lower bound of S * (k-th best exact score), 0 = none yet
    const bool track = bound > 0;
    const int ne = s_ne;
    // crossing test in one unsigned compare: old < tq <= old + wq  <=>  tq - 1 - old < wq  (wraps to a huge value
    // when old >= tq; without a bound tq1 = 2^32-1: ~old is never below a packed weight)
    const uint32_t tq1 = track ? (uint32_t)max(bound - es - ne, 1) - 1u : 0xffffffffu;
    // Lanes without a posting add 0 to a private spare slot behind the accumulators (no branch around the atomic,
    // no same-address serialisation); crossings are rare: the caller votes and only then takes the push path.
    const uint32_t spare = (uint32_t)(kBmRange + lane);
    auto apply = [&](uint32_t x) -> bool {
        const uint32_t wq = x & kPkWMask;
#if EZR_BM25_PK_BRANCHY      // A/B switch: predicate the atomic instead (idle lanes issue nothing)
        if (x == 0u) return false;
        const uint32_t dl = x >> kPkWBits;
#else
        const uint32_t dl = x != 0u ? (x >> kPkWBits) : spare;
#endif
        const uint32_t old = atomicAdd(&acc[dl], wq);
        return tq1 - old < wq;                           // weights are non-negative: a document crosses once
    };
    auto push = [&](uint32_t x) {
        const uint32_t dl = x >> kPkWBits;
        if (want == -1 || p.doc_group[rbase + (int)dl] == want) {
            const int idx = atomicAdd(&s_cnt, 1);
            if (idx < local_cap) s_wi[idx] = (int)dl;
        }
    };
    for (int tb = 0; tb < m; tb += 32) {
        if (tb > 0) load_seg(tb, beg, len);
        // exclusive prefix of piece counts over the 32 tokens of this batch (a piece = kPkPiece postings of one
        // token: kPkUnroll loads per lane in flight, the piece -> token mapping is paid once per piece)
        const int nch = (len + kPkPiece - 1) / kPkPiece;
        int inc = nch;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int v = __shfl_up_sync(0xffffffffu, inc, o);
            if (lane >= o) inc += v;
        }
        const int pre = inc - nch;
        const int total = __shfl_sync(0xffffffffu, inc, 31);
        for (int g = warp; g < total; g += kPkWarps) {
            // token whose piece range contains g: the last lane with pre <= g (empty tokens share a prefix with
            // their successor and are skipped by taking the last one)
            const unsigned mask = __ballot_sync(0xffffffffu, pre <= g);
            const int j = 31 - __clz(mask);
            const int jb = __shfl_sync(0xffffffffu, beg, j);
            const int jl = __shfl_sync(0xffffffffu, len, j);
            const int jp = __shfl_sync(0xffffffffu, pre, j);
            const int o0 = (g - jp) * kPkPiece + lane;
            const uint32_t* src = pk + jb + o0;
            // 32-posting slots this piece really has (warp-uniform).  Most segments of a (query, range) are short
            // (a rare term has a handful of postings in 8192 documents), so the work item comes in three sizes --
            // 1, 4 or kPkUnroll slots -- behind a warp-uniform branch: a short segment executes one load + one atomic
            // instead of kPkUnroll predicated-off copies of them.
            const int n_u = (jl - (g - jp) * kPkPiece + 31) >> 5;
            auto run = [&](auto tag) {
                constexpr int NU = decltype(tag)::value;
                uint32_t x[NU];
#pragma unroll
                for (int u = 0; u < NU; ++u) x[u] = (o0 + u * 32 < jl) ? __ldg(src + u * 32) : 0u;
#if EZR_BM25_PK_VOTE_EACH    // A/B switch: one warp vote per posting slot (the first version)
#pragma unroll
                for (int u = 0; u < NU; ++u) {
                    const bool crossed = apply(x[u]);
                    if (__any_sync(0xffffffffu, crossed)) {  // warp-uniform branch; almost never taken
                        if (crossed) push(x[u]);
                    }
                }
#else
                // one vote per work item: crossings are collected in a bit mask; the (rare) push path re-reads its
                // posting instead of keeping all loaded words live across the vote
                unsigned crossed = 0u;
#pragma unroll
                for (int u = 0; u < NU; ++u) crossed |= (apply(x[u]) ? 1u : 0u) << u;
                if (__any_sync(0xffffffffu, crossed != 0u)) {
#pragma unroll 1
                    for (int u = 0; u < NU; ++u)
                        if ((crossed >> u) & 1u) push(__ldg(src + u * 32));
                }
#endif
            };
            if (n_u <= 1) run(std::integral_constant<int, 1>{});
            else if (n_u <= 4 && kPkUnroll > 4) run(std::integral_constant<int, 4>{});
            else run(std::integral_constant<int, kPkUnroll>{});
        }
    }
    __syncthreads();                                     // every contribution of this (query, range) is in acc

    const int slack = m + es;
    if (!track) {
        // No bound yet (first ranges of a query): k-th largest of 32 disjoint group maxima = G, then compact.
        constexpr int kPer = kBmRange / kPkThreads;
        uint32_t tmax = 0u;
        if constexpr (DEEP) {
            // G = the exact k-th best sum of the range's documents in the query's group (the others are zeroed
            // first; the documents past n_docs hold 0 and never reach doc_group)
            if (want != -1) {
#pragma unroll 4
                for (int i = 0; i < kPer; ++i) {
                    const int doc = tid + i * kPkThreads;
                    if (acc[doc] != 0u && p.doc_group[rbase + doc] != want) acc[doc] = 0u;
                }
                __syncthreads();
            }
#pragma unroll
            for (int i = 0; i < kPer; ++i) tmax = max(tmax, acc[tid + i * kPkThreads]);
            const uint32_t kth = block_kth_largest<kPkThreads>([&](int i) { return acc[i]; }, kBmRange, p.k, s_hist);
            if (tid == 0) s_thr = (int)kth;
            __syncthreads();
        } else if (want == -1) {
#pragma unroll
            for (int i = 0; i < kPer; ++i) tmax = max(tmax, acc[tid + i * kPkThreads]);
        } else {
#pragma unroll 4
            for (int i = 0; i < kPer; ++i) {
                const int doc = tid + i * kPkThreads;
                const uint32_t v = acc[doc];
                if (v > tmax && p.doc_group[rbase + doc] == want) tmax = v;
            }
        }
        if constexpr (!DEEP) {
            uint32_t gmax = tmax;
#pragma unroll
            for (int o = kPkGroup / 2; o > 0; o >>= 1) gmax = max(gmax, __shfl_xor_sync(0xffffffffu, gmax, o));
            if ((lane & (kPkGroup - 1)) == 0) s_wi[tid / kPkGroup] = (int)gmax;
            if (tid == 0) s_thr = 0;
            __syncthreads();
            if (warp == 0) {
                const int mine = s_wi[lane];
                int rank = 0;
#pragma unroll
                for (int j = 0; j < 32; ++j) {
                    const int o = s_wi[j];
                    rank += (o > mine || (o == mine && j < lane)) ? 1 : 0;
                }
                if (rank == p.k - 1) s_thr = mine;       // 0 when fewer than k groups hold a positive score
            }
            __syncthreads();
        }
        const int g = s_thr;
        const int bl = g > 0 ? g - slack : 0;            // B from this range alone
        const uint32_t tl = (uint32_t)max(bl - es, 1);
        __syncthreads();                                 // s_wi is reused as the candidate list
        if (tmax >= tl) {
#pragma unroll 4
            for (int i = 0; i < kPer; ++i) {
                const int doc = tid + i * kPkThreads;
                if (acc[doc] >= tl && (want == -1 || p.doc_group[rbase + doc] == want)) {
                    const int idx = atomicAdd(&s_cnt, 1);
                    if (idx < local_cap) s_wi[idx] = doc;
                }
            }
        }
        if (tid == 0 && bl > 0) atomicMax(c.thr_q + q, bl);
        __syncthreads();
    }
    const int n = s_cnt;
    if (n == 0) return;
    if (n > local_cap) {
        if (tid == 0) c.ovf[q] = 1;
        return;
    }
    // Skipped (non-essential) tokens: the documents above crossed the RELAXED threshold B - e - NE on their essential
    // tokens alone.  Complete their sums here -- one thread per (document, skipped token) binary-searches the token's
    // packed postings of this range -- so that the test below is the exact one (Q >= B - e) and the candidates carry
    // their full integer score: the candidate set and the bound updates are then exactly those of a pass that read
    // every posting, and only the handful of near-candidates pays for the long lists.
    const uint32_t nm = (uint32_t)s_nm;
    if (nm != 0u) {                                      // block-uniform
        for (int idx = tid; idx < n * 32; idx += kPkThreads) {
            const int tk = idx & 31;
            if (!((nm >> tk) & 1u) || tk >= m) continue;
            const int t = p.q_terms[qs + tk];
            if (t < 0 || t >= p.vocab) continue;
            const uint32_t dl = (uint32_t)s_wi[idx >> 5];
            const uint32_t* ro = p.range_off + (int64_t)t * (p.n_ranges + 1) + r;
            const int base = (int)__ldg(p.indptr + t);
            int lo = base + (int)__ldg(ro), hi = base + (int)__ldg(ro + 1);
            const int end = hi;
            while (lo < hi) {                            // lower_bound on the document bits (ascending inside a term)
                const int mid = lo + ((hi - lo) >> 1);
                if ((__ldg(pk + mid) >> kPkWBits) < dl) lo = mid + 1; else hi = mid;
            }
            if (lo < end) {
                const uint32_t x = __ldg(pk + lo);
                if ((x >> kPkWBits) == dl) atomicAdd(&acc[dl], x & kPkWMask);
            }
        }
        __syncthreads();
    }
    for (int i = tid; i < n; i += kPkThreads) {
        const int dl = s_wi[i];
        const uint32_t mine = acc[dl];
        if (nm != 0u && (int)mine < bound - es) continue;  // crossed only the relaxed threshold
        const int slot = atomicAdd(c.cand_cnt + q, 1);
        if (slot < list_cap) {
            c.cand_ids[(int64_t)q * list_cap + slot] = rbase + dl;
            c.cand_q[(int64_t)q * list_cap + slot] = (int)mine;
            c.cand_u[(int64_t)q * list_cap + slot] = (int)mine;       // full sums: lower and upper bound coincide
        } else {
            c.ovf[q] = 1;
        }
        if constexpr (!DEEP) {
            if (track && n >= p.k) {                     // this range alone holds k documents above the bound
                int rank = 0;
                for (int j = 0; j < n; ++j) {
                    const uint32_t o = acc[s_wi[j]];
                    rank += (o > mine || (o == mine && j < i)) ? 1 : 0;
                }
                if (rank == p.k - 1 && (int)mine - slack > bound) atomicMax(c.thr_q + q, (int)mine - slack);
            }
        }
    }
    if constexpr (DEEP) {
        if (track && n >= p.k) {                         // block-uniform: the same raise, by a select
            __syncthreads();                             // relaxed crossers were dropped above, acc is final
            const int kth = (int)block_kth_largest<kPkThreads>([&](int i) { return acc[s_wi[i]]; }, n, p.k, s_hist);
            if (tid == 0 && kth - slack > bound) atomicMax(c.thr_q + q, kth - slack);
        }
    }
}


inline size_t pk_deep_cand_smem(int k) { return (size_t)(kBmRange + 32 + kPkHist + pk_deep_local_cap(k)) * 4; }

// ---- between range chunks: raise every query's bound to the k-th best of ALL candidates so far, drop the rest ----
// (a single range only knows its own k-th best; the bound that keeps later ranges quiet is the running global one)
constexpr int kBdThreads = 128;

// DEEP: the list has pk_deep_list_cap(k) slots, staged in dynamic shared memory, and the k-th largest lower bound
// comes from a radix select instead of pairwise ranks.
template <bool DEEP, typename S>
__device__ __forceinline__ void bm25_bound_body(const Bm25Params& p, const PkParams& c) {
    __shared__ int s_q_fixed[DEEP ? 1 : kPkListCap];
    __shared__ int s_u_fixed[DEEP ? 1 : kPkListCap];
    __shared__ int s_id_fixed[DEEP ? 1 : kPkListCap];
    __shared__ int s_kth, s_n2;
    extern __shared__ __align__(16) unsigned char pk_smem_raw[];
    const int list_cap = DEEP ? pk_deep_list_cap(p.k) : kPkListCap;
    // DEEP: [kPkHist] select scratch | s_q | s_u | s_id, list_cap each
    int* s_hist = reinterpret_cast<int*>(pk_smem_raw);
    int* s_q = DEEP ? s_hist + kPkHist : s_q_fixed;
    int* s_u = DEEP ? s_hist + kPkHist + list_cap : s_u_fixed;
    int* s_id = DEEP ? s_hist + kPkHist + 2 * list_cap : s_id_fixed;
    const int q = blockIdx.x, tid = threadIdx.x;
    const int n = c.cand_cnt[q];
    if (c.ovf[q] != 0 || n < p.k) return;                // block-uniform
    if (n > list_cap) {
        if (tid == 0) c.ovf[q] = 1;
        return;
    }
    for (int i = tid; i < n; i += kBdThreads) {
        s_q[i] = c.cand_q[(int64_t)q * list_cap + i];
        s_u[i] = c.cand_u[(int64_t)q * list_cap + i];
        s_id[i] = c.cand_ids[(int64_t)q * list_cap + i];
    }
    if (tid == 0) s_n2 = 0;
    __syncthreads();
    if constexpr (DEEP) {
        // lower bounds are >= 1 (candidates pass a threshold of at least 1), so the select sees all n of them
        const int kth = (int)block_kth_largest<kBdThreads>([&](int i) { return (uint32_t)s_q[i]; }, n, p.k, s_hist);
        if (tid == 0) s_kth = kth;
    } else {
        for (int i = tid; i < n; i += kBdThreads) {
            const int mine = s_q[i];
            int rank = 0;
            for (int j = 0; j < n; ++j) {
                const int o = s_q[j];
                rank += (o > mine || (o == mine && j < i)) ? 1 : 0;
            }
            if (rank == p.k - 1) s_kth = mine;           // ranks are a permutation: exactly one writer
        }
    }
    __syncthreads();
    const int qs = p.q_ptr[q];
    const int m = p.q_ptr[q + 1] - qs;
    const int es = PkSlack<S>::e(m);
    const int b = max(s_kth - (m + es), c.thr_q[q]);     // the k-th largest LOWER bound is a valid bound
    for (int i = tid; i < n; i += kBdThreads) {
        if (s_u[i] >= b - es) {                          // keep what may still reach it: UPPER bounds decide
            const int pos = atomicAdd(&s_n2, 1);
            c.cand_q[(int64_t)q * list_cap + pos] = s_q[i];
            c.cand_u[(int64_t)q * list_cap + pos] = s_u[i];
            c.cand_ids[(int64_t)q * list_cap + pos] = s_id[i];
        }
    }
    __syncthreads();
    if (tid == 0) {
        c.thr_q[q] = b;
        c.cand_cnt[q] = s_n2;
    }
    // Non-essential tokens for the ranges still to come (first 32 tokens; one warp): ascending by term maximum,
    // the longest prefix whose sum stays within kPkNeNum/kPkNeDen of b - e.
    if (kPkNeNum > 0 && c.term_max != nullptr && tid < 32 && b > es) {
        const int lane = tid;
        uint32_t gm = 0xffffffffu;                       // lanes without a token sort last and are never chosen
        bool have = false;
        if (lane < m) {
            const int t = p.q_terms[qs + lane];
            have = true;
            gm = (t >= 0 && t < p.vocab) ? __ldg(c.term_max + t) : 0u;   // unknown terms contribute nothing
        }
        int rank = 0;
        for (int j = 0; j < 32; ++j) {
            const uint32_t o = __shfl_sync(0xffffffffu, gm, j);
            rank += (o < gm || (o == gm && j < lane)) ? 1 : 0;
        }
        unsigned long long pre = 0ull;                   // sum of the maxima ranked at or before this lane
        for (int j = 0; j < 32; ++j) {
            const uint32_t o = __shfl_sync(0xffffffffu, gm, j);
            const int r = __shfl_sync(0xffffffffu, rank, j);
            const bool hj = __shfl_sync(0xffffffffu, have ? 1 : 0, j) != 0;
            if (hj && r <= rank) pre += o;
        }
        const unsigned long long budget = (unsigned long long)(b - es) * kPkNeNum / kPkNeDen;
        const bool skip = have && pre <= budget;
        const uint32_t mask = __ballot_sync(0xffffffffu, skip);
        unsigned long long ne = skip ? (unsigned long long)gm : 0ull;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) ne += __shfl_xor_sync(0xffffffffu, ne, o);
        if (lane == 0) {
            c.ne_mask[q] = mask;
            c.ne_sum[q] = (int)ne;
        }
    }
}

template <typename S>
__global__ void __launch_bounds__(kBdThreads)
bm25_bound_kernel(const Bm25Params p, const PkParams c) {
    bm25_bound_body<false, S>(p, c);
}

template <typename S>
__global__ void __launch_bounds__(kBdThreads)
bm25_bound_deep_kernel(const Bm25Params p, const PkParams c) {
    bm25_bound_body<true, S>(p, c);
}

inline size_t pk_deep_bound_smem(int k) { return (size_t)(kPkHist + 3 * pk_deep_list_cap(k)) * 4; }

// ---- phase 2: exact scores of the candidates in token order, canonical top-k ----
constexpr int kRsThreads = 128;
constexpr int kRsTok = 64;     // tokens whose (term, base) are staged in shared memory
constexpr int kRsU = 4;        // candidates a warp scores at once (independent binary searches in flight)

// DEEP: out_scores is a [Q][pk_deep_list_cap(k)] row of exact scores beside the candidate ids (ids past the
// query's candidates set to -1), from which the caller's select takes the canonical top-k.
// S: the index's score type; contributions of that type are added with its round-to-nearest add.
template <typename S> __device__ __forceinline__ S add_rn(S a, S b);
template <> __device__ __forceinline__ double add_rn<double>(double a, double b) { return __dadd_rn(a, b); }
template <> __device__ __forceinline__ float add_rn<float>(float a, float b) { return __fadd_rn(a, b); }

template <bool DEEP, typename S>
__device__ __forceinline__ void bm25_rescore_body(const Bm25Params& p, const PkParams& c,
                                                  S* __restrict__ out_scores, int32_t* __restrict__ out_ids,
                                                  int32_t* __restrict__ out_counts) {
    __shared__ S s_sc[DEEP ? 1 : kPkListCap];
    __shared__ int s_id[DEEP ? 1 : kPkListCap];
    __shared__ int s_t[kRsTok];
    __shared__ int s_base[kRsTok];
    __shared__ int s_pos;
    const int list_cap = DEEP ? pk_deep_list_cap(p.k) : kPkListCap;
    const int q = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int n = c.cand_cnt[q];
    if (c.ovf[q] != 0 || n > list_cap) {                 // block-uniform
        if (tid == 0) c.ovf_list[atomicAdd(c.ovf_n, 1)] = q;
        return;
    }
    const int qs = p.q_ptr[q];
    const int m = p.q_ptr[q + 1] - qs;
    if (tid == 0) s_pos = 0;
    for (int j = tid; j < min(m, kRsTok); j += kRsThreads) {
        const int t = p.q_terms[qs + j];
        const bool ok = t >= 0 && t < p.vocab;
        s_t[j] = ok ? t : -1;
        s_base[j] = ok ? (int)p.indptr[t] : 0;
    }
    __syncthreads();
    const S* __restrict__ post_w = reinterpret_cast<const S*>(p.post_w);
    // A warp scores kRsU candidates at once (lane = token): the kRsU binary searches of a lane are independent, so
    // their loads are in flight together -- the kernel is bound by the latency of those dependent L2 reads, not by
    // their count.  The sums stay per candidate, in token order.
    for (int cb = warp * kRsU; cb < n; cb += (kRsThreads / 32) * kRsU) {
        int doc[kRsU];
        S s[kRsU];
#pragma unroll
        for (int u = 0; u < kRsU; ++u) {
            doc[u] = cb + u < n ? c.cand_ids[(int64_t)q * list_cap + cb + u] : -1;
            s[u] = (S)0;
        }
        for (int c0 = 0; c0 < m; c0 += 32) {
            const int j = c0 + lane;
            S wv[kRsU];
#pragma unroll
            for (int u = 0; u < kRsU; ++u) wv[u] = (S)0;
            int t = -1, base = 0;
            if (j < m) {
                if (j < kRsTok) { t = s_t[j]; base = s_base[j]; }
                else {
                    t = p.q_terms[qs + j];
                    if (t < 0 || t >= p.vocab) t = -1;
                    base = t >= 0 ? (int)p.indptr[t] : 0;
                }
            }
            if (t >= 0) {
                int lo[kRsU], hi[kRsU], end[kRsU];
#pragma unroll
                for (int u = 0; u < kRsU; ++u) {
                    lo[u] = hi[u] = end[u] = 0;
                    if (doc[u] >= 0) {
                        const uint32_t* ro = p.range_off + (int64_t)t * (p.n_ranges + 1) + doc[u] / kBmRange;
                        lo[u] = base + (int)ro[0];
                        hi[u] = end[u] = base + (int)ro[1];
                    }
                }
                bool more = true;
                while (more) {                           // lower_bound of doc[u] in the term's postings of its range
                    more = false;
                    int got[kRsU], mid[kRsU];
#pragma unroll
                    for (int u = 0; u < kRsU; ++u) {
                        mid[u] = lo[u] + ((hi[u] - lo[u]) >> 1);     // lo + hi can pass 2^31 on a 2^30+ posting shard
                        got[u] = lo[u] < hi[u] ? __ldg(p.post_doc + mid[u]) : 0;
                    }
#pragma unroll
                    for (int u = 0; u < kRsU; ++u) {
                        if (lo[u] < hi[u]) {
                            if (got[u] < doc[u]) lo[u] = mid[u] + 1; else hi[u] = mid[u];
                            more |= lo[u] < hi[u];
                        }
                    }
                }
#pragma unroll
                for (int u = 0; u < kRsU; ++u)
                    if (lo[u] < end[u] && __ldg(p.post_doc + lo[u]) == doc[u]) wv[u] = __ldg(post_w + lo[u]);
            }
            const int cnt = min(32, m - c0);
            for (int jj = 0; jj < cnt; ++jj) {
#pragma unroll
                for (int u = 0; u < kRsU; ++u) s[u] = add_rn<S>(s[u], __shfl_sync(0xffffffffu, wv[u], jj));   // token order
            }
        }
        if (lane == 0) {
#pragma unroll
            for (int u = 0; u < kRsU; ++u) {
                if (cb + u < n) {
                    if constexpr (DEEP) out_scores[(int64_t)q * list_cap + cb + u] = s[u];
                    else { s_sc[cb + u] = s[u]; s_id[cb + u] = doc[u]; }
                }
            }
        }
    }
    if constexpr (DEEP) {
        for (int i = n + tid; i < list_cap; i += kRsThreads) c.cand_ids[(int64_t)q * list_cap + i] = -1;
        return;
    }
    __syncthreads();
    for (int i = tid; i < n; i += kRsThreads) {
        const S ms = s_sc[i];
        const int mi = s_id[i];
        if (ms > (S)0) {                                 // retrievers.py:195-196: only positive scores qualify
            atomicAdd(&s_pos, 1);
            int rank = 0;
            for (int j = 0; j < n; ++j) rank += better<S>(s_sc[j], s_id[j], ms, mi) ? 1 : 0;
            if (rank < p.k) {
                out_scores[(int64_t)q * p.k + rank] = ms;
                out_ids[(int64_t)q * p.k + rank] = mi + p.id_base;
            }
        }
    }
    __syncthreads();
    const int have = min(s_pos, p.k);
    for (int i = have + tid; i < p.k; i += kRsThreads) {
        out_scores[(int64_t)q * p.k + i] = ScoreTraits<S>::lowest();
        out_ids[(int64_t)q * p.k + i] = -1;
    }
    if (tid == 0) out_counts[q] = have;
}

template <typename S>
__global__ void __launch_bounds__(kRsThreads)
bm25_rescore_kernel(const Bm25Params p, const PkParams c, S* __restrict__ out_scores,
                    int32_t* __restrict__ out_ids, int32_t* __restrict__ out_counts) {
    bm25_rescore_body<false, S>(p, c, out_scores, out_ids, out_counts);
}

template <typename S>
__global__ void __launch_bounds__(kRsThreads)
bm25_rescore_deep_kernel(const Bm25Params p, const PkParams c, S* __restrict__ rows) {
    bm25_rescore_body<true, S>(p, c, rows, nullptr, nullptr);
}

}  // namespace ezr
