// BM25-Extract context compression: many (query, context) groups per launch, one CTA per group.
//
// Replaces the reference compressor's per-context route (compressors.py:32-55: cut the context into sentences,
// build a throw-away BM25 index over them, score the query, keep the best sentences until their characters reach
// rate * len(context)).  A group is one context's sentences plus its query; all token ids come from one vocabulary
// for the whole batch.  Everything happens in shared memory:
//
//   1. count   (term, position) keys sorted (bitonic_sort_u64); a term's run of keys lists its positions in order,
//              so its sentences come in order too: tf = length of a same-sentence sub-run, df = number of sub-runs,
//              first position = the run's head.  fdf[first position] = df marks each distinct term once, in
//              first-seen order.
//   2. idf     exactly as Bm25Stats.from_counts computes it for a corpus of N = the group's sentence count, with no
//              logarithm on the device.  rank_bm25: L[N-n] - L[n] with the host table L[j] = log(j + 0.5) (N-n+0.5 is
//              exact, so this is CPython's math.log(N - n + 0.5) - math.log(n + 0.5) bit for bit); idf_sum is a
//              sequential __dadd_rn over the distinct terms in first-seen order; negative idf -> epsilon *
//              (idf_sum / n_terms).  bm25s: the host's float32 table for this N.
//   3. score   query tokens in order (duplicates repeat), contribution bm25_contribution() as in the index build;
//              float64 sums (rank_bm25) or float32 sums of the float32 weights from +0.0f (bm25s).  A query token
//              of the batch vocabulary that does not occur in this group has df = 0 here and adds nothing
//              (rank_bm25: idf.get(q) or 0).
//   4. select  order = score descending, then sentence index descending (the canonical order, numpy
//              argsort(kind="stable")[::-1]).  The entry of rank r is kept iff r == 0 or the characters of the
//              entries ranked before it do not yet reach ctx_chars * rate: the same set as walking the order and
//              stopping at the first entry whose running sum is >= the threshold.  Rank and running sum of every
//              sentence come from one pass over all sentences (N <= kExtMaxSents).
#include "ezr_common.cuh"
#include "bm25_common.cuh"
#include "../../include/easyrag_b200.h"

namespace ezr {

constexpr int kExtThreads = 512;
constexpr int kExtMaxTokens = 8192;      // tokens of a group (64 KB of sort keys)
constexpr int kExtMaxSents = 1024;       // sentences of a group
constexpr int kExtEmpty = -1;            // out_counts codes: a group without sentences ...
constexpr int kExtBad = -2;              // ... or with bad input (token id out of range, larger than max_tokens/max_sents)

struct ExtParams {
    const int64_t* sent_ptr;     // [G+1] sentence range of each group
    const int64_t* tok_ptr;      // [S+1] token range of each sentence
    const int32_t* tokens;
    const int64_t* sent_chars;   // [S]
    const int64_t* ctx_chars;    // [G]
    const int64_t* q_ptr;        // [G+1]
    const int32_t* q_tokens;     // < 0: not in the vocabulary
    const void* idf_tab;         // rank_bm25: double L[j] = log(j + 0.5); bm25s: float idf per (N, df)
    const int64_t* idf_off;      // bm25s: [G] offset of the group's table (df = 0..N) in idf_tab
    int64_t idf_len;
    int32_t vocab;
    int32_t max_tokens, max_sents, key_cap;
    double k1, b, one_minus_b, num_scale, epsilon, rate;
    void* out_scores;            // [S] or NULL
    uint8_t* out_keep;           // [S]
    int32_t* out_counts;         // [G]
};

size_t ext_smem_bytes(int key_cap, int max_sents, int max_tokens) {
    return (size_t)key_cap * 8 + (size_t)max_sents * 16 + align_up((size_t)(max_sents + 1) * 4, 8) +
           (size_t)max_tokens * 2;
}

// sentence holding position pos: the largest s < n with lp[s] <= pos (empty sentences have lp[s] == lp[s+1])
__device__ __forceinline__ int ext_sentence_of(const int* lp, int n, int pos) {
    int lo = 0, hi = n;
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (lp[mid] <= pos) lo = mid; else hi = mid;
    }
    return lo;
}

__device__ __forceinline__ int ext_lower_bound(const unsigned long long* key, int n, unsigned long long v) {
    int lo = 0, hi = n;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (key[mid] < v) lo = mid + 1; else hi = mid;
    }
    return lo;
}

template <typename S>
__global__ void __launch_bounds__(kExtThreads)
bm25_extract_kernel(const ExtParams p) {
    extern __shared__ __align__(16) unsigned char ext_smem[];
    __shared__ int s_bad, s_terms, s_kept;
    __shared__ double s_avg;
    const int g = blockIdx.x, tid = threadIdx.x, lane = tid & 31;
    const int64_t s0 = p.sent_ptr[g];
    const int64_t n64 = p.sent_ptr[g + 1] - s0;
    if (n64 == 0) {
        if (tid == 0) p.out_counts[g] = kExtEmpty;
        return;
    }
    const int64_t t0 = p.tok_ptr[s0];
    const int64_t len64 = p.tok_ptr[s0 + n64] - t0;
    const bool f64 = sizeof(S) == 8;
    if (n64 < 0 || n64 > p.max_sents || len64 < 0 || len64 > p.max_tokens ||
        (f64 ? n64 >= p.idf_len : p.idf_off[g] < 0 || p.idf_off[g] + n64 >= p.idf_len)) {
        if (tid == 0) p.out_counts[g] = kExtBad;
        return;
    }
    const int N = (int)n64, T = (int)len64;
    unsigned long long* key = reinterpret_cast<unsigned long long*>(ext_smem);     // [key_cap]
    S* acc = reinterpret_cast<S*>(key + p.key_cap);                                 // [max_sents] (8-byte slots)
    double* kd = reinterpret_cast<double*>(key + p.key_cap) + p.max_sents;          // [max_sents], then characters
    long long* chars = reinterpret_cast<long long*>(kd);
    int* lp = reinterpret_cast<int*>(kd + p.max_sents);                             // [N+1] local token offsets
    unsigned short* fdf = reinterpret_cast<unsigned short*>(
        reinterpret_cast<unsigned char*>(lp) + (((p.max_sents + 1) * 4 + 7) & ~7));  // [T] df at first positions

    const int64_t q0 = p.q_ptr[g];
    const int m = (int)(p.q_ptr[g + 1] - q0);
    if (tid == 0) { s_bad = 0; s_terms = 0; s_kept = 0; }
    __syncthreads();
    for (int i = tid; i <= N; i += kExtThreads) {
        const int64_t o = p.tok_ptr[s0 + i] - t0;
        lp[i] = (int)o;
        if (o < 0 || o > T || (i > 0 && p.tok_ptr[s0 + i - 1] > p.tok_ptr[s0 + i])) s_bad = 1;
    }
    int n2 = 1;
    while (n2 < T) n2 <<= 1;
    for (int i = tid; i < n2; i += kExtThreads) {
        unsigned long long k = ~0ull;                                   // padding sorts last
        if (i < T) {
            const int t = p.tokens[t0 + i];
            if (t < 0 || t >= p.vocab) s_bad = 1;
            k = ((unsigned long long)(unsigned)t << 32) | (unsigned)i;
            fdf[i] = 0;
        }
        key[i] = k;
    }
    for (int j = tid; j < m; j += kExtThreads)
        if (p.q_tokens[q0 + j] >= p.vocab) s_bad = 1;
    __syncthreads();
    if (s_bad) {
        if (tid == 0) p.out_counts[g] = kExtBad;
        return;
    }
    bitonic_sort_u64(key, n2, tid, kExtThreads);

    // 1. per distinct term: df, written at its first position
    for (int i = tid; i < T; i += kExtThreads) {
        const unsigned term = (unsigned)(key[i] >> 32);
        if (i > 0 && (unsigned)(key[i - 1] >> 32) == term) continue;
        int df = 0, s = -1;
        for (int j = i; j < T && (unsigned)(key[j] >> 32) == term; ++j) {
            const int pos = (int)(unsigned)key[j];
            if (s < 0 || pos >= lp[s + 1]) { s = ext_sentence_of(lp, N, pos); ++df; }
        }
        fdf[(unsigned)key[i]] = (unsigned short)df;
        atomicAdd(&s_terms, 1);
    }
    __syncthreads();

    // 2. rank_bm25's mean idf (warp 0, first-seen order) while the other warps set up the sentences
    const double* L = reinterpret_cast<const double*>(p.idf_tab);
    if (f64 && tid < 32) {
        double sum = 0.0;
        for (int base = 0; base < T; base += 32) {
            const int i = base + lane;
            const int df = i < T ? fdf[i] : 0;
            const double v = df ? __dsub_rn(L[N - df], L[df]) : 0.0;
            unsigned mk = __ballot_sync(0xffffffffu, df != 0);
            while (mk) {
                const int src = __ffs(mk) - 1;
                mk &= mk - 1;
                sum = __dadd_rn(sum, __shfl_sync(0xffffffffu, v, src));
            }
        }
        if (lane == 0) s_avg = s_terms ? __ddiv_rn(sum, (double)s_terms) : 0.0;
    }
    const double avgdl = __ddiv_rn((double)T, (double)N);
    for (int s = tid; s < N; s += kExtThreads) {
        acc[s] = (S)0;
        kd[s] = bm25_doc_norm((double)(lp[s + 1] - lp[s]), p.k1, p.b, p.one_minus_b, avgdl);
    }
    __syncthreads();

    // 3. scores, query tokens in order; each (term, sentence) pair belongs to one thread
    const float* idf32 = reinterpret_cast<const float*>(p.idf_tab) + (f64 ? 0 : p.idf_off[g]);
    for (int j = 0; j < m; ++j) {
        const int t = p.q_tokens[q0 + j];
        if (t < 0) continue;
        const unsigned long long k0 = (unsigned long long)(unsigned)t << 32;
        const int a = ext_lower_bound(key, T, k0);
        const int e = ext_lower_bound(key, T, k0 + (1ull << 32));
        if (a == e) continue;                                           // df = 0 in this group
        const int df = fdf[(unsigned)key[a]];
        double idf;
        if (f64) {
            idf = __dsub_rn(L[N - df], L[df]);
            if (idf < 0) idf = __dmul_rn(p.epsilon, s_avg);
        } else {
            idf = (double)idf32[df];
        }
        for (int i = a + tid; i < e; i += kExtThreads) {
            const int pos = (int)(unsigned)key[i];
            const int s = ext_sentence_of(lp, N, pos);
            if (i > a && (int)(unsigned)key[i - 1] >= lp[s]) continue;   // not the term's first key in sentence s
            int tf = 1;
            while (i + tf < e && (int)(unsigned)key[i + tf] < lp[s + 1]) ++tf;
            const double w = bm25_contribution(idf, (double)tf, kd[s], p.num_scale);
            if (f64) acc[s] = (S)__dadd_rn((double)acc[s], w);
            else acc[s] = (S)__fadd_rn((float)acc[s], (float)w);
        }
        __syncthreads();
    }
    for (int s = tid; s < N; s += kExtThreads) {
        if (p.out_scores) reinterpret_cast<S*>(p.out_scores)[s0 + s] = acc[s];
        chars[s] = p.sent_chars[s0 + s];                                // kd is no longer needed
    }
    __syncthreads();

    // 4. selection
    const double thr = __dmul_rn((double)p.ctx_chars[g], p.rate);
    int kept = 0;
    for (int s = tid; s < N; s += kExtThreads) {
        const S v = acc[s];
        int rank = 0;
        long long before = 0;
        for (int u = 0; u < N; ++u) {
            const S x = acc[u];
            if (x > v || (x == v && u > s)) { ++rank; before += chars[u]; }
        }
        const bool keep = rank == 0 || !((double)before >= thr);
        p.out_keep[s0 + s] = keep ? 1 : 0;
        kept += keep;
    }
    if (kept) atomicAdd(&s_kept, kept);
    __syncthreads();
    if (tid == 0) p.out_counts[g] = s_kept;
}

}  // namespace ezr

using namespace ezr;

extern "C" {

int ezr_bm25_extract_caps(int32_t* max_tokens_host, int32_t* max_sents_host) {
    EZR_CHECK_ARG(max_tokens_host && max_sents_host, "bm25_extract_caps: NULL argument");
    *max_tokens_host = kExtMaxTokens;
    *max_sents_host = kExtMaxSents;
    return EZR_OK;
}

int ezr_bm25_extract(const int64_t* sent_ptr, const int64_t* tok_ptr, const int32_t* tokens, int32_t vocab,
                     const int64_t* sent_chars, const int64_t* ctx_chars, const int64_t* q_ptr,
                     const int32_t* q_tokens, int32_t n_groups, int32_t max_tokens, int32_t max_sents,
                     const void* idf_tab, int64_t idf_len, const int64_t* idf_off, double k1, double b,
                     double epsilon, double rate, int32_t score_type, void* out_scores, uint8_t* out_keep,
                     int32_t* out_counts, void* stream) {
    EZR_CHECK_ARG(score_type == EZR_F64 || score_type == EZR_F32, "bm25_extract: bad score_type");
    EZR_CHECK_ARG(n_groups >= 0 && vocab >= 1, "bm25_extract: bad n_groups / vocab");
    EZR_CHECK_ARG(max_tokens >= 0 && max_tokens <= kExtMaxTokens, "bm25_extract: max_tokens=%d out of [0,%d]",
                  max_tokens, kExtMaxTokens);
    EZR_CHECK_ARG(max_sents >= 1 && max_sents <= kExtMaxSents, "bm25_extract: max_sents=%d out of [1,%d]",
                  max_sents, kExtMaxSents);
    if (n_groups == 0) return EZR_OK;
    EZR_CHECK_ARG(sent_ptr && tok_ptr && (tokens || max_tokens == 0) && sent_chars && ctx_chars && q_ptr &&
                  out_keep && out_counts && idf_tab, "bm25_extract: NULL argument");
    EZR_CHECK_ARG(score_type == EZR_F64 ? idf_len > max_sents : idf_off != nullptr,
                  "bm25_extract: the idf table does not cover the groups");
    int key_cap = 1;
    while (key_cap < max_tokens) key_cap <<= 1;
    const size_t smem = ext_smem_bytes(key_cap, max_sents, max_tokens);
    static bool attr_done = false;
    if (!attr_done) {
        const int full = (int)ext_smem_bytes(kExtMaxTokens, kExtMaxSents, kExtMaxTokens);
        EZR_CUDA(cudaFuncSetAttribute(bm25_extract_kernel<double>, cudaFuncAttributeMaxDynamicSharedMemorySize, full));
        EZR_CUDA(cudaFuncSetAttribute(bm25_extract_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, full));
        attr_done = true;
    }
    ExtParams p;
    p.sent_ptr = sent_ptr; p.tok_ptr = tok_ptr; p.tokens = tokens; p.sent_chars = sent_chars;
    p.ctx_chars = ctx_chars; p.q_ptr = q_ptr; p.q_tokens = q_tokens; p.idf_tab = idf_tab; p.idf_off = idf_off;
    p.idf_len = idf_len; p.vocab = vocab; p.max_tokens = max_tokens; p.max_sents = max_sents; p.key_cap = key_cap;
    p.k1 = k1; p.b = b; p.one_minus_b = 1.0 - b; p.epsilon = epsilon; p.rate = rate;
    p.num_scale = score_type == EZR_F64 ? k1 + 1.0 : 1.0;
    p.out_scores = out_scores; p.out_keep = out_keep; p.out_counts = out_counts;
    cudaStream_t st = (cudaStream_t)stream;
    if (score_type == EZR_F64)
        bm25_extract_kernel<double><<<(unsigned)n_groups, kExtThreads, smem, st>>>(p);
    else
        bm25_extract_kernel<float><<<(unsigned)n_groups, kExtThreads, smem, st>>>(p);
    EZR_LAUNCH_CHECK();
    return EZR_OK;
}

}  // extern "C"
