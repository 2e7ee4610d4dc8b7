// Reranker hand-off on the device (SURVEY.md 8(f).4): the coarse ranker's fused top-k ids -> the token sequences
// the LLM reranker scores, in the reference's layout and slice order, without a round trip through Python lists.
//
// Reference: LLMRerank._postprocess_nodes walks the coarse list in slices of embed_bs = 32 (rerankers.py:309-322)
// and get_inputs / get_inputs_v2_5 (rerankers.py:196-293) builds, per (query, passage) pair,
//     [bos] + tok("A: " + query)[: 3/4 max_length]  |  sep + tok("B: " + passage)   (the pair truncated to max_length,
//     'only_second': the passage side gives way)     |  sep + prompt
// Here the passages ("B: ..." already tokenised once at index time, CSR on the device), the queries ("A: ...",
// CSR per batch) and the sep / prompt ids are device arrays; pair p = q * k + r is candidate r of query q.
// Output is PACKED (no padding): ids[T] + cu_seqlens[P + 1] (the layout this library's encoder kernels consume;
// a padded [32, L] view is a copy with cu as the index), plus the per-pair query_lengths of get_inputs_v2_5.
// Both packers keep an int32 copy of cu, so their plans refuse T >= 2^31 rather than let the offsets wrap.
#include "ezr_common.cuh"
#include "../../include/easyrag_b200.h"

namespace ezr {

struct RerankParams {
    const int32_t* cand_ids;    // [Q, k_stride] document ids in rank order (-1 padded)
    const int32_t* cand_cnt;    // [Q]
    int n_queries, k, k_stride, id_base, n_docs;
    const int32_t* q_ptr;       // [Q + 1] into q_tok
    const int32_t* q_tok;       // query tokens WITHOUT bos
    const int64_t* p_ptr;       // [n_docs + 1] into p_tok
    const int32_t* p_tok;
    const int32_t* sep;         // [n_sep]
    const int32_t* prompt;      // [n_prompt]
    int n_sep, n_prompt, bos, max_length;
};

// tokens of the three parts of pair p: head = bos + query (<= 3/4 max_length query tokens), body = sep + passage
// truncated so that head + body <= max_length, tail = sep + prompt.  False for a padding slot (*bad_id stays false)
// and for an id outside [id_base, id_base + n_docs) (*bad_id set); p_ptr is read for neither.
__device__ __forceinline__ bool pair_parts(const RerankParams& a, int p, int& doc, int& nq, int& npass,
                                           bool* bad_id = nullptr) {
    const int q = p / a.k, r = p % a.k;
    doc = -1; nq = 0; npass = 0;
    if (r >= a.cand_cnt[q]) return false;
    doc = a.cand_ids[(int64_t)q * a.k_stride + r] - a.id_base;
    if (doc < 0 || doc >= a.n_docs) {
        if (bad_id) *bad_id = true;
        return false;
    }
    nq = min(a.q_ptr[q + 1] - a.q_ptr[q], a.max_length * 3 / 4);
    const int64_t plen = a.p_ptr[doc + 1] - a.p_ptr[doc];
    const int head = 1 + nq;
    const int room = a.max_length - head - a.n_sep;              // 'only_second': the passage gives way
    npass = (int)min((int64_t)max(room, 0), min(plen, (int64_t)a.max_length));
    return true;
}

// per pair: the length and get_inputs_v2_5's query length (0 for padding); ids outside the passage range count
// into *bad
__global__ void rerank_len_kernel(const RerankParams a, int64_t* __restrict__ len, int32_t* __restrict__ query_len,
                                  unsigned long long* __restrict__ bad) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= a.n_queries * a.k) return;
    int doc, nq, npass;
    bool bad_id = false;
    if (!pair_parts(a, p, doc, nq, npass, &bad_id)) {
        len[p] = 0; query_len[p] = 0;
        if (bad_id) atomicAdd(bad, 1ull);
        return;
    }
    len[p] = 1 + nq + a.n_sep + npass + a.n_sep + a.n_prompt;
    query_len[p] = 1 + nq + a.n_sep;                             // get_inputs_v2_5: len([bos] + query + sep)
}

// one warp per pair
__global__ void rerank_fill_kernel(const RerankParams a, const int64_t* __restrict__ cu, int32_t* __restrict__ ids,
                                   int32_t* __restrict__ cu32) {
    const int p = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    const int n_pairs = a.n_queries * a.k;
    if (p > n_pairs) return;
    if (lane == 0) cu32[p] = (int32_t)cu[p];
    if (p == n_pairs) return;
    int doc, nq, npass;
    if (!pair_parts(a, p, doc, nq, npass)) return;
    const int q = p / a.k;
    int32_t* o = ids + cu[p];
    if (lane == 0) o[0] = a.bos;
    const int32_t* qs = a.q_tok + a.q_ptr[q];
    for (int i = lane; i < nq; i += 32) o[1 + i] = qs[i];
    o += 1 + nq;
    for (int i = lane; i < a.n_sep; i += 32) o[i] = a.sep[i];
    o += a.n_sep;
    const int32_t* ps = a.p_tok + a.p_ptr[doc];
    for (int i = lane; i < npass; i += 32) o[i] = ps[i];
    o += npass;
    for (int i = lane; i < a.n_sep; i += 32) o[i] = a.sep[i];
    o += a.n_sep;
    for (int i = lane; i < a.n_prompt; i += 32) o[i] = a.prompt[i];
}

// exclusive scan of int64 lengths (one CTA; P is at most a few hundred thousand pairs)
__global__ void __launch_bounds__(1024)
rerank_scan_kernel(const int64_t* __restrict__ len, int n, int64_t* __restrict__ cu) {
    __shared__ long long s_warp[32];
    __shared__ long long s_carry;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) { s_carry = 0; cu[0] = 0; }
    __syncthreads();
    for (int base = 0; base < n; base += 1024) {
        const int i = base + tid;
        long long v = i < n ? (long long)len[i] : 0;
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
        if (i < n) cu[i + 1] = incl;
        __syncthreads();
        if (tid == 1023) s_carry = incl;
        __syncthreads();
    }
}

static int fill_params(RerankParams& a, const int32_t* cand_ids, const int32_t* cand_cnt, int n_queries, int k, int k_stride,
                       int id_base, int n_docs, const int32_t* q_ptr, const int32_t* q_tok, const int64_t* p_ptr,
                       const int32_t* p_tok,
                       const int32_t* sep, int n_sep, const int32_t* prompt, int n_prompt, int bos, int max_length) {
    EZR_CHECK_ARG(cand_ids && cand_cnt && q_ptr && p_ptr && (q_tok || true) && p_tok, "rerank_pack: NULL argument");
    EZR_CHECK_ARG(n_queries >= 0 && k >= 1 && k_stride >= k && n_docs >= 0,
                  "rerank_pack: bad n_queries / k / stride / n_docs");
    EZR_CHECK_ARG(n_sep >= 0 && n_prompt >= 0 && (n_sep == 0 || sep) && (n_prompt == 0 || prompt) && max_length >= 8,
                  "rerank_pack: bad sep / prompt / max_length");
    EZR_CHECK_ARG((int64_t)n_queries * k < ((int64_t)1 << 30), "rerank_pack: too many pairs");
    EZR_CHECK_ARG(1 + max_length * 3 / 4 + n_sep <= max_length,
                  "rerank_pack: max_length=%d leaves no room for bos + query + sep (%d sep ids)", max_length, n_sep);
    a.cand_ids = cand_ids; a.cand_cnt = cand_cnt; a.n_queries = n_queries; a.k = k; a.k_stride = k_stride;
    a.id_base = id_base; a.n_docs = n_docs; a.q_ptr = q_ptr; a.q_tok = q_tok; a.p_ptr = p_ptr; a.p_tok = p_tok;
    a.sep = sep; a.prompt = prompt;
    a.n_sep = n_sep; a.n_prompt = n_prompt; a.bos = bos; a.max_length = max_length;
    return EZR_OK;
}

// ------------------------------------------------------------------------------------------------------------------
// Cross-encoder pairs (SentenceTransformerRerank -> CrossEncoder.predict, rerankers.py:15-99): the fast tokenizer's
// pair encoding with truncation="longest_first" at max_length, built from query and passage ids tokenised once
// without special tokens.  Layout [cls] q' [sep] x n_mid p' [sep]; token type 0 up to the first [sep], type_b after;
// positions pos_offset + i.  Only the real pairs are written (candidate r of query q with r < counts[q]), compacted in
// query order: pair pair_off[q] + r.
struct CrossParams {
    const int32_t* cand_ids;    // [Q, k_stride] document ids in rank order
    const int32_t* cand_cnt;    // [Q]
    int n_queries, k, k_stride, id_base, n_docs;
    const int32_t* q_ptr;       // [Q + 1] into q_tok
    const int32_t* q_tok;
    const int64_t* p_ptr;       // [n_docs + 1] into p_tok
    const int32_t* p_tok;
    int cls, sep, n_mid, type_b, pos_offset, max_length;
};

__device__ __forceinline__ int cross_count(const CrossParams& a, int q) { return min(max(a.cand_cnt[q], 0), a.k); }

// the truncated lengths (a', b') of the tokenizer's longest_first rule with room T = max_length - specials
__device__ __forceinline__ void cross_lengths(const CrossParams& a, int q, int doc, int& na, int& nb) {
    const int64_t qa = a.q_ptr[q + 1] - a.q_ptr[q];
    const int64_t pb = a.p_ptr[doc + 1] - a.p_ptr[doc];
    const int64_t room = a.max_length - 2 - a.n_mid;
    if (qa + pb <= room) { na = (int)qa; nb = (int)pb; }
    else if (qa > pb) { nb = (int)min(pb, room / 2); na = (int)(room - nb); }
    else { na = (int)min(qa, room / 2); nb = (int)(room - na); }
}

// per slot s = q * k + r: the pair length (0 for padding slots) and, once per query, the query's pair count.
// A document id outside [id_base, id_base + n_docs) counts into *bad and gives an empty pair.
__global__ void cross_len_kernel(const CrossParams a, int64_t* __restrict__ len, int64_t* __restrict__ n_pairs,
                                 int32_t* __restrict__ bad) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= a.n_queries * a.k) return;
    const int q = s / a.k, r = s % a.k;
    const int n = cross_count(a, q);
    if (r == 0) n_pairs[q] = n;
    len[s] = 0;
    if (r >= n) return;
    const int doc = a.cand_ids[(int64_t)q * a.k_stride + r] - a.id_base;
    if (doc < 0 || doc >= a.n_docs) { atomicAdd(bad, 1); return; }
    int na, nb;
    cross_lengths(a, q, doc, na, nb);
    len[s] = 2 + a.n_mid + na + nb;
}

// pair_off (int32 [Q + 1]) and the compacted int32 cu [P + 1] from the two scans; slot_cu[Q * k] = T
__global__ void cross_compact_kernel(const CrossParams a, const int64_t* __restrict__ slot_cu,
                                     const int64_t* __restrict__ pair_off64, int32_t* __restrict__ pair_off,
                                     int32_t* __restrict__ cu32, int64_t* __restrict__ totals) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    const int n_slots = a.n_queries * a.k;
    if (s > n_slots) return;
    if (s == n_slots) {
        cu32[pair_off64[a.n_queries]] = (int32_t)slot_cu[n_slots];
        totals[0] = slot_cu[n_slots];
        totals[1] = pair_off64[a.n_queries];
        return;
    }
    const int q = s / a.k, r = s % a.k;
    if (r == 0) pair_off[q] = (int32_t)pair_off64[q];
    if (q == 0 && r == 0) pair_off[a.n_queries] = (int32_t)pair_off64[a.n_queries];
    if (r < cross_count(a, q)) cu32[pair_off64[q] + r] = (int32_t)slot_cu[s];
}

// one warp per slot
__global__ void cross_fill_kernel(const CrossParams a, const int64_t* __restrict__ slot_cu, int32_t* __restrict__ ids,
                                  int32_t* __restrict__ types, int32_t* __restrict__ pos) {
    const int s = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (s >= a.n_queries * a.k) return;
    const int64_t o = slot_cu[s], n = slot_cu[s + 1] - o;
    if (n == 0) return;
    const int q = s / a.k, r = s % a.k;
    const int doc = a.cand_ids[(int64_t)q * a.k_stride + r] - a.id_base;
    int na, nb;
    cross_lengths(a, q, doc, na, nb);
    const int32_t* qs = a.q_tok + a.q_ptr[q];
    const int32_t* ps = a.p_tok + a.p_ptr[doc];
    const int b0 = 1 + na + a.n_mid;                           // first passage token
    for (int i = lane; i < n; i += 32) {
        int t;
        if (i == 0) t = a.cls;
        else if (i <= na) t = qs[i - 1];
        else if (i < b0) t = a.sep;
        else if (i < b0 + nb) t = ps[i - b0];
        else t = a.sep;
        ids[o + i] = t;
        types[o + i] = i <= na + 1 ? 0 : a.type_b;
        pos[o + i] = a.pos_offset + i;
    }
}

// both packers hand the encoder int32 cu_seqlens: a batch holds fewer than 2^31 tokens
constexpr int64_t kMaxPackTokens = (int64_t)1 << 31;

static int cross_params(CrossParams& a, const int32_t* cand_ids, const int32_t* cand_cnt, int n_queries, int k,
                        int k_stride, int id_base, int n_docs, const int32_t* q_ptr, const int32_t* q_tok,
                        const int64_t* p_ptr, const int32_t* p_tok, int cls, int sep, int n_mid, int type_b,
                        int pos_offset, int max_length) {
    EZR_CHECK_ARG(cand_ids && cand_cnt && q_ptr && p_ptr, "cross_pack: NULL argument");
    EZR_CHECK_ARG(n_queries >= 0 && k >= 1 && k_stride >= k && n_docs >= 0, "cross_pack: bad n_queries / k / stride");
    EZR_CHECK_ARG((int64_t)n_queries * k < ((int64_t)1 << 30), "cross_pack: too many pairs");
    EZR_CHECK_ARG(n_mid == 1 || n_mid == 2, "cross_pack: n_mid must be 1 (BERT) or 2 (RoBERTa)");
    EZR_CHECK_ARG(type_b == 0 || type_b == 1, "cross_pack: type_b must be 0 or 1");
    EZR_CHECK_ARG(max_length >= 2 + n_mid && pos_offset >= 0, "cross_pack: max_length=%d leaves no room for the %d "
                  "special tokens", max_length, 2 + n_mid);
    a.cand_ids = cand_ids; a.cand_cnt = cand_cnt; a.n_queries = n_queries; a.k = k; a.k_stride = k_stride;
    a.id_base = id_base; a.n_docs = n_docs; a.q_ptr = q_ptr; a.q_tok = q_tok; a.p_ptr = p_ptr; a.p_tok = p_tok;
    a.cls = cls; a.sep = sep; a.n_mid = n_mid; a.type_b = type_b; a.pos_offset = pos_offset; a.max_length = max_length;
    return EZR_OK;
}

}  // namespace ezr

using namespace ezr;

extern "C" {

size_t ezr_cross_pack_workspace(int32_t n_queries, int32_t k) {
    const size_t n_slots = (size_t)n_queries * k;
    return align_up((2 * n_slots + 1) * 8, 256) + align_up(((size_t)2 * n_queries + 1) * 8, 256) + 256;
}

int ezr_cross_pack_plan(const int32_t* cand_ids, const int32_t* cand_cnt, int32_t n_queries, int32_t k,
                        int32_t k_stride, int32_t id_base, int32_t n_docs, const int32_t* q_ptr, const int64_t* p_ptr,
                        int32_t n_mid, int32_t max_length, int32_t* out_pair_off, int32_t* out_cu,
                        int64_t* totals_host, void* workspace, size_t ws_bytes, void* stream) {
    CrossParams a;
    int rc = cross_params(a, cand_ids, cand_cnt, n_queries, k, k_stride, id_base, n_docs, q_ptr, nullptr, p_ptr,
                          nullptr, 0, 0, n_mid, 0, 0, max_length);
    if (rc) return rc;
    EZR_CHECK_ARG(out_pair_off && out_cu && totals_host, "cross_pack_plan: NULL output");
    EZR_CHECK_ARG(workspace && ws_bytes >= ezr_cross_pack_workspace(n_queries, k), "cross_pack_plan: workspace too small");
    cudaStream_t st = (cudaStream_t)stream;
    const int n_slots = n_queries * k;
    if (n_queries == 0) {
        totals_host[0] = totals_host[1] = 0;
        EZR_CUDA(cudaMemsetAsync(out_pair_off, 0, 4, st));
        EZR_CUDA(cudaMemsetAsync(out_cu, 0, 4, st));
        return EZR_OK;
    }
    // workspace: len[n_slots] slot_cu[n_slots + 1] | n_pairs[Q] pair_off64[Q + 1] | totals[2] bad
    char* w = static_cast<char*>(workspace);
    int64_t* len = reinterpret_cast<int64_t*>(w);
    int64_t* slot_cu = len + n_slots;
    w += align_up((2 * (size_t)n_slots + 1) * 8, 256);
    int64_t* n_pairs = reinterpret_cast<int64_t*>(w);
    int64_t* pair_off64 = n_pairs + n_queries;
    w += align_up(((size_t)2 * n_queries + 1) * 8, 256);
    int64_t* totals = reinterpret_cast<int64_t*>(w);
    int32_t* bad = reinterpret_cast<int32_t*>(totals + 2);
    EZR_CUDA(cudaMemsetAsync(bad, 0, 4, st));
    cross_len_kernel<<<ceil_div(n_slots, 256), 256, 0, st>>>(a, len, n_pairs, bad);
    EZR_LAUNCH_CHECK();
    rerank_scan_kernel<<<1, 1024, 0, st>>>(len, n_slots, slot_cu);
    EZR_LAUNCH_CHECK();
    rerank_scan_kernel<<<1, 1024, 0, st>>>(n_pairs, n_queries, pair_off64);
    EZR_LAUNCH_CHECK();
    cross_compact_kernel<<<ceil_div(n_slots + 1, 256), 256, 0, st>>>(a, slot_cu, pair_off64, out_pair_off, out_cu,
                                                                       totals);
    EZR_LAUNCH_CHECK();
    int64_t h[3] = {0, 0, 0};
    EZR_CUDA(cudaMemcpyAsync(h, totals, 16 + 4, cudaMemcpyDeviceToHost, st));
    EZR_CUDA(cudaStreamSynchronize(st));
    const int32_t n_bad = *reinterpret_cast<const int32_t*>(h + 2);
    EZR_CHECK_ARG(n_bad == 0, "cross_pack_plan: %d candidate ids outside [id_base, id_base + n_docs) = [%d, %lld)", n_bad,
                  id_base, (long long)id_base + n_docs);
    EZR_CHECK_ARG(h[0] < kMaxPackTokens, "cross_pack_plan: T=%lld tokens in %lld pairs; the int32 cu_seqlens hold fewer "
                  "than 2^31 (split the queries)", (long long)h[0], (long long)h[1]);
    totals_host[0] = h[0];
    totals_host[1] = h[1];
    return EZR_OK;
}

int ezr_cross_pack_fill(const int32_t* cand_ids, const int32_t* cand_cnt, int32_t n_queries, int32_t k,
                        int32_t k_stride, int32_t id_base, int32_t n_docs, const int32_t* q_ptr, const int32_t* q_tok,
                        const int64_t* p_ptr, const int32_t* p_tok, int32_t cls, int32_t sep, int32_t n_mid,
                        int32_t type_b, int32_t pos_offset, int32_t max_length, const void* workspace,
                        int32_t* out_ids, int32_t* out_types, int32_t* out_pos, void* stream) {
    CrossParams a;
    int rc = cross_params(a, cand_ids, cand_cnt, n_queries, k, k_stride, id_base, n_docs, q_ptr, q_tok, p_ptr, p_tok,
                          cls, sep, n_mid, type_b, pos_offset, max_length);
    if (rc) return rc;
    EZR_CHECK_ARG(q_tok && p_tok && workspace && out_ids && out_types && out_pos, "cross_pack_fill: NULL argument");
    const int n_slots = n_queries * k;
    if (n_slots == 0) return EZR_OK;
    const int64_t* slot_cu = static_cast<const int64_t*>(workspace) + n_slots;
    cross_fill_kernel<<<ceil_div(n_slots, 8), 256, 0, (cudaStream_t)stream>>>(a, slot_cu, out_ids, out_types, out_pos);
    EZR_LAUNCH_CHECK();
    return EZR_OK;
}

int ezr_rerank_pack_plan(const int32_t* cand_ids, const int32_t* cand_cnt, int32_t n_queries, int32_t k, int32_t k_stride,
                         int32_t id_base, int32_t n_docs, const int32_t* q_ptr, const int64_t* p_ptr, int32_t n_sep,
                         int32_t n_prompt, int32_t max_length, int64_t* out_len, int64_t* out_cu,
                         int32_t* out_query_len, int64_t* total_host, void* stream) {
    RerankParams a;
    int rc = fill_params(a, cand_ids, cand_cnt, n_queries, k, k_stride, id_base, n_docs, q_ptr, nullptr, p_ptr,
                         reinterpret_cast<const int32_t*>(1), n_sep ? reinterpret_cast<const int32_t*>(1) : nullptr, n_sep,
                         n_prompt ? reinterpret_cast<const int32_t*>(1) : nullptr, n_prompt, 0, max_length);
    if (rc) return rc;
    EZR_CHECK_ARG(out_len && out_cu && out_query_len && total_host, "rerank_pack_plan: NULL output");
    cudaStream_t st = (cudaStream_t)stream;
    const int n_pairs = n_queries * k;
    if (n_pairs == 0) { *total_host = 0; return EZR_OK; }
    // out_cu[0] counts the bad ids until the scan writes its 0; the count is copied out before that, in stream order
    unsigned long long* bad = reinterpret_cast<unsigned long long*>(out_cu);
    EZR_CUDA(cudaMemsetAsync(bad, 0, 8, st));
    rerank_len_kernel<<<ceil_div(n_pairs, 256), 256, 0, st>>>(a, out_len, out_query_len, bad);
    EZR_LAUNCH_CHECK();
    int64_t h[2] = {0, 0};
    EZR_CUDA(cudaMemcpyAsync(h, bad, 8, cudaMemcpyDeviceToHost, st));
    rerank_scan_kernel<<<1, 1024, 0, st>>>(out_len, n_pairs, out_cu);
    EZR_LAUNCH_CHECK();
    EZR_CUDA(cudaMemcpyAsync(h + 1, out_cu + n_pairs, 8, cudaMemcpyDeviceToHost, st));
    EZR_CUDA(cudaStreamSynchronize(st));
    EZR_CHECK_ARG(h[0] == 0, "rerank_pack_plan: %lld candidate ids outside [id_base, id_base + n_docs) = [%d, %lld)",
                  (long long)h[0], id_base, (long long)id_base + n_docs);
    EZR_CHECK_ARG(h[1] < kMaxPackTokens, "rerank_pack_plan: T=%lld tokens in %d pairs; the int32 cu_seqlens hold fewer "
                  "than 2^31 (split the queries)", (long long)h[1], n_pairs);
    *total_host = h[1];
    return EZR_OK;
}

int ezr_rerank_pack_fill(const int32_t* cand_ids, const int32_t* cand_cnt, int32_t n_queries, int32_t k, int32_t k_stride,
                         int32_t id_base, int32_t n_docs, const int32_t* q_ptr, const int32_t* q_tok, const int64_t* p_ptr,
                         const int32_t* p_tok, const int32_t* sep, int32_t n_sep, const int32_t* prompt, int32_t n_prompt,
                         int32_t bos, int32_t max_length, const int64_t* cu, int32_t* out_ids, int32_t* out_cu32,
                         void* stream) {
    RerankParams a;
    int rc = fill_params(a, cand_ids, cand_cnt, n_queries, k, k_stride, id_base, n_docs, q_ptr, q_tok, p_ptr, p_tok, sep,
                         n_sep, prompt, n_prompt, bos, max_length);
    if (rc) return rc;
    EZR_CHECK_ARG(cu && out_ids && out_cu32 && q_tok, "rerank_pack_fill: NULL argument");
    cudaStream_t st = (cudaStream_t)stream;
    const int n_pairs = n_queries * k;
    rerank_fill_kernel<<<ceil_div(n_pairs + 1, 8), 256, 0, st>>>(a, cu, out_ids, out_cu32);
    EZR_LAUNCH_CHECK();
    return EZR_OK;
}

}  // extern "C"
