/*
 * easyrag_b200 -- C ABI of the H100-native coarse-ranking path.
 *
 * The reference (BUAADreamer/EasyRAG) has no native code and therefore no FFI
 * for this path: its boundary is the Python class surface of
 * src/easyrag/custom/retrievers.py.  Each entry point below replaces the
 * arithmetic behind one of those methods; the Python classes in
 * easyrag_b200/retrievers.py keep the reference's signatures and call these
 * through ctypes (see INTEGRATION.md for the binding a maintainer would add).
 *
 * Conventions
 *   - every function returns 0 on success, a negative ezr_status otherwise;
 *     ezr_last_error() returns a thread-local message for the last failure.
 *   - all pointers are DEVICE pointers unless the name ends in _host.
 *   - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream).
 *   - launch functions never allocate: outputs and the workspace are caller-owned
 *     (query the size with the *_workspace call).  The one exception is the
 *     attention entry points (ezr_attn_bidir / ezr_attn_causal), which draw their
 *     small per-call plan from the stream-ordered memory pool of the launch stream
 *     (cudaMallocAsync / cudaFreeAsync: no device-wide wait, graph-capturable).
 *     They do not synchronise, except where a function says so
 *     (ezr_dense_s8_topk, the rerank packers below).
 *   - document ids are int32, local to the shard the index was built over;
 *     `id_base` is added on output so a row-sharded corpus yields global ids.
 *   - canonical rank order everywhere: score descending, then id descending
 *     (== numpy argsort(kind="stable")[::-1], SURVEY.md 8(c)).
 *   - the library targets sm_90a only; ezr_device_check() fails elsewhere.
 */
#ifndef EASYRAG_B200_H
#define EASYRAG_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum ezr_status {
    EZR_OK = 0,
    EZR_ERR_INVALID = -1,
    EZR_ERR_CUDA = -2,
    EZR_ERR_WORKSPACE = -3,
    EZR_ERR_UNSUPPORTED = -4,
    EZR_ERR_ARCH = -5
} ezr_status;

typedef enum ezr_score_type {
    EZR_F64 = 0, /* rank_bm25.BM25Okapi, bm25_type 0 (retrievers.py:113-118) */
    EZR_F32 = 1  /* bm25s, bm25_type 1 (retrievers.py:107-111); dense cosine */
} ezr_score_type;

int ezr_version(void);
const char* ezr_last_error(void);
/* fails with EZR_ERR_ARCH unless the current device is compute capability 10.x */
int ezr_device_check(void);

/* ------------------------------------------------------------------ BM25 --
 * Term-major (CSC) posting lists with per-posting precomputed contribution
 *   w = idf[t] * tf*(k1+1) / (tf + k1*((1-b) + b*dl/avgdl))
 * evaluated with IEEE round-to-nearest, no FMA contraction, in exactly the
 * operation order numpy applies to rank_bm25's expression (oracle/bm25.py).
 * Documents are cut into ranges of `range_size` ids; range_off[t*(n_ranges+1)+r]
 * is the offset (relative to indptr[t]) of the first posting of term t whose
 * document id is >= r*range_size.
 */
typedef struct ezr_bm25_index {
    int64_t n_docs;
    int64_t n_postings;
    int32_t vocab;
    int32_t score_type;        /* ezr_score_type of post_w */
    int32_t range_size;        /* ezr_bm25_range_size(): 8192 in this build */
    int32_t n_ranges;          /* ceil(n_docs / range_size) */
    const int64_t* indptr;     /* [vocab+1] */
    const int32_t* post_doc;   /* [n_postings] ascending inside a term */
    const void* post_w;        /* [n_postings] double or float */
    const uint32_t* range_off; /* [vocab*(n_ranges+1)] */
    const int32_t* doc_group;  /* [n_docs] metadata class of each document, or NULL */
    int32_t monotone;          /* 1 if every post_w >= 0 (no negative idf): enables crossing-based selection */
    int32_t pk_scale_log2;     /* e of ezr_bm25_pack / ezr_bm25_pack_f32 (informational) */
    const uint32_t* post_pk;   /* [n_postings] packed postings from ezr_bm25_pack (F64 post_w) or ezr_bm25_pack_f32
                                  (F32 post_w), or NULL: enables the two-phase top-k (integer candidate pass + exact
                                  rescoring in the index's score type) for a monotone index */
    const uint32_t* term_max;  /* [vocab] from ezr_bm25_term_max, or NULL: lets the candidate pass skip the posting
                                  lists of a query's lowest-weight terms (MaxScore); results are unchanged */
} ezr_bm25_index;

/* documents per range the library was built for (the `range_size` an index must use) */
int ezr_bm25_range_size(void);

/* K_d[i] = k1 * (one_minus_b + (b*doc_len[i]) / avgdl)   -- rank_bm25 get_scores denominator term */
int ezr_bm25_doc_norm(const int32_t* doc_len, int64_t n_docs, double k1, double b, double one_minus_b,
                      double avgdl, double* out_kd, void* stream);

/* out_w[p] = (S)( idf[term(p)] * ((tf*num_scale) / (tf + K_d[doc])) ); num_scale = k1+1 (Okapi) or 1 (bm25s) */
int ezr_bm25_weights(const int64_t* indptr, const int32_t* post_doc, const int32_t* post_tf, int32_t vocab,
                     int64_t n_postings, const double* idf, const double* kd, double num_scale,
                     int32_t score_type, void* out_w, void* stream);

int ezr_bm25_range_index(const int64_t* indptr, const int32_t* post_doc, int32_t vocab, int32_t range_size,
                         int32_t n_ranges, uint32_t* out_range_off, void* stream);

/* ---- index construction (replaces the dict building of BM25Retriever.__init__, retrievers.py:98-118) ----
 * Corpus = int32 term ids tokens[n_tokens] + int64 doc_ptr[n_docs+1] (device).  Two phases because the number of
 * postings is only known after counting:
 *   count: df[vocab], indptr[vocab+1] (int64), first_pos[vocab] (uint64 corpus position of each term's first
 *          occurrence, ~0 = absent: rank_bm25 sums idf in first-seen term order) + the workspace for phase two.
 *          Documents longer than 8192 tokens sort in the global scratch long_keys (long_docs[n_long] document indices,
 *          long_off[n_long] key offsets, sum(next_pow2(len)) uint64 keys); NULL / 0 when there are none.
 *          *status_host = 0, or 1 + the index of a document holding a token id outside [0, vocab).  Synchronises.
 *   fill : post_doc / post_tf [indptr[vocab]], term-major, ascending document id inside a term (no sort: documents
 *          are placed block by block in order).
 * ezr_bm25_shard_*: postings of documents [doc_lo, doc_hi) of a built index (ids rebased to doc_lo). */
int ezr_bm25_build_block(void);
size_t ezr_bm25_build_workspace(int64_t n_docs, int64_t n_tokens, int32_t vocab);
int ezr_bm25_build_count(const int32_t* tokens, const int64_t* doc_ptr, int64_t n_docs, int64_t n_tokens, int32_t vocab,
                         int32_t max_doc_len, int64_t* out_df, int64_t* out_indptr, uint64_t* out_first_pos,
                         const int32_t* long_docs, const int64_t* long_off, uint64_t* long_keys, int32_t n_long,
                         void* workspace, size_t workspace_bytes, int32_t* status_host, void* stream);
int ezr_bm25_build_fill(const int64_t* doc_ptr, int64_t n_docs, int64_t n_tokens, int32_t vocab, const int64_t* indptr,
                        int32_t* out_post_doc, int32_t* out_post_tf, void* workspace, size_t workspace_bytes,
                        void* stream);
int ezr_bm25_shard_count(const int64_t* indptr, const int32_t* post_doc, int32_t vocab, int32_t doc_lo, int32_t doc_hi,
                         int64_t* out_first, int64_t* out_df_local, int64_t* out_indptr_local, void* stream);
int ezr_bm25_shard_copy(const int64_t* first, const int64_t* indptr_local, const int32_t* post_doc,
                        const int32_t* post_tf, int32_t vocab, int32_t doc_lo, int32_t* out_post_doc,
                        int32_t* out_post_tf, void* stream);

/* Packed postings for the candidate pass of ezr_bm25_topk: out_pk[p] = (post_doc[p] mod range_size) << W |
 * ceil(post_w[p] * 2^e), W = 32 - log2(range_size), e chosen from the largest weight so that every field fits
 * (returned in *out_scale_log2).  Rounding up makes the integer sums upper bounds of the float64 scores; the
 * exact scores of the surviving candidates are recomputed from post_w in token order, so results stay
 * bit-identical to rank_bm25 (retrievers.py:128-151).  Needs non-negative finite weights (else EZR_ERR_INVALID).
 * scratch16: 16 bytes of device memory.  Synchronises the stream (index-build time). */
int ezr_bm25_pack(const int32_t* post_doc, const double* post_w, int64_t n_postings, int32_t range_size,
                  uint32_t* out_pk, int32_t* out_scale_log2, void* scratch16, void* stream);

/* The same packed postings from float32 (bm25s) weights, widened to double exactly; the same scale rule and checks.
 * With them ezr_bm25_topk rescores candidates as float32 sums in token order, bit-identical to bm25s get_scores. */
int ezr_bm25_pack_f32(const int32_t* post_doc, const float* post_w, int64_t n_postings, int32_t range_size,
                      uint32_t* out_pk, int32_t* out_scale_log2, void* scratch16, void* stream);

/* out_term_max[t] = largest packed weight among term t's postings (0 for an empty list). */
int ezr_bm25_term_max(const int64_t* indptr, const uint32_t* post_pk, int32_t vocab, uint32_t* out_term_max,
                      void* stream);

/* 1: the candidate pass of ezr_bm25_topk may skip non-essential terms when the index carries term_max;
 * 0 (default): it reads every posting.  Results are identical either way; the extra candidates it produces
 * cost rescoring time that can exceed what the skipped postings save, hence the default. */
int ezr_bm25_set_skipping(int32_t on);

/* 1 (default): every candidate launch is preceded by a plan kernel that resolves token -> posting segment for all its
 * (query, range) pairs in parallel; 0: the candidate CTAs walk that chain of dependent loads themselves (A/B switch;
 * results are identical). */
int ezr_bm25_set_plan(int32_t on);

/* Document ranges of the FIRST candidate launch (default 4; then the same number again, then doubling up to 32).  A
 * tuning switch: fewer, larger launches on short shards; results are identical for every value. */
int ezr_bm25_set_span(int32_t first_ranges);

/* candidates per query the two-phase path can hold before it hands a query to the ordered kernel (0: not built) */
int ezr_bm25_cand_capacity(void);

/* BM25Retriever.get_scores + .filter for a batch of queries (retrievers.py:128-151,191-210):
 * query i has terms q_terms[q_ptr[i] .. q_ptr[i+1]) in token order (duplicates repeat, <0 or >=vocab = unknown).
 * Only documents with score > 0 qualify (retrievers.py:195-196); q_group[i] >= 0 additionally requires
 * doc_group[d] == q_group[i] (filter_dict, retrievers.py:198-202); -1 = no filter.
 * Outputs: out_scores[Q*k] (double/float per index->score_type), out_ids[Q*k] (-1 padded), out_counts[Q].
 * k <= 32 runs fused (accumulators never leave shared memory); with packed postings on a monotone index (float64,
 * or float32 packed by ezr_bm25_pack_f32) it runs the two-phase path.  32 < k <= 1024 on such an index
 * runs the deep form of the two-phase path: its candidate lists hold 4k + 1024 entries
 * per query, and a query that overflows them (or one list of 2k + 512 for a range of 8192 documents) is answered
 * from its score row.  That path reads the number of such queries back to the host once per call (a 4-byte copy
 * and a stream synchronisation), so it cannot be captured into a CUDA graph.  Every other k > 32 case takes the
 * top-k from score rows computed in blocks of queries whose rows stay within 1 GiB.
 * ezr_bm25_topk_workspace therefore grows with Q * k for every index type (plus that one block of score rows). */
size_t ezr_bm25_topk_workspace(const ezr_bm25_index* index, int32_t n_queries, int32_t k);
int ezr_bm25_topk(const ezr_bm25_index* index, const int32_t* q_ptr, const int32_t* q_terms, int32_t n_queries,
                  int32_t k, const int32_t* q_group, int32_t id_base, void* out_scores, int32_t* out_ids,
                  int32_t* out_counts, void* workspace, size_t workspace_bytes, void* stream);

/* BM25Retriever.get_scores (retrievers.py:128-151): full score rows, out_scores[Q * n_docs] */
int ezr_bm25_scores(const ezr_bm25_index* index, const int32_t* q_ptr, const int32_t* q_terms,
                    int32_t n_queries, void* out_scores, void* stream);

/* ---- BM25-Extract context compression (the reference's ContextCompressor, compressors.py:32-55) ----
 * G groups in one launch.  Group g is a context's sentences [sent_ptr[g], sent_ptr[g+1]) (tokens of sentence s:
 * tokens[tok_ptr[s] .. tok_ptr[s+1]), ids in [0, vocab) shared by the whole batch) and its query
 * q_tokens[q_ptr[g] .. q_ptr[g+1]) (a negative id = not in the vocabulary).  Each group is scored as if a throw-away
 * index were built over its own sentences (BM25Retriever.get_scores(query, docs), bit for bit), the sentences are
 * ordered by score descending then index descending, and out_keep[s] = 1 for the leading entries up to and
 * including the first whose running sum of sent_chars is >= ctx_chars[g] * rate (all of them if none is).
 *   score_type EZR_F64: idf_tab = double L[j] = log(j + 0.5) for j < idf_len, idf_len > max_sents; idf_off unused.
 *   score_type EZR_F32: idf_tab = float bm25s idf; the group of N sentences reads idf_tab[idf_off[g] + df], df <= N.
 * out_scores [S] (double / float, may be NULL), out_keep [S], out_counts[g] = number kept, or -1 for a group with no
 * sentences, or -2 for a group with bad input (a token id out of range, more than max_tokens tokens or max_sents
 * sentences, an idf table that does not cover it); such groups write nothing else.
 * max_tokens / max_sents: the largest group of the batch; they size shared memory and may not exceed the caps of
 * ezr_bm25_extract_caps (larger groups need a throw-away index and ezr_bm25_scores).  No workspace, no synchronisation. */
int ezr_bm25_extract_caps(int32_t* max_tokens_host, int32_t* max_sents_host);
int ezr_bm25_extract(const int64_t* sent_ptr, const int64_t* tok_ptr, const int32_t* tokens, int32_t vocab,
                     const int64_t* sent_chars, const int64_t* ctx_chars, const int64_t* q_ptr,
                     const int32_t* q_tokens, int32_t n_groups, int32_t max_tokens, int32_t max_sents,
                     const void* idf_tab, int64_t idf_len, const int64_t* idf_off, double k1, double b,
                     double epsilon, double rate, int32_t score_type, void* out_scores, uint8_t* out_keep,
                     int32_t* out_counts, void* stream);

/* ------------------------------------------------------- generic top-k --
 * Row-wise top-k of a score matrix (k <= 1024): scores[q*row_stride + j], j < n_cols.
 * positive_only != 0 keeps only scores > 0 (BM25Retriever.filter). */
size_t ezr_select_rows_workspace(int32_t n_rows, int64_t n_cols, int32_t k, int32_t score_type);
int ezr_select_rows(const void* scores, int32_t score_type, int32_t n_rows, int64_t n_cols, int64_t row_stride,
                    int32_t k, int32_t positive_only, const int32_t* doc_group, const int32_t* q_group,
                    int32_t id_base, void* out_scores, int32_t* out_ids, int32_t* out_counts, void* workspace,
                    size_t workspace_bytes, void* stream);

/* Merge per-shard / per-partition candidate lists: row q has n_cand (score,id) pairs at q*cand_stride,
 * id < 0 = empty slot.  Used after the all-gather of per-shard top-k (SURVEY.md 8(e)). k <= 1024. */
size_t ezr_merge_topk_workspace(int32_t n_rows, int32_t n_cand, int32_t k, int32_t score_type);
int ezr_merge_topk(const void* cand_scores, const int32_t* cand_ids, int32_t score_type, int32_t n_rows,
                   int32_t n_cand, int64_t cand_stride, int32_t k, void* out_scores, int32_t* out_ids,
                   int32_t* out_counts, void* workspace, size_t workspace_bytes, void* stream);

/* Same merge over candidates that sit in n_parts separate segments: segment p of row q starts at
 * (char*)cand_x + p*part_stride_bytes + q*cand_stride*sizeof(elem) and holds n_cand entries.  This is the layout of
 * the all-gathered per-shard records (easyrag_b200/dist.py: one byte record per rank, gathered back to back), so
 * the shard merge reads the NCCL output in place -- no unpack / transpose kernels.  k <= 32. */
int ezr_merge_topk_parts(const void* cand_scores, const int32_t* cand_ids, int32_t score_type, int32_t n_rows,
                         int32_t n_cand, int64_t cand_stride, int32_t n_parts, int64_t part_stride_bytes, int32_t k,
                         void* out_scores, int32_t* out_ids, int32_t* out_counts, void* stream);

/* Merge of SORTED per-shard lists, k <= 1024 (csrc/merge.cu).  n_parts lists per row, read in place from the gathered
 * records (addressing as ezr_merge_topk_parts).  Each part's slots are in canonical order (score desc, id desc) up to
 * its first id < 0, and hold only ids < 0 after it; ids are distinct across parts (disjoint shards).  Output: the
 * canonical top-k of the union at row q * out_stride, counts = min(k, total valid); slots [count, out_stride) get
 * id -1 and score -inf.  k, n_cand <= 1024, n_parts * n_cand <= 8192, out_stride >= k. */
int ezr_merge_sorted_parts(const void* cand_scores, const int32_t* cand_ids, int32_t score_type, int32_t n_rows,
                           int32_t n_cand, int64_t cand_stride, int32_t n_parts, int64_t part_stride_bytes, int32_t k,
                           void* out_scores, int32_t* out_ids, int32_t* out_counts, int64_t out_stride, void* stream);

/* ------------------------------------------------------------- dense ----
 * QdrantRetriever (retrievers.py:37-52) over a COSINE collection (ingestion.py:180-182):
 * corpus rows and queries are L2-normalised bf16; score = fp32-accumulated dot product.
 * ld_* are row strides in elements.  q_group / doc_group implement the `dir` payload filter
 * (ingestion.py:207-216).  Rows short of k are padded with id -1, score -inf. */
size_t ezr_dense_topk_workspace(int64_t n_rows, int32_t dim, int32_t n_queries, int32_t k);
int ezr_dense_topk(const void* corpus_bf16, int64_t n_rows, int32_t dim, int64_t ld_corpus,
                   const void* queries_bf16, int32_t n_queries, int64_t ld_queries, int32_t k,
                   const int32_t* doc_group, const int32_t* q_group, int32_t id_base, float* out_scores,
                   int32_t* out_ids, int32_t* out_counts, void* workspace, size_t workspace_bytes,
                   void* stream);
/* Insert path of the in-HBM vector store: out[r] = bf16(x[r] / max(||x[r]||, 1e-12)) in fp32 math (what a
 * Distance.COSINE collection does at insert, ingestion.py:180-182).  x is float32 (x_is_f32 != 0) or bf16; strides
 * in elements; out may be a slice of a larger preallocated corpus matrix (append without rebuilding). */
int ezr_normalize_rows(const void* x, int32_t x_is_f32, int64_t ldx, int64_t n_rows, int32_t dim, void* out_bf16,
                       int64_t ldo, void* stream);
/* 0 = pick automatically, 1 = force the generic SIMT kernel, 2 = force the wgmma kernel with 128-query blocks
 * (dim <= 768; the automatic choice there), 3 = force the wgmma kernel with 64-query blocks (the automatic choice
 * above 768), 4 = 64-query blocks and 128-row corpus tiles, 5 = 4 run in cluster pairs (two neighbouring query blocks
 * on the same corpus split; each CTA loads half of every corpus tile and TMA-multicasts it to both), 6 = wgmma score
 * rows of a query block, then the generic row top-k (any dim % 64 == 0, any k <= 1024; never chosen automatically);
 * 2-6 error if the shape is unsupported */
int ezr_dense_set_kernel(int32_t which);
/* name of the kernel the last ezr_dense_topk call on this thread launched
 * ("wgmma" / "wgmma-q64" / "wgmma-q64-n128" / "wgmma-q64-n128-mc2" / "wgmma-scores" / "simt") */
const char* ezr_dense_last_kernel(void);
/* Workspace of form 6 run in query blocks of block_queries queries: their fp32 score rows plus the select workspace
 * (of the smaller last block too).  Form 6 runs the largest block whose bytes fit the workspace it is given, so this
 * many bytes run blocks of block_queries queries; ezr_dense_topk_workspace's bytes run blocks at least as large as
 * the SIMT kernel's (256 MB of score rows).  Fewer bytes than block_queries = 1 needs: EZR_ERR_WORKSPACE. */
size_t ezr_dense_wide_workspace(int64_t n_rows, int32_t n_queries, int32_t k, int32_t block_queries);

/* Cap the TMA ring of the wgmma kernel at `stages` stages (0 = use all shared memory, the default).  A capped
 * ring leaves shared memory on an SM for kernels of another stream only when the resident query block is small; a
 * 128-query block of dim 768 fills the SM either way, and the cap then only shortens the ring. */
int ezr_dense_set_stage_cap(int32_t stages);

/* Measurement probes for the wgmma kernel (results become garbage; never use outside bench experiments):
 * bit mask: 1 = pipeline without TMA loads, 2 = one k-chunk of MMAs per tile, 4 = epilogue without the
 * insertion path. */
int ezr_dense_set_probe(int32_t probe);

/* Dense top-k over an int8 copy of the corpus (easyrag_b200/csrc/dense_s8.cu has the definition and the bound).
 * The result is the canonical top-k under rescore(q, r): the fp32 dot product of the bf16 query and bf16 row in
 * increasing coordinate order, one __fmul_rn and one __fadd_rn per coordinate (no FMA contraction), -0.0 returned
 * as +0.0, over every row that passes the filter -- never an approximation.
 *
 * quantize_rows: per row of bf16 x, scale = max|x_i| / 127 (fp32), out_s8 = clamp(rint(x_i / scale), +-127) (a zero
 * row: scale 0, R 0), err and norm = ||x - scale R||_2 and ||scale R||_2 evaluated in fp64 and rounded up to fp32 (the
 * bound of dense_s8.cu allows for the fp64 rounding).  Strides in
 * elements, as ezr_normalize_rows.  maxima (device float[2] = {max err, max norm}, may be NULL) is raised atomically:
 * zero it before the first rows of an index, keep it across appends. */
int ezr_dense_quantize_rows(const void* x_bf16, int64_t ldx, int64_t n_rows, int32_t dim, int8_t* out_s8, int64_t ldo,
                            float* scale, float* err, float* norm, float* maxima, void* stream);
/* The arguments of ezr_dense_topk, plus the int8 rows (ld_s8 in bytes, a multiple of 16), their per-row scales, the
 * maxima of quantize_rows, and out_cand_counts ([n_queries] or NULL: candidates the int8 pass emitted per query;
 * more than the capacity = overflowed, answered by the full scan; an overflowed query stops emitting, so its count
 * then only tells that it overflowed).  dim % 128 == 0, dim <= 1024; k <= 16 runs the
 * int8 pass + rescoring, 16 < k <= 1024 the full scan.  The call waits for the int8 pass to learn how many queries
 * overflowed (one stream synchronisation). */
size_t ezr_dense_s8_topk_workspace(int64_t n_rows, int32_t dim, int32_t n_queries, int32_t k);
int ezr_dense_s8_topk(const void* corpus_bf16, int64_t n_rows, int32_t dim, int64_t ld_corpus,
                      const void* queries_bf16, int32_t n_queries, int64_t ld_queries, int32_t k,
                      const int32_t* doc_group, const int32_t* q_group, int32_t id_base, float* out_scores,
                      int32_t* out_ids, int32_t* out_counts, const int8_t* corpus_s8, int64_t ld_s8,
                      const float* row_scale, const float* maxima, int32_t* out_cand_counts, void* workspace,
                      size_t workspace_bytes, void* stream);
/* Candidates per query the int8 pass may buffer (0 = the default, 4096).  Results never depend on it: a query that
 * emits more is answered by the full scan.  The workspace size depends on it; query the workspace after setting. */
int ezr_dense_s8_set_capacity(int32_t cap);   /* per host thread */

/* Dense top-k without score rows, "the candidate form" (easyrag_b200/csrc/dense_cand.cu; DESIGN §4.3b).  The arguments,
 * filters, id_base, padding and canonical order of ezr_dense_topk; the result is the canonical top-k under form 6's
 * scores (ezr_dense_set_kernel(6)), bit for bit.  The encoder's wgmma GEMM mainloop runs over the corpus in chunks
 * that double in size, and its epilogue appends to a per-query candidate buffer only the scores at or above the
 * query's current k-th score; a bound step between chunks keeps the top-k of each buffer and raises that threshold.
 * Memory grows with n_queries * (k + capacity) instead of n_queries * n_rows, and the whole batch shares one pass
 * over the corpus.
 *
 * A query whose buffer overflows is answered by form 6 inside the call (gathered, scored, scattered back); the call
 * waits for the candidate pass to learn how many did (one 4-byte copy and one stream synchronisation).
 * out_cand_counts ([n_queries] or NULL): the candidates each query emitted over the whole call, or -1 for a query
 * form 6 answered.  dim % 64 == 0, row strides % 8 == 0 and 16-byte aligned rows, else EZR_ERR_UNSUPPORTED (no
 * silent fall-back to another form); fewer workspace bytes than ezr_dense_cand_topk_workspace: EZR_ERR_WORKSPACE.
 * n_rows == 0 and n_queries == 0 behave as in ezr_dense_topk. */
size_t ezr_dense_cand_topk_workspace(int64_t n_rows, int32_t dim, int32_t n_queries, int32_t k);
int ezr_dense_cand_topk(const void* corpus_bf16, int64_t n_rows, int32_t dim, int64_t ld_corpus,
                        const void* queries_bf16, int32_t n_queries, int64_t ld_queries, int32_t k,
                        const int32_t* doc_group, const int32_t* q_group, int32_t id_base, float* out_scores,
                        int32_t* out_ids, int32_t* out_counts, int32_t* out_cand_counts, void* workspace,
                        size_t workspace_bytes, void* stream);
/* Candidate slots per query of ezr_dense_cand_topk (0 = the default, 4k + 1024, as the BM25 deep list; at most 2^20).
 * Results never depend on it: a query that emits more is answered by form 6.  The workspace size depends on it; query
 * the workspace after setting. */
int ezr_dense_cand_set_capacity(int32_t cap);   /* per host thread */

/* ------------------------------------------------------------- fusion ---
 * HybridRetriever.reciprocal_rank_fusion (retrievers.py:256-274): list a first, then list b
 * (the reference passes [sparse, dense], retrievers.py:290); score += 1/(rank+K), rank from 1, fp64;
 * key = canon[id] (documents with identical text share a key, retrievers.py:263-265; NULL = identity);
 * the returned id is the LAST occurrence of the key (text_to_node overwrite, :264); ties keep
 * first-insertion order (stable sort, :266).  ids_x is [Q][stride_in], cnt_x[Q] valid entries each. */
int ezr_rrf_fuse(const int32_t* ids_a, const int32_t* cnt_a, const int32_t* ids_b, const int32_t* cnt_b,
                 int32_t n_queries, int32_t stride_in, const int32_t* canon, int32_t canon_base, int32_t K,
                 int32_t k_out, int32_t* out_ids, double* out_scores, int32_t* out_counts, void* stream);

/* HybridRetriever.fusion (retrievers.py:239-253): concatenate, drop later items whose text was seen,
 * stable sort by raw score descending, keep k_out. */
int ezr_fusion_simple(const int32_t* ids_a, const double* scores_a, const int32_t* cnt_a, const int32_t* ids_b,
                      const double* scores_b, const int32_t* cnt_b, int32_t n_queries, int32_t stride_in,
                      const int32_t* canon, int32_t canon_base, int32_t k_out, int32_t* out_ids,
                      double* out_scores, int32_t* out_counts, void* stream);

/* Both fusions over ANY number of rank lists (the reference's loops take a list of lists, retrievers.py:243,261;
 * the pipeline passes two).  ids_host / scores_host / cnt_host are HOST arrays of n_lists DEVICE pointers (each list
 * laid out like ids_a / scores_a / cnt_a above; scores_host may be NULL for RRF); list order = insertion order.
 * rrf != 0: reciprocal_rank_fusion, else fusion.  n_lists <= 8, n_lists * stride_in <= 2048. */
int ezr_fuse_lists(int32_t rrf, int32_t n_lists, const int32_t* const* ids_host, const double* const* scores_host,
                   const int32_t* const* cnt_host, int32_t n_queries, int32_t stride_in, const int32_t* canon,
                   int32_t canon_base, int32_t K, int32_t k_out, int32_t* out_ids, double* out_scores,
                   int32_t* out_counts, void* stream);

/* ------------------------------------------------- reranker hand-off ---
 * The coarse ranker's fused top-k -> the token sequences LLMRerank scores (rerankers.py:196-293 get_inputs /
 * get_inputs_v2_5, sliced 32 at a time by _postprocess_nodes :309-322), built on the device.  Pair p = q*k + r is
 * candidate r of query q: [bos] + query[: 3/4 max_length] + sep + passage (the pair truncated to max_length, the
 * passage gives way) + sep + prompt.  Queries ("A: ..." ids, q_ptr/q_tok) and passages ("B: ..." ids of every chunk,
 * tokenised once at index time, n_docs of them, ids id_base ..., p_ptr/p_tok) are device CSR arrays.  Output is packed:
 * ids[T], cu[P+1]; pairs past a query's count are empty.  plan: lengths, their scan (int64) and get_inputs_v2_5's
 * query_lengths; *total_host = T (synchronises; a candidate id outside the passage range, or T >= 2^31, is
 * EZR_ERR_INVALID).  fill: the tokens + an int32 copy of cu (the cu_seqlens format of the encoder kernels). */
int ezr_rerank_pack_plan(const int32_t* cand_ids, const int32_t* cand_cnt, int32_t n_queries, int32_t k, int32_t k_stride,
                         int32_t id_base, int32_t n_docs, const int32_t* q_ptr, const int64_t* p_ptr, int32_t n_sep,
                         int32_t n_prompt, int32_t max_length, int64_t* out_len, int64_t* out_cu,
                         int32_t* out_query_len, int64_t* total_host, void* stream);
int ezr_rerank_pack_fill(const int32_t* cand_ids, const int32_t* cand_cnt, int32_t n_queries, int32_t k, int32_t k_stride,
                         int32_t id_base, int32_t n_docs, const int32_t* q_ptr, const int32_t* q_tok, const int64_t* p_ptr,
                         const int32_t* p_tok, const int32_t* sep, int32_t n_sep, const int32_t* prompt, int32_t n_prompt,
                         int32_t bos, int32_t max_length, const int64_t* cu, int32_t* out_ids, int32_t* out_cu32,
                         void* stream);

/* ---------------------------------------------------- cross-encoder rerank ---
 * SentenceTransformerRerank (rerankers.py:15-99): CrossEncoder.predict over (query, passage) pairs, then the stable
 * descending sort of the sigmoid scores.  Pairs are built on the device from the coarse [Q, k] ids exactly as the
 * fast tokenizer encodes a pair with truncation="longest_first" at max_length: with a, b the query / passage lengths
 * (no specials) and T = max_length - 2 - n_mid, both stay if a + b <= T, else the longer side is cut to T - the other,
 * where the other keeps min(its length, T/2); tokens are cut from the end.  Layout [cls] q [sep] x n_mid p [sep]
 * (BERT n_mid = 1, types 0 | type_b = 1 after the first [sep]; RoBERTa / XLM-R n_mid = 2, type_b = 0), positions
 * pos_offset + i (0 for BERT, padding_idx + 1 for RoBERTa).  Queries (q_ptr / q_tok) and passages (p_ptr / p_tok,
 * n_docs of them, ids id_base ...) are device CSR arrays of ids tokenised without special tokens.
 * Only the real pairs (candidate r < counts[q]) are packed: pair pair_off[q] + r, P = pair_off[Q] in all.
 * plan: pair_off int32 [Q + 1], cu int32 [P + 1] (the caller sizes it Q * k + 1), totals_host = {T, P}
 *       (synchronises; a candidate id outside the passage range, or T >= 2^31, is EZR_ERR_INVALID).
 * fill: ids / types / positions int32 [T], reading the plan's workspace. */
size_t ezr_cross_pack_workspace(int32_t n_queries, int32_t k);
int ezr_cross_pack_plan(const int32_t* cand_ids, const int32_t* cand_cnt, int32_t n_queries, int32_t k,
                        int32_t k_stride, int32_t id_base, int32_t n_docs, const int32_t* q_ptr, const int64_t* p_ptr,
                        int32_t n_mid, int32_t max_length, int32_t* out_pair_off, int32_t* out_cu,
                        int64_t* totals_host, void* workspace, size_t ws_bytes, void* stream);
int ezr_cross_pack_fill(const int32_t* cand_ids, const int32_t* cand_cnt, int32_t n_queries, int32_t k,
                        int32_t k_stride, int32_t id_base, int32_t n_docs, const int32_t* q_ptr, const int32_t* q_tok,
                        const int64_t* p_ptr, const int32_t* p_tok, int32_t cls, int32_t sep, int32_t n_mid,
                        int32_t type_b, int32_t pos_offset, int32_t max_length, const void* workspace,
                        int32_t* out_ids, int32_t* out_types, int32_t* out_pos, void* stream);
/* The rest of the head and the order, one CTA per query: dense = the [P, d] bf16 rows Linear(d, d) + bias made from
 * the pairs' CLS rows; score = sigmoid(tanh(dense) . w_out + b_out) in fp32.  out_all [Q, k] holds every pair's
 * score (-inf past the query's count); out_scores / out_ids [Q, top_n] the top_n by score descending, ties in coarse
 * rank order (ids from cand_ids, -1 / -inf padded); out_counts [Q].  k <= 1024. */
int ezr_cross_score_topk(const void* dense, int64_t ldd, const int32_t* pair_off, int32_t n_queries, int32_t k,
                         const int32_t* cand_ids, int32_t k_stride, const float* w_out, float b_out, int32_t dim,
                         int32_t top_n, float* out_all, float* out_scores, int32_t* out_ids, int32_t* out_counts,
                         void* stream);
/* ezr_cross_score_topk in two steps, bit-identical to it, for pairs scored on several devices.
 * pair_scores: out_sig[p] = sigmoid(tanh(dense[p]) . w_out + b_out) for the n_pairs contiguous [n_pairs, dim] bf16
 *              rows of dense (one warp per pair).
 * order_topk:  from sig float32 [P] (pair pair_off[q] + r = candidate r of query q), the outputs of
 *              ezr_cross_score_topk (one CTA per query).  k <= 1024. */
int ezr_cross_pair_scores(const void* dense, int32_t dim, int32_t n_pairs, const float* w_out, float b_out,
                          float* out_sig, void* stream);
int ezr_cross_order_topk(const float* sig, const int32_t* pair_off, int32_t n_queries, int32_t k,
                         const int32_t* cand_ids, int32_t k_stride, int32_t top_n, float* out_all, float* out_scores,
                         int32_t* out_ids, int32_t* out_counts, void* stream);
/* Rerank fusion (generation_with_rerank_fusion, pipeline.py:393-452): two coarse lists per query reranked separately,
 * their pairs packed and encoded once as the union of the two lists.
 * pair_union:  per query, the distinct DOCUMENT ids (not canon keys: the reranker scores each id's own passage) of
 *              list a's slots [0, cnt_a) then list b's [0, cnt_b), in first-appearance order -- the lists disjoint,
 *              that is list a followed by list b.  out_ids int32 [Q, k_a + k_b] (-1 past the count), out_counts [Q],
 *              out_map_a [Q, k_a] / out_map_b [Q, k_b] the union index of every list slot (-1 past the list's count).
 *              Each list holds distinct ids (a coarse top-k); a repeated id maps its slots to one union entry.
 *              Counts are clamped to [0, k].  k_a + k_b <= 1024, else EZR_ERR_INVALID.  One CTA per query.
 * order_topk_mapped: ezr_cross_order_topk for one list from the union's scores: sig float32 [P] holds the union's
 *              pairs (pair pair_off[q] + u = union entry u of query q), slot_map [Q][map_stride] the list's map
 *              (pair_union's out_map_x); list slot r scores sig[pair_off[q] + slot_map[q, r]].  The list's count is
 *              the map's leading run of entries in [0, pair count of q).  Outputs and order are those of
 *              ezr_cross_order_topk on the list alone (cand_ids / k_stride: the list's ids).  k <= 1024. */
int ezr_pair_union(const int32_t* ids_a, const int32_t* cnt_a, int32_t k_a, int32_t stride_a, const int32_t* ids_b,
                   const int32_t* cnt_b, int32_t k_b, int32_t stride_b, int32_t n_queries, int32_t* out_ids,
                   int32_t* out_counts, int32_t* out_map_a, int32_t* out_map_b, void* stream);
int ezr_cross_order_topk_mapped(const float* sig, const int32_t* pair_off, int32_t n_queries, int32_t k,
                                const int32_t* slot_map, int32_t map_stride, const int32_t* cand_ids, int32_t k_stride,
                                int32_t top_n, float* out_all, float* out_scores, int32_t* out_ids,
                                int32_t* out_counts, void* stream);

/* ------------------------------------------------------------ encoder ---
 * Building blocks of the chunk/query embedding forward pass (GTEEmbedding._embed, gte_embeddings.py:59-72 ->
 * Qwen2Model.forward, modeling_qwen.py:956-1116; HuggingFaceEmbedding._embed, hf_embeddings.py:112-123 ->
 * a BERT-shaped encoder).  Activations are bf16, row-major, PACKED: sequence b owns rows
 * [cu_seqlens[b], cu_seqlens[b+1]) -- no padding tokens.  The Python classes in easyrag_b200/encoder.py chain
 * these per layer on one stream. */

/* out[M,N'] = epi(A[M,K] . W[N,K]^T + bias) (+ residual); wgmma + TMA.  epilogue: 0 none, 1 GELU(erf),
 * 2 SwiGLU (W rows interleaved per 256: 128 gate rows then the matching 128 up rows; N' = N/2).  K % 64 == 0. */
int ezr_gemm_bf16(const void* a, int32_t m, int32_t k, int64_t lda, const void* w, int32_t n, int64_t ldw,
                  const void* bias, const void* residual, int64_t ldr, void* out, int64_t ldo, int32_t epilogue,
                  void* stream);
/* FP8 (opt-in precision of the encoders).  e4m3 operands, fp32 accumulation promoted every 128 K, bf16 output:
 *   out[M,N'] = epi(diag(sa) . A8[M,K] . W8[N,K]^T . diag(sw) + bias) (+ residual)
 * sa float32 [M] (one power-of-two scale per activation row), sw float32 [N] (one per weight row / output channel),
 * epilogues as ezr_gemm_bf16 except SwiGLU: W8 (and bias) rows interleaved per 128: 64 gate rows then the matching
 * 64 up rows.  K % 128 == 0; lda, ldw (bytes) multiples of 16; A8 / W8 16-byte aligned.  out may alias residual. */
int ezr_gemm_fp8(const void* a8, const float* sa, int32_t m, int32_t k, int64_t lda, const void* w8, const float* sw,
                 int32_t n, int64_t ldw, const void* bias, const void* residual, int64_t ldr, void* out, int64_t ldo,
                 int32_t epilogue, void* stream);
/* bf16 [rows, cols] -> e4m3 [rows, cols] (row stride ldo bytes) and float32 scales [rows]: per row
 * s = 2^ceil(log2(amax / 448)) (1 for an all-zero row), q = e4m3_rn(x / s).  One warp per row.  cols, ldx, ldo
 * multiples of 8; x 16-byte, out 8-byte aligned.  Inf / NaN inputs are not supported. */
int ezr_quant_rows_fp8(const void* x, int64_t ldx, int32_t rows, int32_t cols, void* out_e4m3, int64_t ldo,
                       float* out_scale, void* stream);
/* the same for an nn.Linear weight [n, k]: one scale per output channel (row); run once when a model loads */
int ezr_quant_weight_fp8(const void* w, int64_t ldw, int32_t n, int32_t k, void* out_e4m3, int64_t ldo,
                         float* out_scale, void* stream);
/* ezr_rmsnorm / ezr_layernorm rounded to bf16 exactly as they are, stored to out when out != NULL, and that bf16 row
 * quantised as ezr_quant_rows_fp8 does, in the same kernel.  dim % 8 == 0, dim <= 4096; x / out / gamma / beta
 * 16-byte aligned, out_e4m3 8-byte aligned, strides multiples of 8. */
int ezr_rmsnorm_fp8(const void* x, int64_t ldx, const void* gamma, float eps, int32_t n_rows, int32_t dim, void* out,
                    int64_t ldo, void* out_e4m3, int64_t ldq, float* out_scale, void* stream);
int ezr_layernorm_fp8(const void* x, int64_t ldx, const void* gamma, const void* beta, float eps, int32_t n_rows,
                      int32_t dim, void* out, int64_t ldo, void* out_e4m3, int64_t ldq, float* out_scale,
                      void* stream);
/* non-causal attention over packed q|k|v rows ([n_tokens, (H + 2*KV) * hd], row stride ld); head_dim 64 or 128; GQA
 * via n_kv_heads.  Default kernel: wgmma (S = QK^T and O += PV on the tensor cores, S/P/O in registers,
 * Q/K/V tiles by TMA).  n_tokens bounds the TMA tensor map (tiles that run past the last token are zero-filled).
 * n_seq <= 65535 per call (both kernels).  The wgmma kernel's query-block plan (16 bytes per 128-row block) is
 * allocated on `stream` from its device's default memory pool and freed on it after the kernel, so calls on
 * different streams, from any thread, never share one; the call can be captured into a CUDA graph. */
int ezr_attn_bidir(const void* qkv, int64_t n_tokens, int64_t ld, const int32_t* cu_seqlens, int32_t n_seq,
                   int32_t max_len, int32_t n_heads, int32_t n_kv_heads, int32_t head_dim, float softmax_scale, void* out,
                   int64_t ldo, void* stream);
/* causal attention over the same packed layout, same arguments and checks: query row r of a sequence sees its keys
 * 0..r (Qwen2Model.forward(is_causal=True) on a padding-free batch).  wgmma kernel only: under
 * ezr_attn_set_kernel(1) it returns EZR_ERR_INVALID, the mma.sync kernel being bidirectional only. */
int ezr_attn_causal(const void* qkv, int64_t n_tokens, int64_t ld, const int32_t* cu_seqlens, int32_t n_seq,
                    int32_t max_len, int32_t n_heads, int32_t n_kv_heads, int32_t head_dim, float softmax_scale, void* out,
                    int64_t ldo, void* stream);
/* 0 = wgmma kernel (default), 1 = the warp-level mma.sync kernel (kept as an independent cross-check) */
int ezr_attn_set_kernel(int32_t which);
/* "wgmma" / "wgmma-causal" / "mma.sync": what the last ezr_attn_bidir / ezr_attn_causal call on this thread launched */
const char* ezr_attn_last_kernel(void);
int ezr_embed_gather(const int32_t* ids, int32_t n_tokens, const void* table, int64_t ldt, int32_t vocab, int32_t dim,
                     void* out, int64_t ldo, void* stream);
/* BERT embeddings: LayerNorm(word[id] + type[0] + position[pos]) */
int ezr_bert_embed(const int32_t* ids, const int32_t* positions, int32_t n_tokens, const void* word, const void* pos,
                   const void* type0, const void* gamma, const void* beta, float eps, int32_t vocab, int32_t max_pos,
                   int32_t dim, void* out, void* stream);
/* the same with a per-token segment: LayerNorm(word[id] + type_table[types[t]] + position[pos]), n_types table rows
 * (same rounding order: word + type, then + position, each rounded to bf16) */
int ezr_bert_embed_typed(const int32_t* ids, const int32_t* positions, const int32_t* types, int32_t n_tokens,
                         const void* word, const void* pos, const void* type_table, int32_t n_types, const void* gamma,
                         const void* beta, float eps, int32_t vocab, int32_t max_pos, int32_t dim, void* out,
                         void* stream);
/* Qwen2RMSNorm (modeling_qwen.py:91-96) */
int ezr_rmsnorm(const void* x, int64_t ldx, const void* gamma, float eps, int32_t n_rows, int32_t dim, void* out,
                int64_t ldo, void* stream);
int ezr_layernorm(const void* x, int64_t ldx, const void* gamma, const void* beta, float eps, int32_t n_rows,
                  int32_t dim, void* out, int64_t ldo, void* stream);
/* rotary embedding in place on the q and k heads of packed qkv rows (modeling_qwen.py:137-169); bf16 cos/sin tables
 * [max_pos, head_dim/2] */
int ezr_rope(void* qkv, int64_t ld, const int32_t* positions, const void* cos_table, const void* sin_table,
             int32_t max_pos, int32_t n_heads_qk, int32_t head_dim, int32_t n_tokens, void* stream);
/* pooling (0 last token, 1 first/CLS, 2 mean) + optional final RMSNorm of the pooled row + L2 normalisation
 * (l2_mode 0 none, 1 bf16 semantics of gte_embeddings.py:70, 2 fp32 semantics); writes bf16 [n_seq, dim] and,
 * if out_f32 != NULL, the float copy the embedding API returns */
int ezr_pool_normalize(const void* hidden, int64_t ldh, const int32_t* cu_seqlens, int32_t n_seq, int32_t pool,
                       int32_t final_norm, const void* gamma, float eps, int32_t l2_mode, int32_t dim, void* out_bf16,
                       float* out_f32, void* stream);

/* ------------------------------------------------------ string interning --
 * csrc/vocab.cu (easyrag_b200/vocab.py, DESIGN.md §4.9): the id a Python dict filled in first-seen order gives each
 * string (d.setdefault(s, len(d))) and the global index of its first occurrence, for chunks of n_strings UTF-8 strings
 * joined by single NUL bytes (n_bytes bytes, exactly n_strings - 1 NULs; zero-length strings are keys too).
 * State, all caller-owned device memory:
 *   table     ezr_vocab_table_bytes(capacity) bytes, capacity a power of two in [2, 2^40]; it records the hash bits
 *             in force when ezr_vocab_table_init made it, and ezr_vocab_table_grow keeps them.
 *   arena     the bytes of every id in id order; arena_off int64 [id_capacity + 1] (arena_off[0] = 0): id i's bytes
 *             are arena[arena_off[i] .. arena_off[i + 1]).  id_first int64 [id_capacity]: id i's first index.
 *   state_host int64 [2] on the host: {ids, arena bytes used}; ezr_vocab_insert updates it.
 * insert: interns the chunk (its strings have global indices first_index ..) and writes out_ids int32 [n_strings] and,
 *   when out_first != NULL, out_first int64 [n_strings].  Needs 2 * (ids + n_strings) <= capacity (grow the table
 *   first), else EZR_ERR_WORKSPACE.  New ids past id_capacity or new bytes past arena_capacity: EZR_ERR_WORKSPACE; an
 *   id past INT32_MAX: EZR_ERR_INVALID; the table is then left as it was.  Synchronises the stream once.
 * lookup: the same ids without inserting; -1 (and first index -1) for a string the table does not hold.  Synchronises.
 * A separator count other than n_strings - 1 is EZR_ERR_INVALID and writes no output.  Chunks: n_bytes < 2^32.
 * read: copies arena_off[id_lo .. id_hi] to off_host and the bytes of ids [id_lo, id_hi) to bytes_host (synchronises).
 * set_hash_bits: hash bits (1..64, default 64) of tables made afterwards on this host thread; fewer bits make equal
 *   hashes of different strings common (tests of the byte comparison).  Results are the same at every setting. */
int ezr_vocab_set_hash_bits(int32_t bits);
size_t ezr_vocab_table_bytes(int64_t capacity);
size_t ezr_vocab_workspace(int64_t n_strings, int64_t n_bytes);
int ezr_vocab_table_init(void* table, int64_t capacity, void* stream);
int ezr_vocab_table_grow(const void* table, int64_t capacity, void* new_table, int64_t new_capacity, void* stream);
int ezr_vocab_insert(void* table, int64_t capacity, const uint8_t* bytes, int64_t n_bytes, int64_t n_strings,
                     int64_t first_index, uint8_t* arena, int64_t arena_capacity, int64_t* arena_off,
                     int64_t* id_first, int64_t id_capacity, int64_t* state_host, int32_t* out_ids,
                     int64_t* out_first, void* workspace, size_t ws_bytes, void* stream);
int ezr_vocab_lookup(const void* table, int64_t capacity, const uint8_t* bytes, int64_t n_bytes, int64_t n_strings,
                     const uint8_t* arena, const int64_t* arena_off, const int64_t* id_first, int32_t* out_ids,
                     int64_t* out_first, void* workspace, size_t ws_bytes, void* stream);
int ezr_vocab_read(const uint8_t* arena, const int64_t* arena_off, int64_t id_lo, int64_t id_hi, uint8_t* bytes_host,
                   size_t bytes_cap, int64_t* off_host, void* stream);

/* ----------------------------------------------------------- profiling ---
 * Per-kernel CUDA-event timing on the launching stream, for bench.py's roofline figures.
 * ezr_profile_read synchronises on the recorded events and returns the summed duration of the
 * kernel launches recorded in `slot` since the last reset. */
typedef enum ezr_prof_slot {
    EZR_PROF_BM25_SCORE = 0, /* bm25_score_kernel (fused top-k or score rows) */
    EZR_PROF_DENSE_TC = 1,   /* dense_wgmma_kernel */
    EZR_PROF_DENSE_SIMT = 2, /* dense_scores_simt_kernel */
    EZR_PROF_MERGE = 3,      /* merge / select kernels */
    EZR_PROF_FUSE = 4,       /* rrf / simple fusion */
    EZR_PROF_ENC_GEMM = 5,   /* encoder GEMMs (not form 6's score rows: EZR_PROF_DENSE_WIDE) */
    EZR_PROF_ENC_ATTN = 6,   /* encoder attention */
    EZR_PROF_ENC_OTHER = 7,  /* encoder norms / elementwise */
    EZR_PROF_BM25_CAND = 8,  /* bm25_cand_kernel (integer candidate pass over packed postings) */
    EZR_PROF_BM25_RESCORE = 9, /* bm25_rescore_kernel (exact float64 rescoring + top-k of the candidates) */
    EZR_PROF_DENSE_S8_SCAN = 10,    /* dense_s8_prep_kernel + dense_s8_scan_kernel (int8 candidate pass) */
    EZR_PROF_DENSE_S8_RESCORE = 11, /* dense_s8_rescore_kernel (exact rescoring + top-k of the candidates) */
    EZR_PROF_DENSE_S8_FULL = 12,    /* full scan of overflowed queries / k > 16 (gather + score rows + select) */
    EZR_PROF_DENSE_WIDE = 13,       /* gemm_wgmma_kernel's score-row instance (form 6; the select counts as merge) */
    EZR_PROF_BM25_BOUND = 14,       /* bm25_bound_kernel between candidate chunks (also inside EZR_PROF_BM25_CAND) */
    EZR_PROF_DENSE_CAND_GEMM = 15,  /* dense_cand_kernel (the candidate form's GEMM + threshold epilogue) */
    EZR_PROF_DENSE_CAND_BOUND = 16, /* dense_cand_init_kernel + dense_cand_bound_kernel (bound steps, outputs); the
                                     * candidate form's form 6 fallback: EZR_PROF_DENSE_WIDE (+ its select: merge) */
    EZR_PROF_COUNT = 17
} ezr_prof_slot;
/* kernels launched by this library since it was loaded (every launch site counts itself) */
long long ezr_launch_count(void);
int ezr_profile_enable(int32_t on);
int ezr_profile_reset(void);
int ezr_profile_read(int32_t slot, double* total_ms, int32_t* launches);

#ifdef __cplusplus
}
#endif
#endif /* EASYRAG_B200_H */
