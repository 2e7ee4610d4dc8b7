"""GPU parity tests: CUDA path (through the C ABI) vs the CPU oracle on the same seeded inputs.

Bar (BASELINE.json north_star): bit-exact doc-id rank lists and scores for BM25 / RRF / fusion;
cosine scores within 1e-3 for the bf16 dense route (and bit-exact where the inputs make the
dot products exactly representable).
"""
import numpy as np
import pytest
import torch

from oracle import bm25 as obm
from oracle import retrieve as ort
from easyrag_b200 import synth, _lib, batched
from easyrag_b200.index import Bm25Index, Bm25Stats, DenseIndex

pytestmark = pytest.mark.gpu
DEV = "cuda"
COS_TOL = 1e-3          # north_star: "cosine scores within 1e-3 for bf16 embedding"


@pytest.fixture(scope="module", autouse=True)
def _lib_ready(lib_built):
    _lib.require_cuda()


def _pad_ids(ids, k):
    out = np.full(k, -1, dtype=np.int64)
    out[:len(ids)] = ids
    return out


def _check_bm25_topk(res, rows, k, allowed=None, id_base=0):
    ids = res.ids.cpu().numpy()
    sc = res.scores.cpu().numpy()
    cnt = res.counts.cpu().numpy()
    for q, row in enumerate(rows):
        al = None
        if allowed is not None:
            al = allowed[q] if isinstance(allowed, list) else allowed
        ref_i, ref_s = ort.bm25_topk_ids(row, k, al)
        assert cnt[q] == ref_i.size, f"query {q}: count {cnt[q]} != {ref_i.size}"
        assert np.array_equal(ids[q, :cnt[q]], ref_i + id_base), f"query {q}: ids differ"
        assert sc[q, :cnt[q]].tobytes() == ref_s.astype(sc.dtype).tobytes(), f"query {q}: scores not bit-exact"
        assert (ids[q, cnt[q]:] == -1).all()


# ------------------------------------------------------------------ BM25 ----
@pytest.fixture(scope="module")
def c1():
    """BASELINE config 1 shape: 10k chunks, V=50k, 100 queries of 4-12 terms."""
    corpus = synth.make_sparse_corpus(10_000, 50_000, 20240922 + 1)
    queries = synth.make_queries(corpus, 100, 20240922 + 101)
    oracle = obm.OkapiCSR(corpus.doc_lists(), corpus.vocab)
    stats = Bm25Stats.from_tokens(corpus.tokens, corpus.doc_ptr, corpus.vocab, bm25_type=0)
    groups = synth.make_groups(corpus.n_docs, 4, 7)
    index = Bm25Index(stats, device=DEV, doc_group=groups)
    rows = [oracle.get_scores([int(t) for t in terms]) for terms in queries.term_lists()]
    return dict(corpus=corpus, queries=queries, oracle=oracle, stats=stats, index=index, rows=rows, groups=groups)


def test_bm25_weights_bit_exact(c1):
    o, ix = c1["oracle"], c1["index"]
    w = ix.post_w.cpu().numpy()
    for t in np.random.default_rng(0).choice(np.nonzero(o.df)[0], 200, replace=False):
        s, e = o.indptr[t], o.indptr[t + 1]
        assert w[s:e].tobytes() == o.contributions(int(t)).tobytes()


def test_bm25_score_rows_bit_exact(c1):
    q = c1["queries"]
    got = batched.bm25_scores(c1["index"], q.term_ptr, q.terms).cpu().numpy()
    for i, row in enumerate(c1["rows"]):
        assert got[i].tobytes() == row.tobytes(), f"query {i}"


def test_bm25_score_rows_match_literal_reference_loop(c1):
    # the literal per-term / per-document loop of rank_bm25 (what the reference executes), on a subset
    docs = [list(map(int, d)) for d in c1["corpus"].doc_lists()[:1500]]
    lit = obm.OkapiLiteral(docs)
    sub = synth.SparseCorpus(tokens=c1["corpus"].tokens[:int(c1["corpus"].doc_ptr[1500])],
                             doc_ptr=c1["corpus"].doc_ptr[:1501].clone(), vocab=c1["corpus"].vocab)
    ix = Bm25Index(Bm25Stats.from_tokens(sub.tokens, sub.doc_ptr, sub.vocab), device=DEV)
    q = c1["queries"]
    got = batched.bm25_scores(ix, q.term_ptr[:6], q.terms[:int(q.term_ptr[5])]).cpu().numpy()
    for i, terms in enumerate(q.term_lists()[:5]):
        assert got[i].tobytes() == lit.get_scores([int(t) for t in terms]).tobytes()


@pytest.mark.parametrize("k", [1, 10, 32])
def test_bm25_topk_fused_bit_exact(c1, k):
    q = c1["queries"]
    res = batched.bm25_topk(c1["index"], q.term_ptr, q.terms, k)
    _check_bm25_topk(res, c1["rows"], k)


@pytest.mark.parametrize("k", [33, 192, 1024])
def test_bm25_topk_large_k_bit_exact(c1, k):
    q = c1["queries"]
    nq = 12
    res = batched.bm25_topk(c1["index"], q.term_ptr[:nq + 1], q.terms, k)
    _check_bm25_topk(res, c1["rows"][:nq], k)


@pytest.mark.parametrize("k", [10, 64])
def test_bm25_topk_with_dir_filter(c1, k):
    q = c1["queries"]
    g = c1["groups"].numpy()
    want = np.array([i % 6 - 1 for i in range(q.n)], dtype=np.int32)     # -1 none, 0..3 classes, 4 = no such class
    want[want == 4] = -2
    allowed = [None if w == -1 else (g == w) for w in want]
    res = batched.bm25_topk(c1["index"], q.term_ptr, q.terms, k, q_group=torch.from_numpy(want))
    _check_bm25_topk(res, c1["rows"], k, allowed=allowed)


def test_bm25_edge_queries(c1):
    # empty query, all-unknown query, duplicated term, term id out of range, long query (> 12 terms: two rounds)
    o = c1["oracle"]
    present = np.nonzero(o.df)[0]
    lists = [[], [-1, -1], [int(present[3])] * 3, [c1["corpus"].vocab + 5, int(present[10])],
             [int(t) for t in present[:30]]]
    ptr = torch.tensor(np.cumsum([0] + [len(l) for l in lists]), dtype=torch.int32)
    terms = torch.tensor([t for l in lists for t in l] or [0], dtype=torch.int32)
    rows = [o.get_scores(l) for l in lists]
    res = batched.bm25_topk(c1["index"], ptr, terms, 10)
    _check_bm25_topk(res, rows, 10)
    assert res.counts[0].item() == 0 and res.counts[1].item() == 0
    got = batched.bm25_scores(c1["index"], ptr, terms).cpu().numpy()
    for i, row in enumerate(rows):
        assert got[i].tobytes() == row.tobytes()


@pytest.mark.parametrize("n_docs", [1, 2, 8191, 8192, 8193, 20000])
def test_bm25_ragged_sizes_and_ties(n_docs):
    # documents duplicated pairwise -> exact score ties -> canonical order must put the higher id first
    base = synth.make_sparse_corpus((n_docs + 1) // 2, 300, 77, mean_len=12, min_len=0, max_len=40)
    docs = base.doc_lists()
    docs = (docs + docs)[:n_docs]
    tokens = torch.from_numpy(np.concatenate(docs) if sum(map(len, docs)) else np.zeros(0, np.int32)).to(torch.int32)
    ptr = torch.tensor(np.cumsum([0] + [len(d) for d in docs]), dtype=torch.int64)
    if tokens.numel() == 0:
        pytest.skip("degenerate")
    corpus = synth.SparseCorpus(tokens=tokens, doc_ptr=ptr, vocab=300)
    o = obm.OkapiCSR(docs, 300)
    ix = Bm25Index(Bm25Stats.from_tokens(tokens, ptr, 300), device=DEV)
    qs = synth.make_queries(corpus, 20, 78, min_terms=1, max_terms=5)
    rows = [o.get_scores([int(t) for t in terms]) for terms in qs.term_lists()]
    for k in (3, 10):
        _check_bm25_topk(batched.bm25_topk(ix, qs.term_ptr, qs.terms, k), rows, k)


def test_bm25_massive_ties_take_overflow_path():
    # thousands of identical documents: every score ties, the candidate list overflows and the kernel's
    # warp-shuffle fallback must still return the highest ids first
    one = np.array([1, 2, 3, 4, 5, 1], dtype=np.int32)
    other = np.array([7, 8, 9], dtype=np.int32)
    docs = [one if i % 3 else other for i in range(20_000)]
    tokens = torch.from_numpy(np.concatenate(docs)).to(torch.int32)
    ptr = torch.tensor(np.cumsum([0] + [len(d) for d in docs]), dtype=torch.int64)
    o = obm.OkapiCSR(docs, 12)
    ix = Bm25Index(Bm25Stats.from_tokens(tokens, ptr, 12), device=DEV)
    lists = [[1, 2], [7], [1, 7, 9, 11], [5, 5, 5]]
    qp = torch.tensor(np.cumsum([0] + [len(l) for l in lists]), dtype=torch.int32)
    qt = torch.tensor([t for l in lists for t in l], dtype=torch.int32)
    rows = [o.get_scores(l) for l in lists]
    for k in (1, 10, 32):
        _check_bm25_topk(batched.bm25_topk(ix, qp, qt, k), rows, k)



# ---- two-phase path (packed postings -> integer candidates -> exact rescoring) vs the ordered kernel ----
def test_bm25_pack_matches_definition(c1):
    ix = c1["index"]
    assert ix.post_pk is not None, "float64 Okapi index with non-negative idf must carry packed postings"
    R = _lib.BM25_RANGE
    wbits = 32 - int(np.log2(R))
    w = ix.post_w.cpu().numpy()
    d = ix.post_doc.cpu().numpy()
    pk = ix.post_pk.cpu().numpy().view(np.uint32)
    e = ix.pk_scale_log2
    wq = np.ceil(np.ldexp(w, e)).astype(np.uint64)
    assert wq.max() < (1 << (wbits - 1))
    assert (wq[w > 0] >= 1).all()
    assert np.array_equal(pk >> wbits, (d % R).astype(np.uint32))
    assert np.array_equal(pk & ((1 << wbits) - 1), wq.astype(np.uint32))


def _topk_bytes(res):
    return res.ids.cpu().numpy().tobytes(), res.scores.cpu().numpy().tobytes(), res.counts.cpu().numpy().tobytes()


def test_bm25_two_phase_equals_ordered_kernel_and_oracle():
    # 140k documents = 18 ranges of 8192: three range chunks (4, 4, 10) with two bound updates in between
    corpus = synth.make_sparse_corpus(140_000, 4000, 4242, mean_len=30, min_len=0, max_len=120)
    stats = Bm25Stats.from_tokens(corpus.tokens, corpus.doc_ptr, corpus.vocab, bm25_type=0)
    groups = synth.make_groups(corpus.n_docs, 5, 9)
    a = Bm25Index(stats, device=DEV, doc_group=groups, packed=True)
    b = Bm25Index(stats, device=DEV, doc_group=groups, packed=False)
    assert a.post_pk is not None and b.post_pk is None
    o = obm.OkapiCSR(corpus.doc_lists(), corpus.vocab)
    qs = synth.make_queries(corpus, 200, 4243)
    lists = [[int(t) for t in terms] for terms in qs.term_lists()]
    present = np.nonzero(o.df)[0]
    rng = np.random.default_rng(5)
    lists += [[int(t) for t in rng.choice(present, 40)],          # > kBmMaxT tokens: chunked accumulation
              [int(t) for t in rng.choice(present, 100)],         # > 64 tokens: rescoring reads tokens from global
              [int(present[0])] * 7 + [int(present[1])],          # duplicated tokens
              [], [-1, corpus.vocab + 3]]
    ptr = torch.tensor(np.cumsum([0] + [len(l) for l in lists]), dtype=torch.int32)
    terms = torch.tensor([t for l in lists for t in l], dtype=torch.int32)
    rows = [o.get_scores(l) for l in lists]
    _lib.lib().ezr_profile_enable(1)
    for k in (1, 10, 32):
        _lib.lib().ezr_profile_reset()
        ra = batched.bm25_topk(a, ptr, terms, k, id_base=1000)
        torch.cuda.synchronize()
        assert _lib.profile_read("bm25_cand")[1] == 1 and _lib.profile_read("bm25_rescore")[1] == 1
        rb = batched.bm25_topk(b, ptr, terms, k, id_base=1000)
        assert _topk_bytes(ra) == _topk_bytes(rb)
        _check_bm25_topk(ra, rows, k, id_base=1000)
        # the same with the (default-off) skipping of non-essential terms: fewer postings read, same result
        _lib.check(_lib.lib().ezr_bm25_set_skipping(1))
        try:
            rc = batched.bm25_topk(a, ptr, terms, k, id_base=1000)
        finally:
            _lib.check(_lib.lib().ezr_bm25_set_skipping(0))
        assert _topk_bytes(rc) == _topk_bytes(ra)
        # the launch schedule of the ranges (first launch of 1 / 8 / 18 ranges instead of 4) never changes the result
        for span in (1, 8, 18):
            _lib.check(_lib.lib().ezr_bm25_set_span(span))
            try:
                rd = batched.bm25_topk(a, ptr, terms, k, id_base=1000)
            finally:
                _lib.check(_lib.lib().ezr_bm25_set_span(4))
            assert _topk_bytes(rd) == _topk_bytes(ra), span
    _lib.lib().ezr_profile_enable(0)
    assert a.term_max is not None and int(a.term_max.max()) < (1 << 18)
    g = groups.numpy()
    want = np.array([i % 7 - 1 for i in range(len(lists))], dtype=np.int32)      # 5 = no such class
    allowed = [None if w == -1 else (g == w) for w in want]
    ra = batched.bm25_topk(a, ptr, terms, 10, q_group=torch.from_numpy(want))
    rb = batched.bm25_topk(b, ptr, terms, 10, q_group=torch.from_numpy(want))
    assert _topk_bytes(ra) == _topk_bytes(rb)
    _check_bm25_topk(ra, rows, 10, allowed=allowed)


def test_bm25_two_phase_hands_overflow_and_huge_queries_to_ordered_kernel():
    # half of the corpus is one repeated document (mass ties overflow the candidate list), the rest is random;
    # a batch mixes tie queries, ordinary queries and a query of > 4096 tokens (integer sums could wrap)
    base = synth.make_sparse_corpus(10_000, 500, 31, mean_len=20, min_len=1, max_len=60)
    rnd = base.doc_lists()
    same = np.array([490, 491, 492, 493, 490], dtype=np.int32)
    docs = [same if i % 2 else rnd[i // 2] for i in range(20_000)]
    tokens = torch.from_numpy(np.concatenate(docs)).to(torch.int32)
    ptr = torch.tensor(np.cumsum([0] + [len(d) for d in docs]), dtype=torch.int64)
    o = obm.OkapiCSR(docs, 500)
    stats = Bm25Stats.from_tokens(tokens, ptr, 500)
    a = Bm25Index(stats, device=DEV, packed=True)
    assert a.post_pk is not None
    present = np.nonzero(o.df)[0]
    rng = np.random.default_rng(6)
    lists = [[490, 491], [int(t) for t in rng.choice(present, 6)], [493], [int(t) for t in rng.choice(present, 9)],
             [int(t) for t in rng.choice(present, 4200)], [int(t) for t in rng.choice(present, 4)] + [492]]
    qp = torch.tensor(np.cumsum([0] + [len(l) for l in lists]), dtype=torch.int32)
    qt = torch.tensor([t for l in lists for t in l], dtype=torch.int32)
    rows = [o.get_scores(l) for l in lists]
    for k in (1, 10, 32):
        _check_bm25_topk(batched.bm25_topk(a, qp, qt, k), rows, k)



def test_bm25_negative_idf_index_uses_ordered_kernel():
    # Five terms in ~90% of the documents and one in ~30%: the mean idf is negative, so rank_bm25's epsilon floor
    # (eps * average_idf) is negative too and contributions can be negative.  Partial sums are then not monotone:
    # no packed postings, no crossing-based selection - the ordered kernel must still match the oracle bit for bit.
    rng = np.random.default_rng(17)
    docs = []
    for i in range(20_000):
        d = [t for t in range(5) if rng.random() < 0.9] * int(rng.integers(1, 3))
        if rng.random() < 0.3:
            d += [5] * int(rng.integers(1, 4))
        docs.append(np.array(d if d else [0], dtype=np.int32))
    tokens = torch.from_numpy(np.concatenate(docs)).to(torch.int32)
    ptr = torch.tensor(np.cumsum([0] + [len(d) for d in docs]), dtype=torch.int64)
    o = obm.OkapiCSR(docs, 6)
    assert (o.idf < 0).any() and (o.idf > 0).any()
    ix = Bm25Index(Bm25Stats.from_tokens(tokens, ptr, 6), device=DEV)
    assert not ix.monotone and ix.post_pk is None
    w = ix.post_w.cpu().numpy()
    for t in range(6):
        assert w[o.indptr[t]:o.indptr[t + 1]].tobytes() == o.contributions(t).tobytes()
    assert (w < 0).any() and (w > 0).any()
    lists = [[5], [5, 0], [0, 1, 2], [5, 5, 3], [4, 5, 1, 0, 2, 3]]
    qp = torch.tensor(np.cumsum([0] + [len(l) for l in lists]), dtype=torch.int32)
    qt = torch.tensor([t for l in lists for t in l], dtype=torch.int32)
    rows = [o.get_scores(l) for l in lists]
    assert any((r > 0).any() for r in rows) and any((r < 0).any() for r in rows)
    for k in (1, 10, 32):
        _check_bm25_topk(batched.bm25_topk(ix, qp, qt, k), rows, k)
    got = batched.bm25_scores(ix, qp, qt).cpu().numpy()
    for i, row in enumerate(rows):
        assert got[i].tobytes() == row.tobytes()


def test_bm25s_float32_bit_exact():
    corpus = synth.make_sparse_corpus(9000, 3000, 5, mean_len=60, min_len=1, max_len=200)
    qs = synth.make_queries(corpus, 40, 6)
    o = obm.Bm25sLucene(corpus.doc_lists(), corpus.vocab)
    ix = Bm25Index(Bm25Stats.from_tokens(corpus.tokens, corpus.doc_ptr, corpus.vocab, bm25_type=1), device=DEV)
    assert ix.post_w.dtype == torch.float32
    assert ix.post_w.cpu().numpy().tobytes() == o.post_w.tobytes()
    rows = [o.get_scores([int(t) for t in terms]) for terms in qs.term_lists()]
    got = batched.bm25_scores(ix, qs.term_ptr, qs.terms).cpu().numpy()
    for i, row in enumerate(rows):
        assert got[i].tobytes() == row.tobytes()
    _check_bm25_topk(batched.bm25_topk(ix, qs.term_ptr, qs.terms, 10), rows, 10)


def test_bm25_sharded_index_equals_global(c1):
    # doc-partitioned postings with GLOBAL idf/avgdl: merging shard lists reproduces the unsharded list
    q, k = c1["queries"], 10
    n = c1["stats"].n_docs
    cand_s, cand_i = [], []
    for lo, hi in ((0, 4096), (4096, 8192), (8192, n)):
        ix = Bm25Index(c1["stats"], device=DEV, doc_lo=lo, doc_hi=hi)
        r = batched.bm25_topk(ix, q.term_ptr, q.terms, k)
        cand_s.append(r.scores)
        cand_i.append(r.ids)
    merged = batched.merge_topk(torch.cat(cand_s, 1).contiguous(), torch.cat(cand_i, 1).contiguous(), k)
    _check_bm25_topk(merged, c1["rows"], k)


# --------------------------------------------------------- generic select ----
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("k", [1, 10, 33, 256, 1024])
def test_select_rows_matches_canonical_order(dtype, k):
    g = torch.Generator().manual_seed(k)
    s = (torch.rand(7, 50_000, generator=g, dtype=torch.float64) * 50).round() / 50 - 0.2    # many ties, some <= 0
    s = s.to(dtype)
    res = batched.select_rows(s.to(DEV), k, positive_only=True)
    _check_bm25_topk(res, [r.numpy() for r in s], k)
    res = batched.select_rows(s.to(DEV), k, positive_only=False)
    ids = res.ids.cpu().numpy()
    for q in range(s.shape[0]):
        ref = ort.canonical_order(s[q].numpy())[:k]
        assert np.array_equal(ids[q], ref)


def test_select_rows_single_long_row_uses_parts():
    s = torch.rand(1, 1_000_003, generator=torch.Generator().manual_seed(1), dtype=torch.float64)
    res = batched.select_rows(s.to(DEV), 100)
    assert np.array_equal(res.ids.cpu().numpy()[0], ort.canonical_order(s[0].numpy())[:100])


# ----------------------------------------------------------------- dense ----
def _dense_case(n, d, q, seed, integer=False):
    g = torch.Generator().manual_seed(seed)
    if integer:
        # small integers: every product and partial sum is exact in bf16/fp32 -> any summation order agrees
        c = torch.randint(-2, 3, (n, d), generator=g).float()
        qq = torch.randint(-2, 3, (q, d), generator=g).float()
    else:
        c = synth.make_dense_corpus(n, d, seed).float()
        qq = synth.make_dense_queries(c.to(torch.bfloat16), q, seed + 1).float()
    return c.to(torch.bfloat16), qq.to(torch.bfloat16)


def _check_dense(res, c, qv, k, allowed=None, exact=False, id_base=0):
    cf, qf = c.float().numpy(), qv.float().numpy()
    ref_i, ref_s = ort.dense_topk(cf, qf, k, allowed)
    ids, sc, cnt = res.ids.cpu().numpy(), res.scores.cpu().numpy(), res.counts.cpu().numpy()
    sims = qf @ cf.T
    for q in range(qf.shape[0]):
        n_ref = int((ref_i[q] >= 0).sum())
        assert cnt[q] == n_ref
        if exact:
            assert np.array_equal(ids[q, :n_ref], ref_i[q, :n_ref] + id_base), f"query {q}"
            assert np.array_equal(sc[q, :n_ref], ref_s[q, :n_ref])
            continue
        got = ids[q, :n_ref] - id_base
        # every returned score is the true cosine of the returned id, to 1e-3
        assert np.abs(sc[q, :n_ref] - sims[q, got]).max() <= COS_TOL
        # sorted descending, and the set is the oracle's up to scores closer than the tolerance
        assert (np.diff(sc[q, :n_ref]) <= 0).all()
        if n_ref:
            kth = ref_s[q, n_ref - 1]
            assert (sims[q, got] >= kth - COS_TOL).all()
            assert len(set(got.tolist())) == n_ref
        if allowed is not None:
            m = allowed[q] if allowed.ndim == 2 else allowed
            assert m[got].all()


# 1 = generic SIMT, 2 = wgmma with 128-query blocks (dim <= 768), 3 = wgmma with 64-query blocks, 4 = same with 128-row
# corpus tiles, 5 = 4 in cluster pairs (each CTA loads half of every corpus tile and TMA-multicasts it to both)
KERNEL_NAMES = {1: b"simt", 2: b"wgmma", 3: b"wgmma-q64", 4: b"wgmma-q64-n128", 5: b"wgmma-q64-n128-mc2"}


@pytest.mark.parametrize("kernel", [1, 2, 3, 4, 5])
@pytest.mark.parametrize("n,d,q,k", [(5000, 128, 130, 10), (777, 768, 3, 5), (64, 64, 1, 16), (20_000, 768, 257, 10),
                                     (100, 256, 5, 12)])
def test_dense_exact_integer_inputs(kernel, n, d, q, k):
    c, qv = _dense_case(n, d, q, 100 + n, integer=True)
    L = _lib.lib()
    _lib.check(L.ezr_dense_set_kernel(kernel))
    try:
        res = batched.dense_topk(DenseIndex(c, device=DEV), qv.to(DEV), k)
        assert L.ezr_dense_last_kernel() == KERNEL_NAMES[kernel]
    finally:
        L.ezr_dense_set_kernel(0)
    _check_dense(res, c, qv, k, exact=True)


def test_dense_wide_dims_cluster_pair_kernel():
    c, qv = _dense_case(70_000, 1024, 300, 270, integer=True)      # odd number of query blocks (5), 1024-d, several splits
    L = _lib.lib()
    _lib.check(L.ezr_dense_set_kernel(5))
    try:
        res = batched.dense_topk(DenseIndex(c, device=DEV), qv.to(DEV), 10)
        assert L.ezr_dense_last_kernel() == KERNEL_NAMES[5]
    finally:
        L.ezr_dense_set_kernel(0)
    _check_dense(res, c, qv, 10, exact=True)


@pytest.mark.parametrize("n,d,q,k", [(3000, 1024, 130, 10), (2500, 832, 5, 8), (70_000, 1024, 300, 10)])
def test_dense_wide_dims_use_hybrid_tmem_smem_queries(n, d, q, k):
    # BGE-large is 1024-d (BASELINE config 5): a 128-query block of that width does not fit shared memory beside the
    # corpus ring, so the automatic choice is the 64-query block with 128-row corpus tiles; the 64-row-tile form is
    # forced as well, and the 128-query form refuses the shape
    c, qv = _dense_case(n, d, q, 200 + n, integer=True)
    res = batched.dense_topk(DenseIndex(c, device=DEV), qv.to(DEV), k)
    assert _lib.lib().ezr_dense_last_kernel() == KERNEL_NAMES[4]
    _check_dense(res, c, qv, k, exact=True)
    L = _lib.lib()
    _lib.check(L.ezr_dense_set_kernel(3))
    try:
        res = batched.dense_topk(DenseIndex(c, device=DEV), qv.to(DEV), k)
        assert L.ezr_dense_last_kernel() == KERNEL_NAMES[3]
    finally:
        L.ezr_dense_set_kernel(0)
    _check_dense(res, c, qv, k, exact=True)
    _lib.check(L.ezr_dense_set_kernel(2))
    try:
        with pytest.raises(_lib.EzrError):
            batched.dense_topk(DenseIndex(c, device=DEV), qv.to(DEV), k)      # 128-query blocks stop at 768
    finally:
        L.ezr_dense_set_kernel(0)


@pytest.mark.parametrize("kernel", [1, 2, 3, 4, 5])
def test_dense_unit_vectors_within_tolerance(kernel):
    c, qv = _dense_case(30_000, 768, 200, 7)
    L = _lib.lib()
    _lib.check(L.ezr_dense_set_kernel(kernel))
    try:
        res = batched.dense_topk(DenseIndex(c, device=DEV), qv.to(DEV), 10)
    finally:
        L.ezr_dense_set_kernel(0)
    _check_dense(res, c, qv, 10)


@pytest.mark.parametrize("kernel", [1, 2, 3, 4, 5])
def test_dense_dir_filter_and_id_base(kernel):
    c, qv = _dense_case(9000, 256, 70, 11, integer=True)
    groups = synth.make_groups(9000, 4, 12)
    want = torch.tensor([i % 6 - 1 for i in range(70)], dtype=torch.int32)
    want[want == 4] = -2
    g = groups.numpy()
    allowed = np.stack([np.ones(9000, bool) if w == -1 else (g == w) for w in want.tolist()])
    L = _lib.lib()
    _lib.check(L.ezr_dense_set_kernel(kernel))
    try:
        res = batched.dense_topk(DenseIndex(c, device=DEV, doc_group=groups, row_lo=1000), qv.to(DEV), 10, q_group=want)
    finally:
        L.ezr_dense_set_kernel(0)
    _check_dense(res, c, qv, 10, allowed=allowed, exact=True, id_base=1000)


def test_dense_large_k_goes_through_generic_kernel():
    c, qv = _dense_case(4000, 192, 4, 13, integer=True)       # dim 192 % 64 == 0 but k = 288 > 16
    res = batched.dense_topk(DenseIndex(c, device=DEV), qv.to(DEV), 288)
    assert _lib.lib().ezr_dense_last_kernel() == b"simt"
    _check_dense(res, c, qv, 288, exact=True)
    c, qv = _dense_case(300, 100, 4, 14, integer=True)        # odd dim
    res = batched.dense_topk(DenseIndex(c, device=DEV), qv.to(DEV), 10)
    _check_dense(res, c, qv, 10, exact=True)


def test_dense_fewer_rows_than_k():
    c, qv = _dense_case(7, 64, 3, 15, integer=True)
    res = batched.dense_topk(DenseIndex(c, device=DEV), qv.to(DEV), 10)
    _check_dense(res, c, qv, 10, exact=True)
    assert (res.counts.cpu().numpy() == 7).all()


# ---------------------------------------------------------------- fusion ----
def _random_lists(rng, n_docs, nq, width, dup_frac=0.2):
    canon = synth.make_duplicates(n_docs, dup_frac, int(rng.integers(1 << 30))).numpy()
    ids_a = np.full((nq, width), -1, np.int32)
    ids_b = np.full((nq, width), -1, np.int32)
    cnt_a = rng.integers(0, width + 1, nq).astype(np.int32)
    cnt_b = rng.integers(0, width + 1, nq).astype(np.int32)
    for q in range(nq):
        ids_a[q, :cnt_a[q]] = rng.permutation(n_docs)[:cnt_a[q]]
        ids_b[q, :cnt_b[q]] = rng.permutation(n_docs)[:cnt_b[q]]
    return canon, ids_a, cnt_a, ids_b, cnt_b


@pytest.mark.parametrize("width,k_out", [(10, 10), (10, 4), (37, 256), (288, 256), (1024, 6)])
def test_rrf_bit_exact(width, k_out):
    rng = np.random.default_rng(width)
    n_docs, nq = max(60, width * 2), 50
    canon, ids_a, cnt_a, ids_b, cnt_b = _random_lists(rng, n_docs, nq, width)
    t = lambda a: torch.from_numpy(a).to(DEV)
    res = batched.rrf_fuse(t(ids_a), t(cnt_a), t(ids_b), t(cnt_b), k_out, K=60, canon=t(canon.astype(np.int32)))
    ids, sc, cnt = res.ids.cpu().numpy(), res.scores.cpu().numpy(), res.counts.cpu().numpy()
    for q in range(nq):
        ref_i, ref_s = ort.rrf_ids([ids_a[q, :cnt_a[q]], ids_b[q, :cnt_b[q]]], canon, K=60, topk=k_out)
        assert cnt[q] == ref_i.size
        assert np.array_equal(ids[q, :cnt[q]], ref_i)
        assert sc[q, :cnt[q]].tobytes() == ref_s.tobytes()
        assert (ids[q, cnt[q]:] == -1).all()


@pytest.mark.parametrize("width,k_out", [(10, 10), (192, 256), (50, 7)])
def test_simple_fusion_bit_exact(width, k_out):
    rng = np.random.default_rng(1000 + width)
    n_docs, nq = max(60, width * 2), 40
    canon, ids_a, cnt_a, ids_b, cnt_b = _random_lists(rng, n_docs, nq, width)
    sa = np.round(rng.random((nq, width)) * 20, 0) / 4           # coarse -> ties between the two routes
    sb = np.round(rng.random((nq, width)) * 20, 0) / 4
    t = lambda a: torch.from_numpy(a).to(DEV)
    res = batched.fusion_simple(t(ids_a), t(sa), t(cnt_a), t(ids_b), t(sb), t(cnt_b), k_out,
                                canon=t(canon.astype(np.int32)))
    ids, sc, cnt = res.ids.cpu().numpy(), res.scores.cpu().numpy(), res.counts.cpu().numpy()
    for q in range(nq):
        ref_i, ref_s = ort.fusion_ids([ids_a[q, :cnt_a[q]], ids_b[q, :cnt_b[q]]],
                                      [sa[q, :cnt_a[q]], sb[q, :cnt_b[q]]], canon, topk=k_out)
        assert cnt[q] == ref_i.size
        assert np.array_equal(ids[q, :cnt[q]], ref_i)
        assert sc[q, :cnt[q]].tobytes() == ref_s.tobytes()


@pytest.mark.parametrize("n_lists,width,k_out", [(1, 12, 10), (3, 10, 10), (5, 40, 64), (8, 256, 256)])
def test_fusion_over_any_number_of_lists_bit_exact(n_lists, width, k_out):
    """retrievers.py:243,261 loop over a list of lists: 1, 3, 5 and 8 lists against the oracle's own loops."""
    rng = np.random.default_rng(77 + n_lists)
    n_docs, nq = max(60, width * 2), 30
    canon = np.arange(n_docs)
    dup = rng.random(n_docs) < 0.1
    canon[dup] = rng.integers(0, np.maximum(np.arange(n_docs)[dup], 1))
    canon = canon[canon]                                            # one level of chains is enough for a key map
    ids = [np.full((nq, width), -1, np.int32) for _ in range(n_lists)]
    cnt = [rng.integers(0, width + 1, nq).astype(np.int32) for _ in range(n_lists)]
    sc = [np.round(rng.random((nq, width)) * 20, 0) / 4 for _ in range(n_lists)]
    for l in range(n_lists):
        for q in range(nq):
            ids[l][q, :cnt[l][q]] = rng.choice(n_docs, cnt[l][q], replace=False)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
    cn = t(canon.astype(np.int32))
    for rrf in (True, False):
        res = batched.fuse_lists([t(a) for a in ids], [t(c) for c in cnt], k_out, rrf=rrf, K=60,
                                 scores=[t(x) for x in sc], canon=cn)
        g_ids, g_sc, g_cnt = res.ids.cpu().numpy(), res.scores.cpu().numpy(), res.counts.cpu().numpy()
        for q in range(nq):
            lists = [ids[l][q, :cnt[l][q]] for l in range(n_lists)]
            if rrf:
                ref_i, ref_s = ort.rrf_ids(lists, canon, K=60, topk=k_out)
            else:
                ref_i, ref_s = ort.fusion_ids(lists, [sc[l][q, :cnt[l][q]] for l in range(n_lists)], canon, topk=k_out)
            assert g_cnt[q] == ref_i.size
            assert np.array_equal(g_ids[q, :g_cnt[q]], ref_i)
            assert g_sc[q, :g_cnt[q]].tobytes() == ref_s.tobytes()


# ------------------------------------------------------- index build on the GPU ----
def _assert_counts_equal(st, tokens, ptr, vocab):
    from _host_counts import host_counts
    c = host_counts(tokens, ptr, vocab)
    assert np.array_equal(st.df.cpu().numpy(), c["df"])
    assert np.array_equal(st.indptr.cpu().numpy(), c["indptr"])
    assert np.array_equal(st.post_doc.cpu().numpy(), c["post_doc"])          # term-major, documents ascending
    assert np.array_equal(st.post_tf.cpu().numpy(), c["post_tf"])
    assert np.array_equal(st.doc_len.cpu().numpy(), c["doc_len"])


@pytest.mark.parametrize("n,vocab,mean_len,max_len", [(3000, 700, 40, 200), (20000, 5000, 300, 800), (9000, 64, 12, 40),
                                                       (1, 10, 5, 9)])
def test_index_build_kernels_match_the_host_counting(n, vocab, mean_len, max_len):
    """csrc/bm25_build.cu (per-document sort, block-ordered placement) against the numpy restatement of
    retrievers.py:98-118: df, indptr, postings in (term, document) order, tf, document lengths -- and the idf values
    that depend on the first-seen term order (sequential float64 sum)."""
    from _host_counts import stats_from_host_counts
    corpus = synth.make_sparse_corpus(n, vocab, 900 + n, mean_len=mean_len, min_len=0, max_len=max_len)
    st = Bm25Stats.from_tokens(corpus.tokens, corpus.doc_ptr, vocab)
    assert st.post_doc.is_cuda
    _assert_counts_equal(st, corpus.tokens, corpus.doc_ptr, vocab)
    ref = stats_from_host_counts(corpus.tokens, corpus.doc_ptr, vocab)
    assert st.avgdl == ref.avgdl and st.average_idf == ref.average_idf and st.idf.tobytes() == ref.idf.tobytes()


def test_index_build_long_documents_empty_documents_and_bad_tokens():
    g = torch.Generator().manual_seed(3)
    lens = [0, 5, 9000, 0, 8192, 8193, 20000, 1, 300, 0]           # around the shared-memory sort capacity (8192)
    vocab = 1500
    tokens = torch.randint(0, vocab, (sum(lens),), generator=g, dtype=torch.int32)
    ptr = torch.tensor(np.cumsum([0] + lens), dtype=torch.int64)
    st = Bm25Stats.from_tokens(tokens, ptr, vocab)
    _assert_counts_equal(st, tokens, ptr, vocab)
    bad = tokens.clone()
    bad[9100] = vocab                                                # inside document 4 (tokens 9005..17196)
    with pytest.raises(ValueError, match="document 4"):
        Bm25Stats.from_tokens(bad, ptr, vocab)


def test_index_shard_slice_kernels_equal_a_filter_of_the_global_postings(c1):
    st = c1["stats"]
    n = st.n_docs
    for lo, hi in ((0, n), (0, n // 3), (n // 3, 2 * n // 3 + 5), (n - 7, n), (5, 5)):
        ix = Bm25Index(st, device=DEV, doc_lo=lo, doc_hi=hi, packed=False) if hi > lo else None
        pd, tf, ind = st.post_doc.cpu().numpy(), st.post_tf.cpu().numpy(), st.indptr.cpu().numpy()
        term_of = np.repeat(np.arange(st.vocab), np.diff(ind))
        keep = (pd >= lo) & (pd < hi)
        if ix is None:
            continue
        assert np.array_equal(ix.post_doc.cpu().numpy(), pd[keep] - lo)
        want_ptr = np.zeros(st.vocab + 1, np.int64)
        np.cumsum(np.bincount(term_of[keep], minlength=st.vocab), out=want_ptr[1:])
        assert np.array_equal(ix.indptr.cpu().numpy(), want_ptr)


# ------------------------------------------------------- hybrid, one GPU ----
def test_hybrid_dense_bm25_rrf_matches_oracle(c1):
    n, dim, k = c1["stats"].n_docs, 256, 10
    c, qv = _dense_case(n, dim, c1["queries"].n, 31, integer=True)
    canon = synth.make_duplicates(n, 0.05, 32)
    ranker = batched.CoarseRanker(DenseIndex(c, device=DEV), c1["index"], canon=canon)
    q = c1["queries"]
    fused, sparse, dense = ranker.hybrid(qv.to(DEV), q.term_ptr.to(DEV), q.terms.to(DEV), k, k, k)
    torch.cuda.synchronize()
    _check_bm25_topk(sparse, c1["rows"], k)
    _check_dense(dense, c, qv, k, exact=True)
    d_ref, _ = ort.dense_topk(c.float().numpy(), qv.float().numpy(), k)
    f_ids, f_sc, f_cnt = fused.ids.cpu().numpy(), fused.scores.cpu().numpy(), fused.counts.cpu().numpy()
    for i, row in enumerate(c1["rows"]):
        s_ref, _ = ort.bm25_topk_ids(row, k)
        ref_i, ref_s = ort.rrf_ids([s_ref, d_ref[i]], canon.numpy(), K=60, topk=k)
        assert np.array_equal(f_ids[i, :f_cnt[i]], ref_i)
        assert f_sc[i, :f_cnt[i]].tobytes() == ref_s.tobytes()


@pytest.mark.parametrize("serial", [False, True])
def test_submitted_batches_equal_joined_batches_and_host_pipeline(c1, serial):
    # batch pipelining: six different batches submitted back to back (two result slots, reused three times) must give
    # exactly what hybrid() gives for each batch on its own; then the same through HostPipeline (pinned host buffers)
    n, dim, k = c1["stats"].n_docs, 256, 10
    q = c1["queries"]
    nq = q.n
    ranker = batched.CoarseRanker(DenseIndex(_dense_case(n, dim, 1, 77, integer=True)[0], device=DEV), c1["index"],
                                  overlap=True, serial_routes=serial)
    ptr, terms = q.term_ptr.to(DEV), q.terms.to(DEV)
    qvs = [_dense_case(8, dim, nq, 100 + i, integer=True)[1].to(DEV) for i in range(6)]
    # a different BM25 batch per step too: rotate the queries (term lists of query j move to position j + i)
    tp = q.term_ptr.numpy().astype(np.int64)
    tt = q.terms.numpy()
    bm = []
    for i in range(6):
        order = np.roll(np.arange(nq), i)
        lens = (tp[1:] - tp[:-1])[order]
        nptr = np.zeros(nq + 1, np.int32)
        np.cumsum(lens, out=nptr[1:])
        nterms = np.concatenate([tt[tp[j]:tp[j + 1]] for j in order]) if nq else tt
        bm.append((torch.from_numpy(nptr), torch.from_numpy(nterms.astype(np.int32))))
    want = []
    for i in range(6):
        f, _, _ = ranker.hybrid(qvs[i], bm[i][0].to(DEV), bm[i][1].to(DEV), k, k, k)
        want.append((f.ids.clone(), f.scores.clone(), f.counts.clone()))
    torch.cuda.synchronize()
    got = []
    d_bm = [(a.to(DEV), b.to(DEV)) for a, b in bm]
    torch.cuda.synchronize()
    side = torch.cuda.Stream()                                # the consumer: the caller's stream never waits for a join
    for i in range(6):
        t = ranker.submit(qvs[i], d_bm[i][0], d_bm[i][1], k=k, k_out=k)
        with torch.cuda.stream(side):
            t.wait(side)
            got.append((t.fused.ids.clone(), t.fused.scores.clone(), t.fused.counts.clone()))
            t.release(side)
    ranker.join()
    torch.cuda.synchronize()
    for i in range(6):
        for a, b in zip(got[i], want[i]):
            assert torch.equal(a, b), f"batch {i}"
    assert not torch.equal(want[0][0], want[1][0])          # the batches really differ
    # host pipeline: pinned inputs and outputs, one output buffer per step
    max_terms = max(int(b.numel()) for _, b in bm)
    pipe = batched.HostPipeline(ranker, nq, dim, max_terms, k, k)
    assert pipe.pipelined
    outs = []
    for i in range(6):
        h_ids = torch.empty(nq, k, dtype=torch.int32).pin_memory()
        h_sc = torch.empty(nq, k, dtype=torch.float64).pin_memory()
        pipe.step(qvs[i].cpu().pin_memory(), bm[i][0].pin_memory(), bm[i][1].pin_memory(), h_ids, h_sc)
        outs.append((h_ids, h_sc))
    pipe.drain()
    torch.cuda.synchronize()
    for i in range(6):
        cnt = want[i][2].cpu().numpy()
        wi, ws = want[i][0].cpu().numpy(), want[i][1].cpu().numpy()
        for j in range(nq):
            assert np.array_equal(outs[i][0].numpy()[j, :cnt[j]], wi[j, :cnt[j]])
            assert outs[i][1].numpy()[j, :cnt[j]].tobytes() == ws[j, :cnt[j]].tobytes()


# ----------------------------------------------------- widening (SURVEY 8(f)) ----
def test_index_save_load_roundtrip(c1, tmp_path):
    ix = c1["index"]
    ix.save(str(tmp_path / "bm25"))
    ix2 = Bm25Index.load(str(tmp_path / "bm25"), device=DEV)
    q = c1["queries"]
    a = batched.bm25_topk(ix, q.term_ptr, q.terms, 10)
    b = batched.bm25_topk(ix2, q.term_ptr, q.terms, 10)
    assert torch.equal(a.ids, b.ids) and torch.equal(a.scores, b.scores)
    c, qv = _dense_case(3000, 128, 9, 3, integer=True)
    d = DenseIndex(c, device=DEV, row_lo=5)
    d.save(str(tmp_path / "dense"))
    d2 = DenseIndex.load(str(tmp_path / "dense"), device=DEV)
    x, y = batched.dense_topk(d, qv.to(DEV), 10), batched.dense_topk(d2, qv.to(DEV), 10)
    assert torch.equal(x.ids, y.ids) and torch.equal(x.scores, y.scores)


def test_dual_sparse_route_fusion(c1):
    # pipeline.py:357-365: chunk BM25 (k=192) + path BM25 (k=6) -> HybridRetriever.fusion(topk=256)
    corpus = c1["corpus"]
    n = corpus.n_docs
    # a second, much shorter "knowledge path" text per node: its first 4 tokens
    docs = corpus.doc_lists()
    p_tokens = torch.from_numpy(np.concatenate([d[:4] for d in docs])).to(torch.int32)
    p_ptr = torch.tensor(np.cumsum([0] + [min(4, len(d)) for d in docs]), dtype=torch.int64)
    p_or = obm.OkapiCSR([d[:4] for d in docs], corpus.vocab)
    p_ix = Bm25Index(Bm25Stats.from_tokens(p_tokens, p_ptr, corpus.vocab), device=DEV)
    canon = synth.make_duplicates(n, 0.02, 3)
    q = c1["queries"]
    nq = 20
    qp, qt = q.term_ptr[:nq + 1], q.terms
    res = batched.dual_sparse_fusion(c1["index"], p_ix, qp, qt, qp, qt, 192, 6, 256, canon=canon)
    ids, sc, cnt = res.ids.cpu().numpy(), res.scores.cpu().numpy(), res.counts.cpu().numpy()
    for i, terms in enumerate(q.term_lists()[:nq]):
        a_i, a_s = ort.bm25_topk_ids(c1["rows"][i], 192)
        b_i, b_s = ort.bm25_topk_ids(p_or.get_scores([int(t) for t in terms]), 6)
        ref_i, ref_s = ort.fusion_ids([a_i, b_i], [a_s, b_s], canon.numpy(), topk=256)
        assert cnt[i] == ref_i.size
        assert np.array_equal(ids[i, :cnt[i]], ref_i)
        assert sc[i, :cnt[i]].tobytes() == ref_s.tobytes()
