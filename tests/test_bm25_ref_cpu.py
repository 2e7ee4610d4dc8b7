"""CPU: tests/_bm25_ref.py (the torch restatement of BM25 the benchmark-scale GPU tests compare against) equals the
numpy host counting (tests/_host_counts.py) and the oracle classes (oracle/bm25.py) bit for bit.

Corpora of up to 20k documents with empty documents, repeated tokens inside documents and queries, and a corpus whose
mean idf is negative (rank_bm25's epsilon floor then makes some contributions negative)."""
import numpy as np
import pytest
import torch

from _bm25_ref import FIRST_ABSENT, bm25s_row, bm25s_weights, canonical_topk, counts, okapi_row, okapi_weights
from _host_counts import host_counts
from easyrag_b200 import synth
from easyrag_b200.index import Bm25Stats
from oracle import bm25 as obm
from oracle import retrieve as ort


def _corpus(kind):
    if kind == "zipf":          # empty documents (min_len 0), Zipf tokens repeat inside documents
        return synth.make_sparse_corpus(20_000, 5000, 11, mean_len=40, min_len=0, max_len=200)
    if kind == "short":         # a small vocabulary: long posting lists, high tf
        return synth.make_sparse_corpus(6000, 64, 12, mean_len=12, min_len=0, max_len=40)
    # five terms in ~90% of the documents and one in ~30%: the mean idf is negative
    # (as test_bm25_negative_idf_index_uses_ordered_kernel in tests/test_gpu_retrieval.py)
    rng = np.random.default_rng(17)
    docs = []
    for _ in range(20_000):
        d = [t for t in range(5) if rng.random() < 0.9] * int(rng.integers(1, 3))
        if rng.random() < 0.3:
            d += [5] * int(rng.integers(1, 4))
        docs.append(np.array(d if d else [0], dtype=np.int32))
    return synth.SparseCorpus(tokens=torch.from_numpy(np.concatenate(docs)),
                              doc_ptr=torch.tensor(np.cumsum([0] + [len(d) for d in docs]), dtype=torch.int64), vocab=6)


KINDS = ["zipf", "short", "negidf"]


@pytest.fixture(scope="module", params=KINDS)
def case(request):
    c = _corpus(request.param)
    n, vocab = c.n_docs, c.vocab
    r = counts(c.tokens, c.doc_ptr, vocab)
    indptr = torch.zeros(vocab + 1, dtype=torch.int64)
    torch.cumsum(r["df"], 0, out=indptr[1:])
    total = int(c.doc_ptr[-1])
    first = r["first_pos"].numpy().astype(np.uint64)
    st = Bm25Stats.from_counts(n, vocab, total, r["doc_len"], r["df"], indptr, r["doc"], r["tf"], first)
    st1 = Bm25Stats.from_counts(n, vocab, total, r["doc_len"], r["df"], indptr, r["doc"], r["tf"], first, bm25_type=1)
    dl = r["doc_len"][r["doc"]]
    w = okapi_weights(r["tf"], dl, torch.from_numpy(st.idf)[r["term"]], st.avgdl)
    w32 = bm25s_weights(r["tf"], dl, torch.from_numpy(st1.idf.astype(np.float32))[r["term"]], st1.avgdl)
    qs = synth.make_queries(c, 40, 13, min_terms=1, max_terms=12)
    lists = [[int(t) for t in q] for q in qs.term_lists()]
    lists += [[], [-1, vocab + 3], [lists[0][0]] * 5 + [lists[1][0]], list(range(min(vocab, 40)))]
    return dict(kind=request.param, corpus=c, r=r, indptr=indptr.numpy(), st=st, st1=st1, w=w, w32=w32, lists=lists)


def test_counts_equal_host_counting(case):
    c, r = case["corpus"], case["r"]
    h = host_counts(c.tokens, c.doc_ptr, c.vocab)
    assert np.array_equal(r["df"].numpy(), h["df"])
    assert np.array_equal(case["indptr"], h["indptr"])
    assert np.array_equal(r["doc"].numpy(), h["post_doc"]) and np.array_equal(r["tf"].numpy(), h["post_tf"])
    assert np.array_equal(r["doc_len"].numpy(), h["doc_len"])
    present = h["df"] > 0
    fp = r["first_pos"].numpy()
    assert np.array_equal(fp[present].astype(np.uint64), h["first_pos"][present]) and (fp[~present] == FIRST_ABSENT).all()


def test_counts_in_blocks_concatenate_to_the_whole(case):
    # document blocks (as the GPU file walks the 1M-document corpus) merge back into the term-major postings
    c, r = case["corpus"], case["r"]
    n = c.n_docs
    cuts = sorted({min(x, n) for x in (0, 1, 4096, 8191, 8192, n // 2 + 3, n)})
    parts = [counts(c.tokens, c.doc_ptr, c.vocab, lo, hi) for lo, hi in zip(cuts[:-1], cuts[1:])]
    key = torch.cat([p["key"] for p in parts])
    order = torch.argsort(key)
    assert torch.equal(key[order], r["key"]) and torch.equal(torch.cat([p["tf"] for p in parts])[order], r["tf"])
    assert torch.equal(sum(p["df"] for p in parts), r["df"])
    first = torch.stack([p["first_pos"] for p in parts]).min(0).values
    assert torch.equal(first, r["first_pos"])


def test_okapi_weights_and_rows_equal_okapi_csr(case):
    c = case["corpus"]
    o = obm.OkapiCSR(c.doc_lists(), c.vocab)
    st = case["st"]
    assert st.avgdl == o.avgdl and st.idf.tobytes() == o.idf.tobytes()
    if case["kind"] == "negidf":
        assert (o.idf < 0).any() and (case["w"] < 0).any()
    assert case["w"].numpy().tobytes() == np.concatenate([o.contributions(t) for t in range(c.vocab)]).tobytes()
    for q in case["lists"]:
        got = okapi_row(q, case["indptr"], case["r"]["doc"], case["w"], st.idf, c.n_docs)
        assert got.numpy().tobytes() == o.get_scores(q).tobytes(), q


def test_okapi_row_equals_the_literal_loop_on_a_subset(case):
    c = case["corpus"]
    m = 1500
    docs = c.doc_lists()[:m]
    lit = obm.OkapiLiteral([list(map(int, d)) for d in docs])
    ptr = c.doc_ptr[:m + 1].clone()
    tok = c.tokens[:int(ptr[-1])]
    r = counts(tok, ptr, c.vocab)
    indptr = np.concatenate([[0], np.cumsum(r["df"].numpy())])
    st = Bm25Stats.from_counts(m, c.vocab, int(ptr[-1]), r["doc_len"], r["df"], torch.from_numpy(indptr), r["doc"],
                               r["tf"], r["first_pos"].numpy().astype(np.uint64))
    w = okapi_weights(r["tf"], r["doc_len"][r["doc"]], torch.from_numpy(st.idf)[r["term"]], st.avgdl)
    for q in case["lists"][:6] + case["lists"][-4:]:
        want = lit.get_scores([t for t in q if 0 <= t < c.vocab])       # the literal loop keys a dict: no -1 / OOV
        assert okapi_row(q, indptr, r["doc"], w, st.idf, m).numpy().tobytes() == want.tobytes(), q


def test_bm25s_weights_and_rows_equal_bm25s_lucene(case):
    c = case["corpus"]
    o = obm.Bm25sLucene(c.doc_lists(), c.vocab)
    assert case["w32"].dtype == torch.float32 and case["w32"].numpy().tobytes() == o.post_w.tobytes()
    df = case["r"]["df"].numpy()
    for q in case["lists"]:
        got = bm25s_row(q, case["indptr"], case["r"]["doc"], case["w32"], df, c.n_docs)
        assert got.dtype == torch.float32 and got.numpy().tobytes() == o.get_scores(q).tobytes(), q


# ---------------------------------------------------------------------------------------------- canonical_topk
def _tie_rows(dtype):
    g = torch.Generator().manual_seed(4)
    s = (torch.rand(9, 30_000, generator=g, dtype=torch.float64) * 40).round() / 40 - 0.1     # ~40 distinct values
    s[3] = 0.5                                                     # one value everywhere: the id decides
    s[4] = 0.0                                                     # nothing positive
    s[5, :] = -1.0
    s[5, [7, 29_999, 100]] = 2.0                                   # fewer positive scores than k
    return s.to(dtype)


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
@pytest.mark.parametrize("k", [1, 10, 32, 33, 1024])
def test_canonical_topk_equals_the_oracle_order(dtype, k):
    s = _tie_rows(dtype)
    g = torch.Generator().manual_seed(5)
    groups = torch.randint(0, 4, (s.shape[1],), generator=g)
    want = torch.tensor([-1, 0, 1, 2, 3, -1, 0, 7, -1])            # 7: no such class
    allowed = (want[:, None] == -1) | (groups[None, :] == want[:, None])
    base = 2 ** 31 - 1 - s.shape[1]
    for al in (None, allowed):
        ids, sc, cnt = canonical_topk(s, k, al, id_base=base)
        for q in range(s.shape[0]):
            ref_i, ref_s = ort.bm25_topk_ids(s[q].numpy(), k, None if al is None else al[q].numpy())
            assert int(cnt[q]) == ref_i.size
            assert np.array_equal(ids[q, :ref_i.size].numpy(), ref_i + base) and (ids[q, ref_i.size:] == -1).all()
            assert sc[q, :ref_i.size].numpy().tobytes() == ref_s.tobytes()
    # the all-equal row: the highest ids first
    ids, _, _ = canonical_topk(s, k)
    assert ids[3].tolist() == list(range(s.shape[1] - 1, s.shape[1] - 1 - k, -1))


def test_canonical_topk_with_fewer_columns_than_k():
    s = torch.tensor([[0.5, 0.5, 0.25]], dtype=torch.float64)
    ids, sc, cnt = canonical_topk(s, 5)
    assert ids.tolist() == [[1, 0, 2, -1, -1]] and int(cnt[0]) == 3 and sc[0, :3].tolist() == [0.5, 0.5, 0.25]
