"""CPU: the reference helpers tests/test_gpu_configs4.py adds for a 4M-row corpus, pinned to the plain definitions.

* ``_bm25_ref.postings_of_docs`` (a document range picked out of the whole term-major postings) against
  ``_bm25_ref.counts`` of the same documents and against tests/_host_counts.py;
* ``_topk_ref.fp64_top`` / ``canonical_topk`` past 2^20 rows (a wider id field in the int64 keys) against a numpy
  lexsort, with ties between ids above and below 2^20;
* ``test_gpu_dense_s8.rescore_all`` over row chunks against the unchunked definition, byte for byte.
"""
import numpy as np
import pytest
import torch

from _bm25_ref import counts, postings_of_docs
from _host_counts import host_counts
from _topk_ref import ID_BITS, canonical_keys, canonical_topk, fp64_top, id_bits_for
from easyrag_b200 import synth
from test_gpu_dense_s8 import rescore_all


def test_postings_of_docs_equal_counts_of_the_same_documents():
    n, vocab = 3000, 700
    c = synth.make_sparse_corpus(n, vocab, 5, mean_len=40, min_len=1, max_len=120)
    h = host_counts(c.tokens, c.doc_ptr, vocab)
    indptr = torch.from_numpy(h["indptr"])
    post_doc = torch.from_numpy(h["post_doc"])
    post_tf = torch.from_numpy(h["post_tf"])
    for lo, hi in ((0, n), (0, 1), (17, 1000), (1000, 2048), (2999, 3000), (1234, 1234)):
        got = postings_of_docs(indptr, post_doc, lo, hi)
        want = counts(c.tokens, c.doc_ptr, vocab, lo, hi)
        assert torch.equal(got["term"], want["term"]) and torch.equal(got["doc"], want["doc"]), (lo, hi)
        assert torch.equal(post_tf[got["pos"]].long(), want["tf"]), (lo, hi)
    # the slices of a partition concatenate, term by term, to the whole index
    parts = [postings_of_docs(indptr, post_doc, lo, hi) for lo, hi in ((0, 777), (777, 2000), (2000, n))]
    key = torch.cat([p["term"] * n + p["doc"] for p in parts]).sort().values
    whole = torch.repeat_interleave(torch.arange(vocab), torch.from_numpy(h["df"])) * n + post_doc.long()
    assert torch.equal(key, whole)


def _lexsort_top(s, k):
    """numpy: (score desc, id desc) top-k of integer score rows."""
    ids = np.arange(s.shape[1])
    order = np.lexsort((-ids[None, :].repeat(s.shape[0], 0), -s), axis=1)[:, :k]
    return order, np.take_along_axis(s, order, 1)


def test_fp64_top_past_2_20_rows():
    n, d = (1 << 20) + 4099, 16
    assert id_bits_for(n) == 21 and id_bits_for(1 << 20) == ID_BITS and id_bits_for(4_000_000) == 22
    g = torch.Generator().manual_seed(3)
    c = torch.randint(-2, 3, (n, d), generator=g).to(torch.bfloat16)
    top = torch.full((d,), 2.0, dtype=torch.bfloat16)
    copies = torch.tensor([5, (1 << 20) - 1, 1 << 20, (1 << 20) + 1, n - 1])      # ties on both sides of 2^20
    c[copies] = top
    q = torch.randint(-2, 3, (6, d), generator=g).to(torch.bfloat16)
    q[0] = top
    ids, sc, valid = fp64_top(q, c, 9, integer=True, c_chunk=300_000)
    s = (q.double() @ c.double().T).numpy()
    w_ids, w_sc = _lexsort_top(s, 9)
    assert valid.all() and np.array_equal(ids.numpy(), w_ids) and np.array_equal(sc.numpy(), w_sc)
    assert ids[0, :5].tolist() == sorted(copies.tolist(), reverse=True)
    ci, cs = canonical_topk(torch.from_numpy(s), 9)
    assert np.array_equal(ci.numpy(), w_ids) and np.array_equal(cs.numpy(), w_sc)
    # the 20-bit field cannot hold these ids
    with pytest.raises(AssertionError, match="20-bit"):
        canonical_keys(torch.from_numpy(s[:, -10:]), torch.arange(n - 10, n))


def test_rescore_all_over_row_chunks_is_the_same_bytes():
    c = synth.make_dense_corpus(5000, 256, 9)
    c[::613] = c[7]
    q = synth.make_dense_queries(c, 70, 10)
    q[1] = 0
    whole = rescore_all(q, c)
    for row_chunk in (1, 999, 4096, 5000):
        got = rescore_all(q, c, q_chunk=32, row_chunk=row_chunk)
        assert torch.equal(got.view(torch.int32), whole.view(torch.int32)), row_chunk
