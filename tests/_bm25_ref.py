"""Test infrastructure: BM25 restated in plain torch ops, independent of the library, for CPU and CUDA tensors.

The oracle classes (oracle/bm25.py) loop over documents in Python and are too slow for the benchmark corpus (1M
chunks, 3e8 tokens).  This module computes the same numbers with whole-tensor torch ops, so the GPU tests can check
the kernels at that scale; tests/test_bm25_ref_cpu.py pins it to the oracle classes and to tests/_host_counts.py.

Bit-exactness rules every function here keeps:

* one eager op per arithmetic step, so nothing is contracted into a fused multiply-add;
* divisors are tensors on the operands' device, never Python scalars: on CUDA, torch divides by a CPU scalar as a
  multiplication by its reciprocal, which is not the IEEE quotient;
* score rows add the terms strictly in token order, each as ``row[docs] = row[docs] + w``.  A document appears once
  in a term's postings, so that is the oracle's sequential per-document sum.
"""
import torch

K1, B = 1.5, 0.75                 # retrievers.py:103-104, as oracle/bm25.py
FIRST_ABSENT = torch.iinfo(torch.int64).max


def counts(tokens, doc_ptr, vocab, doc_lo=0, doc_hi=None):
    """Postings of documents ``[doc_lo, doc_hi)``: ``tokens`` int [T], ``doc_ptr`` int64 [N+1] on one device.

    -> dict(term, doc, tf) int64 in (term, document) order, i.e. the block's slice of the term-major postings;
    ``key = term * N + doc`` (N = all documents, so keys of different blocks compare); ``df`` int64 [vocab] of this
    block; ``first_pos`` int64 [vocab]: corpus position of each term's first occurrence in the block (FIRST_ABSENT if
    none); ``doc_len`` int64 [doc_hi - doc_lo]."""
    n = doc_ptr.numel() - 1
    doc_hi = n if doc_hi is None else doc_hi
    dev = tokens.device
    p0, p1 = int(doc_ptr[doc_lo]), int(doc_ptr[doc_hi])
    lens = doc_ptr[doc_lo + 1:doc_hi + 1] - doc_ptr[doc_lo:doc_hi]
    tok = tokens[p0:p1].to(torch.int64)
    if tok.numel() and (int(tok.min()) < 0 or int(tok.max()) >= vocab):
        raise ValueError("token id out of range [0, vocab)")
    doc = torch.repeat_interleave(torch.arange(doc_lo, doc_hi, device=dev), lens)
    key, tf = torch.unique(tok * max(n, 1) + doc, sorted=True, return_counts=True)
    term = key // max(n, 1)
    first = torch.full((vocab,), FIRST_ABSENT, dtype=torch.int64, device=dev)
    first.scatter_reduce_(0, tok, torch.arange(p0, p1, device=dev), reduce="amin")
    return dict(key=key, term=term, doc=key - term * max(n, 1), tf=tf, df=torch.bincount(term, minlength=vocab),
                first_pos=first, doc_len=lens.to(torch.int64))


def postings_of_docs(indptr, post_doc, doc_lo, doc_hi):
    """The postings of documents ``[doc_lo, doc_hi)`` picked out of a whole term-major index (``indptr`` int64 [V+1],
    ``post_doc`` int [P], one device), in the index's order: -> dict(pos, term, doc) int64, ``pos`` the index of each
    posting in the whole arrays.  What :func:`counts` of the same documents lists, and what a row shard holds."""
    pos = torch.nonzero((post_doc >= doc_lo) & (post_doc < doc_hi)).flatten()
    term = torch.searchsorted(indptr[1:], pos, right=True)
    return dict(pos=pos, term=term, doc=post_doc[pos].to(torch.int64))


def _t(x, like):
    """A 0-dim float64 tensor on ``like``'s device (a tensor divisor keeps the division IEEE on CUDA)."""
    return torch.tensor(float(x), dtype=torch.float64, device=like.device)


def okapi_weights(tf, dl, idf, avgdl, k1=K1, b=B):
    """float64 rank_bm25 contribution of each posting, in OkapiCSR's order (oracle/bm25.py:97-100):
    t1 = b*dl; t2 = t1/avgdl; t3 = (1-b)+t2; K = k1*t3; den = tf+K; num = tf*(k1+1); r = num/den; c = idf*r.
    ``tf``, ``dl`` (length of the posting's document) and ``idf`` (of the posting's term) are per-posting tensors."""
    tf, dl, idf = tf.to(torch.float64), dl.to(torch.float64), idf.to(torch.float64)
    t1 = dl * b
    t2 = t1 / _t(avgdl, t1)
    t3 = t2 + (1 - b)
    K = t3 * k1
    den = tf + K
    num = tf * (k1 + 1)
    r = num / den
    return idf * r


def bm25s_weights(tf, dl, idf32, avgdl, k1=K1, b=B):
    """float32 bm25s (lucene) weight of each posting (oracle/bm25.py:174-224): idf float32, tfc = tf/(K + tf) in
    float64 with K as in :func:`okapi_weights`, stored weight = float32(float64(idf32) * tfc)."""
    tf, dl = tf.to(torch.float64), dl.to(torch.float64)
    t1 = dl * b
    t2 = t1 / _t(avgdl, t1)
    t3 = t2 + (1 - b)
    K = t3 * k1
    tfc = tf / (K + tf)
    return (idf32.to(torch.float32).to(torch.float64) * tfc).to(torch.float32)


def _row(query, indptr, post_doc, w, keep, n, dtype):
    """Score row of one query: terms in token order, duplicates repeated, skipped where ``keep(t)`` is False."""
    row = torch.zeros(n, dtype=dtype, device=w.device)
    for t in query:
        t = int(t)
        if t < 0 or t >= len(indptr) - 1 or not keep(t):
            continue
        s, e = int(indptr[t]), int(indptr[t + 1])
        docs = post_doc[s:e].long()
        row[docs] = row[docs] + w[s:e]
    return row


def okapi_row(query, indptr, post_doc, w, idf, n):
    """float64 rank_bm25 ``get_scores``: unknown, out-of-range and idf == 0 tokens are skipped (OkapiCSR).
    ``indptr`` and ``idf`` are host sequences (numpy), ``post_doc`` / ``w`` tensors on the device of the row."""
    return _row(query, indptr, post_doc, w, lambda t: idf[t] != 0.0, n, torch.float64)


def bm25s_row(query, indptr, post_doc, w32, df, n):
    """float32 bm25s ``get_scores``: float32 sums in token order; tokens with df == 0 are dropped."""
    return _row(query, indptr, post_doc, w32, lambda t: df[t] != 0, n, torch.float32)


def canonical_topk(rows, k, allowed=None, id_base=0):
    """The order the top-k kernels promise: positive (and allowed) scores only, score descending, id descending.

    Exact for any ties, at the k-th place included: the row is reversed (ids descending) and then stable-sorted by
    score, so equal scores keep the higher id first.  ``rows`` [Q, n] float32/float64, ``allowed`` bool [Q, n] or
    [n].  -> (ids int64 [Q, k] with id_base added, -1 padded; scores [Q, k], 0 where padded; counts int64 [Q])."""
    q, n = rows.shape
    ok = rows > 0
    if allowed is not None:
        ok = ok & allowed
    masked = torch.where(ok, rows, torch.full_like(rows, float("-inf"))).flip(1)
    vals, idx = torch.sort(masked, dim=1, descending=True, stable=True)
    vals, idx = vals[:, :k], idx[:, :k]
    valid = vals > 0
    ids = torch.where(valid, (n - 1 - idx) + id_base, torch.full_like(idx, -1))
    if ids.shape[1] < k:                                   # fewer columns than k
        pad = k - ids.shape[1]
        ids = torch.cat([ids, torch.full((q, pad), -1, dtype=ids.dtype, device=ids.device)], 1)
        vals = torch.cat([vals, torch.zeros(q, pad, dtype=vals.dtype, device=vals.device)], 1)
        valid = torch.cat([valid, torch.zeros(q, pad, dtype=torch.bool, device=valid.device)], 1)
    return ids, torch.where(valid, vals, torch.zeros_like(vals)), valid.sum(1)
