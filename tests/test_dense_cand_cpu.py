"""Host side of the candidate form of dense top-k (csrc/dense_cand.cu, ``ezr_dense_cand_topk``).  No GPU needed.

1. A numpy restatement of the algorithm -- chunks of roundup(k, 256) rows growing by CAND_GROWTH, emission on
   ``score >= T_q``, a bounded candidate buffer whose overflow hands the query to a full top-k, and the bound step's
   canonical top-k -- against a plain canonical top-k of the whole score table: random and adversarial tables, ties
   across chunk boundaries, rising scores, filters, and every capacity from 1 to n.
2. A negative control: the same algorithm emitting on ``score > T_q`` loses the later of two tied rows.
3. The workspace arithmetic of ``ezr_dense_cand_topk_workspace`` and the argument checks that run before any device
   work (unsupported shapes, short workspaces, the capacity switch), and the Python refusals.
"""
import ctypes as C

import numpy as np
import pytest

from easyrag_b200 import _lib
from easyrag_b200.retrievers import B200VectorStore

GROWTH = 2              # CAND_GROWTH of csrc/dense_cand.cu
EZR_ERR_INVALID, EZR_ERR_WORKSPACE, EZR_ERR_UNSUPPORTED = -1, -3, -4


def _canon(s, ids, k):
    """canonical (score desc, id desc) top-k of one query's (scores, ids)"""
    order = np.lexsort((-ids.astype(np.int64), -s))[:k]
    return s[order], ids[order]


def chunk_bounds(n, k, growth=GROWTH):
    out, row0, rows = [], 0, (k + 255) // 256 * 256
    while row0 < n:
        out.append((row0, min(n, row0 + rows)))
        row0 += rows
        rows *= growth
    return out


def cand_topk(S, k, cap, allowed=None, strict=False, growth=GROWTH):
    """The candidate form on a score table S [Q, n] (fp32) -> (scores, ids, counts, cand_counts) as the library
    writes them: [Q, k] padded with -inf / -1, cand_counts -1 for a query the full top-k answered."""
    Q, n = S.shape
    out_s = np.full((Q, k), -np.inf, np.float32)
    out_i = np.full((Q, k), -1, np.int32)
    counts = np.zeros(Q, np.int32)
    cand = np.zeros(Q, np.int64)
    ids = np.arange(n, dtype=np.int64)
    for q in range(Q):
        T = -np.inf
        keep_s, keep_i = np.empty(0, np.float32), np.empty(0, np.int64)
        emitted, over = 0, False
        for lo, hi in chunk_bounds(n, k, growth):
            s = S[q, lo:hi]
            hit = (s > T) if strict else (s >= T)
            if allowed is not None:
                hit &= allowed[q, lo:hi]
            new_s, new_i = s[hit], ids[lo:hi][hit]
            emitted += new_s.size
            if keep_s.size + new_s.size > cap:                  # the buffer count passed the capacity
                over = True
                break
            keep_s, keep_i = _canon(np.concatenate([keep_s, new_s]), np.concatenate([keep_i, new_i]), k)
            T = keep_s[k - 1] if keep_s.size >= k else -np.inf
        if over:
            row = S[q] if allowed is None else S[q][allowed[q]]
            rid = ids if allowed is None else ids[allowed[q]]
            keep_s, keep_i = _canon(row, rid, k)
            cand[q] = -1
        else:
            cand[q] = emitted
        m = keep_s.size
        out_s[q, :m], out_i[q, :m], counts[q] = keep_s, keep_i, m
    return out_s, out_i, counts, cand


def plain_topk(S, k, allowed=None):
    Q, n = S.shape
    out_s = np.full((Q, k), -np.inf, np.float32)
    out_i = np.full((Q, k), -1, np.int32)
    counts = np.zeros(Q, np.int32)
    ids = np.arange(n)
    for q in range(Q):
        m = np.ones(n, bool) if allowed is None else allowed[q]
        s, i = _canon(S[q][m], ids[m], k)
        out_s[q, :s.size], out_i[q, :s.size], counts[q] = s, i, s.size
    return out_s, out_i, counts


def _check(S, k, cap, allowed=None):
    s, i, c, cand = cand_topk(S, k, cap, allowed)
    rs, ri, rc = plain_topk(S, k, allowed)
    np.testing.assert_array_equal(c, rc)
    np.testing.assert_array_equal(i, ri)
    np.testing.assert_array_equal(s, rs)
    return cand


# ---------------------------------------------------------------------------------------------- 1. the algorithm
@pytest.mark.parametrize("k", [1, 16, 17, 192, 256, 288])
def test_random_tables(k):
    rng = np.random.default_rng(k)
    S = rng.standard_normal((6, 5000)).astype(np.float32)
    cand = _check(S, k, 4 * k + 1024)
    assert (cand >= 0).all()                                  # random scores never overflow the default capacity


@pytest.mark.parametrize("k", [1, 7, 288])
def test_adversarial_tables(k):
    rng = np.random.default_rng(100 + k)
    n = 3000
    tables = [
        rng.integers(-2, 3, (4, n)).astype(np.float32),                 # five values: mass ties everywhere
        np.zeros((2, n), np.float32),                                   # one value
        np.sort(rng.standard_normal((2, n)).astype(np.float32))[:, ::-1].copy(),   # falling with the id
        np.where(rng.random((2, n)) < 0.01, 1.0, -1.0).astype(np.float32),         # a few winners in a sea of ties
    ]
    for S in tables:
        for cap in (1, k, 4 * k + 1024, n):
            _check(S, k, cap)


def test_ties_across_chunk_boundaries():
    # k = 5: chunks [0, 256), [256, 768), [768, 1792), [1792, 3000)
    k, n = 5, 3000
    S = np.full((1, n), -1.0, np.float32)
    dup = [3, 255, 256, 767, 768, 1791, 1792, n - 1]
    S[0, dup] = 0.5
    S[0, [10, 20, 30, 40]] = 0.75
    s, i, c, cand = cand_topk(S, k, 4 * k + 1024)
    assert cand[0] >= 0
    assert i[0].tolist() == [40, 30, 20, 10, n - 1]            # the last copy of the tied k-th row ranks first
    _check(S, k, 4 * k + 1024)


def test_rising_scores_overflow_and_fall_back():
    k, n = 16, 10_000
    S = np.arange(n, dtype=np.float32)[None, :].repeat(3, 0) / n
    for cap in (1, k, 4 * k + 1024):
        cand = _check(S, k, cap)
        assert (cand == -1).all()                              # every later chunk emits all of its rows
    assert (_check(S, k, n) >= 0).all()


def test_every_capacity_gives_the_same_result():
    rng = np.random.default_rng(7)
    n, k = 700, 33
    S = rng.integers(-3, 4, (3, n)).astype(np.float32)
    S[1] = rng.standard_normal(n).astype(np.float32)
    allowed = rng.random((3, n)) < 0.5
    ref = plain_topk(S, k, allowed)
    seen = set()
    for cap in range(1, n + 1):
        s, i, c, cand = cand_topk(S, k, cap, allowed)
        np.testing.assert_array_equal(i, ref[1])
        np.testing.assert_array_equal(s, ref[0])
        np.testing.assert_array_equal(c, ref[2])
        seen.update((cand == -1).tolist())
        if cap == n:
            assert (cand >= 0).all()                            # a buffer of n slots never overflows
    assert seen == {True, False}                                # both routes ran


def test_filters():
    rng = np.random.default_rng(11)
    n, k = 4000, 288
    S = rng.standard_normal((4, n)).astype(np.float32)
    doc = rng.integers(0, 5, n)
    doc[:100] = 5                                              # class 5: fewer rows than k
    q_group = [-1, 2, 5, 9]                                    # none / a class / a short class / a class no row has
    allowed = np.stack([np.ones(n, bool) if g == -1 else doc == g for g in q_group])
    _check(S, k, 4 * k + 1024, allowed)
    s, i, c, cand = cand_topk(S, k, 4 * k + 1024, allowed)
    assert c.tolist() == [k, k, 100, 0] and cand[3] == 0


def test_chunk_schedule():
    assert chunk_bounds(1, 288) == [(0, 1)]
    assert chunk_bounds(512, 288) == [(0, 512)]
    assert chunk_bounds(513, 288) == [(0, 512), (512, 513)]
    b = chunk_bounds(1_000_000, 288)
    assert [hi - lo for lo, hi in b][:4] == [512, 1024, 2048, 4096] and b[-1][1] == 1_000_000
    assert len(b) == 11


# ------------------------------------------------------------------------------------------ 2. negative control
def test_strict_threshold_loses_the_later_tie():
    # k = 1: row 0 and row 600 (second chunk) tie; the canonical top-1 is row 600 (higher id)
    S = np.full((1, 1000), -1.0, np.float32)
    S[0, 0] = S[0, 600] = 2.0
    rs, ri, rc = plain_topk(S, 1)
    assert ri[0, 0] == 600
    s, i, c, cand = cand_topk(S, 1, 1024)
    assert i[0, 0] == 600
    s, i, c, cand = cand_topk(S, 1, 1024, strict=True)
    assert i[0, 0] == 0                                        # '>' drops the tie: wrong
    assert not np.array_equal(i, ri)


# ------------------------------------------------------------------------------------- 3. workspace and refusals
def _align(x):
    return (x + 255) // 256 * 256


def _want_workspace(L, n, d, nq, k, cap):
    fixed = _align(nq * 4) + _align(4)
    cand = 4 * _align(nq * 4) + 2 * _align(nq * cap * 4)
    fb = _align(nq * d * 2) + _align(nq * 4) + 2 * _align(nq * k * 4) + _align(nq * 4)
    fb += L.ezr_dense_wide_workspace(n, nq, k, 1)
    return fixed + max(cand, fb)


@pytest.mark.parametrize("n,d,nq,k", [(1_000_000, 768, 10_000, 288), (1_000_000, 768, 10_000, 1024),
                                      (4_000_000, 1024, 64, 288), (1_000_000, 3584, 4096, 288), (1, 64, 1, 1),
                                      (300, 64, 129, 17)])
def test_workspace_arithmetic(lib_built, n, d, nq, k):
    L = _lib.lib()
    assert L.ezr_dense_cand_topk_workspace(n, d, nq, k) == _want_workspace(L, n, d, nq, k, 4 * k + 1024)
    try:
        assert L.ezr_dense_cand_set_capacity(k) == 0
        assert L.ezr_dense_cand_topk_workspace(n, d, nq, k) == _want_workspace(L, n, d, nq, k, k)
        assert L.ezr_dense_cand_set_capacity(1) == 0
        assert L.ezr_dense_cand_topk_workspace(n, d, nq, k) == _want_workspace(L, n, d, nq, k, 1)
    finally:
        L.ezr_dense_cand_set_capacity(0)
    assert L.ezr_dense_cand_topk_workspace(0, d, nq, k) == 0
    assert L.ezr_dense_cand_topk_workspace(n, d, 0, k) == 0


def test_workspace_grows_with_q_k_not_q_n(lib_built):
    L = _lib.lib()
    # the configs[4] shape and the 1M x 768 x 10k batch: a small fraction of form 6's score rows
    assert L.ezr_dense_cand_topk_workspace(4_000_000, 1024, 64, 288) < 64 * 4_000_000 * 4 // 8
    assert L.ezr_dense_cand_topk_workspace(1_000_000, 768, 10_000, 288) < 200 << 20


def test_capacity_switch(lib_built):
    L = _lib.lib()
    assert L.ezr_dense_cand_set_capacity(-1) == EZR_ERR_INVALID
    assert L.ezr_dense_cand_set_capacity((1 << 20) + 1) == EZR_ERR_INVALID
    assert L.ezr_dense_cand_set_capacity(1 << 20) == 0
    assert L.ezr_dense_cand_set_capacity(0) == 0
    assert L.ezr_dense_set_kernel(7) == EZR_ERR_INVALID         # the candidate form is not a kernel form


def _call(L, n=1000, d=64, ldc=None, nq=4, ldq=None, k=10, corpus=0x10000, queries=0x20000, ws=None, ws_bytes=0,
          doc_group=None, q_group=None):
    p = C.c_void_p
    return L.ezr_dense_cand_topk(p(corpus), n, d, ldc or d, p(queries), nq, ldq or d, k, p(doc_group), p(q_group), 0,
                                 p(0x30000), p(0x40000), p(0x50000), p(0), p(ws), ws_bytes, p(0))


def test_refusals_before_device_work(lib_built):
    # addresses are never dereferenced on these paths: every check runs before the first CUDA call
    L = _lib.lib()
    assert _call(L, k=0) == EZR_ERR_INVALID
    assert _call(L, k=1025) == EZR_ERR_INVALID
    assert _call(L, ldc=32) == EZR_ERR_INVALID
    assert _call(L, q_group=0x60000) == EZR_ERR_INVALID          # q_group without doc_group
    assert _call(L, nq=0) == 0                                   # the empty batch does nothing
    assert _call(L, d=100, ldc=104, ldq=104) == EZR_ERR_UNSUPPORTED
    assert b"dim % 64" in L.ezr_last_error()
    assert _call(L, ldc=68) == EZR_ERR_UNSUPPORTED               # corpus stride % 8 != 0
    assert _call(L, ldq=68) == EZR_ERR_UNSUPPORTED
    assert _call(L, corpus=0x10008) == EZR_ERR_UNSUPPORTED       # rows not 16-byte aligned
    assert _call(L, queries=0x20004) == EZR_ERR_UNSUPPORTED
    need = L.ezr_dense_cand_topk_workspace(1000, 64, 4, 10)
    assert _call(L) == EZR_ERR_WORKSPACE
    assert _call(L, ws=0x70000, ws_bytes=need - 1) == EZR_ERR_WORKSPACE
    assert b"workspace" in L.ezr_last_error()


def test_vector_store_refusals():
    for kw in (dict(dense_form=6), dict(dense_form=1), dict(block_queries=64), dict(quantize=True)):
        with pytest.raises(ValueError, match="dense_cand"):
            B200VectorStore(dense_cand=True, **kw)
    with pytest.raises(ValueError, match="dense_form=6"):
        B200VectorStore(block_queries=64)
    assert B200VectorStore(dense_cand=True).dense_cand

