"""CPU check of the float32 bracket the two-phase BM25 top-k rests on for bm25s indexes (csrc/bm25_pk.cuh header).

bm25s scores a document as a float32 sum rounded after every token (``np.add.at`` per query token, in token order).
The candidate pass accumulates ``Q(d) = sum_j ceil(w_j * 2^e)`` from the same packed postings as for float64 and
keeps a document when ``Q(d) >= B - e(m)``, ``B = (k-th largest Q) - m - e(m)``, with

    e(m) = ceil(gamma_{m-1} * m * 2^18),  gamma_n = n u / (1 - n u),  u = 2^-24.

Restated here with numpy on the ``Bm25sLucene`` contributions (same scale rule as ``ezr_bm25_pack_f32``):

* the constant itself, against exact rational arithmetic, and that the float64 constant 1 covers u = 2^-53;
* the bracket ``Q - m - e(m) <= 2^e * s <= Q + e(m)`` for every (query, document), queries of several hundred
  tokens and repeated tokens included;
* superset: the canonical float32 top-k is contained in ``{d : Q(d) >= B - e(m)}``, with and without skipped tokens;
* negative control: a constructed float32 case in which the float64 constants (e = 1) drop the answer document and
  e(m) keeps it.
"""
import math
from fractions import Fraction

import numpy as np
import pytest

from oracle import bm25 as obm
from oracle import retrieve as ort
from easyrag_b200 import synth

WBITS = 19          # 32 - log2(8192): packed weight field of the default build
MAX_TERMS = 1 << (31 - WBITS)


def e_slack(m: int) -> int:
    """PkSlack<float>::e (bm25_pk.cuh), in the kernel's integer form."""
    n = max(m - 1, 0)
    num, den = n * m * (1 << (WBITS - 1)), (1 << 24) - n
    return -(-num // den)


def _gamma_bound(m: int, u: Fraction) -> Fraction:
    n = max(m - 1, 0)
    return n * u / (1 - n * u) * m * (1 << (WBITS - 1))


def _scale_log2(wmax: float) -> int:
    """ezr_bm25_pack(_f32): wmax < 2^ex (frexp)  ->  e = WBITS - 1 - ex, so ceil(w * 2^e) <= 2^(WBITS-1)."""
    if wmax <= 0:
        return 0
    _, ex = math.frexp(wmax)
    return WBITS - 1 - ex


def test_slack_constant_matches_its_definition():
    u32, u64 = Fraction(1, 1 << 24), Fraction(1, 1 << 53)
    for m in list(range(1, 300)) + [1000, 2047, 4095, MAX_TERMS]:
        assert e_slack(m) == math.ceil(_gamma_bound(m, u32)), m
        assert _gamma_bound(m, u64) < 1                   # the float64 instances' literal 1
    assert (e_slack(1), e_slack(2), e_slack(30), e_slack(MAX_TERMS)) == (0, 1, 14, 1 << 18)
    assert MAX_TERMS * (1 << (WBITS - 1)) + e_slack(MAX_TERMS) < 1 << 31     # integer sums and bounds fit in int32


@pytest.fixture(scope="module")
def case():
    corpus = synth.make_sparse_corpus(6000, 3000, 99, mean_len=60, min_len=1, max_len=200)
    o = obm.Bm25sLucene(corpus.doc_lists(), corpus.vocab)
    assert o.post_w.dtype == np.float32 and (o.post_w > 0).all()      # Lucene idf > 0: monotone
    e = _scale_log2(float(o.post_w.max()))
    queries = synth.make_queries(corpus, 60, 100)
    lists = [[int(t) for t in terms] for terms in queries.term_lists()]
    present = np.nonzero(o.df)[0]
    top = np.argsort(o.df, kind="stable")[-40:]                       # the longest posting lists
    rng = np.random.default_rng(3)
    lists += [[int(t) for t in rng.choice(present, 40)],
              [int(present[0])] * 5 + [int(present[7])],
              [int(t) for t in rng.choice(top, 300)],                 # several hundred tokens, many repeats
              [int(t) for t in rng.choice(present, 700)] + [-1, 10 ** 6],
              [int(top[-1])] * 250]
    return o, e, lists


def _packed(o, t, e):
    s, en = o.indptr[t], o.indptr[t + 1]
    w = o.post_w[s:en].astype(np.float64)                             # widening is exact
    q = np.ceil(np.ldexp(w, e))
    assert (q <= (1 << (WBITS - 1))).all() and (q >= 1).all()
    return q.astype(np.int64)


def _int_scores(o, e, tokens, skip=()):
    q = np.zeros(o.corpus_size, dtype=np.int64)
    for j, t in enumerate(tokens):
        if t < 0 or t >= o.df.shape[0] or o.df[t] == 0 or j in skip:
            continue
        s, en = o.indptr[t], o.indptr[t + 1]
        np.add.at(q, o.post_doc[s:en], _packed(o, t, e))
    return q


def test_integer_scores_bracket_the_float32_scores(case):
    o, e, lists = case
    for tokens in lists:
        s = o.get_scores(tokens)
        assert s.dtype == np.float32
        q = _int_scores(o, e, tokens)
        m = len(tokens)                                   # the kernel uses the token count of the query
        scaled = np.ldexp(s.astype(np.float64), e)        # exact
        es = e_slack(m)
        assert (q - m - es <= scaled).all() and (scaled <= q + es).all(), m


@pytest.mark.parametrize("k", [1, 10, 32, 192, 1024])
def test_candidates_are_a_superset_of_the_exact_topk(case, k):
    o, e, lists = case
    checked = 0
    for tokens in lists:
        s = o.get_scores(tokens)
        ids, _ = ort.bm25_topk_ids(s, k, None)            # canonical exact top-k (positive scores only)
        q = _int_scores(o, e, tokens)
        m = len(tokens)
        if (q > 0).sum() < k:
            continue                                      # fewer than k positives: no bound, everything is kept
        es = e_slack(m)
        bound = int(np.sort(q)[-k]) - m - es
        keep = q >= max(bound - es, 1)
        assert keep[ids].all()
        checked += 1
    assert checked > 0


@pytest.mark.parametrize("k", [10, 192])
def test_skipping_lowest_weight_tokens_keeps_the_superset(case, k):
    o, e, lists = case
    num, den = 3, 10                                      # kPkNeNum / kPkNeDen
    skipped_any = 0
    for tokens in lists:
        if len(tokens) > 32:
            continue                                      # the mask covers the first 32 tokens
        s = o.get_scores(tokens)
        ids, _ = ort.bm25_topk_ids(s, k, None)
        q = _int_scores(o, e, tokens)
        m = len(tokens)
        if (q > 0).sum() < k:
            continue
        es = e_slack(m)
        bound = int(np.sort(q)[-k]) - m - es
        if bound <= es:
            continue
        gm = [int(_packed(o, t, e).max()) if (0 <= t < o.df.shape[0] and o.df[t] > 0) else 0 for t in tokens]
        budget = (bound - es) * num // den
        skip, ne = set(), 0
        for j in sorted(range(len(tokens)), key=lambda j: (gm[j], j)):
            if ne + gm[j] <= budget:
                ne += gm[j]
                skip.add(j)
            else:
                break
        skipped_any += bool(skip)
        q_ess = _int_scores(o, e, tokens, skip=skip)
        assert (q - q_ess <= ne).all()                    # the skipped part never exceeds NE
        keep = q_ess >= max(bound - es - ne, 1)           # the relaxed crossing threshold
        assert keep[ids].all()
    assert skipped_any > 0


def test_float64_slack_loses_a_float32_answer():
    """Two documents share m = 322 tokens.  257 tokens of weight 2 - 4u (u = 2^-17 = 1/S) take both sums to about
    2^26 / S, where a float32 ulp is 8 units.  Then 64 tokens add 2^17 + 5 units to A (each add rounds UP by 3)
    and 2^17 + 11 units to C (each rounds DOWN by 3): the float32 sums stay equal while C's integer sum pulls 384
    units ahead.  A last token of exactly one ulp, in A only, makes A the top-1.  With e = 1 the bound
    Q(C) - m - 1 exceeds Q(A) + 1, so A is dropped; e(m) = 1616 keeps it."""
    u = 2.0 ** -17
    big, na, nc = (2 ** 18 - 4) * u, (2 ** 17 + 5) * u, (2 ** 17 + 11) * u
    w_a = [big] * 257 + [na] * 64 + [8 * u]
    w_c = [big] * 257 + [nc] * 64
    m = len(w_a)
    # postings: token j holds (A=0, w_a[j]) and, for j < len(w_c), (C=1, w_c[j])
    post_doc, post_w, indptr = [], [], [0]
    for j in range(m):
        post_doc.append(0), post_w.append(w_a[j])
        if j < len(w_c):
            post_doc.append(1), post_w.append(w_c[j])
        indptr.append(len(post_doc))
    post_doc, post_w = np.array(post_doc), np.array(post_w, dtype=np.float32)
    assert post_w.astype(np.float64).tolist() == [float(x) for x in post_w] and float(post_w.max()) < 2
    e = _scale_log2(float(post_w.max()))
    assert e == 17
    o = type("Ix", (), {})()
    o.corpus_size, o.indptr, o.post_doc, o.post_w = 2, np.array(indptr), post_doc, post_w
    o.df = np.diff(o.indptr)
    s = obm.Bm25sLucene.get_scores(o, list(range(m)))     # the oracle's float32 sum, token by token
    ids, _ = ort.bm25_topk_ids(s, 1, None)
    assert ids.tolist() == [0] and s[0] > s[1]
    q = _int_scores(o, e, list(range(m)))
    scaled = np.ldexp(s.astype(np.float64), e)
    assert scaled[0] > q[0] + 1                           # the float64 upper bracket fails for float32 sums
    b1 = int(q[1]) - m - 1                                # float64 constants: B = G - m - 1, keep Q >= B - 1
    assert q[0] < b1 - 1
    es = e_slack(m)
    assert es == 1616
    be = int(q[1]) - m - es
    assert q[0] >= be - es and (q - m - es <= scaled).all() and (scaled <= q + es).all()
