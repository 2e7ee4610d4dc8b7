"""CPU model of the deep form of the two-phase BM25 top-k (32 < k <= 1024, easyrag_b200/csrc/bm25_pk.cuh).

The deep candidate pass differs from the k <= 32 one in where its bounds come from:

* a (query, range) without a bound takes G = the exact k-th largest integer sum of the range (radix select,
  ``block_kth_largest``; 0 when fewer than k sums are positive), keeps the documents with Q >= G - m - 2 and raises
  the query's bound B to G - m - 1;
* a range with a bound keeps the documents crossing B - 1 and, when it keeps k or more, raises B to the k-th largest
  of their sums minus m + 1 (the in-range raise, again a select);
* between range chunks the bound step raises B to the k-th largest candidate sum minus m + 1 and drops the
  candidates below B - 1.

Restated here with numpy on the oracle's integer sums (tests/test_bound_math.py has the bracket itself), for
k in {33, 192, 1024}, random and constructed inputs (ties at the k-th place, whole tie groups), ranges in any order:
G really has k documents at Q >= G, the candidates after every step contain the exact top-k, and a bound one step
too high loses an answer document.
"""
import numpy as np
import pytest

from oracle import bm25 as obm
from easyrag_b200 import synth
from test_bound_math import _int_scores, _scale_log2

R = 2048                     # documents per range of the model (the kernels use 8192; the argument does not care)
KS = (33, 192, 1024)


def kth_largest_positive(v, k):
    """block_kth_largest: the k-th largest positive value, duplicates counted; 0 when fewer than k are positive."""
    p = np.sort(v[v > 0])[::-1]
    return int(p[k - 1]) if p.size >= k else 0


def deep_pass(q, m, k, order, chunks, on_step=None, g_shift=0):
    """Candidates {doc: Q} and the final bound of the deep candidate pass over ranges ``order`` cut into ``chunks``.
    ``g_shift`` raises every bound by that many steps (the negative control)."""
    slack = m + 1
    B, cand, done = 0, {}, []
    pos = 0
    for n_r in chunks:
        for r in order[pos:pos + n_r]:
            lo, hi = r * R, min(q.size, (r + 1) * R)
            acc = q[lo:hi]
            if B <= 0:
                G = kth_largest_positive(acc, k)
                if G > 0:
                    assert int((acc >= G).sum()) >= k          # k distinct documents of the range at Q >= G
                bl = G - slack + g_shift if G > 0 else 0
                keep = np.nonzero(acc >= max(bl - 1, 1))[0]
                B = max(B, bl)
            else:
                keep = np.nonzero(acc >= max(B - 1, 1))[0]
                if keep.size >= k:
                    kth = kth_largest_positive(acc[keep], k)
                    if kth - slack + g_shift > B:
                        B = kth - slack + g_shift
            cand.update({lo + int(d): int(acc[d]) for d in keep})
            done.append(r)
            if on_step:
                on_step(cand, done)
        pos += n_r
        if pos < len(order) and len(cand) >= k:                # bm25_bound_kernel
            kth = kth_largest_positive(np.fromiter(cand.values(), np.int64), k)
            B = max(kth - slack + g_shift, B)
            cand = {d: v for d, v in cand.items() if v >= B - 1}
            if on_step:
                on_step(cand, done)
    return cand, B


def exact_topk(s, k):
    """canonical top-k ids: positive scores, score descending, id descending."""
    ids = np.nonzero(s > 0)[0][::-1]
    return set(ids[np.argsort(-s[ids], kind="stable")][:k].tolist())


def check_superset(q, s, m, k, order, chunks):
    want = exact_topk(s, k)

    def step(cand, done):
        seen = [d for d in want if d // R in done]
        missing = [d for d in seen if d not in cand]
        assert not missing, f"k={k} order={order} chunks={chunks}: lost {missing[:5]}"

    cand, _ = deep_pass(q, m, k, order, chunks, step)
    assert want <= set(cand)
    return len(cand)


@pytest.fixture(scope="module")
def case():
    corpus = synth.make_sparse_corpus(12_000, 3000, 71, mean_len=60, min_len=1, max_len=200)
    o = obm.OkapiCSR(corpus.doc_lists(), corpus.vocab)
    assert (o.idf >= 0).all()
    wmax = max(float(o.contributions(int(t)).max()) for t in np.nonzero(o.df)[0])
    e = _scale_log2(wmax)
    queries = synth.make_queries(corpus, 12, 72)
    lists = [[int(t) for t in terms] for terms in queries.term_lists()]
    present = np.nonzero(o.df)[0]
    common = np.argsort(o.df, kind="stable")[-20:]
    rng = np.random.default_rng(5)
    lists += [[int(t) for t in rng.choice(common, 6)], [int(common[-1])] * 3 + [int(present[3])],
              [int(t) for t in rng.choice(present, 40)]]
    return o, e, lists


def _orders(n_r, rng):
    yield list(range(n_r)), [1] * n_r
    yield list(range(n_r)), [n_r]
    yield list(range(n_r))[::-1], [2] + [1] * (n_r - 2)
    for _ in range(2):
        yield [int(x) for x in rng.permutation(n_r)], [1, n_r - 1]


@pytest.mark.parametrize("k", KS)
def test_deep_candidates_contain_the_exact_topk(case, k):
    o, e, lists = case
    rng = np.random.default_rng(k)
    n_r = -(-o.corpus_size // R)
    deep_enough = 0
    for tokens in lists:
        s = o.get_scores(tokens)
        q, _ = _int_scores(o, e, tokens)
        deep_enough += int((s > 0).sum() > k)
        for order, chunks in _orders(n_r, rng):
            check_superset(q, s, len(tokens), k, order, chunks)
    assert deep_enough >= 3                                    # the top-k is a real cut, not every positive document


def _tie_case(k, rng, n=6 * R):
    """integer sums with a tie group straddling the k-th place, a whole tie group of 3k documents further down, and
    distinct values elsewhere; the exact score equals the sum (m = 1 keeps the bracket trivially true)."""
    q = rng.permutation(np.arange(1, n + 1, dtype=np.int64) * 5)
    top = np.argsort(-q, kind="stable")
    q[top[k - 20:k + 40]] = q[top[k - 20]]                     # 60 ties across the k-th place
    q[top[2 * k:5 * k]] = q[top[2 * k]]
    return q


@pytest.mark.parametrize("k", KS)
def test_ties_at_the_kth_place(k):
    rng = np.random.default_rng(100 + k)
    q = _tie_case(k, rng)
    s = q.astype(np.float64)
    n_r = q.size // R
    for order, chunks in _orders(n_r, rng):
        check_superset(q, s, 1, k, order, chunks)
    # one whole tie group holding every positive document
    q2 = np.zeros(6 * R, np.int64)
    q2[rng.choice(q2.size, 3 * k, replace=False)] = 77
    check_superset(q2, q2.astype(np.float64), 1, k, list(range(6)), [1] * 6)


@pytest.mark.parametrize("k", KS)
def test_bound_one_step_too_high_loses_an_answer(k):
    # The bracket is tight: k documents with Q = G whose exact scaled scores sit at its bottom (G - m - 1), and one
    # document e with Q = G - m - 2 = B - 1 whose exact score sits at its top (Q + 1 = G - m - 1).  All k + 1 tie
    # exactly; e has the highest id, so it is in the canonical top-k.  B = G - m - 1 keeps it (Q >= B - 1); B + 1
    # does not.
    m, G = 3, 1000
    rng = np.random.default_rng(7 + k)
    q = rng.integers(1, 500, 3 * R).astype(np.int64)            # everything else far below
    s = q.astype(np.float64)
    at_g = rng.choice(R - 1, k, replace=False)                  # in the first range, below e's id
    e = R - 1
    q[at_g], s[at_g] = G, G - m - 1
    q[e], s[e] = G - m - 2, G - m - 1
    want = exact_topk(s, k)
    assert e in want
    order, chunks = [0, 1, 2], [1, 2]
    cand, _ = deep_pass(q, m, k, order, chunks)
    assert want <= set(cand)
    bad, _ = deep_pass(q, m, k, order, chunks, g_shift=1)
    assert e not in bad and not want <= set(bad)
