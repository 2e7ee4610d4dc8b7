"""CPU: the rerank-fusion oracle (pipeline.py:400-409) on hand-computed cases, the numpy union reference that
ezr_pair_union must reproduce, and the argument checks of ``batched.pair_union``."""
import numpy as np
import pytest
import torch

from oracle import rerank_fusion as orf
from oracle import retrieve as ort
from oracle.retrieve import ONode


def _nodes(texts, ids):
    return [ONode(text=t, idx=i) for t, i in zip(texts, ids)]


def test_ties_at_one_and_zero_keep_coarse_order_then_rrf():
    sparse = _nodes("ABCD", [0, 1, 2, 3])
    dense = _nodes("EBF", [4, 1, 5])
    fused, s, d = orf.rerank_fusion(sparse, dense, [0.0, 1.0, 0.5, 1.0], [1.0, 0.0, 1.0], top_n=3, topk=10)
    # ties at 1.0 keep coarse order; a score of 0.0 sorts last (key 0); sparse's 0.0 falls out at top_n = 3
    assert s == [(1, 1.0), (3, 1.0), (2, 0.5)]
    assert d == [(4, 1.0), (5, 1.0), (1, 0.0)]
    # B: 1/61 + 1/63; E: 1/61; D and F: 1/62 (insertion order keeps D, from the sparse list, first); C: 1/63
    assert fused == [(1, 1 / 61 + 1 / 63), (4, 1 / 61), (3, 1 / 62), (5, 1 / 62), (2, 1 / 63)]


def test_short_and_empty_routes():
    fused, s, d = orf.rerank_fusion(_nodes("AB", [0, 1]), [], [0.25, 0.75], [], top_n=6, topk=6)
    assert s == [(1, 0.75), (0, 0.25)] and d == []
    assert fused == [(1, 1 / 61), (0, 1 / 62)]
    fused, s, d = orf.rerank_fusion([], _nodes("C", [2]), [], [0.5], top_n=6, topk=1, K=10)
    assert s == [] and d == [(2, 0.5)] and fused == [(2, 1 / 11)]
    assert orf.rerank_fusion([], [], [], [], top_n=6, topk=6) == ([], [], [])


def test_same_text_under_two_ids_merges_by_text():
    # ids 7 and 8 carry the same text; 7 is in the sparse list, 8 in the dense list: RRF keys by text, so they are one
    # item whose node is the last writer (the dense list's 8)
    sparse = _nodes(["X", "Y"], [7, 9])
    dense = _nodes(["Z", "X"], [10, 8])
    fused, s, d = orf.rerank_fusion(sparse, dense, [0.9, 0.1], [0.8, 0.3], top_n=2, topk=3)
    assert s == [(7, 0.9), (9, 0.1)] and d == [(10, 0.8), (8, 0.3)]
    assert fused == [(8, 1 / 61 + 1 / 62), (10, 1 / 61), (9, 1 / 62)]
    # the integer form the GPU fusion is pinned to gives the same list under canon
    canon = np.arange(11)
    canon[8] = 7
    ids, sc = ort.rrf_ids([[i for i, _ in s], [i for i, _ in d]], canon, K=60, topk=3)
    assert ids.tolist() == [i for i, _ in fused] and sc.tolist() == [x for _, x in fused]


def test_union_reference_hand_cases():
    # query 0: disjoint; 1: identical lists in another order; 2: partial overlap; 3: both empty; 4: counts past k and
    # negative; 5: an id repeated inside list a
    ids_a = np.array([[1, 2, 3], [5, 6, 7], [1, 2, 3], [-1, -1, -1], [4, 5, 6], [9, 8, 9]])
    cnt_a = np.array([3, 3, 2, 0, 7, 3])
    ids_b = np.array([[4, 5, -1, -1], [7, 5, 6, -1], [3, 2, 9, -1], [-1, -1, -1, -1], [1, 2, 3, 4], [8, 1, -1, -1]])
    cnt_b = np.array([2, 3, 3, 0, -2, 2])
    out, cnt, ma, mb = orf.pair_union(ids_a, cnt_a, ids_b, cnt_b)
    assert cnt.tolist() == [5, 3, 4, 0, 3, 3]
    assert out.tolist() == [[1, 2, 3, 4, 5, -1, -1], [5, 6, 7, -1, -1, -1, -1], [1, 2, 3, 9, -1, -1, -1],
                            [-1] * 7, [4, 5, 6, -1, -1, -1, -1], [9, 8, 1, -1, -1, -1, -1]]
    assert ma.tolist() == [[0, 1, 2], [0, 1, 2], [0, 1, -1], [-1, -1, -1], [0, 1, 2], [0, 1, 0]]
    assert mb.tolist() == [[3, 4, -1, -1], [2, 0, 1, -1], [2, 1, 3, -1], [-1] * 4, [-1] * 4, [1, 2, -1, -1]]
    # every slot reads its own id back through the map
    for q in range(6):
        for lst, c, m in ((ids_a, cnt_a, ma), (ids_b, cnt_b, mb)):
            n = min(max(c[q], 0), lst.shape[1])
            assert all(out[q, m[q, r]] == lst[q, r] for r in range(n))


def test_union_reference_random_invariants():
    rng = np.random.default_rng(5)
    nq, ka, kb, n_docs = 200, 19, 29, 60
    ids_a = np.stack([rng.choice(n_docs, ka, replace=False) for _ in range(nq)])
    ids_b = np.stack([rng.choice(n_docs, kb, replace=False) for _ in range(nq)])
    cnt_a, cnt_b = rng.integers(0, ka + 1, nq), rng.integers(0, kb + 1, nq)
    out, cnt, ma, mb = orf.pair_union(ids_a, cnt_a, ids_b, cnt_b)
    for q in range(nq):
        a, b = ids_a[q, :cnt_a[q]], ids_b[q, :cnt_b[q]]
        expect = list(a) + [i for i in b if i not in set(a)]
        assert out[q, :cnt[q]].tolist() == expect and (out[q, cnt[q]:] == -1).all()
        assert ma[q, :cnt_a[q]].tolist() == list(range(cnt_a[q])) and (ma[q, cnt_a[q]:] == -1).all()
        assert [expect[u] for u in mb[q, :cnt_b[q]]] == list(b) and (mb[q, cnt_b[q]:] == -1).all()


def test_pair_union_refuses_bad_shapes_before_any_launch():
    from easyrag_b200 import batched
    z = lambda *s: torch.zeros(*s, dtype=torch.int32)
    with pytest.raises(ValueError, match="queries"):
        batched.pair_union(z(3, 4), z(3), z(2, 4), z(2))
    with pytest.raises(ValueError, match="queries"):
        batched.pair_union(z(3, 4), z(2), z(3, 4), z(3))
    with pytest.raises(ValueError, match="1024"):
        batched.pair_union(z(1, 512), z(1), z(1, 513), z(1))
    with pytest.raises(ValueError, match=">= 1"):
        batched.pair_union(z(1, 0), z(1), z(1, 4), z(1))
    with pytest.raises(ValueError, match=r"\[Q, k\]"):
        batched.pair_union(z(4), z(1), z(1, 4), z(1))
