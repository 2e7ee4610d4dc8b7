"""Oracle: rerank fusion of the reference (``generation_with_rerank_fusion``, pipeline.py:393-452).  TEST
INFRASTRUCTURE ONLY.

* ``rerank_fusion`` restates pipeline.py:400-409 on per-pair scores: each route's nodes scored and sorted as
  ``SentenceTransformerRerank._postprocess_nodes`` does (rerankers.py:94-96) and cut to ``top_n``, then
  ``HybridRetriever.reciprocal_rank_fusion([sparse, dense], topk=r_topk_1)`` keyed by text.
* ``pair_union`` is the per-query union that ``ezr_pair_union`` must produce: distinct ids in first-appearance order
  over list a's slots then list b's, and each slot's union index.
"""
from __future__ import annotations

from typing import List, Sequence, Tuple

import numpy as np

from .retrieve import ONode, OScored, reciprocal_rank_fusion


def rerank_fusion(sparse: Sequence[ONode], dense: Sequence[ONode], sparse_scores: Sequence[float],
                  dense_scores: Sequence[float], top_n: int, topk: int, K: int = 60
                  ) -> Tuple[List[Tuple[int, float]], List[Tuple[int, float]], List[Tuple[int, float]]]:
    """``sparse`` / ``dense``: each route's coarse nodes in rank order, ``*_scores`` the reranker's score of each.
    -> (fused, sparse top_n, dense top_n) as (node idx, score) lists.  The route lists are read before the fusion,
    which overwrites the scores of the nodes it returns (retrievers.py:270-272)."""
    def postprocess(nodes, scores):
        scored = [OScored(node=n, score=float(s)) for n, s in zip(nodes, scores)]
        return sorted(scored, key=lambda x: -x.score if x.score else 0)[:top_n]

    node_with_scores_dense = postprocess(dense, dense_scores)
    node_with_scores_sparse = postprocess(sparse, sparse_scores)
    routes = [[(x.node.idx, x.score) for x in lst] for lst in (node_with_scores_sparse, node_with_scores_dense)]
    fused = reciprocal_rank_fusion([node_with_scores_sparse, node_with_scores_dense], K=K, topk=topk)
    return [(x.node.idx, x.score) for x in fused], routes[0], routes[1]


def pair_union(ids_a: np.ndarray, cnt_a: np.ndarray, ids_b: np.ndarray, cnt_b: np.ndarray):
    """ids_x int [Q, k_x], cnt_x [Q] (clamped to [0, k_x]) -> (ids int32 [Q, k_a + k_b] -1 padded, counts [Q],
    map_a int32 [Q, k_a], map_b [Q, k_b], -1 past each list's count)."""
    nq, ka = ids_a.shape
    kb = ids_b.shape[1]
    out = np.full((nq, ka + kb), -1, np.int32)
    counts = np.zeros(nq, np.int32)
    map_a = np.full((nq, ka), -1, np.int32)
    map_b = np.full((nq, kb), -1, np.int32)
    for q in range(nq):
        index = {}
        for lst, cnt, k, slot_map in ((ids_a, cnt_a, ka, map_a), (ids_b, cnt_b, kb, map_b)):
            for r in range(min(max(int(cnt[q]), 0), k)):
                i = int(lst[q, r])
                if i not in index:
                    index[i] = len(index)
                    out[q, index[i]] = i
                slot_map[q, r] = index[i]
        counts[q] = len(index)
    return out, counts, map_a, map_b
