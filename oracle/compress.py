"""Oracle: the reference's BM25-Extract compressor (compressors.py:32-55) over pre-split sentences.  TEST
INFRASTRUCTURE ONLY.

Scores come from :class:`oracle.bm25.OkapiLiteral` (bm25_type 0) / :class:`oracle.bm25.Bm25sLucene` (bm25_type 1),
built over the context's own sentences as ``BM25Retriever.get_scores(query, sentences)`` builds its throw-away
index.  Two selection orders:

* literal:   ``scores.argsort()[::-1]`` exactly as the reference writes it (numpy's default, unstable sort);
* canonical: score descending, then sentence index descending (``argsort(kind="stable")[::-1]``), the order
             easyrag_b200 uses everywhere.  The two agree whenever no two scores are equal.
"""
from __future__ import annotations

from typing import Dict, List, Sequence

import numpy as np

from .bm25 import B, EPSILON, K1, Bm25sLucene, OkapiLiteral


def scores(query: Sequence[str], sentences: Sequence[Sequence[str]], bm25_type: int = 0) -> np.ndarray:
    """get_scores(query, sentences): float64 (rank_bm25) or float32 (bm25s)."""
    if bm25_type == 0:
        return OkapiLiteral([list(s) for s in sentences], k1=K1, b=B, epsilon=EPSILON).get_scores(list(query))
    vocab: Dict[str, int] = {}
    docs = [np.array([vocab.setdefault(w, len(vocab)) for w in s], dtype=np.int64) for s in sentences]
    return Bm25sLucene(docs, max(len(vocab), 1), k1=K1, b=B).get_scores([vocab.get(w, -1) for w in query])


def kept(sc: np.ndarray, sentences: Sequence[str], ctx_len: int, rate: float, literal: bool = False) -> List[int]:
    """compressors.py:44-51: indices of the kept sentences, ascending."""
    sorted_idx = sc.argsort()[::-1] if literal else np.argsort(sc, kind="stable")[::-1]
    i, now_len = 0, 0
    for i, idx in enumerate(sorted_idx):
        now_len += len(sentences[idx])
        if now_len >= ctx_len * rate:
            break
    sorted_idx = sorted_idx[:i + 1]
    return sorted(int(x) for x in sorted_idx)


def compress(query: Sequence[str], sentence_tokens: Sequence[Sequence[str]], sentences: Sequence[str], ctx_len: int,
             rate: float, bm25_type: int = 0, literal: bool = False) -> str:
    """compressors.py:32-55 over a tokenised query and pre-split (stripped, non-empty) sentences."""
    keep = kept(scores(query, sentence_tokens, bm25_type), sentences, ctx_len, rate, literal)
    return "".join(sentences[i] for i in keep)
