"""Hand-off of the coarse ranker's candidates to the fine-ranking stage (SURVEY.md 8(f).4).

The reference's ``LLMRerank._postprocess_nodes`` (rerankers.py:298-376) walks the coarse list in slices of
``embed_bs`` (32, yaml:28) and tokenises ``(query, get_node_content(node, embed_type))`` pairs per slice, then
overwrites ``node.score`` in place.  The reranker itself is outside this repository's scope; what belongs to
the coarse path is producing its input in exactly that layout, without re-deriving anything on the way:

* ``rerank_batches``   - the drop-in view: a fused ``List[NodeWithScore]`` -> the same slices of pairs.
* ``candidate_batches`` - the batched view: the ``[Q, k]`` id tensor of ``CoarseRanker`` -> per-query slices of
  document ids in rank order (one D2H copy for the whole batch; texts are looked up by the caller).

* ``RerankPacker``      - the device path: the fused ``[Q, k]`` ids never leave the GPU; the token sequences
  ``get_inputs`` / ``get_inputs_v2_5`` (rerankers.py:196-293) would build for every (query, candidate) pair are
  gathered by a kernel from the passages tokenised ONCE at index time, packed (ids + cu_seqlens, the layout this
  library's encoder kernels consume), in the reference's rank order and 32-pair slices.

The first two are host-side Python (strings and lists), like the code they feed.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Iterator, List, Optional, Sequence, Tuple

import torch

from . import _lib
from .retrievers import get_node_content

DEFAULT_RERANK_BATCH = 32      # yaml:28 (embed_bs of the reranker)


def rerank_batches(nodes: Sequence, query_str: str, embed_type: int = 0,
                   batch_size: int = DEFAULT_RERANK_BATCH) -> Iterator[Tuple[int, int, List[Tuple[str, str]]]]:
    """Yield ``(begin, end, [(query, text), ...])`` exactly as rerankers.py:309-322 slices the coarse list.

    ``nodes`` are ``NodeWithScore``-like objects (``.node``); the caller scores a slice and writes
    ``nodes[begin + i].score`` back, which is what the reference does (rerankers.py:365-370).
    """
    if batch_size < 1:
        raise ValueError("batch_size must be positive")
    n = len(nodes)
    for begin in range(0, n, batch_size):
        end = min(begin + batch_size, n)
        yield begin, end, [(query_str, get_node_content(nw.node, embed_type)) for nw in nodes[begin:end]]


def candidate_batches(ids, counts, batch_size: int = DEFAULT_RERANK_BATCH) -> Iterator[Tuple[int, int, List[int]]]:
    """Yield ``(query index, begin, [doc ids])`` for every slice of every query's candidate list, rank order kept.

    ``ids`` is ``[Q, k]`` (torch tensor on any device, or array-like) with ``-1`` padding, ``counts`` is ``[Q]``:
    the ``TopK`` a ``CoarseRanker`` / ``ShardedCoarseRanker`` returns.  One transfer for the whole batch.
    """
    if batch_size < 1:
        raise ValueError("batch_size must be positive")
    ids_h = ids.cpu().tolist() if hasattr(ids, "cpu") else [list(r) for r in ids]
    cnt_h = counts.cpu().tolist() if hasattr(counts, "cpu") else list(counts)
    for q, (row, c) in enumerate(zip(ids_h, cnt_h)):
        row = row[:c]
        for begin in range(0, c, batch_size):
            yield q, begin, row[begin:begin + batch_size]


@dataclass
class PackedRerankInput:
    """Pair p = q * k + r (candidate r of query q); pairs past a query's count are empty (length 0)."""
    ids: torch.Tensor          # int32 [T] packed token ids
    cu: torch.Tensor           # int32 [P + 1] cu_seqlens
    query_len: torch.Tensor    # int32 [P] len([bos] + query + sep)   (get_inputs_v2_5's query_lengths)
    prompt_len: int            # len(sep + prompt)                     (get_inputs_v2_5's prompt_lengths)
    n_queries: int
    k: int

    def slices(self, batch_size: int = DEFAULT_RERANK_BATCH) -> Iterator[Tuple[int, int, int]]:
        """(query, first pair, last pair + 1) of every slice rerankers.py:309-312 would form, in its order."""
        for q in range(self.n_queries):
            for r in range(0, self.k, batch_size):
                yield q, q * self.k + r, q * self.k + min(r + batch_size, self.k)


class RerankPacker:
    """Holds the corpus passages as token ids on the device and packs reranker inputs for fused candidate lists.

    ``passage_tokens[i]`` = the reranker tokenizer's ids of ``"B: " + get_node_content(node_i, embed_type)``
    (``add_special_tokens=False``), tokenised once when the index is built; ``sep`` / ``prompt`` = ids of ``"\n"`` and
    of the instruction prompt (rerankers.py:253-262).  ``pack`` takes query ids of ``"A: " + query``.
    """

    def __init__(self, passage_tokens: Sequence[Sequence[int]], sep: Sequence[int], prompt: Sequence[int], bos: int,
                 max_length: int = 1024, device="cuda", id_base: int = 0):
        _lib.require_cuda()
        self.device = torch.device(device)
        ptr = [0]
        for t in passage_tokens:
            ptr.append(ptr[-1] + len(t))
        flat = [int(x) for t in passage_tokens for x in t]
        self.n_docs = len(ptr) - 1
        self.p_ptr = torch.tensor(ptr, dtype=torch.int64, device=self.device)
        self.p_tok = torch.tensor(flat if flat else [0], dtype=torch.int32, device=self.device)
        self.sep = torch.tensor(list(sep) or [0], dtype=torch.int32, device=self.device)
        self.prompt = torch.tensor(list(prompt) or [0], dtype=torch.int32, device=self.device)
        self.n_sep, self.n_prompt = len(sep), len(prompt)
        self.bos, self.max_length, self.id_base = int(bos), int(max_length), int(id_base)

    def pack(self, cand_ids: torch.Tensor, cand_counts: torch.Tensor, q_ptr: torch.Tensor, q_tok: torch.Tensor,
             stream=None) -> PackedRerankInput:
        """``cand_ids`` int32 [Q, k] / ``cand_counts`` int32 [Q]: a ``TopK`` of the coarse ranker (device tensors);
        ``q_ptr`` int32 [Q+1] / ``q_tok`` int32: the batch's query ids (CSR, without bos).  Raises before any token
        buffer is allocated if a candidate id inside a query's count lies outside
        ``[id_base, id_base + len(passage_tokens))``, or if the pack would hold 2^31 tokens or more."""
        import ctypes
        L = _lib.lib()
        dev = self.device
        ids = cand_ids.to(device=dev, dtype=torch.int32)
        assert ids.dim() == 2 and ids.stride(1) == 1
        nq, k = ids.shape
        cnt = cand_counts.to(device=dev, dtype=torch.int32).contiguous()
        qp = q_ptr.to(device=dev, dtype=torch.int32).contiguous()
        qt = q_tok.to(device=dev, dtype=torch.int32).contiguous()
        if qt.numel() == 0:
            qt = torch.zeros(1, dtype=torch.int32, device=dev)
        n_pairs = nq * k
        ln = torch.empty(max(n_pairs, 1), dtype=torch.int64, device=dev)
        cu64 = torch.empty(n_pairs + 1, dtype=torch.int64, device=dev)
        qlen = torch.zeros(max(n_pairs, 1), dtype=torch.int32, device=dev)
        total = ctypes.c_int64(0)
        st = _lib.stream_ptr(stream)
        with torch.cuda.device(dev):
            _lib.check(L.ezr_rerank_pack_plan(_lib.ptr(ids), _lib.ptr(cnt), nq, k, ids.stride(0), self.id_base,
                                              self.n_docs, _lib.ptr(qp), _lib.ptr(self.p_ptr), self.n_sep,
                                              self.n_prompt, self.max_length, _lib.ptr(ln), _lib.ptr(cu64),
                                              _lib.ptr(qlen), ctypes.byref(total), st), "ezr_rerank_pack_plan")
            out = torch.empty(max(int(total.value), 1), dtype=torch.int32, device=dev)
            cu32 = torch.zeros(n_pairs + 1, dtype=torch.int32, device=dev)
            if n_pairs:
                _lib.check(L.ezr_rerank_pack_fill(_lib.ptr(ids), _lib.ptr(cnt), nq, k, ids.stride(0), self.id_base,
                                                  self.n_docs, _lib.ptr(qp), _lib.ptr(qt), _lib.ptr(self.p_ptr),
                                                  _lib.ptr(self.p_tok), _lib.ptr(self.sep), self.n_sep,
                                                  _lib.ptr(self.prompt), self.n_prompt, self.bos, self.max_length,
                                                  _lib.ptr(cu64), _lib.ptr(out), _lib.ptr(cu32), st),
                           "ezr_rerank_pack_fill")
        return PackedRerankInput(ids=out[:int(total.value)], cu=cu32, query_len=qlen[:n_pairs],
                                 prompt_len=self.n_sep + self.n_prompt, n_queries=nq, k=k)
