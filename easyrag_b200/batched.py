"""Batched tensor API over the C ABI: the throughput path beside the drop-in retrievers.

``NodeWithScore`` lists cannot be produced at 100k queries/s (SURVEY.md section 7), so the
retriever classes in :mod:`easyrag_b200.retrievers` are thin per-query views over this module.
Everything here takes and returns torch CUDA tensors used purely as device buffers; the
arithmetic is in easyrag_b200/csrc/*.cu.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Optional, Sequence, Tuple

import torch

from . import _lib
from .index import Bm25Index, DenseIndex


def _i32(t: Optional[torch.Tensor], device) -> Optional[torch.Tensor]:
    if t is None:
        return None
    return t.to(device=device, dtype=torch.int32).contiguous()


class Workspace:
    """Grow-only device scratch buffer (launch functions never allocate)."""

    def __init__(self, device):
        self.device = device
        self.buf = torch.empty(0, dtype=torch.uint8, device=device)

    def get(self, nbytes: int) -> torch.Tensor:
        if self.buf.numel() < nbytes:
            self.buf = torch.empty(int(nbytes * 1.25) + 256, dtype=torch.uint8, device=self.device)
        return self.buf


@dataclass
class TopK:
    scores: torch.Tensor     # [Q, k] float32 (dense, bm25s) or float64 (Okapi, fusion)
    ids: torch.Tensor        # [Q, k] int32, -1 padded
    counts: torch.Tensor     # [Q] int32


def dense_topk(index: DenseIndex, queries: torch.Tensor, k: int, q_group: Optional[torch.Tensor] = None,
               id_base: Optional[int] = None, ws: Optional[Workspace] = None, stream=None,
               out: Optional[TopK] = None, cand_counts: Optional[torch.Tensor] = None, form: Optional[int] = None,
               block_queries: Optional[int] = None) -> TopK:
    """QdrantRetriever._aretrieve's search for a batch (retrievers.py:37-52): cosine top-k, ids descending on ties.

    A quantized index runs ``ezr_dense_s8_topk`` (int8 candidate pass + exact rescoring; its scores are the
    fixed-order fp32 ``rescore`` of csrc/dense_s8.cu).  ``cand_counts`` (int32 [Q] on the device, quantized indexes
    only) receives the candidates per query of the int8 pass.

    ``form`` forces a kernel form of ``ezr_dense_set_kernel`` for this call (the calling thread's switch is set back
    to 0, automatic, afterwards); form 6 (wgmma score rows + select) takes any dim % 64 == 0 and k <= 1024.
    ``block_queries`` (form 6 only) runs it in query blocks of that many queries, with a workspace of
    ``ezr_dense_wide_workspace`` bytes; by default the block is the largest that ``ezr_dense_topk_workspace`` holds."""
    if block_queries is not None:
        if form != 6:
            raise ValueError("block_queries needs form=6 (the wgmma score-row form)")
        if getattr(index, "quantized", False):
            raise ValueError("block_queries does not apply to a quantized index")
        if block_queries < 1:
            raise ValueError(f"block_queries={block_queries} must be >= 1")
    if form is None:
        return _dense_topk(index, queries, k, q_group, id_base, ws, stream, out, cand_counts, None, None)
    L = _lib.lib()
    _lib.check(L.ezr_dense_set_kernel(int(form)), "ezr_dense_set_kernel")
    try:
        return _dense_topk(index, queries, k, q_group, id_base, ws, stream, out, cand_counts, form, block_queries)
    finally:
        L.ezr_dense_set_kernel(0)


def _dense_topk(index, queries, k, q_group, id_base, ws, stream, out, cand_counts, form, block_queries) -> TopK:
    L = _lib.lib()
    dev = index.device
    q = queries
    if q.dtype != torch.bfloat16 or q.device != dev or not q.is_contiguous():
        q = queries.to(device=dev, dtype=torch.bfloat16).contiguous()
    nq, dim = q.shape
    if dim != index.dim:
        raise ValueError(f"query dim {dim} != corpus dim {index.dim}")
    qg = _i32(q_group, dev)
    if qg is not None and index.doc_group is None:
        raise ValueError("q_group given but the index has no doc_group")
    if out is None:
        out = TopK(torch.empty(nq, k, dtype=torch.float32, device=dev), torch.empty(nq, k, dtype=torch.int32, device=dev),
                   torch.empty(nq, dtype=torch.int32, device=dev))
    quantized = getattr(index, "quantized", False)
    if cand_counts is not None and not quantized:
        raise ValueError("cand_counts needs a quantized index")
    if block_queries is not None:
        need = L.ezr_dense_wide_workspace(index.n_rows, nq, k, block_queries)
    else:
        need = (L.ezr_dense_s8_topk_workspace if quantized else L.ezr_dense_topk_workspace)(index.n_rows, dim, nq, k)
    ws = ws or Workspace(dev)
    buf = ws.get(need)
    # form 6 runs the largest query block the bytes it is given hold: give it exactly the bytes sized above, so that
    # the block does not depend on what the grow-only buffer held before
    ws_bytes = need if form == 6 else buf.numel()
    base = index.row_lo if id_base is None else id_base
    with torch.cuda.device(dev):
        if quantized:
            _lib.check(L.ezr_dense_s8_topk(
                _lib.ptr(index.vectors), index.n_rows, dim, index.vectors.stride(0), _lib.ptr(q), nq, q.stride(0), k,
                _lib.ptr(index.doc_group if qg is not None else None), _lib.ptr(qg), base, _lib.ptr(out.scores),
                _lib.ptr(out.ids), _lib.ptr(out.counts), _lib.ptr(index.rows_s8), index.rows_s8.stride(0),
                _lib.ptr(index.row_scale), _lib.ptr(index.maxima), _lib.ptr(cand_counts), _lib.ptr(buf), buf.numel(),
                _lib.stream_ptr(stream)), "ezr_dense_s8_topk")
            return out
        _lib.check(L.ezr_dense_topk(_lib.ptr(index.vectors), index.n_rows, dim, index.vectors.stride(0), _lib.ptr(q), nq,
                                    q.stride(0), k, _lib.ptr(index.doc_group if qg is not None else None), _lib.ptr(qg),
                                    base, _lib.ptr(out.scores), _lib.ptr(out.ids), _lib.ptr(out.counts), _lib.ptr(buf),
                                    ws_bytes, _lib.stream_ptr(stream)), "ezr_dense_topk")
    return out


def dense_topk_cand(index: DenseIndex, queries: torch.Tensor, k: int, q_group: Optional[torch.Tensor] = None,
                    id_base: Optional[int] = None, ws: Optional[Workspace] = None, stream=None,
                    out: Optional[TopK] = None, cand_counts: Optional[torch.Tensor] = None) -> TopK:
    """Cosine top-k of the bf16 rows without score rows (``ezr_dense_cand_topk``, csrc/dense_cand.cu): the canonical
    top-k under form 6's scores, bit-identical to ``dense_topk(..., form=6)``, for any dim % 64 == 0 and k <= 1024.

    Its workspace grows with Q * (k + capacity) where form 6's grows with Q * n_rows, and the whole batch shares one
    pass over the corpus.  ``cand_counts`` (int32 [Q] on the device) receives the candidates each query emitted, or -1
    for a query whose buffer overflowed and that form 6 answered inside the call.  A quantized index is searched on
    its bf16 rows."""
    L = _lib.lib()
    dev = index.device
    q = queries
    if q.dtype != torch.bfloat16 or q.device != dev or not q.is_contiguous():
        q = queries.to(device=dev, dtype=torch.bfloat16).contiguous()
    nq, dim = q.shape
    if dim != index.dim:
        raise ValueError(f"query dim {dim} != corpus dim {index.dim}")
    qg = _i32(q_group, dev)
    if qg is not None and index.doc_group is None:
        raise ValueError("q_group given but the index has no doc_group")
    if cand_counts is not None and (cand_counts.dtype != torch.int32 or cand_counts.numel() < nq
                                    or cand_counts.device != q.device or not cand_counts.is_contiguous()):
        raise ValueError("cand_counts must be an int32 device tensor with one slot per query")
    if out is None:
        out = TopK(torch.empty(nq, k, dtype=torch.float32, device=dev), torch.empty(nq, k, dtype=torch.int32, device=dev),
                   torch.empty(nq, dtype=torch.int32, device=dev))
    need = L.ezr_dense_cand_topk_workspace(index.n_rows, dim, nq, k)
    ws = ws or Workspace(dev)
    buf = ws.get(need)
    base = index.row_lo if id_base is None else id_base
    with torch.cuda.device(dev):
        _lib.check(L.ezr_dense_cand_topk(
            _lib.ptr(index.vectors), index.n_rows, dim, index.vectors.stride(0), _lib.ptr(q), nq, q.stride(0), k,
            _lib.ptr(index.doc_group if qg is not None else None), _lib.ptr(qg), base, _lib.ptr(out.scores),
            _lib.ptr(out.ids), _lib.ptr(out.counts), _lib.ptr(cand_counts), _lib.ptr(buf), buf.numel(),
            _lib.stream_ptr(stream)), "ezr_dense_cand_topk")
    return out


def bm25_topk(index: Bm25Index, q_ptr: torch.Tensor, q_terms: torch.Tensor, k: int,
              q_group: Optional[torch.Tensor] = None, id_base: Optional[int] = None,
              ws: Optional[Workspace] = None, stream=None, out: Optional[TopK] = None) -> TopK:
    """BM25Retriever.get_scores + filter for a batch (retrievers.py:128-151,191-210)."""
    L = _lib.lib()
    dev = index.device
    qp, qt = _i32(q_ptr, dev), _i32(q_terms, dev)
    nq = qp.numel() - 1
    qg = _i32(q_group, dev)
    if qg is not None and index.doc_group is None:
        raise ValueError("q_group given but the index has no doc_group")
    if out is None:
        out = TopK(torch.empty(nq, k, dtype=index.score_dtype, device=dev),
                   torch.empty(nq, k, dtype=torch.int32, device=dev), torch.empty(nq, dtype=torch.int32, device=dev))
    need = L.ezr_bm25_topk_workspace(index.struct, nq, k)
    ws = ws or Workspace(dev)
    buf = ws.get(need)
    base = index.doc_lo if id_base is None else id_base
    with torch.cuda.device(dev):
        _lib.check(L.ezr_bm25_topk(index.struct, _lib.ptr(qp), _lib.ptr(qt), nq, k, _lib.ptr(qg), base,
                                   _lib.ptr(out.scores), _lib.ptr(out.ids), _lib.ptr(out.counts), _lib.ptr(buf),
                                   buf.numel(), _lib.stream_ptr(stream)), "ezr_bm25_topk")
    return out


def bm25_scores(index: Bm25Index, q_ptr: torch.Tensor, q_terms: torch.Tensor, stream=None) -> torch.Tensor:
    """BM25Retriever.get_scores (retrievers.py:128-151): [Q, n_docs] score rows."""
    L = _lib.lib()
    dev = index.device
    qp, qt = _i32(q_ptr, dev), _i32(q_terms, dev)
    nq = qp.numel() - 1
    out = torch.empty(nq, index.n_docs, dtype=index.score_dtype, device=dev)
    with torch.cuda.device(dev):
        _lib.check(L.ezr_bm25_scores(index.struct, _lib.ptr(qp), _lib.ptr(qt), nq, _lib.ptr(out),
                                     _lib.stream_ptr(stream)), "ezr_bm25_scores")
    return out


@dataclass
class Extract:
    keep: torch.Tensor               # uint8 [S]: sentence kept
    counts: torch.Tensor             # int32 [G]: sentences kept; -1 = the group has no sentences
    scores: Optional[torch.Tensor]   # [S] float64 (Okapi) / float32 (bm25s), when asked for


def extract_caps() -> Tuple[int, int]:
    """(tokens, sentences) of the largest group :func:`bm25_extract` answers in its one launch."""
    import ctypes
    t, s = ctypes.c_int32(0), ctypes.c_int32(0)
    _lib.check(_lib.lib().ezr_bm25_extract_caps(ctypes.byref(t), ctypes.byref(s)), "ezr_bm25_extract_caps")
    return t.value, s.value


_LOG_HALF: dict = {}      # device -> float64 L[j] = math.log(j + 0.5)
_IDF_BM25S: dict = {}     # device -> float32 bm25s idf of (N, df) at N*(N+1)/2 + df, 0 <= df <= N


def log_half_table(n: int):
    """float64 L[j] = math.log(j + 0.5), j < n: rank_bm25's idf of df n among N documents is L[N - n] - L[n] bit for
    bit, because N - n + 0.5 is exact."""
    import numpy as np
    return np.array([math.log(j + 0.5) for j in range(n)], dtype=np.float64)


def _log_half(n: int, dev) -> torch.Tensor:
    t = _LOG_HALF.get(dev)
    if t is None or t.numel() < n:
        t = torch.from_numpy(log_half_table(max(n, 2 * (t.numel() if t is not None else 0), 1024))).to(dev)
        _LOG_HALF[dev] = t
    return t


def _bm25s_idf_table(max_n: int, dev) -> torch.Tensor:
    from .index import bm25s_idf
    t = _IDF_BM25S.get(dev)
    have = 0 if t is None else int((math.isqrt(8 * t.numel() + 1) - 1) // 2)    # t covers N < have
    if have <= max_n:
        top = max(max_n + 1, 2 * have, 256)
        vals = [0.0 if d == 0 else bm25s_idf(n, d) for n in range(top) for d in range(n + 1)]
        t = torch.tensor(vals, dtype=torch.float64).to(torch.float32).to(dev)
        _IDF_BM25S[dev] = t
    return t


def _select_host(scores, chars, ctx_chars: int, rate: float):
    """The reference's walk (compressors.py:44-50) in the canonical order: score descending, then index descending."""
    import numpy as np
    order = np.argsort(scores, kind="stable")[::-1]
    run = np.cumsum(np.asarray(chars, dtype=np.int64)[order])
    hit = np.nonzero(run >= ctx_chars * rate)[0]
    keep = np.zeros(len(scores), dtype=np.uint8)
    keep[order[:(hit[0] + 1) if hit.size else len(order)]] = 1
    return keep


def bm25_extract(sent_ptr, tok_ptr, tokens, sent_chars, ctx_chars, q_ptr, q_tokens, vocab: int, rate: float = 0.5,
                 bm25_type: int = 0, k1: Optional[float] = None, b: Optional[float] = None,
                 epsilon: Optional[float] = None, scores: bool = False, device="cuda", stream=None) -> Extract:
    """BM25-Extract over a batch of groups (``ezr_bm25_extract``): group g is a context's sentences
    ``[sent_ptr[g], sent_ptr[g+1])`` with tokens ``tokens[tok_ptr[s]:tok_ptr[s+1]]`` (ids < ``vocab``, one vocabulary for
    the batch) and its query ``q_tokens[q_ptr[g]:q_ptr[g+1]]`` (-1 = unknown).  Each group's scores are those of
    ``BM25Retriever.get_scores(query, sentences)``; ``keep`` marks the sentences the reference compressor keeps.

    ``sent_ptr`` / ``tok_ptr`` are read on the host (pass CPU tensors or arrays: the call then does not synchronise).
    Groups within :func:`extract_caps` run in one launch; larger ones are answered one by one through a throw-away
    index and ``ezr_bm25_scores`` with the selection on the host, which synchronises."""
    import numpy as np
    from .index import B as B_, EPSILON as EPS_, K1 as K1_, Bm25Stats
    k1 = K1_ if k1 is None else k1
    b = B_ if b is None else b
    epsilon = EPS_ if epsilon is None else epsilon
    if bm25_type not in (0, 1):
        raise ValueError("bm25_type must be 0 (BM25Okapi) or 1 (bm25s)")
    dev = torch.device(device)
    sp = torch.as_tensor(sent_ptr).to(torch.int64).cpu()
    tp = torch.as_tensor(tok_ptr).to(torch.int64).cpu()
    G = sp.numel() - 1
    n_sent = sp[1:] - sp[:-1]
    n_tok = tp[sp[1:]] - tp[sp[:-1]]
    cap_t, cap_s = extract_caps()
    over = (n_tok > cap_t) | (n_sent > cap_s)
    inside = ~over
    max_t = int(n_tok[inside].max()) if bool(inside.any()) else 0
    max_s = max(int(n_sent[inside].max()) if bool(inside.any()) else 1, 1)

    def dv(x, dtype):
        return torch.as_tensor(x).to(device=dev, dtype=dtype).contiguous()

    with torch.cuda.device(dev):
        d_sp, d_tp = dv(sp, torch.int64), dv(tp, torch.int64)
        d_tok, d_chars = dv(tokens, torch.int32), dv(sent_chars, torch.int64)
        d_ctx, d_qp, d_qt = dv(ctx_chars, torch.int64), dv(q_ptr, torch.int64), dv(q_tokens, torch.int32)
        n_total = int(tp.numel() - 1)
        sdt = torch.float64 if bm25_type == 0 else torch.float32
        out = Extract(torch.empty(n_total, dtype=torch.uint8, device=dev), torch.empty(G, dtype=torch.int32, device=dev),
                      torch.empty(n_total, dtype=sdt, device=dev) if scores else None)
        if bm25_type == 0:
            tab, off = _log_half(max_s + 1, dev), None
        else:
            tab = _bm25s_idf_table(max_s, dev)
            off = dv(n_sent * (n_sent + 1) // 2, torch.int64)
        if G:
            _lib.check(_lib.lib().ezr_bm25_extract(
                _lib.ptr(d_sp), _lib.ptr(d_tp), _lib.ptr(d_tok), int(vocab), _lib.ptr(d_chars), _lib.ptr(d_ctx),
                _lib.ptr(d_qp), _lib.ptr(d_qt), G, max_t, max_s, _lib.ptr(tab), tab.numel(), _lib.ptr(off), k1, b,
                epsilon, rate, _lib.F64 if bm25_type == 0 else _lib.F32, _lib.ptr(out.scores), _lib.ptr(out.keep),
                _lib.ptr(out.counts), _lib.stream_ptr(stream)), "ezr_bm25_extract")
        over_ids = torch.nonzero(over).flatten().tolist()
        if over_ids:
            qp = torch.as_tensor(q_ptr).to(torch.int64).cpu()
            chars_h = torch.as_tensor(sent_chars).to(torch.int64).cpu().numpy()
            ctx_h = torch.as_tensor(ctx_chars).to(torch.int64).cpu().numpy()
            for g in over_ids:
                s_lo, s_hi = int(sp[g]), int(sp[g + 1])
                t_lo, t_hi = int(tp[s_lo]), int(tp[s_hi])
                stats = Bm25Stats.from_tokens(d_tok[t_lo:t_hi], d_tp[s_lo:s_hi + 1] - t_lo, int(vocab),
                                              bm25_type=bm25_type, k1=k1, b=b, epsilon=epsilon, device=dev)
                index = Bm25Index(stats, device=dev, k1=k1, b=b, packed=False)
                q = d_qt[int(qp[g]):int(qp[g + 1])]
                row = bm25_scores(index, torch.tensor([0, q.numel()], dtype=torch.int32), q, stream=stream)[0]
                keep = _select_host(row.cpu().numpy(), chars_h[s_lo:s_hi], int(ctx_h[g]), rate)
                out.keep[s_lo:s_hi].copy_(torch.from_numpy(keep))
                out.counts[g] = int(keep.sum())
                if scores:
                    out.scores[s_lo:s_hi].copy_(row)
    return out


def select_rows(scores: torch.Tensor, k: int, positive_only: bool = False, doc_group: Optional[torch.Tensor] = None,
                q_group: Optional[torch.Tensor] = None, id_base: int = 0, ws: Optional[Workspace] = None,
                stream=None) -> TopK:
    L = _lib.lib()
    dev = scores.device
    assert scores.dim() == 2 and scores.stride(1) == 1
    st = _lib.F64 if scores.dtype == torch.float64 else _lib.F32
    if scores.dtype not in (torch.float64, torch.float32):
        raise TypeError("scores must be float32 or float64")
    nq, n = scores.shape
    out = TopK(torch.empty(nq, k, dtype=scores.dtype, device=dev), torch.empty(nq, k, dtype=torch.int32, device=dev),
               torch.empty(nq, dtype=torch.int32, device=dev))
    need = L.ezr_select_rows_workspace(nq, n, k, st)
    ws = ws or Workspace(dev)
    buf = ws.get(need)
    dg, qg = _i32(doc_group, dev), _i32(q_group, dev)
    with torch.cuda.device(dev):
        _lib.check(L.ezr_select_rows(_lib.ptr(scores), st, nq, n, scores.stride(0), k, int(positive_only), _lib.ptr(dg),
                                     _lib.ptr(qg), id_base, _lib.ptr(out.scores), _lib.ptr(out.ids), _lib.ptr(out.counts),
                                     _lib.ptr(buf), buf.numel(), _lib.stream_ptr(stream)), "ezr_select_rows")
    return out


def merge_topk_parts(cand_scores: torch.Tensor, cand_ids: torch.Tensor, n_parts: int, part_stride_bytes: int, k: int,
                     out: Optional[TopK] = None, stream=None) -> TopK:
    """Merge ``n_parts`` per-shard top-k lists per query, read in place from an all-gathered byte record.

    ``cand_scores`` / ``cand_ids``: [Q, k_in] views of part 0 inside the gathered buffer; part p of the same
    arrays lies ``p * part_stride_bytes`` further (easyrag_b200/dist.py)."""
    L = _lib.lib()
    dev = cand_scores.device
    assert cand_scores.shape == cand_ids.shape and cand_scores.stride(1) == 1 and cand_ids.stride(1) == 1
    assert cand_ids.dtype == torch.int32 and cand_scores.stride(0) == cand_ids.stride(0)
    st = _lib.F64 if cand_scores.dtype == torch.float64 else _lib.F32
    nq, c = cand_scores.shape
    if out is None:
        out = TopK(torch.empty(nq, k, dtype=cand_scores.dtype, device=dev),
                   torch.empty(nq, k, dtype=torch.int32, device=dev), torch.empty(nq, dtype=torch.int32, device=dev))
    with torch.cuda.device(dev):
        _lib.check(L.ezr_merge_topk_parts(_lib.ptr(cand_scores), _lib.ptr(cand_ids), st, nq, c, cand_scores.stride(0),
                                          n_parts, part_stride_bytes, k, _lib.ptr(out.scores), _lib.ptr(out.ids),
                                          _lib.ptr(out.counts), _lib.stream_ptr(stream)), "ezr_merge_topk_parts")
    return out


def merge_sorted_parts(cand_scores: torch.Tensor, cand_ids: torch.Tensor, n_parts: int, part_stride_bytes: int,
                       k: int, out: Optional[TopK] = None, stream=None) -> TopK:
    """:func:`merge_topk_parts` for k <= 1024, over parts that are each in canonical order up to their first id < 0
    (what every route writes) with ids distinct across parts (disjoint shards): ``ezr_merge_sorted_parts``.

    ``out``: result buffers whose rows may be wider than ``k`` (``out.ids.shape[1]`` = the row stride); the slots past
    each row's count get id -1 and score -inf, so two routes of different depths can share one width."""
    L = _lib.lib()
    dev = cand_scores.device
    assert cand_scores.shape == cand_ids.shape and cand_scores.stride(1) == 1 and cand_ids.stride(1) == 1
    assert cand_ids.dtype == torch.int32 and cand_scores.stride(0) == cand_ids.stride(0)
    st = _lib.F64 if cand_scores.dtype == torch.float64 else _lib.F32
    nq, c = cand_scores.shape
    if out is None:
        out = TopK(torch.empty(nq, k, dtype=cand_scores.dtype, device=dev),
                   torch.empty(nq, k, dtype=torch.int32, device=dev), torch.empty(nq, dtype=torch.int32, device=dev))
    assert out.scores.dtype == cand_scores.dtype and out.ids.dtype == torch.int32 and out.ids.shape[0] == nq
    assert out.scores.shape == out.ids.shape and out.scores.is_contiguous() and out.ids.is_contiguous()
    with torch.cuda.device(dev):
        _lib.check(L.ezr_merge_sorted_parts(_lib.ptr(cand_scores), _lib.ptr(cand_ids), st, nq, c,
                                            cand_scores.stride(0), n_parts, part_stride_bytes, k, _lib.ptr(out.scores),
                                            _lib.ptr(out.ids), _lib.ptr(out.counts), out.ids.shape[1],
                                            _lib.stream_ptr(stream)), "ezr_merge_sorted_parts")
    return out


def merge_topk(cand_scores: torch.Tensor, cand_ids: torch.Tensor, k: int, stream=None) -> TopK:
    """Merge candidate lists [Q, C] (id < 0 = empty) into the canonical top-k."""
    L = _lib.lib()
    dev = cand_scores.device
    assert cand_scores.shape == cand_ids.shape and cand_scores.is_contiguous() and cand_ids.is_contiguous()
    st = _lib.F64 if cand_scores.dtype == torch.float64 else _lib.F32
    nq, c = cand_scores.shape
    cand_ids = cand_ids.to(torch.int32)
    out = TopK(torch.empty(nq, k, dtype=cand_scores.dtype, device=dev), torch.empty(nq, k, dtype=torch.int32, device=dev),
               torch.empty(nq, dtype=torch.int32, device=dev))
    with torch.cuda.device(dev):
        _lib.check(L.ezr_merge_topk(_lib.ptr(cand_scores), _lib.ptr(cand_ids), st, nq, c, c, k,
                                    _lib.ptr(out.scores), _lib.ptr(out.ids), _lib.ptr(out.counts), None, 0,
                                    _lib.stream_ptr(stream)), "ezr_merge_topk")
    return out


def rrf_fuse(ids_a: torch.Tensor, cnt_a: torch.Tensor, ids_b: torch.Tensor, cnt_b: torch.Tensor, k_out: int,
             K: int = 60, canon: Optional[torch.Tensor] = None, stream=None, out: Optional[TopK] = None) -> TopK:
    """HybridRetriever.reciprocal_rank_fusion (retrievers.py:256-274) for a batch; list a = sparse, b = dense."""
    L = _lib.lib()
    dev = ids_a.device
    canon = _device_canon(canon, dev)
    assert ids_a.shape == ids_b.shape and ids_a.dtype == torch.int32 and ids_b.dtype == torch.int32
    nq, stride = ids_a.shape
    if out is None:
        out = TopK(torch.empty(nq, k_out, dtype=torch.float64, device=dev),
                   torch.empty(nq, k_out, dtype=torch.int32, device=dev), torch.empty(nq, dtype=torch.int32, device=dev))
    with torch.cuda.device(dev):
        _lib.check(L.ezr_rrf_fuse(_lib.ptr(ids_a.contiguous()), _lib.ptr(cnt_a), _lib.ptr(ids_b.contiguous()),
                                  _lib.ptr(cnt_b), nq, stride, _lib.ptr(canon), 0, K, k_out, _lib.ptr(out.ids),
                                  _lib.ptr(out.scores), _lib.ptr(out.counts), _lib.stream_ptr(stream)), "ezr_rrf_fuse")
    return out


MAX_UNION = 1024           # k_a + k_b of ezr_pair_union: the pair packer's and the reranker head's per-query limit


@dataclass
class PairUnion:
    ids: torch.Tensor        # [Q, k_a + k_b] int32: distinct ids of list a then list b, first appearance; -1 padded
    counts: torch.Tensor     # [Q] int32
    map_a: torch.Tensor      # [Q, k_a] int32: union index of each list-a slot, -1 past its count
    map_b: torch.Tensor      # [Q, k_b] int32


def pair_union(ids_a: torch.Tensor, cnt_a: torch.Tensor, ids_b: torch.Tensor, cnt_b: torch.Tensor,
               stream=None) -> PairUnion:
    """The per-query union of two candidate lists by document id (``ezr_pair_union``): list a = sparse, b = dense, the
    order of ``rrf_fuse``.  ``ids_x`` int32 [Q, k_x] on the device (row stride may exceed k_x), ``cnt_x`` [Q]."""
    if ids_a.dim() != 2 or ids_b.dim() != 2:
        raise ValueError("ids_a and ids_b must be [Q, k]")
    (nq, ka), (nqb, kb) = ids_a.shape, ids_b.shape
    if nqb != nq or cnt_a.numel() != nq or cnt_b.numel() != nq:
        raise ValueError(f"list a has {nq} queries ({cnt_a.numel()} counts), list b {nqb} ({cnt_b.numel()} counts)")
    if ka < 1 or kb < 1 or ka + kb > MAX_UNION:
        raise ValueError(f"k_a={ka}, k_b={kb}: each must be >= 1 and k_a + k_b <= {MAX_UNION}")
    L = _lib.lib()
    dev = ids_a.device
    ids_a, ids_b = (t.to(torch.int32) for t in (ids_a, ids_b))
    ids_a, ids_b = (t if t.stride(1) == 1 and t.stride(0) >= t.shape[1] else t.contiguous() for t in (ids_a, ids_b))
    cnt_a, cnt_b = _i32(cnt_a, dev), _i32(cnt_b, dev)
    out = PairUnion(torch.empty(nq, ka + kb, dtype=torch.int32, device=dev), torch.empty(nq, dtype=torch.int32, device=dev),
                    torch.empty(nq, ka, dtype=torch.int32, device=dev), torch.empty(nq, kb, dtype=torch.int32, device=dev))
    with torch.cuda.device(dev):
        _lib.check(L.ezr_pair_union(_lib.ptr(ids_a), _lib.ptr(cnt_a), ka, ids_a.stride(0), _lib.ptr(ids_b),
                                    _lib.ptr(cnt_b), kb, ids_b.stride(0), nq, _lib.ptr(out.ids), _lib.ptr(out.counts),
                                    _lib.ptr(out.map_a), _lib.ptr(out.map_b), _lib.stream_ptr(stream)),
                   "ezr_pair_union")
    return out


def _device_canon(canon: Optional[torch.Tensor], dev) -> Optional[torch.Tensor]:
    """The kernels read ``canon`` on the device: a host tensor is copied over (a host address is not valid there)."""
    return None if canon is None else canon.to(device=dev, dtype=torch.int32).contiguous()


def fusion_simple(ids_a: torch.Tensor, sc_a: torch.Tensor, cnt_a: torch.Tensor, ids_b: torch.Tensor, sc_b: torch.Tensor,
                  cnt_b: torch.Tensor, k_out: int, canon: Optional[torch.Tensor] = None, stream=None) -> TopK:
    """HybridRetriever.fusion (retrievers.py:239-253) for a batch."""
    L = _lib.lib()
    dev = ids_a.device
    canon = _device_canon(canon, dev)
    nq, stride = ids_a.shape
    sa = sc_a.to(torch.float64).contiguous()
    sb = sc_b.to(torch.float64).contiguous()
    out = TopK(torch.empty(nq, k_out, dtype=torch.float64, device=dev),
               torch.empty(nq, k_out, dtype=torch.int32, device=dev), torch.empty(nq, dtype=torch.int32, device=dev))
    with torch.cuda.device(dev):
        _lib.check(L.ezr_fusion_simple(_lib.ptr(ids_a.contiguous()), _lib.ptr(sa), _lib.ptr(cnt_a),
                                       _lib.ptr(ids_b.contiguous()), _lib.ptr(sb), _lib.ptr(cnt_b), nq, stride,
                                       _lib.ptr(canon), 0, k_out, _lib.ptr(out.ids), _lib.ptr(out.scores),
                                       _lib.ptr(out.counts), _lib.stream_ptr(stream)), "ezr_fusion_simple")
    return out


def fuse_lists(ids: Sequence[torch.Tensor], counts: Sequence[torch.Tensor], k_out: int, rrf: bool = True, K: int = 60,
               scores: Optional[Sequence[torch.Tensor]] = None, canon: Optional[torch.Tensor] = None, stream=None) -> TopK:
    """``reciprocal_rank_fusion`` / ``fusion`` over ANY number of rank lists (retrievers.py:239-274 loop over a list
    of lists).  ``ids[l]`` int32 [Q, width], ``counts[l]`` int32 [Q], ``scores[l]`` float64 [Q, width] (fusion only);
    all lists share ``width``."""
    import ctypes as C
    L = _lib.lib()
    n = len(ids)
    dev = ids[0].device
    canon = _device_canon(canon, dev)
    nq, width = ids[0].shape
    ids = [t.contiguous() for t in ids]
    assert all(t.shape == (nq, width) and t.dtype == torch.int32 for t in ids) and len(counts) == n
    sc = None
    if not rrf:
        sc = [t.to(torch.float64).contiguous() for t in scores]
        assert all(t.shape == (nq, width) for t in sc)
    out = TopK(torch.empty(nq, k_out, dtype=torch.float64, device=dev),
               torch.empty(nq, k_out, dtype=torch.int32, device=dev), torch.empty(nq, dtype=torch.int32, device=dev))
    arr = lambda ts: (C.c_void_p * n)(*[t.data_ptr() for t in ts])
    with torch.cuda.device(dev):
        _lib.check(L.ezr_fuse_lists(int(rrf), n, arr(ids), arr(sc) if sc is not None else None, arr(counts), nq, width,
                                    _lib.ptr(canon), 0, K, k_out, _lib.ptr(out.ids), _lib.ptr(out.scores),
                                    _lib.ptr(out.counts), _lib.stream_ptr(stream)), "ezr_fuse_lists")
    return out


class CoarseRanker:
    """dense + BM25 + RRF for query batches on one GPU (``HybridRetriever._aretrieve``, retrievers.py:276-291).

    The two routes are independent until the fusion.  ``overlap=True`` issues them on two CUDA streams and
    lets the RRF kernel join them; the default issues them back to back on the caller's stream (the dense
    kernel occupies all shared memory of every SM, so the routes cannot co-reside anyway and per-kernel
    timing stays clean).  All buffers are preallocated per (batch size, k) and reused.
    """

    def __init__(self, dense: DenseIndex, sparse: Bm25Index, canon: Optional[torch.Tensor] = None,
                 overlap: bool = False, depth: int = 2, serial_routes: bool = False):
        assert dense.device == sparse.device
        self.dense, self.sparse = dense, sparse
        self.device = dense.device
        self.canon = None if canon is None else canon.to(device=self.device, dtype=torch.int32).contiguous()
        self.overlap = overlap
        # submit() only: both routes on ONE side stream (BM25, then dense with its full shared-memory ring) instead of
        # side by side; the join still runs on its own stream under the next batch's routes
        self.serial_routes = bool(serial_routes)
        self.depth = max(int(depth), 1)
        self.s_dense = torch.cuda.Stream(device=self.device) if overlap else None
        self.s_sparse = torch.cuda.Stream(device=self.device) if overlap else None
        # the join of a submitted batch (collective, merges, RRF): short kernels, scheduled ahead of the next
        # batch's route CTAs whenever an SM has room
        self.s_tail = torch.cuda.Stream(device=self.device, priority=-1) if overlap else None
        self.ws_dense = Workspace(self.device)
        self.ws_sparse = Workspace(self.device)
        self._bufs = {}
        self._slots = {}
        self._n_submit = 0

    def _buffers(self, nq, kd, ks, ko):
        key = (nq, kd, ks, ko)
        if key not in self._bufs:
            dev = self.device
            mk = lambda dt, *shape: torch.empty(*shape, dtype=dt, device=dev)
            self._bufs[key] = (
                TopK(mk(torch.float32, nq, kd), mk(torch.int32, nq, kd), mk(torch.int32, nq)),
                TopK(mk(self.sparse.score_dtype, nq, ks), mk(torch.int32, nq, ks), mk(torch.int32, nq)),
                TopK(mk(torch.float64, nq, ko), mk(torch.int32, nq, ko), mk(torch.int32, nq)),
            )
        return self._bufs[key]

    def routes(self, queries: torch.Tensor, q_ptr: torch.Tensor, q_terms: torch.Tensor, k: int, k_out: int,
               q_group: Optional[torch.Tensor] = None, d_out: Optional[TopK] = None,
               s_out: Optional[TopK] = None) -> Tuple[TopK, TopK, TopK]:
        """Both routes over this ranker's (shard of the) corpus -> (dense, sparse, fused-output buffer).

        ``d_out`` / ``s_out``: caller-owned result buffers (the sharded ranker passes views of its exchange
        record, so the kernels write straight into the message)."""
        nq = queries.shape[0]
        d_own, s_own, f_out = self._buffers(nq, k, k, k_out)
        d_out = d_own if d_out is None else d_out
        s_out = s_own if s_out is None else s_out
        cur = torch.cuda.current_stream(self.device)
        if self.overlap:
            self.s_dense.wait_stream(cur)
            self.s_sparse.wait_stream(cur)
            # dense first: its persistent CTAs (one per SM) must be resident before the BM25 grid starts filling
            # whatever shared memory / registers / issue slots they leave free
            with torch.cuda.stream(self.s_dense):
                dense_topk(self.dense, queries, k, q_group=q_group, ws=self.ws_dense, stream=self.s_dense, out=d_out)
            with torch.cuda.stream(self.s_sparse):
                bm25_topk(self.sparse, q_ptr, q_terms, k, q_group=q_group, ws=self.ws_sparse, stream=self.s_sparse,
                          out=s_out)
            cur.wait_stream(self.s_sparse)
            cur.wait_stream(self.s_dense)
        else:
            bm25_topk(self.sparse, q_ptr, q_terms, k, q_group=q_group, ws=self.ws_sparse, stream=cur, out=s_out)
            dense_topk(self.dense, queries, k, q_group=q_group, ws=self.ws_dense, stream=cur, out=d_out)
        return d_out, s_out, f_out

    def hybrid(self, queries: torch.Tensor, q_ptr: torch.Tensor, q_terms: torch.Tensor, k_dense: int = 10,
               k_sparse: int = 10, k_out: int = 10, K: int = 60, q_group: Optional[torch.Tensor] = None
               ) -> Tuple[TopK, TopK, TopK]:
        """Returns (fused, sparse, dense).  Inputs must already be on the device."""
        if k_dense != k_sparse:
            raise ValueError("the fused path keeps both routes at the same k (pad the shorter list upstream)")
        d_out, s_out, f_out = self.routes(queries, q_ptr, q_terms, k_dense, k_out, q_group=q_group)
        rrf_fuse(s_out.ids, s_out.counts, d_out.ids, d_out.counts, k_out, K=K, canon=self.canon, out=f_out)
        return f_out, s_out, d_out

    # ---- batch pipelining: submit() returns before the batch is joined to the caller's stream -------------------
    def _slot(self, key, make):
        """Result buffers + events of the next in-flight batch (``depth`` of them per key, used round robin)."""
        if key not in self._slots:
            self._slots[key] = [dict(make(), ev_in=torch.cuda.Event(), ev_d=torch.cuda.Event(),
                                     ev_s=torch.cuda.Event(), done=torch.cuda.Event(), free=torch.cuda.Event())
                                for _ in range(self.depth)]
        slot = self._slots[key][self._n_submit % self.depth]
        self._n_submit += 1
        return slot

    def launch_routes(self, slot, queries, q_ptr, q_terms, k, q_group, d_out: TopK, s_out: TopK) -> None:
        """Both routes on their streams, ordered after (a) the caller's stream at this point (the inputs), (b) the
        join that last read this slot's buffers and (c) the consumer's release of the slot.  Nothing is joined back
        to the caller's stream: ``slot['ev_d']`` / ``slot['ev_s']`` mark the two routes' results."""
        if not self.overlap:
            raise RuntimeError("submit() needs CoarseRanker(overlap=True): the routes and the join run on own streams")
        cur = torch.cuda.current_stream(self.device)
        slot["ev_in"].record(cur)
        s_sp = self.s_dense if self.serial_routes else self.s_sparse
        for st in ((self.s_dense,) if self.serial_routes else (self.s_dense, self.s_sparse)):
            st.wait_event(slot["ev_in"])
            st.wait_event(slot["done"])          # never-recorded events do not block
            st.wait_event(slot["free"])
        if self.serial_routes:
            with torch.cuda.stream(s_sp):
                bm25_topk(self.sparse, q_ptr, q_terms, k, q_group=q_group, ws=self.ws_sparse, stream=s_sp, out=s_out)
                slot["ev_s"].record(s_sp)
        with torch.cuda.stream(self.s_dense):
            dense_topk(self.dense, queries, k, q_group=q_group, ws=self.ws_dense, stream=self.s_dense, out=d_out)
            slot["ev_d"].record(self.s_dense)
        if not self.serial_routes:
            with torch.cuda.stream(s_sp):
                bm25_topk(self.sparse, q_ptr, q_terms, k, q_group=q_group, ws=self.ws_sparse, stream=s_sp, out=s_out)
                slot["ev_s"].record(s_sp)

    def submit(self, queries: torch.Tensor, q_ptr: torch.Tensor, q_terms: torch.Tensor, k: int = 10, k_out: int = 10,
               K: int = 60, q_group: Optional[torch.Tensor] = None) -> "Ticket":
        """:meth:`hybrid` for a stream of independent batches: the same kernels, but the batch is NOT joined to the
        caller's stream, so the routes of the next submitted batch start while this batch's RRF (and, sharded, its
        all-gather and merges) are still running.  Up to ``depth`` batches are in flight; a slot's buffers are
        rewritten ``depth`` submits later, after its join has finished and -- if the consumer reads them on another
        stream -- after :meth:`Ticket.release`.  Read the results after :meth:`Ticket.wait` or :meth:`join`."""
        nq = queries.shape[0]

        def make():
            mk = lambda dt, *shape: torch.empty(*shape, dtype=dt, device=self.device)
            return dict(d=TopK(mk(torch.float32, nq, k), mk(torch.int32, nq, k), mk(torch.int32, nq)),
                        s=TopK(mk(self.sparse.score_dtype, nq, k), mk(torch.int32, nq, k), mk(torch.int32, nq)),
                        f=TopK(mk(torch.float64, nq, k_out), mk(torch.int32, nq, k_out), mk(torch.int32, nq)))
        slot = self._slot((nq, k, k_out), make)
        self.launch_routes(slot, queries, q_ptr, q_terms, k, q_group, slot["d"], slot["s"])
        with torch.cuda.stream(self.s_tail):
            self.s_tail.wait_event(slot["ev_d"])
            self.s_tail.wait_event(slot["ev_s"])
            rrf_fuse(slot["s"].ids, slot["s"].counts, slot["d"].ids, slot["d"].counts, k_out, K=K, canon=self.canon,
                     out=slot["f"], stream=self.s_tail)
            slot["done"].record(self.s_tail)
        return Ticket(slot["f"], slot["s"], slot["d"], slot)

    def join(self) -> None:
        """The caller's stream waits for every submitted batch."""
        cur = torch.cuda.current_stream(self.device)
        for st in (self.s_tail, self.s_dense, self.s_sparse):
            if st is not None:
                cur.wait_stream(st)


class Ticket:
    """A submitted batch: result buffers (valid once ``done`` has fired) and the slot they live in."""
    __slots__ = ("fused", "sparse", "dense", "_slot")

    def __init__(self, fused: TopK, sparse: TopK, dense: TopK, slot: dict):
        self.fused, self.sparse, self.dense, self._slot = fused, sparse, dense, slot

    @property
    def done(self) -> torch.cuda.Event:
        return self._slot["done"]

    def wait(self, stream: Optional[torch.cuda.Stream] = None) -> None:
        (stream or torch.cuda.current_stream(self.fused.ids.device)).wait_event(self._slot["done"])

    def release(self, stream: Optional[torch.cuda.Stream] = None) -> None:
        """Call on the stream that read the results, after the reads: the slot may be rewritten once they finish."""
        self._slot["free"].record(stream or torch.cuda.current_stream(self.fused.ids.device))


class HostPipeline:
    """Host-buffer front end of the batched path: pinned host inputs in, pinned host results out, every call.

    ``step`` enqueues, without blocking the host: H2D of the query vectors / term pointers / term ids on a copy
    stream, both routes + (all-gather, merge) + RRF on the caller's stream, D2H of the fused ids and float64 scores
    on a second copy stream.  Inputs are double buffered on the device, so the copies of step i+1 run under the
    kernels of step i; a result buffer is only reused once its D2H has completed.  With a ranker built with
    ``overlap=True`` the steps are *submitted* (``CoarseRanker.submit``): the join and the D2H of step i run under the
    route kernels of step i+1.  ``ranker`` is a
    :class:`CoarseRanker` or an :class:`easyrag_b200.dist.ShardedCoarseRanker`.
    """

    def __init__(self, ranker, n_queries: int, dim: int, max_terms: int, k: int = 10, k_out: int = 10, depth: int = 2,
                 pipelined: Optional[bool] = None):
        base = getattr(ranker, "ranker", ranker)
        self.ranker, self.k, self.k_out = ranker, k, k_out
        # pipelined (default whenever the ranker runs its routes on own streams): steps are submitted, not joined
        self.pipelined = bool(base.overlap) if pipelined is None else bool(pipelined)
        self.device = dev = base.device
        self.sharded = base is not ranker
        self.s_in = torch.cuda.Stream(device=dev)
        self.s_out = torch.cuda.Stream(device=dev)
        self.slots = []
        for _ in range(depth):
            self.slots.append(dict(
                qvec=torch.empty(n_queries, dim, dtype=torch.bfloat16, device=dev),
                ptr=torch.empty(n_queries + 1, dtype=torch.int32, device=dev),
                terms=torch.empty(max(max_terms, 1), dtype=torch.int32, device=dev),
                ev_in=torch.cuda.Event(), ev_free=torch.cuda.Event()))
        self.ev_done = torch.cuda.Event()
        self.ev_out = torch.cuda.Event()
        self.n = 0

    def step(self, h_qvec: torch.Tensor, h_ptr: torch.Tensor, h_terms: torch.Tensor, h_ids_out: torch.Tensor,
             h_scores_out: torch.Tensor, q_group: Optional[torch.Tensor] = None) -> None:
        """One batch.  ``h_*`` are pinned host tensors: bf16 [Q, D], int32 [Q+1], int32 [T] in; int32 [Q, k_out] and
        float64 [Q, k_out] out (valid after :meth:`drain` or a synchronize)."""
        slot = self.slots[self.n % len(self.slots)]
        self.n += 1
        nq, nt = h_qvec.shape[0], h_terms.numel()
        if nq != slot["qvec"].shape[0] or nt > slot["terms"].numel():
            raise ValueError("HostPipeline is sized at construction: same batch size, at most max_terms term ids")
        cur = torch.cuda.current_stream(self.device)
        with torch.cuda.stream(self.s_in):
            self.s_in.wait_event(slot["ev_free"])            # the kernels that last read this slot have finished
            slot["qvec"].copy_(h_qvec, non_blocking=True)
            slot["ptr"].copy_(h_ptr, non_blocking=True)
            slot["terms"][:nt].copy_(h_terms, non_blocking=True)
            slot["ev_in"].record(self.s_in)
        cur.wait_event(slot["ev_in"])
        if self.pipelined:
            # the batch is not joined to the caller's stream: the routes of the next step start while this step's
            # join (all-gather, merges, RRF) and its D2H are still running
            if self.sharded:
                t = self.ranker.submit(slot["qvec"], slot["ptr"], slot["terms"], k=self.k, k_out=self.k_out,
                                       q_group=q_group)
            else:
                t = self.ranker.submit(slot["qvec"], slot["ptr"], slot["terms"], self.k, self.k_out, q_group=q_group)
            slot["ev_free"] = t.done                         # both routes have read the inputs once the join has run
            with torch.cuda.stream(self.s_out):
                t.wait(self.s_out)
                h_ids_out.copy_(t.fused.ids, non_blocking=True)
                h_scores_out.copy_(t.fused.scores, non_blocking=True)
                t.release(self.s_out)                        # the result slot may be rewritten after these copies
                self.ev_out.record(self.s_out)
            return
        cur.wait_event(self.ev_out)                          # the previous results have left the fused buffer
        if self.sharded:
            fused = self.ranker.hybrid(slot["qvec"], slot["ptr"], slot["terms"], k=self.k, k_out=self.k_out,
                                       q_group=q_group)[0]
        else:
            fused = self.ranker.hybrid(slot["qvec"], slot["ptr"], slot["terms"], self.k, self.k, self.k_out,
                                       q_group=q_group)[0]
        slot["ev_free"].record(cur)
        self.ev_done.record(cur)
        with torch.cuda.stream(self.s_out):
            self.s_out.wait_event(self.ev_done)
            h_ids_out.copy_(fused.ids, non_blocking=True)
            h_scores_out.copy_(fused.scores, non_blocking=True)
            self.ev_out.record(self.s_out)

    def drain(self) -> None:
        """Make the caller's stream wait for every copy enqueued so far (then a stream / event sync covers them)."""
        torch.cuda.current_stream(self.device).wait_event(self.ev_out)


def dual_sparse_fusion(chunk_index: Bm25Index, path_index: Bm25Index, q_ptr: torch.Tensor, q_terms: torch.Tensor,
                       path_q_ptr: torch.Tensor, path_q_terms: torch.Tensor, k_chunk: int, k_path: int, k_out: int,
                       canon: Optional[torch.Tensor] = None, q_group: Optional[torch.Tensor] = None,
                       ws: Optional[Workspace] = None) -> TopK:
    """The reference's maintained coarse ranker as one batched op (pipeline.py:357-365): chunk-text BM25
    (k = f_topk_2) and knowledge-path BM25 (k = f_topk_3) over the same nodes, merged by ``HybridRetriever.fusion``
    (text-dedup, stable sort by raw score).  The two indexes have their own vocabularies, hence two term lists."""
    dev = chunk_index.device
    a = bm25_topk(chunk_index, q_ptr, q_terms, k_chunk, q_group=q_group, ws=ws)
    b = bm25_topk(path_index, path_q_ptr, path_q_terms, k_path, q_group=q_group, ws=ws)
    width = max(k_chunk, k_path)

    def pad(t: TopK, k: int):
        if k == width:
            return t.ids, t.scores.to(torch.float64)
        ids = torch.full((t.ids.shape[0], width), -1, dtype=torch.int32, device=dev)
        sc = torch.zeros(t.ids.shape[0], width, dtype=torch.float64, device=dev)
        ids[:, :k] = t.ids
        sc[:, :k] = t.scores
        return ids, sc
    ia, sa = pad(a, k_chunk)
    ib, sb = pad(b, k_path)
    return fusion_simple(ia, sa, a.counts, ib, sb, b.counts, k_out, canon=canon)
