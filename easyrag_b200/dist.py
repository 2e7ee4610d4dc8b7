"""Row-sharded coarse ranking (SURVEY.md section 8(e)) and pair-split fine ranking across the GPUs of one box.

The reference is single-process; this is new.  Corpus rows (and the BM25 document axis) are cut
into contiguous shards, one per rank; queries are replicated.  Corpus-global BM25 statistics
(idf, avgdl) are shared, so every shard scores exactly as the unsharded index would.  Each rank
computes its local dense and BM25 top-k with *global* ids straight into one byte record and a
SINGLE all-gather (NCCL over NVLink on GPUs, gloo in the CPU tests) exchanges the records;
every rank then merges G*k candidates per route under the canonical order -- the same order
the 1-GPU path uses, hence identical rank lists -- reading the gathered buffer in place, and
runs RRF.  ``hybrid`` / ``submit`` merge lists of k <= 32 (``ezr_merge_topk_parts``);
``pipeline_hybrid`` and :class:`ShardedDualSparseRanker` run the pipeline's depths (k <= 1024 per route) and merge the
sorted per-shard lists by rank (``ezr_merge_sorted_parts``).

Fine ranking (:class:`ShardedCrossEncoderReranker`) splits the other way: every rank holds the whole cross-encoder and
the same candidate lists, the (query, candidate) pairs are cut into token-balanced runs, one per rank, and ONE
all-reduce of a [P] fp32 score vector gives every rank every pair's score; each rank then orders all queries.  Its
``rerank_fusion`` splits the pairs of the union of two candidate lists the same way.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.distributed as dist


def shard_bounds(n_rows: int, world: int, rank: int, align: int = 1) -> Tuple[int, int]:
    """Contiguous, ordered, exhaustive, BALANCED split of ``n_rows``.

    The rows are cut into ``ceil(n_rows / align)`` units of ``align`` rows (the last may be short); every rank gets
    ``units // world`` of them and the first ``units % world`` ranks one more, so shard sizes differ by at most
    ``align`` rows.  Shard-local indexes use local ids (ranges and tiles restart at the shard's first row), so
    nothing requires a coarse alignment: the default is 1."""
    units = -(-n_rows // align)
    base, extra = divmod(units, world)
    lo_u = rank * base + min(rank, extra)
    hi_u = lo_u + base + (1 if rank < extra else 0)
    return min(n_rows, lo_u * align), min(n_rows, hi_u * align)


def _packed(sizes):
    """Offsets of arrays of ``sizes`` bytes placed back to back, each at a 16-byte boundary -> (offsets, total)."""
    o, out = 0, []
    for s in sizes:
        out.append(o)
        o += (s + 15) // 16 * 16
    return out, o


@dataclass
class RecordLayout:
    """Byte layout of one rank's contribution: dense scores f32 | dense ids i32 | sparse scores | sparse ids i32.

    The dense arrays are [Q, k], the sparse ones [Q, k_sparse] (``None``: the same k)."""
    n_queries: int
    k: int
    sparse_bytes: int      # 8 for BM25Okapi (float64), 4 for bm25s (float32)
    k_sparse: Optional[int] = None

    @property
    def ks(self) -> int:
        return self.k if self.k_sparse is None else self.k_sparse

    @property
    def sizes(self):
        n, ns = self.n_queries * self.k, self.n_queries * self.ks
        return (n * 4, n * 4, ns * self.sparse_bytes, ns * 4)

    @property
    def offsets(self):
        return _packed(self.sizes)

    @property
    def nbytes(self) -> int:
        return self.offsets[1]


def record_views(layout: RecordLayout, buf: torch.Tensor):
    """The four per-route arrays of one rank's record as typed views of the byte buffer ``buf`` (dense scores f32
    and ids i32 [Q, k], sparse scores f64/f32 and ids i32 [Q, k_sparse]): writing through them fills the message in
    place, reading them from a gathered buffer needs no unpacking."""
    offs, _ = layout.offsets
    q, k, ks = layout.n_queries, layout.k, layout.ks
    sdt = torch.float64 if layout.sparse_bytes == 8 else torch.float32
    out = []
    for off, size, dt, w in zip(offs, layout.sizes, (torch.float32, torch.int32, sdt, torch.int32), (k, k, ks, ks)):
        out.append(buf[off:off + size].view(dt).view(q, w))
    return out


MAX_DEEP_K = 1024          # per-route depth of the deep merge (ezr_merge_sorted_parts)


def _check_depth(name: str, k: int) -> None:
    if not 1 <= k <= MAX_DEEP_K:
        raise ValueError(f"{name}={k} out of [1, {MAX_DEEP_K}]")


def _merged(nq: int, width: int, score_dtype, dev):
    """A [Q, width] result buffer of the deep merge (rows wider than a route's k are padded with id -1)."""
    from .batched import TopK
    return TopK(torch.empty(nq, width, dtype=score_dtype, device=dev), torch.empty(nq, width, dtype=torch.int32, device=dev),
                torch.empty(nq, dtype=torch.int32, device=dev))


def _narrow(t, k: int):
    from .batched import TopK
    return TopK(t.scores[:, :k], t.ids[:, :k], t.counts)


class ShardedCoarseRanker:
    """dense + BM25 + RRF over a row-sharded corpus; every rank returns the full fused result.

    Per (batch size, k) one record buffer and one gather buffer are allocated once.  The two route kernels write
    their top-k straight into the record (typed views), ONE ``all_gather_into_tensor`` exchanges the records, and the
    merge kernel reads the gathered buffer in place (``ezr_merge_topk_parts``): no pack/unpack kernels, no per-step
    allocations.
    """

    def __init__(self, ranker, group=None):
        """``ranker``: :class:`easyrag_b200.batched.CoarseRanker` over this rank's shard (indexes built with
        ``row_lo`` / ``doc_lo`` = the shard's first global row)."""
        self.ranker = ranker
        self.group = group
        self.world = dist.get_world_size(group)
        self.rank = dist.get_rank(group)
        self._state = {}

    def _make(self, nq: int, k: int, sparse_dtype):
        from .batched import TopK
        dev = self.ranker.device
        layout = RecordLayout(nq, k, 8 if sparse_dtype == torch.float64 else 4)
        record = torch.zeros(layout.nbytes, dtype=torch.uint8, device=dev)
        gathered = torch.zeros(self.world * layout.nbytes, dtype=torch.uint8, device=dev)
        ds, di, ss, si = record_views(layout, record)
        cnt = lambda: torch.empty(nq, dtype=torch.int32, device=dev)
        mk = lambda dt: torch.empty(nq, k, dtype=dt, device=dev)
        return dict(
            layout=layout, record=record, gathered=gathered,
            d_local=TopK(ds, di, cnt()), s_local=TopK(ss, si, cnt()),
            views=record_views(layout, gathered[:layout.nbytes]),
            dense=TopK(mk(torch.float32), mk(torch.int32), cnt()),
            sparse=TopK(mk(sparse_dtype), mk(torch.int32), cnt()))

    def _buffers(self, nq: int, k: int, sparse_dtype):
        key = (nq, k, sparse_dtype)
        if key not in self._state:
            self._state[key] = self._make(nq, k, sparse_dtype)
        return self._state[key]

    def _join(self, st, k: int, k_out: int, K: int, canon, f_out, stream=None):
        """all-gather of the records, per-route merge of the world's lists, RRF -- on the current stream."""
        from . import batched
        dist.all_gather_into_tensor(st["gathered"], st["record"], group=self.group)   # the one collective
        g_ds, g_di, g_ss, g_si = st["views"]
        nbytes = st["layout"].nbytes
        dense = batched.merge_topk_parts(g_ds, g_di, self.world, nbytes, k, out=st["dense"], stream=stream)
        sparse = batched.merge_topk_parts(g_ss, g_si, self.world, nbytes, k, out=st["sparse"], stream=stream)
        fused = batched.rrf_fuse(sparse.ids, sparse.counts, dense.ids, dense.counts, k_out, K=K, canon=canon, out=f_out,
                                 stream=stream)
        return fused, sparse, dense

    def hybrid(self, queries, q_ptr, q_terms, k: int = 10, k_out: int = 10, K: int = 60, q_group=None,
               canon: Optional[torch.Tensor] = None):
        from . import batched
        r = self.ranker
        nq = queries.shape[0]
        if k > 32:
            raise ValueError("the sharded path merges per-shard lists of k <= 32")
        st = self._buffers(nq, k, r.sparse.score_dtype)
        _, _, f_out = r.routes(queries, q_ptr, q_terms, k, k_out, q_group=q_group, d_out=st["d_local"],
                               s_out=st["s_local"])
        return self._join(st, k, k_out, K, canon if canon is not None else r.canon, f_out)

    def submit(self, queries, q_ptr, q_terms, k: int = 10, k_out: int = 10, K: int = 60, q_group=None,
               canon: Optional[torch.Tensor] = None):
        """:meth:`hybrid` without the join to the caller's stream (see ``CoarseRanker.submit``): the all-gather, the
        merges and the RRF of this batch run on the ranker's join stream while the routes of the next submitted
        batch already occupy the SMs.  Every rank must submit the same sequence of batches (one collective each)."""
        from . import batched
        r = self.ranker
        nq = queries.shape[0]
        if k > 32:
            raise ValueError("the sharded path merges per-shard lists of k <= 32")

        def make():
            st = self._make(nq, k, r.sparse.score_dtype)
            st["f"] = batched.TopK(torch.empty(nq, k_out, dtype=torch.float64, device=r.device),
                                   torch.empty(nq, k_out, dtype=torch.int32, device=r.device),
                                   torch.empty(nq, dtype=torch.int32, device=r.device))
            return st
        slot = r._slot(("sharded", id(self), nq, k, k_out), make)
        r.launch_routes(slot, queries, q_ptr, q_terms, k, q_group, slot["d_local"], slot["s_local"])
        with torch.cuda.stream(r.s_tail):
            r.s_tail.wait_event(slot["ev_d"])
            r.s_tail.wait_event(slot["ev_s"])
            fused, sparse, dense = self._join(slot, k, k_out, K, canon if canon is not None else r.canon, slot["f"],
                                              stream=r.s_tail)
            slot["done"].record(r.s_tail)
        return batched.Ticket(fused, sparse, dense, slot)

    def join(self) -> None:
        self.ranker.join()

    def pipeline_hybrid(self, queries, q_ptr, q_terms, k_dense: int = 288, k_sparse: int = 192, k_out: int = 256,
                        K: int = 60, q_group=None, canon: Optional[torch.Tensor] = None, dense_cand: bool = False):
        """dense top-``k_dense`` + BM25 top-``k_sparse`` + RRF to ``k_out`` at the pipeline's depths (pipeline.py's
        f_topk_1 / f_topk_2 / f_topk), each route k in [1, 1024] -> (fused, sparse, dense), bit-identical to one GPU
        running ``dense_topk(k_dense)`` + ``bm25_topk(k_sparse)`` + ``fuse_lists`` over the whole corpus.

        Both routes run on the caller's stream and write straight into one record (:class:`RecordLayout` with
        ``k_sparse``); ONE ``all_gather_into_tensor`` exchanges it; ``ezr_merge_sorted_parts`` merges each route's G
        sorted lists in place into a [Q, W] buffer, W = max(k_dense, k_sparse), the one width the RRF kernel takes.
        ``sparse`` / ``dense`` are [Q, k] views of those buffers.  Buffers are allocated once per shape.

        Memory: the gathered buffer holds G * Q * (8 * k_dense + (S + 4) * k_sparse) bytes, S the BM25 score size (8
        for Okapi, 4 for bm25s): 369 MB at G = 8, Q = 10k, 288 / 192, float64.  Batches are not split into query
        blocks, so a very large Q needs the caller to split it.

        ``dense_cand=True`` runs the dense route with ``dense_topk_cand`` (form 6's scores without score rows) on every
        shard; the result is then bit-identical to one GPU running ``dense_topk_cand`` in place of ``dense_topk``."""
        from . import batched
        _check_depth("k_dense", k_dense)
        _check_depth("k_sparse", k_sparse)
        if k_out < 1:
            raise ValueError(f"k_out={k_out} must be >= 1")
        r = self.ranker
        nq = queries.shape[0]
        key = ("deep", nq, k_dense, k_sparse, k_out)
        if key not in self._state:
            dev, sdt = r.device, r.sparse.score_dtype
            layout = RecordLayout(nq, k_dense, 8 if sdt == torch.float64 else 4, k_sparse=k_sparse)
            record = torch.zeros(layout.nbytes, dtype=torch.uint8, device=dev)
            gathered = torch.zeros(self.world * layout.nbytes, dtype=torch.uint8, device=dev)
            ds, di, ss, si = record_views(layout, record)
            cnt = lambda: torch.empty(nq, dtype=torch.int32, device=dev)
            width = max(k_dense, k_sparse)
            self._state[key] = dict(
                layout=layout, record=record, gathered=gathered,
                d_local=batched.TopK(ds, di, cnt()), s_local=batched.TopK(ss, si, cnt()),
                views=record_views(layout, gathered[:layout.nbytes]),
                dense=_merged(nq, width, torch.float32, dev), sparse=_merged(nq, width, sdt, dev),
                fused=_merged(nq, k_out, torch.float64, dev))
        st = self._state[key]
        batched.bm25_topk(r.sparse, q_ptr, q_terms, k_sparse, q_group=q_group, ws=r.ws_sparse, out=st["s_local"])
        if dense_cand:
            batched.dense_topk_cand(r.dense, queries, k_dense, q_group=q_group, ws=r.ws_dense, out=st["d_local"])
        else:
            batched.dense_topk(r.dense, queries, k_dense, q_group=q_group, ws=r.ws_dense, out=st["d_local"])
        dist.all_gather_into_tensor(st["gathered"], st["record"], group=self.group)   # the one collective
        g_ds, g_di, g_ss, g_si = st["views"]
        nbytes = st["layout"].nbytes
        dense = batched.merge_sorted_parts(g_ds, g_di, self.world, nbytes, k_dense, out=st["dense"])
        sparse = batched.merge_sorted_parts(g_ss, g_si, self.world, nbytes, k_sparse, out=st["sparse"])
        fused = batched.rrf_fuse(sparse.ids, sparse.counts, dense.ids, dense.counts, k_out, K=K,
                                 canon=canon if canon is not None else r.canon, out=st["fused"])
        return fused, _narrow(sparse, k_sparse), _narrow(dense, k_dense)


class ShardedDualSparseRanker:
    """``batched.dual_sparse_fusion`` over a row-sharded corpus (the reference's default coarse ranker, pipeline.py:
    357-365: chunk-text BM25 top-k_chunk + knowledge-path BM25 top-k_path + ``HybridRetriever.fusion``); every rank
    returns the full result, bit-identical to ``dual_sparse_fusion`` over the unsharded indexes.

    Both indexes are this rank's shard (``doc_lo`` / ``doc_hi``, corpus-global statistics, global ids).  The two
    lists go into one record, ONE ``all_gather_into_tensor`` exchanges it, ``ezr_merge_sorted_parts`` merges each
    list's G sorted parts in place, and ``ezr_fusion_simple`` fuses the merged lists.  Record and gather buffers are
    allocated once per shape; the gathered buffer holds G * Q * (S_c + 4) * k_chunk + G * Q * (S_p + 4) * k_path bytes
    (S the score size of each index: 8 for Okapi, 4 for bm25s)."""

    def __init__(self, chunk_index, path_index, canon: Optional[torch.Tensor] = None, group=None):
        from .batched import Workspace
        assert chunk_index.device == path_index.device
        self.chunk, self.path = chunk_index, path_index
        self.device = chunk_index.device
        self.canon = None if canon is None else canon.to(device=self.device, dtype=torch.int32).contiguous()
        self.group = group
        self.world = dist.get_world_size(group)
        self.rank = dist.get_rank(group)
        self.ws = Workspace(self.device)
        self._state = {}

    def _make(self, nq: int, k_chunk: int, k_path: int):
        from .batched import TopK
        dev = self.device
        dts = (self.chunk.score_dtype, torch.int32, self.path.score_dtype, torch.int32)
        shapes = ((nq, k_chunk), (nq, k_chunk), (nq, k_path), (nq, k_path))
        sizes = [q * k * torch.empty(0, dtype=dt).element_size() for (q, k), dt in zip(shapes, dts)]
        offs, nbytes = _packed(sizes)
        record = torch.zeros(nbytes, dtype=torch.uint8, device=dev)
        gathered = torch.zeros(self.world * nbytes, dtype=torch.uint8, device=dev)

        def views(buf):
            return [buf[o:o + s].view(dt).view(*shp) for o, s, dt, shp in zip(offs, sizes, dts, shapes)]
        cs, ci, ps, pi = views(record)
        cnt = lambda: torch.empty(nq, dtype=torch.int32, device=dev)
        width = max(k_chunk, k_path)
        return dict(nbytes=nbytes, record=record, gathered=gathered, c_local=TopK(cs, ci, cnt()),
                    p_local=TopK(ps, pi, cnt()), views=views(gathered[:nbytes]),
                    chunk=_merged(nq, width, self.chunk.score_dtype, dev),
                    path=_merged(nq, width, self.path.score_dtype, dev))

    def fuse(self, q_ptr, q_terms, path_q_ptr, path_q_terms, k_chunk: int = 192, k_path: int = 6, k_out: int = 256,
             q_group=None):
        """Same arguments and result as ``batched.dual_sparse_fusion`` (the term lists of each index's vocabulary);
        ``k_chunk`` and ``k_path`` in [1, 1024]."""
        from . import batched
        _check_depth("k_chunk", k_chunk)
        _check_depth("k_path", k_path)
        if k_out < 1:
            raise ValueError(f"k_out={k_out} must be >= 1")
        nq = q_ptr.numel() - 1
        if path_q_ptr.numel() - 1 != nq:
            raise ValueError(f"{nq} chunk queries but {path_q_ptr.numel() - 1} path queries")
        key = (nq, k_chunk, k_path)
        if key not in self._state:
            self._state[key] = self._make(nq, k_chunk, k_path)
        st = self._state[key]
        batched.bm25_topk(self.chunk, q_ptr, q_terms, k_chunk, q_group=q_group, ws=self.ws, out=st["c_local"])
        batched.bm25_topk(self.path, path_q_ptr, path_q_terms, k_path, q_group=q_group, ws=self.ws, out=st["p_local"])
        dist.all_gather_into_tensor(st["gathered"], st["record"], group=self.group)   # the one collective
        g_cs, g_ci, g_ps, g_pi = st["views"]
        a = batched.merge_sorted_parts(g_cs, g_ci, self.world, st["nbytes"], k_chunk, out=st["chunk"])
        b = batched.merge_sorted_parts(g_ps, g_pi, self.world, st["nbytes"], k_path, out=st["path"])
        return batched.fusion_simple(a.ids, a.scores, a.counts, b.ids, b.scores, b.counts, k_out, canon=self.canon)


def token_balanced_ranges(cu_h: Sequence[int], world: int) -> List[Tuple[int, int]]:
    """Contiguous, ordered, exhaustive runs ``[lo, hi)`` of whole pairs, one per rank, with about equal token counts.

    ``cu_h`` int [P + 1] holds the pairs' token offsets (T = ``cu_h[-1]``).  Rank r's run starts at the first pair whose
    start token is >= r T / world, so a run holds less than T / world tokens plus the length of its last pair.  A run is
    empty when P < world or when a long pair spans a whole share."""
    if world < 1:
        raise ValueError(f"world={world} must be >= 1")
    cu = np.asarray(cu_h, dtype=np.int64)
    n, t = cu.size - 1, int(cu[-1])
    starts = cu[:-1] * world                          # start * world >= r * T  <=>  start >= r * T / world, exactly
    bounds = [int(np.searchsorted(starts, r * t, side="left")) for r in range(world)] + [n]
    return [(bounds[r], bounds[r + 1]) for r in range(world)]


def exchange_pair_scores(sig: torch.Tensor, group=None) -> torch.Tensor:
    """In place: each rank's ``sig`` float32 [P] holds the scores of its own run of pairs and +0.0 everywhere else;
    afterwards every rank holds all P scores, bit for bit.

    One ``all_reduce(SUM)``.  It is exact in any reduction order: every element has at most one contribution that is not
    +0.0, a sigmoid is never negative (an underflow gives +0.0, never -0.0), and x + (+0.0) == x for every x >= +0.0.
    Compared with an all-gather it needs no padding to the longest run and no copy into place afterwards: the scoring
    kernel writes straight into the buffer that is reduced.  The message is 4 bytes per pair either way."""
    dist.all_reduce(sig, op=dist.ReduceOp.SUM, group=group)
    return sig


def check_replicated(values: Sequence[int], what: str, group=None, device="cpu") -> None:
    """Raise ``ValueError`` on every rank unless every rank passed the same ``values`` (one small all-gather)."""
    world = dist.get_world_size(group)
    mine = torch.tensor(list(values), dtype=torch.int64, device=device)
    every = torch.empty(world * mine.numel(), dtype=torch.int64, device=device)
    dist.all_gather_into_tensor(every, mine, group=group)
    rows = every.view(world, -1).cpu()
    if not bool((rows == rows[0]).all()):
        raise ValueError(f"{what} differ across ranks (one row per rank): {rows.tolist()}; every rank must pass "
                         f"the same input")


class ShardedCrossEncoderReranker:
    """:class:`easyrag_b200.rerank.CrossEncoderReranker` with the pairs split across ranks; every rank returns the full
    result, bit-identical to one GPU's.

    Every rank packs all pairs (deterministic and cheap, and it gives every rank the pairs' token offsets), then encodes
    only its run of them (:func:`token_balanced_ranges`): the chunked encoder, the CLS rows, Linear + bias and the
    per-pair sigmoid (``ezr_cross_pair_scores``) into its slice of a zeroed [P] fp32 buffer.  One
    :func:`exchange_pair_scores` per batch completes the buffer and every rank orders all queries
    (``ezr_cross_order_topk``).  A pair's score does not depend on the encoder pass it is in, hence the bit-identity.

    ``cand``, ``q_ptr`` and ``q_tok`` must be the same on every rank (``ShardedCoarseRanker``'s output is); the
    candidate shape and the pair and token totals are compared across ranks with one small all-gather per call.  With
    no process group, or a group of one, this is the wrapped reranker on one GPU.
    """

    def __init__(self, reranker, group=None):
        """``reranker``: a :class:`easyrag_b200.rerank.CrossEncoderReranker` on this rank's device (same model and
        passages on every rank)."""
        self.reranker = reranker
        self.group = group
        self.distributed = dist.is_available() and dist.is_initialized()
        self.world = dist.get_world_size(group) if self.distributed else 1
        self.rank = dist.get_rank(group) if self.distributed else 0
        nccl = self.distributed and dist.get_backend(group) == dist.Backend.NCCL
        self._check_device = reranker.device if nccl else "cpu"

    def rerank(self, cand, q_ptr: torch.Tensor, q_tok: torch.Tensor, top_n: int,
               events: Optional[List[torch.cuda.Event]] = None):
        """Same arguments and results as ``CrossEncoderReranker.rerank``.  The stage events bracket: packing and the
        cross-rank input check; this rank's encoder run; its head, the score exchange (which waits for the slowest
        rank) and the order."""
        from . import _lib
        from .batched import TopK
        from .encoder import gemm
        from .rerank import MAX_CANDIDATES, _mark
        L = _lib.lib()
        rr = self.reranker
        m, dev = rr.model, rr.device
        if cand.ids.dim() == 2 and cand.ids.shape[1] > MAX_CANDIDATES:
            raise ValueError(f"k={cand.ids.shape[1]} candidates per query; at most {MAX_CANDIDATES} are supported")
        if top_n < 1:
            raise ValueError("top_n must be >= 1")
        _mark(events)
        pairs = rr.pack(cand.ids, cand.counts, q_ptr, q_tok)
        nq, k, n_pairs, d = pairs.n_queries, pairs.k, pairs.n_pairs, m.cfg.hidden_size
        if self.distributed:
            check_replicated((nq, k, n_pairs, int(pairs.cu_h[-1])), "candidate shape [Q, k], pair and token totals",
                             self.group, self._check_device)
        _mark(events)
        lo, hi = token_balanced_ranges(pairs.cu_h, self.world)[self.rank]
        out = TopK(torch.empty(nq, top_n, dtype=torch.float32, device=dev),
                   torch.empty(nq, top_n, dtype=torch.int32, device=dev), torch.empty(nq, dtype=torch.int32, device=dev))
        all_scores = torch.empty(nq, k, dtype=torch.float32, device=dev)
        sig = torch.zeros(n_pairs, dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            if hi > lo:
                cls = torch.empty(hi - lo, d, dtype=torch.bfloat16, device=dev)
                for p0, p1 in rr.chunks(pairs.cu_h[lo:hi + 1]):
                    rr._encode_cls(pairs, lo + p0, lo + p1, cls[p0:p1])
            _mark(events)
            if hi > lo:
                dense = gemm(cls, m.w1, bias=m.b1)
                _lib.check(L.ezr_cross_pair_scores(_lib.ptr(dense), d, hi - lo, _lib.ptr(m.w2), m.b2,
                                                   _lib.ptr(sig[lo:hi]), _lib.stream_ptr()), "ezr_cross_pair_scores")
            if self.distributed and n_pairs:
                exchange_pair_scores(sig, self.group)
            _lib.check(L.ezr_cross_order_topk(_lib.ptr(sig), _lib.ptr(pairs.pair_off), nq, k, _lib.ptr(pairs.cand_ids),
                                              pairs.cand_ids.stride(0), top_n, _lib.ptr(all_scores),
                                              _lib.ptr(out.scores), _lib.ptr(out.ids), _lib.ptr(out.counts),
                                              _lib.stream_ptr()), "ezr_cross_order_topk")
            _mark(events)
        return out, all_scores

    def rerank_fusion(self, sparse, dense, q_ptr: torch.Tensor, q_tok: torch.Tensor, top_n: int, k_out: int,
                      K: int = 60, canon: Optional[torch.Tensor] = None,
                      events: Optional[List[torch.cuda.Event]] = None):
        """Same arguments and result as ``CrossEncoderReranker.rerank_fusion``, bit-identical to it: every rank builds
        and packs the union of the two lists, encodes its token-balanced run of the union's pairs, and after one
        :func:`exchange_pair_scores` orders both routes and fuses them.  The cross-rank check covers both list shapes
        and the union's pair and token totals.  Stage events as in :meth:`rerank`."""
        from .rerank import _mark
        rr = self.reranker
        _mark(events)
        union, pairs = rr._union_pack(sparse, dense, q_ptr, q_tok, top_n, k_out)
        if self.distributed:
            check_replicated((pairs.n_queries, union.map_a.shape[1], union.map_b.shape[1], pairs.n_pairs,
                              int(pairs.cu_h[-1])), "list shapes [Q, k_sparse], [Q, k_dense], union pair and token "
                             "totals", self.group, self._check_device)
        _mark(events)
        lo, hi = token_balanced_ranges(pairs.cu_h, self.world)[self.rank]
        sig = torch.zeros(pairs.n_pairs, dtype=torch.float32, device=rr.device)
        with torch.cuda.device(rr.device):
            rr._score_run(pairs, lo, hi, sig, events)
            if self.distributed and pairs.n_pairs:
                exchange_pair_scores(sig, self.group)
            out = rr._fusion_orders(sig, pairs, union, sparse, dense, top_n, k_out, K, canon)
            _mark(events)
        return out
