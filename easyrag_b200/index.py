"""Index construction for the two coarse-ranking routes.

* :class:`Bm25Stats` -- corpus statistics exactly as ``rank_bm25.BM25Okapi.__init__`` /
  ``bm25s.BM25.index`` derive them (reference call sites retrievers.py:98-118): document
  frequencies, ``avgdl``, ``idf`` with the epsilon floor.  The transcendental part (``math.log``)
  and the order-sensitive float64 sum stay on the host so they are bit-identical to CPython
  (SURVEY.md section 7 "hard parts"); counting tf/df, sorting and placing the postings run in this
  library's own kernels (csrc/bm25_build.cu: per-document shared-memory sort, block-ordered placement).
* :class:`Bm25Index` -- device-resident term-major postings with the per-posting contribution
  precomputed by ``ezr_bm25_weights`` (CUDA, round-to-nearest, no FMA), plus the range table the
  query kernel uses.  Needs a GPU; there is no CPU path.
* :class:`DenseIndex` -- the bf16 corpus matrix that replaces the Qdrant collection
  (ingestion.py:155-191), with the optional ``dir`` class per row for payload filters.
"""
from __future__ import annotations

import json
import math
import os
from dataclasses import dataclass
from typing import Optional

import numpy as np
import torch

from . import _lib

K1, B, EPSILON = 1.5, 0.75, 0.25     # retrievers.py:103-105


def bm25s_idf(n_docs: int, df: int) -> float:
    """bm25s' idf of a term found in ``df`` of ``n_docs`` documents, in float64 (indexes store its float32)."""
    return math.log(1 + (n_docs - df + 0.5) / (df + 0.5))


@dataclass
class Bm25Stats:
    n_docs: int
    vocab: int
    bm25_type: int                 # 0 = BM25Okapi (float64), 1 = bm25s lucene (float32)
    avgdl: float
    doc_len: torch.Tensor          # int32 [N]
    df: torch.Tensor               # int64 [V]
    idf: np.ndarray                # float64 [V] (type 1: float32 values widened)
    indptr: torch.Tensor           # int64 [V+1]
    post_doc: torch.Tensor         # int32 [P], ascending within a term
    post_tf: torch.Tensor          # int32 [P]
    average_idf: float = 0.0

    @staticmethod
    def from_tokens(tokens: torch.Tensor, doc_ptr: torch.Tensor, vocab: int, bm25_type: int = 0,
                    k1: float = K1, b: float = B, epsilon: float = EPSILON, device=None) -> "Bm25Stats":
        """``tokens`` int32/int64 [T] term ids, ``doc_ptr`` int64 [N+1].  Counting, sorting and placing run in this
        library's own kernels (csrc/bm25_build.cu); there is no CPU implementation."""
        n = doc_ptr.numel() - 1
        if n == 0:
            raise ZeroDivisionError("division by zero")      # rank_bm25: avgdl = num_doc / corpus_size
        _lib.require_cuda()
        L = _lib.lib()
        if device is None:
            device = tokens.device if tokens.is_cuda else torch.device("cuda")
        device = torch.device(device)
        import ctypes
        with torch.cuda.device(device):
            tok = tokens.to(device=device, dtype=torch.int32).contiguous()
            ptr = doc_ptr.to(device=device, dtype=torch.int64).contiguous()
            lens = ptr[1:] - ptr[:-1]
            total = int(ptr[-1])
            max_len = int(lens.max())
            cap = 8192                                       # kBuildCap: longer documents sort in a global scratch
            long_docs = long_off = long_keys = None
            n_long = 0
            if max_len > cap:
                idx = torch.nonzero(lens > cap).flatten()
                n_long = int(idx.numel())
                ll = lens[idx].cpu().tolist()
                sizes = [1 << (int(x) - 1).bit_length() for x in ll]
                offs = [0]
                for z in sizes[:-1]:
                    offs.append(offs[-1] + z)
                long_docs = idx.to(torch.int32).contiguous()
                long_off = torch.tensor(offs, dtype=torch.int64, device=device)
                long_keys = torch.empty(sum(sizes), dtype=torch.int64, device=device)
            ws = torch.empty(L.ezr_bm25_build_workspace(n, total, vocab), dtype=torch.uint8, device=device)
            df = torch.empty(vocab, dtype=torch.int64, device=device)
            indptr = torch.empty(vocab + 1, dtype=torch.int64, device=device)
            first_pos = torch.empty(vocab, dtype=torch.int64, device=device)
            status = ctypes.c_int32(0)
            st = _lib.stream_ptr()
            _lib.check(L.ezr_bm25_build_count(_lib.ptr(tok), _lib.ptr(ptr), n, total, vocab, max_len, _lib.ptr(df),
                                              _lib.ptr(indptr), _lib.ptr(first_pos), _lib.ptr(long_docs),
                                              _lib.ptr(long_off), _lib.ptr(long_keys), n_long, _lib.ptr(ws), ws.numel(),
                                              ctypes.byref(status), st), "ezr_bm25_build_count")
            if status.value != 0:
                raise ValueError(f"token id out of range [0, vocab) in document {status.value - 1}")
            n_post = int(indptr[-1])
            post_doc = torch.empty(n_post, dtype=torch.int32, device=device)
            post_tf = torch.empty(n_post, dtype=torch.int32, device=device)
            _lib.check(L.ezr_bm25_build_fill(_lib.ptr(ptr), n, total, vocab, _lib.ptr(indptr), _lib.ptr(post_doc),
                                             _lib.ptr(post_tf), _lib.ptr(ws), ws.numel(), st), "ezr_bm25_build_fill")
            torch.cuda.current_stream().synchronize()
            del ws
        return Bm25Stats.from_counts(n, vocab, total, lens.to(torch.int32), df, indptr, post_doc, post_tf,
                                     first_pos.cpu().numpy(), bm25_type=bm25_type, epsilon=epsilon)

    @staticmethod
    def from_counts(n_docs: int, vocab: int, total_tokens: int, doc_len: torch.Tensor, df: torch.Tensor,
                    indptr: torch.Tensor, post_doc: torch.Tensor, post_tf: torch.Tensor, first_pos: np.ndarray,
                    bm25_type: int = 0, epsilon: float = EPSILON) -> "Bm25Stats":
        """The host-exact part of the index build: ``avgdl`` and ``idf`` exactly as rank_bm25 / bm25s derive them
        from the counted arrays (``math.log`` per term, a sequential float64 sum in first-seen term order).
        ``first_pos[t]``: corpus position of term t's first occurrence (only its ORDER matters)."""
        n = n_docs
        avgdl = total_tokens / n
        df_host = df.cpu().numpy()
        present = np.nonzero(df_host)[0]
        idf = np.zeros(vocab, dtype=np.float64)
        average_idf = 0.0
        if bm25_type == 0:
            # rank_bm25 _calc_idf: idf = log(N - n + 0.5) - log(n + 0.5); sequential float64 sum over
            # terms in first-seen order; negatives replaced by epsilon * mean.
            vals = np.array([math.log(n - int(d) + 0.5) - math.log(int(d) + 0.5) for d in df_host[present]],
                            dtype=np.float64)
            idf[present] = vals
            if present.size:
                order = np.argsort(np.asarray(first_pos)[present].astype(np.uint64), kind="stable")
                seq = np.cumsum(vals[order])          # np.cumsum is a plain left-to-right float64 sum
                average_idf = float(seq[-1]) / present.size
                neg = present[vals < 0]
                idf[neg] = epsilon * average_idf
        elif bm25_type == 1:
            vals = np.array([bm25s_idf(n, int(d)) for d in df_host[present]], dtype=np.float64).astype(np.float32)
            idf[present] = vals.astype(np.float64)
        else:
            raise ValueError("bm25_type must be 0 (BM25Okapi) or 1 (bm25s)")
        return Bm25Stats(n_docs=n, vocab=vocab, bm25_type=bm25_type, avgdl=avgdl, doc_len=doc_len.to(torch.int32),
                         df=df, idf=idf, indptr=indptr, post_doc=post_doc, post_tf=post_tf,
                         average_idf=average_idf)


INDEX_FORMAT_VERSION = 1


def _save_arrays(path: str, meta: dict, arrays: dict) -> None:
    os.makedirs(path, exist_ok=True)
    for name, t in arrays.items():
        np.save(os.path.join(path, name + ".npy"), t.detach().cpu().view(torch.int16).numpy()
                if t.dtype == torch.bfloat16 else t.detach().cpu().numpy())
    meta = dict(meta, format_version=INDEX_FORMAT_VERSION,
                bf16=[n for n, t in arrays.items() if t.dtype == torch.bfloat16])
    with open(os.path.join(path, "meta.json"), "w") as f:
        json.dump(meta, f)


def _load_arrays(path: str):
    with open(os.path.join(path, "meta.json")) as f:
        meta = json.load(f)
    if meta.get("format_version") != INDEX_FORMAT_VERSION:
        raise ValueError(f"{path}: index format {meta.get('format_version')} != {INDEX_FORMAT_VERSION}")

    def get(name):
        # start-up is an mmap, not a re-tokenise: a private copy-on-write mapping of the .npy payload; the pages go
        # from the page cache straight into the H2D copy (no intermediate host array)
        a = np.load(os.path.join(path, name + ".npy"), mmap_mode="c")
        t = torch.from_numpy(a)
        return t.view(torch.bfloat16) if name in meta.get("bf16", []) else t
    return meta, get


class Bm25Index:
    """Device-resident BM25 index over documents ``[doc_lo, doc_hi)`` of a corpus described by ``stats``.

    Global statistics (idf, avgdl) always come from the whole corpus so that a row-sharded index
    scores exactly like the unsharded one (SURVEY.md 8(e)).

    ``packed``: build the 4-byte packed postings that let ``ezr_bm25_topk`` run the two-phase path (integer
    candidate pass + exact rescoring) for 1 <= k <= 1024.  ``None`` (default) packs float64 (Okapi) indexes and
    leaves float32 (bm25s) ones on the ordered kernel; ``True`` packs either type; ``False`` packs neither.  Results
    are the same bytes either way.
    """

    def __init__(self, stats: Bm25Stats, device=None, doc_lo: int = 0, doc_hi: Optional[int] = None,
                 doc_group: Optional[torch.Tensor] = None, k1: float = K1, b: float = B,
                 packed: Optional[bool] = None):
        _lib.require_cuda()
        self._packed_opt = packed
        L = _lib.lib()
        device = torch.device(device if device is not None else "cuda")
        doc_hi = stats.n_docs if doc_hi is None else doc_hi
        self.stats = stats
        self.doc_lo, self.doc_hi = doc_lo, doc_hi
        self.n_docs = doc_hi - doc_lo
        self.vocab = stats.vocab
        self.score_type = _lib.F64 if stats.bm25_type == 0 else _lib.F32
        self.score_dtype = torch.float64 if stats.bm25_type == 0 else torch.float32
        self.device = device
        with torch.cuda.device(device):
            post_doc = stats.post_doc.to(device).contiguous()
            post_tf = stats.post_tf.to(device).contiguous()
            indptr = stats.indptr.to(device).contiguous()
            if doc_lo != 0 or doc_hi != stats.n_docs:
                # a row shard's postings are a contiguous sub-segment of every term's (document-sorted) list
                first = torch.empty(stats.vocab, dtype=torch.int64, device=device)
                df_local = torch.empty(stats.vocab, dtype=torch.int64, device=device)
                ind_local = torch.empty(stats.vocab + 1, dtype=torch.int64, device=device)
                _lib.check(L.ezr_bm25_shard_count(_lib.ptr(indptr), _lib.ptr(post_doc), stats.vocab, doc_lo, doc_hi,
                                                  _lib.ptr(first), _lib.ptr(df_local), _lib.ptr(ind_local),
                                                  _lib.stream_ptr()), "ezr_bm25_shard_count")
                n_local = int(ind_local[-1])
                doc_l = torch.empty(n_local, dtype=torch.int32, device=device)
                tf_l = torch.empty(n_local, dtype=torch.int32, device=device)
                _lib.check(L.ezr_bm25_shard_copy(_lib.ptr(first), _lib.ptr(ind_local), _lib.ptr(post_doc),
                                                 _lib.ptr(post_tf), stats.vocab, doc_lo, _lib.ptr(doc_l), _lib.ptr(tf_l),
                                                 _lib.stream_ptr()), "ezr_bm25_shard_copy")
                indptr, post_doc, post_tf = ind_local, doc_l, tf_l
            self.indptr = indptr.contiguous()
            self.post_doc = post_doc.contiguous()
            self.n_postings = int(self.post_doc.numel())
            st = _lib.stream_ptr()
            doc_len = stats.doc_len[doc_lo:doc_hi].to(device).contiguous()
            kd = torch.empty(self.n_docs, dtype=torch.float64, device=device)
            _lib.check(L.ezr_bm25_doc_norm(_lib.ptr(doc_len), self.n_docs, k1, b, 1 - b, stats.avgdl,
                                           _lib.ptr(kd), st), "ezr_bm25_doc_norm")
            idf_dev = torch.from_numpy(stats.idf).to(device)
            self.post_w = torch.empty(self.n_postings, dtype=self.score_dtype, device=device)
            num_scale = (k1 + 1) if stats.bm25_type == 0 else 1.0
            _lib.check(L.ezr_bm25_weights(_lib.ptr(self.indptr), _lib.ptr(self.post_doc), _lib.ptr(post_tf.contiguous()),
                                          self.vocab, self.n_postings, _lib.ptr(idf_dev), _lib.ptr(kd), num_scale,
                                          self.score_type, _lib.ptr(self.post_w), st), "ezr_bm25_weights")
            self.n_ranges = (self.n_docs + _lib.BM25_RANGE - 1) // _lib.BM25_RANGE
            self.range_off = torch.empty(self.vocab * (self.n_ranges + 1), dtype=torch.int32, device=device)
            _lib.check(L.ezr_bm25_range_index(_lib.ptr(self.indptr), _lib.ptr(self.post_doc), self.vocab,
                                              _lib.BM25_RANGE, self.n_ranges, _lib.ptr(self.range_off), st),
                       "ezr_bm25_range_index")
            self.doc_group = None
            if doc_group is not None:
                self.doc_group = doc_group[doc_lo:doc_hi].to(device=device, dtype=torch.int32).contiguous()
            # rank_bm25 replaces negative idf by epsilon * average_idf, which is negative only when the mean idf is
            self.monotone = bool((stats.idf >= 0).all())
            self._build_packed()
            torch.cuda.current_stream().synchronize()
        self._struct = None
        self.refresh_struct()

    def _build_packed(self):
        """4-byte packed postings for the candidate pass of ``ezr_bm25_topk`` (derived data, never stored on disk).

        Only indices with non-negative contributions qualify.  With ``packed=None`` float64 indices are packed
        unless ``EASYRAG_B200_BM25_PACKED=0`` (keeps the ordered single-pass kernel, A/B measurements) and float32
        (bm25s) ones are not; ``packed=True`` packs both (float32 weights through ``ezr_bm25_pack_f32``)."""
        self.post_pk, self.pk_scale_log2, self.term_max = None, 0, None
        want = getattr(self, "_packed_opt", None)
        if want is None:
            want = self.score_type == _lib.F64 and os.environ.get("EASYRAG_B200_BM25_PACKED", "1") != "0"
        if not want or not self.monotone or self.n_postings == 0 or _lib.lib().ezr_bm25_cand_capacity() == 0:
            return
        import ctypes
        pack = _lib.lib().ezr_bm25_pack if self.score_type == _lib.F64 else _lib.lib().ezr_bm25_pack_f32
        with torch.cuda.device(self.device):
            pk = torch.empty(self.n_postings, dtype=torch.int32, device=self.device)
            scratch = torch.empty(2, dtype=torch.int64, device=self.device)
            e = ctypes.c_int32(0)
            _lib.check(pack(_lib.ptr(self.post_doc), _lib.ptr(self.post_w), self.n_postings, _lib.BM25_RANGE,
                            _lib.ptr(pk), ctypes.byref(e), _lib.ptr(scratch), _lib.stream_ptr()), "ezr_bm25_pack")
            # per-term maximum of the packed weights: lets the candidate pass skip a query's lowest-weight terms
            tmax = torch.empty(self.vocab, dtype=torch.int32, device=self.device)
            _lib.check(_lib.lib().ezr_bm25_term_max(_lib.ptr(self.indptr), _lib.ptr(pk), self.vocab, _lib.ptr(tmax),
                                                    _lib.stream_ptr()), "ezr_bm25_term_max")
        self.post_pk, self.pk_scale_log2, self.term_max = pk, int(e.value), tmax

    def refresh_struct(self):
        s = _lib.Bm25IndexStruct()
        s.n_docs, s.n_postings, s.vocab = self.n_docs, self.n_postings, self.vocab
        s.score_type, s.range_size, s.n_ranges = self.score_type, _lib.BM25_RANGE, self.n_ranges
        s.indptr = self.indptr.data_ptr()
        s.post_doc = self.post_doc.data_ptr()
        s.post_w = self.post_w.data_ptr()
        s.range_off = self.range_off.data_ptr()
        s.doc_group = self.doc_group.data_ptr() if self.doc_group is not None else None
        s.monotone = int(self.monotone)
        s.pk_scale_log2 = int(self.pk_scale_log2)
        s.post_pk = self.post_pk.data_ptr() if self.post_pk is not None else None
        s.term_max = self.term_max.data_ptr() if getattr(self, "term_max", None) is not None else None
        self._struct = s

    def ordered_view(self) -> "Bm25Index":
        """The same device arrays without the packed postings: ``ezr_bm25_topk`` then runs the ordered kernel (float64
        or float32).  Two independent kernel paths over one index = a full-size self-check (bench.py --self-check)."""
        import copy
        v = copy.copy(self)
        v._packed_opt = False
        v.post_pk, v.pk_scale_log2, v.term_max = None, 0, None
        v._struct = None
        v.refresh_struct()
        return v

    def set_doc_group(self, doc_group: Optional[torch.Tensor]):
        self.doc_group = None if doc_group is None else doc_group.to(device=self.device, dtype=torch.int32).contiguous()
        self.refresh_struct()

    @property
    def struct(self):
        import ctypes
        return ctypes.byref(self._struct)

    def index_bytes(self) -> int:
        return (self.post_doc.numel() * 4 + self.post_w.numel() * self.post_w.element_size()
                + self.range_off.numel() * 4 + self.indptr.numel() * 8
                + (self.post_pk.numel() * 4 + self.term_max.numel() * 4 if self.post_pk is not None else 0))

    # ---- on-disk format (SURVEY.md 8(f).1: the reference rebuilds the BM25 index in RAM on every start,
    # retrievers.py:98-118).  A directory of .npy arrays + meta.json; loading needs no tokenisation and no log().
    def save(self, path: str) -> None:
        arrays = dict(indptr=self.indptr, post_doc=self.post_doc, post_w=self.post_w, range_off=self.range_off)
        if self.doc_group is not None:
            arrays["doc_group"] = self.doc_group
        _save_arrays(path, dict(kind="bm25", n_docs=self.n_docs, vocab=self.vocab, score_type=self.score_type,
                                doc_lo=self.doc_lo, doc_hi=self.doc_hi, n_ranges=self.n_ranges,
                                range_size=_lib.BM25_RANGE, monotone=bool(self.monotone)), arrays)

    @classmethod
    def load(cls, path: str, device=None, packed: Optional[bool] = None) -> "Bm25Index":
        _lib.require_cuda()
        meta, get = _load_arrays(path)
        if meta["kind"] != "bm25" or meta["range_size"] != _lib.BM25_RANGE:
            raise ValueError(f"{path}: not a BM25 index of this build")
        self = cls.__new__(cls)
        self._packed_opt = packed
        device = torch.device(device if device is not None else "cuda")
        self.stats = None
        self.device = device
        self.n_docs, self.vocab, self.score_type = meta["n_docs"], meta["vocab"], meta["score_type"]
        self.doc_lo, self.doc_hi, self.n_ranges = meta["doc_lo"], meta["doc_hi"], meta["n_ranges"]
        self.score_dtype = torch.float64 if self.score_type == _lib.F64 else torch.float32
        self.indptr = get("indptr").to(device)
        self.post_doc = get("post_doc").to(device)
        self.post_w = get("post_w").to(device)
        self.range_off = get("range_off").to(device)
        self.n_postings = int(self.post_doc.numel())
        self.monotone = bool(meta.get("monotone", False))
        self.doc_group = get("doc_group").to(device) if os.path.exists(os.path.join(path, "doc_group.npy")) else None
        self._build_packed()
        self._struct = None
        self.refresh_struct()
        return self


def normalize_rows(x: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    """out (bf16 [n, d], may be a slice of a larger matrix) = L2-normalised rows of x (float32 or bf16, on the device)."""
    assert x.dim() == 2 and out.shape == x.shape and x.stride(1) == 1 and out.stride(1) == 1
    assert out.dtype == torch.bfloat16 and x.dtype in (torch.float32, torch.bfloat16) and x.device == out.device
    with torch.cuda.device(x.device):
        _lib.check(_lib.lib().ezr_normalize_rows(_lib.ptr(x), int(x.dtype == torch.float32), x.stride(0), x.shape[0],
                                                 x.shape[1], _lib.ptr(out), out.stride(0), _lib.stream_ptr()),
                   "ezr_normalize_rows")
    return out


def check_quantizable(dim: int) -> None:
    """The int8 scan (csrc/dense_s8.cu) takes 128-byte k-chunks of at most 1024 values."""
    if dim % 128 != 0 or not 128 <= dim <= 1024:
        raise ValueError(f"a quantized dense index needs dim % 128 == 0 and dim <= 1024 (got {dim})")


class DenseIndex:
    """Row-major bf16 matrix of L2-normalised chunk embeddings (rows ``[row_lo, row_hi)`` of the corpus).

    The matrix lives in a buffer with spare capacity: :meth:`reserve` + :meth:`rows_for_append` hand out slices
    the encoder writes into directly (``embed_packed`` -> slice, no Python lists, no rebuild), :meth:`append`
    copies / normalises a block of new rows behind the existing ones in amortised O(new rows).

    ``quantized=True`` keeps an int8 mirror of the rows (per-row scale, error and norm bounds, and the corpus-wide
    maxima of the last two) in step with the bf16 rows: :func:`easyrag_b200.batched.dense_topk` then runs the
    certified int8 pass + exact rescoring of ``ezr_dense_s8_topk``, which returns the same kind of exact result.
    Rows written in place through :meth:`rows_for_append` are quantized at :meth:`commit`.  The quantized search is
    currently slower than the bf16 one on unit-vector corpora (its certified margin admits too many candidates; see
    the README) and synchronises its stream once per call.
    """

    def __init__(self, vectors: Optional[torch.Tensor], device=None, row_lo: int = 0,
                 doc_group: Optional[torch.Tensor] = None, normalize: bool = False, dim: Optional[int] = None,
                 capacity: int = 0, quantized: bool = False):
        _lib.require_cuda()
        device = torch.device(device if device is not None else "cuda")
        self.device = device
        self.row_lo = row_lo
        self.quantized = bool(quantized)
        if vectors is None and dim is None:
            raise ValueError("DenseIndex: pass vectors or dim")
        if self.quantized:
            check_quantizable(dim if vectors is None else vectors.shape[1])
        if vectors is None:
            if dim is None:
                raise ValueError("DenseIndex: pass vectors or dim")
            self._buf = torch.empty(max(capacity, 0), dim, dtype=torch.bfloat16, device=device)
            self.n_rows, self.dim = 0, dim
        else:
            v = vectors.to(device)
            if normalize:
                src = v if v.dtype in (torch.float32, torch.bfloat16) else v.float()
                buf = torch.empty(max(capacity, v.shape[0]), v.shape[1], dtype=torch.bfloat16, device=device)
                normalize_rows(src.contiguous(), buf[:v.shape[0]])
            elif capacity > v.shape[0]:
                buf = torch.empty(capacity, v.shape[1], dtype=torch.bfloat16, device=device)
                buf[:v.shape[0]].copy_(v)
            else:
                buf = v.to(torch.bfloat16).contiguous()
            self._buf = buf
            self.n_rows, self.dim = v.shape
        self.doc_group = None if doc_group is None else doc_group.to(device=device, dtype=torch.int32).contiguous()
        if self.quantized:
            self._alloc_mirror(self._buf.shape[0])
            self._quantize(0, self.n_rows)

    @property
    def vectors(self) -> torch.Tensor:
        """The live rows (a view of the capacity buffer)."""
        return self._buf[:self.n_rows]

    # ---- int8 mirror: rows, per-row scale / error bound / norm bound, maxima = [max error, max norm]
    def _alloc_mirror(self, cap: int) -> None:
        dev = self.device
        self._s8 = torch.empty(cap, self.dim, dtype=torch.int8, device=dev)
        self._scale = torch.empty(cap, dtype=torch.float32, device=dev)
        self._err = torch.empty(cap, dtype=torch.float32, device=dev)
        self._norm = torch.empty(cap, dtype=torch.float32, device=dev)
        self.maxima = torch.zeros(2, dtype=torch.float32, device=dev)

    def _quantize(self, lo: int, hi: int) -> None:
        if hi <= lo:
            return
        x = self._buf[lo:hi]
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().ezr_dense_quantize_rows(
                _lib.ptr(x), x.stride(0), hi - lo, self.dim, _lib.ptr(self._s8[lo:hi]), self._s8.stride(0),
                _lib.ptr(self._scale[lo:hi]), _lib.ptr(self._err[lo:hi]), _lib.ptr(self._norm[lo:hi]),
                _lib.ptr(self.maxima), _lib.stream_ptr()), "ezr_dense_quantize_rows")

    @property
    def rows_s8(self) -> torch.Tensor:
        return self._s8[:self.n_rows]

    @property
    def row_scale(self) -> torch.Tensor:
        return self._scale[:self.n_rows]

    @property
    def row_err(self) -> torch.Tensor:
        return self._err[:self.n_rows]

    @property
    def row_norm(self) -> torch.Tensor:
        return self._norm[:self.n_rows]

    def index_bytes(self) -> int:
        """Device bytes of the live rows (bf16, plus the int8 mirror and its per-row floats when quantized)."""
        n = self.n_rows * self.dim * 2
        if self.quantized:
            n += self.n_rows * (self.dim + 12) + 8
        return n

    def reserve(self, n_rows: int) -> None:
        """Make room for ``n_rows`` rows in total (geometric growth, one copy of the live rows when it grows)."""
        if n_rows <= self._buf.shape[0]:
            return
        cap = max(n_rows, int(self._buf.shape[0] * 1.5) + 64)
        buf = torch.empty(cap, self.dim, dtype=torch.bfloat16, device=self.device)
        buf[:self.n_rows].copy_(self._buf[:self.n_rows])
        self._buf = buf
        if self.quantized:
            old = (self._s8, self._scale, self._err, self._norm, self.maxima)
            self._alloc_mirror(cap)
            for dst, src in zip((self._s8, self._scale, self._err, self._norm), old[:4]):
                dst[:self.n_rows].copy_(src[:self.n_rows])
            self.maxima = old[4]

    def rows_for_append(self, n: int) -> torch.Tensor:
        """A writable [n, dim] bf16 slice right behind the live rows; call :meth:`commit` once it is filled."""
        self.reserve(self.n_rows + n)
        return self._buf[self.n_rows:self.n_rows + n]

    def commit(self, n: int) -> None:
        if self.quantized:
            self._quantize(self.n_rows, self.n_rows + n)
        self.n_rows += n
        self.doc_group = None            # per-row classes are rebuilt by the owner (they depend on the filter keys)

    def append(self, vectors: torch.Tensor, normalize: bool = False) -> None:
        v = vectors.to(self.device)
        if v.shape[1] != self.dim:
            raise ValueError(f"append: dim {v.shape[1]} != {self.dim}")
        dst = self.rows_for_append(v.shape[0])
        if normalize:
            normalize_rows((v if v.dtype in (torch.float32, torch.bfloat16) else v.float()).contiguous(), dst)
        else:
            dst.copy_(v)
        self.commit(v.shape[0])

    def save(self, path: str) -> None:
        arrays = dict(vectors=self.vectors)
        if self.doc_group is not None:
            arrays["doc_group"] = self.doc_group
        if self.quantized:
            arrays.update(rows_s8=self.rows_s8, row_scale=self.row_scale, row_err=self.row_err,
                          row_norm=self.row_norm, maxima=self.maxima)
        _save_arrays(path, dict(kind="dense", n_rows=self.n_rows, dim=self.dim, row_lo=self.row_lo,
                                quantized=self.quantized), arrays)

    @classmethod
    def load(cls, path: str, device=None) -> "DenseIndex":
        """A directory saved with the int8 mirror loads quantized (the mirror as saved); one without loads bf16."""
        meta, get = _load_arrays(path)
        if meta["kind"] != "dense":
            raise ValueError(f"{path}: not a dense index")
        dg = get("doc_group") if os.path.exists(os.path.join(path, "doc_group.npy")) else None
        self = cls(get("vectors"), device=device, row_lo=meta["row_lo"], doc_group=dg)
        if meta.get("quantized", False):
            check_quantizable(self.dim)
            self.quantized = True
            self._alloc_mirror(self._buf.shape[0])
            for dst, name in ((self._s8, "rows_s8"), (self._scale, "row_scale"), (self._err, "row_err"),
                              (self._norm, "row_norm")):
                dst[:self.n_rows].copy_(get(name))
            self.maxima.copy_(get("maxima"))
        return self
