"""Fine ranking with a cross-encoder on the GPU: ``SentenceTransformerRerank`` (reference: rerankers.py:15-99).

The reference scores every (query, candidate) pair with ``CrossEncoder(model, max_length=512).predict`` -- a BERT or
XLM-RoBERTa ``*ForSequenceClassification`` with one label, sigmoid on the logit -- and keeps the ``top_n`` candidates
by ``sorted(nodes, key=lambda x: -x.score if x.score else 0)``.  Here:

* ``CrossEncoderModel``     - the checkpoint: the encoder stack is this library's ``BertEncoder`` (wgmma GEMMs and
  attention), plus the classification head's weights.
* ``CrossEncoderReranker``  - the batched device path: a ``[Q, k]`` ``TopK`` of the coarse ranker -> the pairs packed
  on the device from passages tokenised once (csrc/handoff.cu), the encoder run in chunks of whole pairs under a
  token budget, the CLS rows through Linear + bias (ezr_pool_normalize + ezr_gemm_bf16), then tanh / dot / sigmoid
  and the per-query order in one kernel (csrc/rerank.cu).  ``rerank_fusion`` reranks a sparse and a dense list
  separately and fuses them by RRF (pipeline.py:393-452), encoding the pairs of both lists once (csrc/rerank_fusion.cu).
* ``SentenceTransformerRerank`` - the drop-in node postprocessor, built on the batched path with one query.
"""
from __future__ import annotations

import ctypes
from dataclasses import dataclass
from typing import Any, Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib
from .batched import TopK, Workspace
from .encoder import POOL_CLS, BertConfig, BertEncoder, PackedBatch, gemm, random_state
from .schema import BaseNodePostprocessor, Field, MetadataMode, NodeWithScore, PrivateAttr, QueryBundle

DEFAULT_SENTENCE_TRANSFORMER_MAX_LENGTH = 512
DEFAULT_MAX_TOKENS = 65536
MAX_CANDIDATES = 1024          # candidates per query the ordering kernel holds (one CTA per query)
MAX_CHUNK_PAIRS = 65535        # sequences one attention call takes (ezr_attn_bidir refuses more, for either kernel)

# family -> (separators between the two segments, token type of the second segment); see ezr_cross_pack_plan
_TEMPLATES = {"bert": (1, 1), "roberta": (2, 0)}


class CrossEncoderModel:
    """A one-label BERT / (XLM-)RoBERTa sequence classifier on the GPU.

    ``state`` uses transformers' ``BertForSequenceClassification`` names (``bert.*``, ``bert.pooler.dense.*``,
    ``classifier.*``) or ``(XLM)RobertaForSequenceClassification`` names (``roberta.*``, ``classifier.dense.*``,
    ``classifier.out_proj.*``).  ``cls_id`` / ``sep_id`` are the tokenizer's ``[CLS]`` / ``[SEP]`` (``<s>`` / ``</s>``)
    ids; ``pad_id`` is RoBERTa's ``padding_idx``, from which its position ids start (``pad_id + 1``).
    """

    def __init__(self, family: str, cfg: BertConfig, state: Dict[str, torch.Tensor], cls_id: int, sep_id: int,
                 pad_id: int = 1, device="cuda"):
        if family not in _TEMPLATES:
            raise ValueError(f"family must be 'bert' or 'roberta', not {family!r}")
        if cfg.hidden_size % cfg.num_attention_heads or cfg.head_dim not in (64, 128):
            raise ValueError(f"head_dim {cfg.hidden_size / cfg.num_attention_heads:g} is not supported: the attention "
                             f"kernels take head_dim 64 or 128")
        prefix = "bert." if family == "bert" else "roberta."
        if family == "bert":
            w1, b1 = state["bert.pooler.dense.weight"], state["bert.pooler.dense.bias"]
            w2, b2 = state["classifier.weight"], state["classifier.bias"]
        else:
            w1, b1 = state["classifier.dense.weight"], state["classifier.dense.bias"]
            w2, b2 = state["classifier.out_proj.weight"], state["classifier.out_proj.bias"]
        if w2.shape[0] != 1:
            raise ValueError(f"the classifier has {w2.shape[0]} labels; a cross-encoder reranker needs num_labels == 1")
        body = {k[len(prefix):]: v for k, v in state.items() if k.startswith(prefix)}
        self.encoder = BertEncoder(cfg, body, device=device, pooling="cls")
        self.cfg, self.family, self.device = cfg, family, self.encoder.device
        self.cls_id, self.sep_id, self.pad_id = int(cls_id), int(sep_id), int(pad_id)
        self.n_mid, self.type_b = _TEMPLATES[family]
        self.pos_offset = 0 if family == "bert" else self.pad_id + 1
        dev = self.device
        self.w1 = w1.detach().to(device=dev, dtype=torch.bfloat16).contiguous()
        self.b1 = b1.detach().to(device=dev, dtype=torch.bfloat16).contiguous()
        self.w2 = w2.detach()[0].to(device=dev, dtype=torch.float32).contiguous()
        self.b2 = float(b2.detach().float()[0])

    @staticmethod
    def from_pretrained(model_dir: str, device="cuda") -> "CrossEncoderModel":
        """A local checkpoint directory (weights, config.json and tokenizer files), read through transformers
        without any download."""
        from transformers import AutoModelForSequenceClassification, AutoTokenizer
        hf = AutoModelForSequenceClassification.from_pretrained(model_dir, local_files_only=True,
                                                                dtype=torch.float32)
        c = hf.config
        if c.model_type == "bert":
            family = "bert"
        elif c.model_type in ("roberta", "xlm-roberta"):
            family = "roberta"
        else:
            raise ValueError(f"model_type {c.model_type!r}: only BERT and (XLM-)RoBERTa cross-encoders are supported")
        if c.num_labels != 1:
            raise ValueError(f"the classifier has {c.num_labels} labels; a cross-encoder reranker needs num_labels == 1")
        if getattr(c, "hidden_act", "gelu") != "gelu":
            raise ValueError(f"hidden_act {c.hidden_act!r}: the encoder kernels implement erf GELU only")
        cfg = BertConfig(vocab_size=c.vocab_size, hidden_size=c.hidden_size, intermediate_size=c.intermediate_size,
                         num_hidden_layers=c.num_hidden_layers, num_attention_heads=c.num_attention_heads,
                         max_position_embeddings=c.max_position_embeddings, layer_norm_eps=c.layer_norm_eps)
        tok = AutoTokenizer.from_pretrained(model_dir, local_files_only=True)
        return CrossEncoderModel(family, cfg, hf.state_dict(), tok.cls_token_id, tok.sep_token_id,
                                 pad_id=c.pad_token_id if c.pad_token_id is not None else 1, device=device)

    def flops(self, lens: Sequence[int]) -> float:
        """Encoder FLOPs of pairs of these lengths (the head adds 2 d^2 per pair)."""
        return self.encoder.flops(lens)


def _mark(events: Optional[list]) -> None:
    if events is not None:
        ev = torch.cuda.Event(enable_timing=True)
        ev.record()
        events.append(ev)


@dataclass
class CrossPairs:
    """Packed pairs: pair ``pair_off[q] + r`` is candidate r of query q (r < its count); no empty pairs."""
    cand_ids: torch.Tensor     # int32 [Q, k] (row stride may exceed k)
    pair_off: torch.Tensor     # int32 [Q + 1]
    ids: torch.Tensor          # int32 [T]
    types: torch.Tensor        # int32 [T]
    positions: torch.Tensor    # int32 [T]
    cu_h: np.ndarray           # int64 [P + 1], host copy of the pairs' cu_seqlens
    n_queries: int
    k: int

    @property
    def n_pairs(self) -> int:
        return self.cu_h.size - 1


@dataclass
class RerankFusion:
    """Result of :meth:`CrossEncoderReranker.rerank_fusion`: each route reranked on its own, and the two fused."""
    fused: TopK                # [Q, k_out], float64 RRF scores of the two reranked top_n lists (sparse first on ties)
    sparse: TopK               # [Q, top_n], float32 sigmoid scores, as ``rerank`` returns for the sparse list
    dense: TopK                # [Q, top_n]
    sparse_all: torch.Tensor   # float32 [Q, k_sparse], -inf padded
    dense_all: torch.Tensor    # float32 [Q, k_dense]
    n_pairs: int               # distinct (query, passage) pairs encoded
    route_pairs: torch.Tensor  # int64 [] on the device: the pairs of both routes, read by ``n_route_pairs``

    @property
    def n_route_pairs(self) -> int:
        """The pairs two ``rerank`` calls would encode (reading it synchronises with the device)."""
        return int(self.route_pairs)


class CrossEncoderReranker:
    """Batched fine ranking of coarse candidate lists on the GPU.

    ``passage_tokens[i]`` = the cross-encoder tokenizer's ids of passage ``id_base + i`` without special tokens,
    tokenised once.  ``max_tokens`` bounds the tokens one encoder pass holds (activation memory); it must fit one
    pair of ``max_length``.  Scores do not depend on it.
    """

    def __init__(self, model: CrossEncoderModel, passage_tokens: Sequence[Sequence[int]],
                 max_length: int = DEFAULT_SENTENCE_TRANSFORMER_MAX_LENGTH, max_tokens: int = DEFAULT_MAX_TOKENS,
                 id_base: int = 0):
        _lib.require_cuda()
        if max_length < 2 + model.n_mid:
            raise ValueError(f"max_length={max_length} leaves no room for the {2 + model.n_mid} special tokens")
        if model.pos_offset + max_length > model.cfg.max_position_embeddings:
            raise ValueError(f"max_length={max_length} needs positions up to {model.pos_offset + max_length - 1}; the "
                             f"model has {model.cfg.max_position_embeddings}")
        if max_tokens < max_length:
            raise ValueError(f"max_tokens={max_tokens} must hold one pair of max_length={max_length} tokens")
        self.model, self.device = model, model.device
        self.max_length, self.max_tokens, self.id_base = int(max_length), int(max_tokens), int(id_base)
        lens = np.fromiter((len(t) for t in passage_tokens), dtype=np.int64, count=len(passage_tokens))
        ptr = np.zeros(lens.size + 1, np.int64)
        np.cumsum(lens, out=ptr[1:])
        flat = np.fromiter((int(x) for t in passage_tokens for x in t), dtype=np.int32, count=int(ptr[-1]))
        self.n_docs = int(lens.size)
        self.p_ptr = torch.from_numpy(ptr).to(self.device)
        self.p_tok = torch.from_numpy(flat if flat.size else np.zeros(1, np.int32)).to(self.device)
        self.ws = Workspace(self.device)

    def pack(self, cand_ids: torch.Tensor, cand_counts: torch.Tensor, q_ptr: torch.Tensor, q_tok: torch.Tensor
             ) -> CrossPairs:
        """The real (query, candidate) pairs of ``cand_ids`` int32 [Q, k] / ``cand_counts`` [Q] as the encoder
        consumes them.  One device-to-host copy: the totals and ``cu``, which size the buffers and cut the chunks."""
        L = _lib.lib()
        m, dev = self.model, self.device
        ids = cand_ids.to(device=dev, dtype=torch.int32)
        if ids.dim() != 2:
            raise ValueError("cand_ids must be [Q, k]")
        if ids.stride(1) != 1:
            ids = ids.contiguous()
        nq, k = ids.shape
        cnt = cand_counts.to(device=dev, dtype=torch.int32).contiguous()
        qp = q_ptr.to(device=dev, dtype=torch.int32).contiguous()
        qt = q_tok.to(device=dev, dtype=torch.int32).contiguous()
        if qt.numel() == 0:
            qt = torch.zeros(1, dtype=torch.int32, device=dev)
        if qp.numel() != nq + 1 or cnt.numel() != nq:
            raise ValueError(f"q_ptr ({qp.numel()}) / counts ({cnt.numel()}) do not match {nq} queries")
        ws = self.ws.get(L.ezr_cross_pack_workspace(nq, k))
        pair_off = torch.empty(nq + 1, dtype=torch.int32, device=dev)
        cu = torch.empty(nq * k + 1, dtype=torch.int32, device=dev)
        totals = (ctypes.c_int64 * 2)()
        common = (_lib.ptr(ids), _lib.ptr(cnt), nq, k, ids.stride(0), self.id_base, self.n_docs, _lib.ptr(qp))
        with torch.cuda.device(dev):
            st = _lib.stream_ptr()
            _lib.check(L.ezr_cross_pack_plan(*common, _lib.ptr(self.p_ptr), m.n_mid, self.max_length,
                                             _lib.ptr(pair_off), _lib.ptr(cu), totals, _lib.ptr(ws), ws.numel(), st),
                       "ezr_cross_pack_plan")
            n_tok, n_pairs = int(totals[0]), int(totals[1])
            tok = torch.empty(max(n_tok, 1), dtype=torch.int32, device=dev)
            types = torch.empty_like(tok)
            pos = torch.empty_like(tok)
            _lib.check(L.ezr_cross_pack_fill(*common, _lib.ptr(qt), _lib.ptr(self.p_ptr), _lib.ptr(self.p_tok),
                                             m.cls_id, m.sep_id, m.n_mid, m.type_b, m.pos_offset, self.max_length,
                                             _lib.ptr(ws), _lib.ptr(tok), _lib.ptr(types), _lib.ptr(pos), st),
                       "ezr_cross_pack_fill")
        cu_h = cu[:n_pairs + 1].cpu().numpy().astype(np.int64)
        return CrossPairs(ids[:, :k], pair_off, tok[:n_tok], types[:n_tok], pos[:n_tok], cu_h, nq, k)

    def rerank(self, cand: TopK, q_ptr: torch.Tensor, q_tok: torch.Tensor, top_n: int,
               events: Optional[List[torch.cuda.Event]] = None) -> Tuple[TopK, torch.Tensor]:
        """``cand``: ids int32 [Q, k] (-1 padded) and counts [Q] of a coarse ranker, on the device; ``q_ptr`` int32
        [Q + 1] / ``q_tok`` int32: the queries' ids without special tokens (CSR).
        -> (top_n per query: float32 sigmoid scores, document ids, counts;  all_scores float32 [Q, k], -inf padded).
        ``events``: if a list, timing events are recorded into it at the start, after packing, after the encoder and
        at the end (stage times for benchmarks)."""
        L = _lib.lib()
        m, dev = self.model, self.device
        if cand.ids.dim() == 2 and cand.ids.shape[1] > MAX_CANDIDATES:
            raise ValueError(f"k={cand.ids.shape[1]} candidates per query; at most {MAX_CANDIDATES} are supported")
        if top_n < 1:
            raise ValueError("top_n must be >= 1")
        _mark(events)
        pairs = self.pack(cand.ids, cand.counts, q_ptr, q_tok)
        _mark(events)
        nq, k = pairs.n_queries, pairs.k
        out = TopK(torch.empty(nq, top_n, dtype=torch.float32, device=dev),
                   torch.empty(nq, top_n, dtype=torch.int32, device=dev), torch.empty(nq, dtype=torch.int32, device=dev))
        all_scores = torch.empty(nq, k, dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            dense = None
            if pairs.n_pairs:
                cls = torch.empty(pairs.n_pairs, m.cfg.hidden_size, dtype=torch.bfloat16, device=dev)
                for p0, p1 in self.chunks(pairs.cu_h):
                    self._encode_cls(pairs, p0, p1, cls[p0:p1])
            _mark(events)
            if pairs.n_pairs:
                dense = gemm(cls, m.w1, bias=m.b1)
            _lib.check(L.ezr_cross_score_topk(_lib.ptr(dense), m.cfg.hidden_size, _lib.ptr(pairs.pair_off), nq, k,
                                              _lib.ptr(pairs.cand_ids), pairs.cand_ids.stride(0), _lib.ptr(m.w2), m.b2,
                                              m.cfg.hidden_size, top_n, _lib.ptr(all_scores), _lib.ptr(out.scores),
                                              _lib.ptr(out.ids), _lib.ptr(out.counts), _lib.stream_ptr()),
                       "ezr_cross_score_topk")
            _mark(events)
        return out, all_scores

    def rerank_fusion(self, sparse: TopK, dense: TopK, q_ptr: torch.Tensor, q_tok: torch.Tensor, top_n: int,
                      k_out: int, K: int = 60, canon: Optional[torch.Tensor] = None,
                      events: Optional[List[torch.cuda.Event]] = None) -> RerankFusion:
        """``generation_with_rerank_fusion`` (pipeline.py:393-452) for a batch: the sparse and the dense coarse lists
        (ids int32 [Q, k_sparse] / [Q, k_dense], -1 padded, and counts [Q]) each reranked to ``top_n``, then
        ``rrf_fuse(sparse, dense)`` to ``k_out`` (``canon``: as in ``rrf_fuse``).  Every output is bit-identical to two
        :meth:`rerank` calls and ``rrf_fuse``, but a document in both lists is packed and encoded once: the pairs are
        those of ``batched.pair_union`` (one pack, one encoder run, one head), and each route is ordered from the
        union's scores through its slot map.  k_sparse + k_dense <= 1024.  ``events``: as in :meth:`rerank` (the
        union is in the first stage)."""
        _mark(events)
        union, pairs = self._union_pack(sparse, dense, q_ptr, q_tok, top_n, k_out)
        _mark(events)
        sig = torch.empty(pairs.n_pairs, dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            self._score_run(pairs, 0, pairs.n_pairs, sig, events)
            out = self._fusion_orders(sig, pairs, union, sparse, dense, top_n, k_out, K, canon)
            _mark(events)
        return out

    def _union_pack(self, sparse: TopK, dense: TopK, q_ptr: torch.Tensor, q_tok: torch.Tensor, top_n: int,
                    k_out: int):
        """The checks of :meth:`rerank_fusion`, the union of the two lists and its pack -> (PairUnion, CrossPairs)."""
        from .batched import pair_union
        if top_n < 1 or k_out < 1:
            raise ValueError(f"top_n={top_n} and k_out={k_out} must be >= 1")
        dev = self.device
        union = pair_union(sparse.ids.to(dev), sparse.counts.to(dev), dense.ids.to(dev), dense.counts.to(dev))
        return union, self.pack(union.ids, union.counts, q_ptr, q_tok)

    def _score_run(self, pairs: CrossPairs, lo: int, hi: int, sig: torch.Tensor,
                   events: Optional[List[torch.cuda.Event]]) -> None:
        """Pairs [lo, hi) through the chunked encoder (then an event), Linear + bias and the sigmoid into sig[lo:hi]."""
        m, d = self.model, self.model.cfg.hidden_size
        if hi > lo:
            cls = torch.empty(hi - lo, d, dtype=torch.bfloat16, device=self.device)
            for p0, p1 in self.chunks(pairs.cu_h[lo:hi + 1]):
                self._encode_cls(pairs, lo + p0, lo + p1, cls[p0:p1])
        _mark(events)
        if hi > lo:
            rows = gemm(cls, m.w1, bias=m.b1)
            _lib.check(_lib.lib().ezr_cross_pair_scores(_lib.ptr(rows), d, hi - lo, _lib.ptr(m.w2), m.b2,
                                                        _lib.ptr(sig[lo:hi]), _lib.stream_ptr()),
                       "ezr_cross_pair_scores")

    def _fusion_orders(self, sig: torch.Tensor, pairs: CrossPairs, union, sparse: TopK, dense: TopK, top_n: int,
                       k_out: int, K: int, canon: Optional[torch.Tensor]) -> RerankFusion:
        """Both routes ordered from the union's pair scores ``sig`` (``ezr_cross_order_topk_mapped``), then RRF."""
        from .batched import rrf_fuse
        L, dev, nq = _lib.lib(), self.device, pairs.n_queries
        routes = []
        for cand, slot_map in ((sparse, union.map_a), (dense, union.map_b)):
            ids = cand.ids.to(device=dev, dtype=torch.int32)
            if ids.stride(1) != 1:
                ids = ids.contiguous()
            k = ids.shape[1]
            top = TopK(torch.empty(nq, top_n, dtype=torch.float32, device=dev),
                       torch.empty(nq, top_n, dtype=torch.int32, device=dev),
                       torch.empty(nq, dtype=torch.int32, device=dev))
            all_scores = torch.empty(nq, k, dtype=torch.float32, device=dev)
            _lib.check(L.ezr_cross_order_topk_mapped(_lib.ptr(sig), _lib.ptr(pairs.pair_off), nq, k, _lib.ptr(slot_map),
                                                     slot_map.stride(0), _lib.ptr(ids), ids.stride(0), top_n,
                                                     _lib.ptr(all_scores), _lib.ptr(top.scores), _lib.ptr(top.ids),
                                                     _lib.ptr(top.counts), _lib.stream_ptr()),
                       "ezr_cross_order_topk_mapped")
            routes.append((top, all_scores, cand.counts.to(dev).clamp(0, k).sum()))
        (s, s_all, s_n), (d, d_all, d_n) = routes
        fused = rrf_fuse(s.ids, s.counts, d.ids, d.counts, k_out, K=K, canon=canon)
        return RerankFusion(fused, s, d, s_all, d_all, pairs.n_pairs, s_n + d_n)

    def chunks(self, cu_h: np.ndarray) -> List[Tuple[int, int]]:
        """Consecutive runs [p0, p1) of whole pairs holding at most ``max_tokens`` tokens and at most
        ``MAX_CHUNK_PAIRS`` pairs each."""
        out, p0, n = [], 0, cu_h.size - 1
        while p0 < n:
            p1 = int(np.searchsorted(cu_h, cu_h[p0] + self.max_tokens, side="right")) - 1
            p1 = min(max(p1, p0 + 1), n, p0 + MAX_CHUNK_PAIRS)
            out.append((p0, p1))
            p0 = p1
        return out

    def _encode_cls(self, pairs: CrossPairs, p0: int, p1: int, cls_out: torch.Tensor) -> None:
        """Encoder over pairs [p0, p1); their CLS rows -> ``cls_out``."""
        m, cu_h = self.model, pairs.cu_h
        t0, t1 = int(cu_h[p0]), int(cu_h[p1])
        max_len = int(np.diff(cu_h[p0:p1 + 1]).max())
        batch = PackedBatch(ids=pairs.ids[t0:t1],
                            cu=torch.from_numpy((cu_h[p0:p1 + 1] - t0).astype(np.int32)).to(self.device),
                            positions=pairs.positions[t0:t1], max_len=max_len, n_seq=p1 - p0,
                            max_pos=m.pos_offset + max_len, types=pairs.types[t0:t1])
        h = m.encoder.hidden(batch)
        _lib.check(_lib.lib().ezr_pool_normalize(_lib.ptr(h), h.stride(0), _lib.ptr(batch.cu), batch.n_seq, POOL_CLS, 0,
                                                 None, 0.0, 0, m.cfg.hidden_size, _lib.ptr(cls_out), None,
                                                 _lib.stream_ptr()), "ezr_pool_normalize")


def random_cross_encoder_state(family: str, cfg: BertConfig, seed: int, std: float = 0.02) -> Dict[str, torch.Tensor]:
    """Random-init classifier weights of the right shapes and names (there are no checkpoints offline); values
    bf16-representable.  RoBERTa has one token type."""
    body = random_state("bert", cfg, seed, std)
    g = torch.Generator().manual_seed(seed + 1)
    rn = lambda *shape, s=std: (torch.randn(*shape, generator=g) * s).to(torch.bfloat16).float()
    d = cfg.hidden_size
    if family == "bert":
        st = {"bert." + k: v for k, v in body.items()}
        st.update({"bert.pooler.dense.weight": rn(d, d), "bert.pooler.dense.bias": rn(d),
                   "classifier.weight": rn(1, d, s=0.1), "classifier.bias": rn(1)})
    else:
        body["embeddings.token_type_embeddings.weight"] = body["embeddings.token_type_embeddings.weight"][:1]
        st = {"roberta." + k: v for k, v in body.items()}
        st.update({"classifier.dense.weight": rn(d, d), "classifier.dense.bias": rn(d),
                   "classifier.out_proj.weight": rn(1, d, s=0.1), "classifier.out_proj.bias": rn(1)})
    return st


class SentenceTransformerRerank(BaseNodePostprocessor):
    """Drop-in for the reference's ``SentenceTransformerRerank`` (rerankers.py:15-99), scoring on the GPU.

    ``model`` is a local checkpoint directory (loaded with :meth:`CrossEncoderModel.from_pretrained` and its
    tokenizer), unless ``encoder`` (a :class:`CrossEncoderModel`) and ``tokenizer`` (a HF tokenizer) are given.
    """
    model: str = Field(description="Sentence transformer model name.")
    top_n: int = Field(description="Number of nodes to return sorted by score.")
    device: str = Field(default="cuda", description="Device to use for sentence transformer.")
    keep_retrieval_score: bool = Field(default=False, description="Whether to keep the retrieval score in metadata.")
    _model: Any = PrivateAttr()
    _tok: Any = PrivateAttr()

    def __init__(self, top_n: int = 2, model: str = "cross-encoder/stsb-distilroberta-base",
                 device: Optional[str] = None, keep_retrieval_score: Optional[bool] = False, *,
                 encoder: Optional[CrossEncoderModel] = None, tokenizer=None):
        device = device or "cuda"
        if encoder is None:
            encoder = CrossEncoderModel.from_pretrained(model, device=device)
        if tokenizer is None:
            from .embeddings import _loading
            tokenizer = _loading.load_tokenizer(model)
        super().__init__(top_n=top_n, model=model, device=device, keep_retrieval_score=keep_retrieval_score)
        self._model = encoder
        self._tok = tokenizer

    @classmethod
    def class_name(cls) -> str:
        return "SentenceTransformerRerank"

    def _postprocess_nodes(self, nodes: List[NodeWithScore],
                           query_bundle: Optional[QueryBundle] = None) -> List[NodeWithScore]:
        if query_bundle is None:
            raise ValueError("Missing query bundle in extra info.")
        if len(nodes) == 0:
            return []
        texts = [n.node.get_content(metadata_mode=MetadataMode.NONE) for n in nodes]
        passages = self._tok(texts, add_special_tokens=False)["input_ids"]
        query = self._tok([query_bundle.query_str], add_special_tokens=False)["input_ids"][0]
        dev = self._model.device
        n = len(nodes)
        rr = CrossEncoderReranker(self._model, passages, max_length=DEFAULT_SENTENCE_TRANSFORMER_MAX_LENGTH)
        cand = TopK(scores=torch.zeros(1, n, device=dev), ids=torch.arange(n, dtype=torch.int32, device=dev)[None],
                    counts=torch.full((1,), n, dtype=torch.int32, device=dev))
        order, scores = rr.rerank(cand, torch.tensor([0, len(query)], dtype=torch.int32),
                                  torch.tensor(query, dtype=torch.int32), top_n=n)
        scores = scores[0].cpu().tolist()
        for node, score in zip(nodes, scores):
            if self.keep_retrieval_score:
                node.node.metadata["retrieval_score"] = node.score
            node.score = score
        return [nodes[i] for i in order.ids[0].cpu().tolist()][: self.top_n]
