"""Drop-in retrievers: same classes, constructor arguments and methods as the reference's
src/easyrag/custom/retrievers.py, with the arithmetic on the GPU.

  QdrantRetriever   retrievers.py:23-69    -> dense cosine top-k        (csrc/dense*.cu)
  BM25Retriever     retrievers.py:80-220   -> BM25 score + filter       (csrc/bm25.cu)
  HybridRetriever   retrievers.py:223-305  -> RRF / simple fusion       (csrc/fusion.cu)

Host-side work that stays in Python exactly as in the reference: tokenisation through the
caller's ``tokenizer.cut`` and stop-word removal (retrievers.py:72-76), ``get_node_content``
(ingestion.py:34-76) and the construction of ``NodeWithScore`` lists.  There is no CPU
implementation of the scoring: without a CUDA device these classes raise ``EzrError``.
"""
from __future__ import annotations

import logging
from typing import Any, Callable, Dict, List, Optional, Sequence, Tuple, cast

import numpy as np
import torch

from . import _lib, batched
from .index import Bm25Index, Bm25Stats, DenseIndex, K1, B, EPSILON, normalize_rows
from .schema import (BaseEmbedding, BaseNode, BaseRetriever, NodeWithScore, QueryBundle, VectorStoreQuery,
                     VectorStoreQueryResult, filter_conditions)
from .vocab import Vocabulary

logger = logging.getLogger(__name__)

DEFAULT_SIMILARITY_TOP_K = 2      # llama_index.core.constants
MAX_TOP_K = 1024                   # kSelMaxK in csrc/select.cuh


# ------------------------------------------------------------------ text views
def get_node_content(node, embed_type: int = 0, nodes: Optional[list] = None, nodeid2idx: Optional[dict] = None) -> str:
    """Text view selector, semantics of ingestion.py:34-76 (types 0-5; 3/6 image-caption substitution).

    The table-merge branch of type 6 (ingestion.py:36-57) needs the neighbouring nodes and is only
    reachable with ``nodes``/``nodeid2idx``; the retrievers never pass them (retrievers.py:99), neither do we.
    """
    text: str = node.get_content()
    md = node.metadata
    if embed_type == 1:
        if 'file_path' in md:
            text = '###\n' + md['file_path'] + "\n\n" + text
    elif embed_type == 2:
        if 'know_path' in md:
            text = '###\n' + md['know_path'] + "\n\n" + text
    elif embed_type in (3, 6):
        for imgobj in (md.get('imgobjs') or []):
            text = text.replace(f"{imgobj['cap']} {imgobj['title']}\n",
                                f"{imgobj['cap']}.{imgobj['title']}:{imgobj['content']}\n")
    elif embed_type == 4:
        text = md['file_path'] if 'file_path' in md else ""
    elif embed_type == 5:
        text = md['know_path'] if 'know_path' in md else ""
    return text


def tokenize_and_remove_stopwords(tokenizer, text, stopwords):
    """retrievers.py:72-76, unchanged semantics (host side)."""
    words = tokenizer.cut(text)
    return [word for word in words if word not in stopwords and word != ' ']


class _GroupTable:
    """Maps ``filter_dict`` / qdrant equality filters onto small integer classes per document.

    For a tuple of metadata keys every document gets the index of its value tuple; a query's filter
    becomes the index of the wanted tuple (or -2: no document can match).  Built once per key set.
    """

    def __init__(self, nodes: Sequence[Any], missing: Any = None):
        """``missing``: None keeps the reference's BM25 behaviour (a node without the key raises KeyError,
        retrievers.py:200); a sentinel makes such a node match nothing, as a Qdrant payload filter does."""
        self._nodes = nodes
        self._missing = missing
        self._tables: Dict[Tuple[str, ...], Tuple[Dict[tuple, int], torch.Tensor]] = {}

    def resolve(self, conditions: Optional[Dict[str, Any]]):
        """-> (doc_group int32 cpu tensor or None, wanted id)."""
        if not conditions:
            return None, -1
        keys = tuple(conditions.keys())
        if keys not in self._tables:
            table: Dict[tuple, int] = {}
            ids = np.empty(len(self._nodes), dtype=np.int32)
            for i, n in enumerate(self._nodes):
                if self._missing is None:      # a missing key raises KeyError in the reference (retrievers.py:200)
                    tup = tuple(_hashable(n.metadata[k]) for k in keys)
                else:
                    tup = tuple(_hashable(n.metadata.get(k, self._missing)) for k in keys)
                ids[i] = table.setdefault(tup, len(table))
            self._tables[keys] = (table, torch.from_numpy(ids))
        table, ids = self._tables[keys]
        want = table.get(tuple(_hashable(conditions[k]) for k in keys), -2)
        return ids, want


def _hashable(v):
    try:
        hash(v)
        return v
    except TypeError:
        return repr(v)


def _canon_ids(texts: Sequence[str]) -> np.ndarray:
    """canon[i] = first index whose text equals texts[i] (the dict key of retrievers.py:246,263)."""
    first: Dict[str, int] = {}
    out = np.empty(len(texts), dtype=np.int32)
    for i, t in enumerate(texts):
        out[i] = first.setdefault(t, i)
    return out


# ---------------------------------------------------------------- dense route
_MISSING = ("<missing metadata key>",)      # sentinel: a node without the filter key matches no filter value


class B200VectorStore:
    """In-HBM replacement for the Qdrant collection (ingestion.py:155-191): exact cosine search.

    ``query`` / ``aquery`` keep ``QdrantVectorStore``'s call shape used at retrievers.py:44-47,61-64.
    Vectors are L2-normalised at insert, as a Distance.COSINE collection does, and held in bf16.  ``add`` appends
    (amortised O(new nodes)); :meth:`add_embedded` takes the encoder's device tensor directly and
    :meth:`from_embed_model` lets the embedding model write its bf16 rows straight into the corpus matrix -- no
    Python float lists between the encoder and the index.

    ``dense_form`` / ``block_queries`` are passed to :func:`easyrag_b200.batched.dense_topk` as ``form`` /
    ``block_queries`` on every query (``dense_form=6``: wgmma score rows, for wide embeddings such as gte-Qwen2-7B's
    3584 dims or k > 16); the defaults keep the automatic choice.  ``dense_cand=True`` searches with
    :func:`easyrag_b200.batched.dense_topk_cand` instead (form 6's results without its score rows); it excludes
    ``dense_form``, ``block_queries`` and ``quantize``.
    """

    def __init__(self, nodes: Optional[Sequence[Any]] = None, device="cuda", quantize: bool = False,
                 dense_form: Optional[int] = None, block_queries: Optional[int] = None, dense_cand: bool = False):
        if dense_cand and (dense_form is not None or block_queries is not None or quantize):
            raise ValueError("dense_cand=True excludes dense_form, block_queries and quantize")
        if block_queries is not None and (dense_form != 6 or quantize):
            raise ValueError("block_queries needs dense_form=6 and an index that is not quantized")
        self.device = device
        self.dense_form = dense_form
        self.block_queries = block_queries
        self.dense_cand = bool(dense_cand)
        # keep an int8 mirror: exact search through a certified int8 pass (currently slower than bf16, README)
        self.quantize = bool(quantize)
        self.nodes: List[Any] = []
        self.index: Optional[DenseIndex] = None
        self._groups: Optional[_GroupTable] = None
        self._group_cache: Dict[Tuple[str, ...], torch.Tensor] = {}
        self._ws = None
        if nodes:
            self.add(nodes)

    def _ensure_index(self, dim: int) -> DenseIndex:
        if self.index is None:
            self.index = DenseIndex(None, device=self.device, dim=dim, quantized=self.quantize)
            self._ws = batched.Workspace(self.index.device)
        elif self.index.dim != dim:
            raise ValueError(f"embedding dim {dim} != collection dim {self.index.dim}")
        return self.index

    def _registered(self, nodes: Sequence[Any]) -> List[str]:
        self.nodes.extend(nodes)
        self._groups = _GroupTable(self.nodes, missing=_MISSING)
        self._group_cache.clear()
        return [n.node_id for n in nodes]

    def add(self, nodes: Sequence[Any]) -> List[str]:
        """VectorStore.add: nodes carrying ``.embedding`` lists (what the ingestion pipeline produces)."""
        nodes = list(nodes)
        if not nodes:
            return []
        emb = torch.tensor([n.embedding for n in nodes], dtype=torch.float32)        # the new nodes only
        self._ensure_index(emb.shape[1]).append(emb, normalize=True)
        return self._registered(nodes)

    def add_embedded(self, nodes: Sequence[Any], embeddings: torch.Tensor) -> List[str]:
        """Nodes plus their embeddings as a tensor ([n, d] float32 / bf16, host or device): no Python lists."""
        nodes = list(nodes)
        if embeddings.shape[0] != len(nodes):
            raise ValueError("add_embedded: one embedding row per node")
        self._ensure_index(embeddings.shape[1]).append(embeddings, normalize=True)
        return self._registered(nodes)

    @classmethod
    def from_embed_model(cls, nodes: Sequence[Any], embed_model, device="cuda", batch_size: Optional[int] = None,
                         quantize: bool = False, dense_form: Optional[int] = None,
                         block_queries: Optional[int] = None, dense_cand: bool = False) -> "B200VectorStore":
        """Corpus encode written in place (replaces pipeline.py:141-158 + ingestion.py:155-191): every batch of
        ``embed_model.embed_tensor`` lands in its slice of the corpus matrix, normalised on the way."""
        store = cls(device=device, quantize=quantize, dense_form=dense_form, block_queries=block_queries,
                    dense_cand=dense_cand)
        nodes = list(nodes)
        bs = int(batch_size or getattr(embed_model, "embed_batch_size", 128) or 128)
        embed_type = getattr(embed_model, "_embed_type", 0)
        for i in range(0, len(nodes), bs):
            part = nodes[i:i + bs]
            texts = [get_node_content(n, embed_type) for n in part]
            out = embed_model.embed_tensor(texts, "text") if _takes_prompt(embed_model) else embed_model.embed_tensor(texts)
            emb_bf16 = out[0]                                   # (bf16 [B, d], float32 [B, d]) on the device
            index = store._ensure_index(emb_bf16.shape[1])
            if i == 0:
                index.reserve(len(nodes))
            index.append(emb_bf16, normalize=True)
        store._registered(nodes)
        return store

    def _doc_group(self, keys: Tuple[str, ...], ids: torch.Tensor) -> torch.Tensor:
        """Per-row class ids of a filter-key tuple on the device, uploaded once per key set (not per query)."""
        t = self._group_cache.get(keys)
        if t is None:
            t = ids.to(self.index.device)
            self._group_cache[keys] = t
        return t

    def query(self, query: VectorStoreQuery, qdrant_filters=None, **kwargs) -> VectorStoreQueryResult:
        if self.index is None:
            return VectorStoreQueryResult()
        k = int(query.similarity_top_k)
        if not 1 <= k <= MAX_TOP_K:
            raise ValueError(f"similarity_top_k={k} outside [1, {MAX_TOP_K}]")
        dev = self.index.device
        q32 = torch.tensor([query.query_embedding], dtype=torch.float32, device=dev)
        q = normalize_rows(q32, torch.empty(1, self.index.dim, dtype=torch.bfloat16, device=dev))
        conditions = filter_conditions(qdrant_filters)
        doc_group, want = self._groups.resolve(conditions)
        q_group = None
        if doc_group is not None:
            self.index.doc_group = self._doc_group(tuple(conditions.keys()), doc_group)
            q_group = torch.tensor([want], dtype=torch.int32)
        if self.dense_cand:
            res = batched.dense_topk_cand(self.index, q, k, q_group=q_group, ws=self._ws)
        else:
            res = batched.dense_topk(self.index, q, k, q_group=q_group, ws=self._ws, form=self.dense_form,
                                     block_queries=self.block_queries)
        n = int(res.counts[0])
        ids = res.ids[0, :n].tolist()
        sims = res.scores[0, :n].tolist()
        return VectorStoreQueryResult(nodes=[self.nodes[i] for i in ids], similarities=sims,
                                      ids=[self.nodes[i].node_id for i in ids])

    async def aquery(self, query: VectorStoreQuery, qdrant_filters=None, **kwargs) -> VectorStoreQueryResult:
        return self.query(query, qdrant_filters=qdrant_filters, **kwargs)


def _takes_prompt(embed_model) -> bool:
    import inspect
    try:
        return "prompt_name" in inspect.signature(embed_model.embed_tensor).parameters
    except (TypeError, ValueError):
        return False


class QdrantRetriever(BaseRetriever):
    """retrievers.py:23-69.  ``vector_store`` is a :class:`B200VectorStore` (or anything with the same aquery)."""

    def __init__(self, vector_store, embed_model: BaseEmbedding, similarity_top_k: int = 2, filters=None) -> None:
        self._vector_store = vector_store
        self._embed_model = embed_model
        self._similarity_top_k = similarity_top_k
        self.filters = filters
        super().__init__()

    async def _aretrieve(self, query_bundle: QueryBundle) -> List[NodeWithScore]:
        query_embedding = self._embed_model.get_query_embedding(query_bundle.query_str)
        vector_store_query = VectorStoreQuery(query_embedding, similarity_top_k=self._similarity_top_k)
        query_result = await self._vector_store.aquery(vector_store_query, qdrant_filters=self.filters)
        return [NodeWithScore(node=node, score=similarity)
                for node, similarity in zip(query_result.nodes, query_result.similarities)]

    def _retrieve(self, query_bundle: QueryBundle) -> List[NodeWithScore]:
        query_embedding = self._embed_model.get_query_embedding(query_bundle.query_str)
        vector_store_query = VectorStoreQuery(query_embedding, similarity_top_k=self._similarity_top_k)
        query_result = self._vector_store.query(vector_store_query, qdrant_filters=self.filters)
        return [NodeWithScore(node=node, score=similarity)
                for node, similarity in zip(query_result.nodes, query_result.similarities)]


# --------------------------------------------------------------- sparse route
def _encode_corpus(token_lists: Sequence[Sequence[str]]):
    """token strings -> (vocab dict in first-seen order, int32 tokens, int64 doc_ptr)."""
    vocab: Dict[str, int] = {}
    flat: List[int] = []
    ptr = [0]
    for doc in token_lists:
        for w in doc:
            flat.append(vocab.setdefault(w, len(vocab)))
        ptr.append(len(flat))
    return vocab, torch.tensor(flat, dtype=torch.int32), torch.tensor(ptr, dtype=torch.int64)


class BM25Retriever(BaseRetriever):
    """retrievers.py:80-220: jieba-tokenised BM25 (Okapi fp64 / bm25s fp32), k1=1.5 b=0.75 eps=0.25.

    ``packed``: as :class:`Bm25Index` -- ``None`` packs the postings of an Okapi index only, ``True`` also those of a
    bm25s index (its top-k then runs the two-phase path); the results are the same either way."""

    def __init__(self, nodes: List[BaseNode], tokenizer: Optional[Callable[[str], List[str]]],
                 similarity_top_k: int = DEFAULT_SIMILARITY_TOP_K, callback_manager=None, objects=None,
                 object_map: Optional[dict] = None, verbose: bool = False, stopwords: List[str] = [""],
                 embed_type: int = 0, bm25_type: int = 0, device="cuda", packed: Optional[bool] = None) -> None:
        self._nodes = nodes
        self._tokenizer = tokenizer
        self._similarity_top_k = similarity_top_k
        self.embed_type = embed_type
        self._corpus = [tokenize_and_remove_stopwords(self._tokenizer, get_node_content(node, self.embed_type),
                                                      stopwords=stopwords) for node in self._nodes]
        self.bm25_type = bm25_type
        self.k1, self.b, self.epsilon = K1, B, EPSILON
        self._device = device
        # the corpus is interned on the device (easyrag_b200.vocab): the same ids and dict as _encode_corpus
        vocab = Vocabulary(device)
        tokens, doc_ptr = vocab.intern(self._corpus)
        self._vocab = vocab.to_dict()
        self.bm25 = self._build(tokens, doc_ptr, len(self._vocab), packed=packed)
        self.filter_dict = None
        self.stopwords = stopwords
        self._groups = _GroupTable(self._nodes)
        self._group_keys: Optional[Tuple[str, ...]] = None
        self.canon = Vocabulary(device).first_index([n.get_content() for n in self._nodes]).to(torch.int32).cpu()
        self._ws = batched.Workspace(self.bm25.device)
        super().__init__(callback_manager=callback_manager, object_map=object_map, objects=objects, verbose=verbose)

    def _build(self, tokens, doc_ptr, vocab, packed: Optional[bool] = None) -> Bm25Index:
        stats = Bm25Stats.from_tokens(tokens, doc_ptr, max(vocab, 1), bm25_type=1 if self.bm25_type == 1 else 0,
                                      k1=self.k1, b=self.b, epsilon=self.epsilon)
        return Bm25Index(stats, device=self._device, k1=self.k1, b=self.b, packed=packed)

    def _query_ids(self, query: str, vocab: Dict[str, int]):
        toks = tokenize_and_remove_stopwords(self._tokenizer, query, stopwords=self.stopwords)
        ids = torch.tensor([vocab.get(t, -1) for t in toks], dtype=torch.int32)
        ptr = torch.tensor([0, len(toks)], dtype=torch.int32)
        return ptr, ids

    def get_scores(self, query, docs=None):
        """retrievers.py:128-151 -> numpy score vector (float64 for bm25_type 0, float32 for 1).  ``docs``: one
        context per call, small enough that its vocabulary stays a host dict (``_encode_corpus``)."""
        if docs is None:
            index, vocab = self.bm25, self._vocab
        else:
            corpus = [tokenize_and_remove_stopwords(self._tokenizer, doc, stopwords=self.stopwords) for doc in docs]
            vocab, tokens, doc_ptr = _encode_corpus(corpus)
            index = self._build(tokens, doc_ptr, len(vocab), packed=False)    # only score rows are read: skip the packed postings
        ptr, ids = self._query_ids(query, vocab)
        return batched.bm25_scores(index, ptr, ids)[0].cpu().numpy()

    @classmethod
    def from_defaults(cls, index=None, nodes: Optional[List[BaseNode]] = None, docstore=None,
                      tokenizer: Optional[Callable[[str], List[str]]] = None,
                      similarity_top_k: int = DEFAULT_SIMILARITY_TOP_K, verbose: bool = False,
                      stopwords: List[str] = [""], embed_type: int = 0, bm25_type: int = 0,
                      packed: Optional[bool] = None) -> "BM25Retriever":
        if sum(bool(val) for val in [index, nodes, docstore]) != 1:
            raise ValueError("Please pass exactly one of index, nodes, or docstore.")
        if index is not None:
            docstore = index.docstore
        if docstore is not None:
            nodes = cast(List[BaseNode], list(docstore.docs.values()))
        assert nodes is not None, "Please pass exactly one of index, nodes, or docstore."
        return cls(nodes=nodes, tokenizer=tokenizer, similarity_top_k=similarity_top_k, verbose=verbose,
                   stopwords=stopwords, embed_type=embed_type, bm25_type=bm25_type, packed=packed)

    def _apply_filter(self):
        doc_group, want = self._groups.resolve(self.filter_dict if self.filter_dict else None)
        keys = tuple(self.filter_dict.keys()) if self.filter_dict else None
        if doc_group is not None and keys != self._group_keys:
            self.bm25.set_doc_group(doc_group)
            self._group_keys = keys
        if doc_group is None:
            return None
        return torch.tensor([want], dtype=torch.int32)

    def _nodes_from(self, res: batched.TopK) -> List[NodeWithScore]:
        n = int(res.counts[0])
        ids = res.ids[0, :n].tolist()
        sc = res.scores[0, :n].tolist()
        nodes = [NodeWithScore(node=self._nodes[ix], score=float(s)) for ix, s in zip(ids, sc)]
        return sorted(nodes, key=lambda x: x.score, reverse=True)    # retrievers.py:209 (already in order)

    def filter(self, scores):
        """retrievers.py:191-210 on a caller-supplied score vector (numpy)."""
        k = int(self._similarity_top_k)
        if not 1 <= k <= MAX_TOP_K:
            raise ValueError(f"similarity_top_k={k} outside [1, {MAX_TOP_K}]")
        q_group = self._apply_filter()
        s = torch.as_tensor(np.ascontiguousarray(scores)).to(self.bm25.device)
        if s.dtype not in (torch.float32, torch.float64):
            s = s.to(torch.float64)
        res = batched.select_rows(s.reshape(1, -1), k, positive_only=True,
                                  doc_group=self.bm25.doc_group if q_group is not None else None,
                                  q_group=q_group, ws=self._ws)
        return self._nodes_from(res)

    def _retrieve(self, query_bundle: QueryBundle) -> List[NodeWithScore]:
        if query_bundle.custom_embedding_strs or query_bundle.embedding:
            logger.warning("BM25Retriever does not support embeddings, skipping...")
        k = int(self._similarity_top_k)
        if not 1 <= k <= MAX_TOP_K:
            raise ValueError(f"similarity_top_k={k} outside [1, {MAX_TOP_K}]")
        ptr, ids = self._query_ids(query_bundle.query_str, self._vocab)
        q_group = self._apply_filter()
        res = batched.bm25_topk(self.bm25, ptr, ids, k, q_group=q_group, ws=self._ws)
        return self._nodes_from(res)


# ------------------------------------------------------------------- fusion
def _fuse_lists(list_of_lists, topk: int, rrf: bool, K: int = 60) -> List[NodeWithScore]:
    """Shared host wrapper: text keys -> integer keys -> ``ezr_fuse_lists`` -> items.

    Any number of rank lists, like the reference's loops (retrievers.py:243-248, 261-265); the pipeline passes two
    (pipeline.py:362,408; retrievers.py:290).  The kernel holds up to 8 lists / 2048 entries per call.
    """
    _lib.require_cuda()
    lists = [list(l) for l in list_of_lists]
    items = [it for l in lists for it in l]
    if not items:
        return []
    if len(lists) > 8:
        raise ValueError("easyrag_b200 fuses at most 8 rank lists per call")
    width = max(max(len(l) for l in lists), 1)
    if width > 1024 or width * len(lists) > 2048:
        raise ValueError("rank lists longer than 1024 entries (2048 over all lists) are not supported")
    keys: Dict[str, int] = {}
    canon = np.empty(len(items), dtype=np.int32)
    for i, it in enumerate(items):
        canon[i] = keys.setdefault(it.get_content(), i)
    dev = torch.device("cuda")
    ids, cnts, scs = [], [], []
    base = 0
    for l in lists:
        row = torch.full((1, width), -1, dtype=torch.int32)
        row[0, :len(l)] = torch.arange(base, base + len(l), dtype=torch.int32)
        ids.append(row.to(dev))
        cnts.append(torch.tensor([len(l)], dtype=torch.int32, device=dev))
        if not rrf:
            sc = torch.zeros(1, width, dtype=torch.float64)
            sc[0, :len(l)] = torch.tensor([float(x.score) for x in l], dtype=torch.float64)
            scs.append(sc.to(dev))
        base += len(l)
    k_out = max(1, min(int(topk), len(items)))
    res = batched.fuse_lists(ids, cnts, k_out, rrf=rrf, K=K, scores=scs if not rrf else None,
                             canon=torch.from_numpy(canon).to(dev))
    n = int(res.counts[0])
    if int(topk) < n:
        n = max(int(topk), 0)
    pos = res.ids[0, :n].tolist()
    out = [items[p] for p in pos]
    if rrf:
        for it, s in zip(out, res.scores[0, :n].tolist()):
            it.score = s                                  # retrievers.py:271
    return out


class HybridRetriever(BaseRetriever):
    """retrievers.py:223-305."""

    def __init__(self, dense_retriever: QdrantRetriever, sparse_retriever: BM25Retriever, retrieval_type=1, topk=256):
        self.dense_retriever = dense_retriever
        self.sparse_retriever = sparse_retriever
        self.retrieval_type = retrieval_type  # 1:dense only 2:sparse only 3:hybrid
        self.filters = None
        self.filter_dict = None
        self.topk = topk
        super().__init__()

    @classmethod
    def fusion(self, list_of_list_ranks_system, topk=256):
        """retrievers.py:239-253."""
        return _fuse_lists(list_of_list_ranks_system, topk, rrf=False)

    @classmethod
    def reciprocal_rank_fusion(self, list_of_list_ranks_system, K=60, topk=256):
        """retrievers.py:256-274."""
        return _fuse_lists(list_of_list_ranks_system, topk, rrf=True, K=K)

    async def _aretrieve(self, query_bundle: QueryBundle) -> List[NodeWithScore]:
        if self.retrieval_type != 1:
            self.sparse_retriever.filter_dict = self.filter_dict
            sparse_nodes = await self.sparse_retriever.aretrieve(query_bundle)
            if self.retrieval_type == 2:
                return sparse_nodes
        if self.retrieval_type != 2:
            self.dense_retriever.filters = self.filters
            dense_nodes = await self.dense_retriever.aretrieve(query_bundle)
            if self.retrieval_type == 1:
                return dense_nodes
        return self.reciprocal_rank_fusion([sparse_nodes, dense_nodes], topk=self.topk)

    def _retrieve(self, query_bundle: QueryBundle) -> List[NodeWithScore]:
        """retrievers.py:293-305 (unmaintained in the reference): id-deduplicated concatenation."""
        sparse_nodes = self.sparse_retriever.retrieve(query_bundle)
        dense_nodes = self.dense_retriever.retrieve(query_bundle)
        all_nodes, node_ids = [], set()
        for n in sparse_nodes + dense_nodes:
            if n.node.node_id not in node_ids:
                all_nodes.append(n)
                node_ids.add(n.node.node_id)
        return all_nodes
