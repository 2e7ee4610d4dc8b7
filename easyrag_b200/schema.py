"""llama_index types the retriever surface is written against.

The reference subclasses llama-index-core 0.10.29's ``BaseRetriever`` / ``BaseEmbedding`` and
passes ``NodeWithScore`` / ``QueryBundle`` around (retrievers.py:6-15).  When llama_index is
importable the real classes are used, so the drop-in retrievers are genuine ``BaseRetriever``
instances (pipeline.py:213-217 wraps one in AutoMergingRetriever).  This image has no
llama_index, so minimal stand-ins with the same attribute surface are defined instead
(SURVEY.md 8(b) lists exactly what pipeline.py touches).
"""
from __future__ import annotations

import asyncio
import uuid
from enum import Enum
from typing import Any, Dict, List, Optional, Sequence, Union

try:  # pragma: no cover - exercised only where llama_index is installed
    from llama_index.core import QueryBundle  # type: ignore
    from llama_index.core.base.base_retriever import BaseRetriever  # type: ignore
    from llama_index.core.base.embeddings.base import BaseEmbedding  # type: ignore
    from llama_index.core.schema import NodeWithScore, TextNode, BaseNode  # type: ignore
    from llama_index.core.bridge.pydantic import Field, PrivateAttr  # type: ignore
    HAVE_LLAMA_INDEX = True
except Exception:  # ModuleNotFoundError here
    HAVE_LLAMA_INDEX = False

    def Field(default=None, **kwargs):
        """Stand-in for pydantic's ``Field``: the class attribute simply holds the default."""
        return default

    def PrivateAttr(default=None, **kwargs):
        return default

    class BaseNode:
        pass

    class TextNode(BaseNode):
        def __init__(self, text: str = "", id_: Optional[str] = None, metadata: Optional[Dict[str, Any]] = None,
                     embedding: Optional[List[float]] = None, relationships: Optional[dict] = None):
            self.text = text
            self.id_ = id_ or str(uuid.uuid4())
            self.metadata = metadata if metadata is not None else {}
            self.embedding = embedding
            self.relationships = relationships if relationships is not None else {}

        @property
        def node_id(self) -> str:
            return self.id_

        def get_content(self, metadata_mode=None) -> str:
            return self.text

        def __repr__(self):
            return f"TextNode(id_={self.id_!r}, text={self.text[:32]!r})"

    class NodeWithScore:
        def __init__(self, node: BaseNode, score: Optional[float] = None):
            self.node = node
            self.score = score

        def get_content(self, metadata_mode=None) -> str:
            return self.node.get_content()

        @property
        def metadata(self) -> Dict[str, Any]:
            return self.node.metadata

        @property
        def node_id(self) -> str:
            return self.node.node_id

        @property
        def text(self) -> str:
            return self.node.text

        def get_score(self, raise_error: bool = False) -> float:
            if self.score is None:
                if raise_error:
                    raise ValueError("Score not set.")
                return 0.0
            return self.score

        def __repr__(self):
            return f"NodeWithScore(score={self.score!r}, node={self.node!r})"

    class QueryBundle:
        def __init__(self, query_str: str, custom_embedding_strs: Optional[List[str]] = None,
                     embedding: Optional[List[float]] = None):
            self.query_str = query_str
            self.custom_embedding_strs = custom_embedding_strs
            self.embedding = embedding

    class BaseRetriever:
        """retrieve/aretrieve wrap _retrieve/_aretrieve; the async default falls back to the sync one."""

        def __init__(self, callback_manager=None, object_map: Optional[dict] = None, objects=None,
                     verbose: bool = False) -> None:
            self.callback_manager = callback_manager
            self.object_map = object_map or {}
            self._verbose = verbose

        def _retrieve(self, query_bundle: QueryBundle) -> List[NodeWithScore]:
            raise NotImplementedError

        async def _aretrieve(self, query_bundle: QueryBundle) -> List[NodeWithScore]:
            return self._retrieve(query_bundle)

        def retrieve(self, str_or_query_bundle: Union[str, QueryBundle]) -> List[NodeWithScore]:
            qb = QueryBundle(str_or_query_bundle) if isinstance(str_or_query_bundle, str) else str_or_query_bundle
            return self._retrieve(qb)

        async def aretrieve(self, str_or_query_bundle: Union[str, QueryBundle]) -> List[NodeWithScore]:
            qb = QueryBundle(str_or_query_bundle) if isinstance(str_or_query_bundle, str) else str_or_query_bundle
            return await self._aretrieve(qb)

    class BaseEmbedding:
        def __init__(self, model_name: str = "unknown", embed_batch_size: int = 10, callback_manager=None,
                     **kwargs: Any) -> None:
            self.model_name = model_name
            self.embed_batch_size = embed_batch_size
            self.callback_manager = callback_manager
            for name, value in kwargs.items():        # the declared fields of a subclass (pydantic would validate them)
                setattr(self, name, value)

        # subclass hooks
        def _get_query_embedding(self, query: str) -> List[float]:
            raise NotImplementedError

        def _get_text_embedding(self, text: str) -> List[float]:
            raise NotImplementedError

        def _get_text_embeddings(self, texts: List[str]) -> List[List[float]]:
            return [self._get_text_embedding(t) for t in texts]

        async def _aget_query_embedding(self, query: str) -> List[float]:
            return self._get_query_embedding(query)

        async def _aget_text_embedding(self, text: str) -> List[float]:
            return self._get_text_embedding(text)

        # public surface used by pipeline.py / retrievers.py
        def get_query_embedding(self, query: str) -> List[float]:
            return self._get_query_embedding(query)

        async def aget_query_embedding(self, query: str) -> List[float]:
            return await self._aget_query_embedding(query)

        def get_text_embedding(self, text: str) -> List[float]:
            return self._get_text_embedding(text)

        def get_text_embedding_batch(self, texts: List[str], show_progress: bool = False, **kwargs: Any
                                     ) -> List[List[float]]:
            out: List[List[float]] = []
            bs = max(1, int(self.embed_batch_size))
            for i in range(0, len(texts), bs):
                out.extend(self._get_text_embeddings(list(texts[i:i + bs])))
            return out

        async def aget_text_embedding_batch(self, texts: List[str], show_progress: bool = False, **kwargs: Any
                                            ) -> List[List[float]]:
            return self.get_text_embedding_batch(texts, show_progress=show_progress, **kwargs)


# the node-postprocessor base of the rerankers (rerankers.py:6-7): its own fallback, since a llama_index install may
# predate or omit the postprocessor module
try:  # pragma: no cover - exercised only where llama_index is installed
    from llama_index.core.postprocessor.types import BaseNodePostprocessor  # type: ignore
    from llama_index.core.schema import MetadataMode  # type: ignore
except Exception:
    class MetadataMode(str, Enum):
        ALL = "all"
        EMBED = "embed"
        LLM = "llm"
        NONE = "none"

    class BaseNodePostprocessor:
        """postprocess_nodes wraps _postprocess_nodes; a bare query string becomes a QueryBundle."""

        def __init__(self, callback_manager=None, **kwargs: Any) -> None:
            self.callback_manager = callback_manager
            for name, value in kwargs.items():        # the declared fields of a subclass (pydantic would validate them)
                setattr(self, name, value)

        def _postprocess_nodes(self, nodes: List[NodeWithScore],
                               query_bundle: Optional[QueryBundle] = None) -> List[NodeWithScore]:
            raise NotImplementedError

        def postprocess_nodes(self, nodes: List[NodeWithScore], query_bundle: Optional[QueryBundle] = None,
                              query_str: Optional[str] = None) -> List[NodeWithScore]:
            if query_str is not None and query_bundle is not None:
                raise ValueError("Cannot specify both query_str and query_bundle")
            if query_str is not None:
                query_bundle = QueryBundle(query_str)
            return self._postprocess_nodes(nodes, query_bundle)


class VectorStoreQuery:
    """llama_index.core.vector_stores.VectorStoreQuery: only the two fields retrievers.py:39-43 sets."""

    def __init__(self, query_embedding=None, similarity_top_k: int = 1, **kwargs):
        self.query_embedding = query_embedding
        self.similarity_top_k = similarity_top_k


class VectorStoreQueryResult:
    def __init__(self, nodes=None, similarities=None, ids=None):
        self.nodes = nodes or []
        self.similarities = similarities or []
        self.ids = ids or []


class _Match:
    def __init__(self, value):
        self.value = value


class _FieldCondition:
    def __init__(self, key, value):
        self.key = key
        self.match = _Match(value)


class PayloadFilter:
    """Shape-compatible with ``qdrant_client.models.Filter(must=[FieldCondition(key, match=MatchValue(value))])``."""

    def __init__(self, must: Sequence[_FieldCondition]):
        self.must = list(must)


def build_qdrant_filters(dir):
    """ingestion.py:207-216."""
    return PayloadFilter([_FieldCondition("dir", dir)])


def filter_conditions(filters) -> Optional[Dict[str, Any]]:
    """Reduce a qdrant ``Filter`` (or our PayloadFilter, or a plain dict) to {key: value} equality terms."""
    if filters is None:
        return None
    if isinstance(filters, dict):
        return dict(filters)
    must = getattr(filters, "must", None)
    if not must:
        return None
    out = {}
    for cond in must:
        out[cond.key] = cond.match.value
    return out
