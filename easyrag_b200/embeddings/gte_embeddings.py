"""Drop-in ``GTEEmbedding`` (reference: src/easyrag/custom/embeddings/gte_embeddings.py:22-112).

Same constructor (``model_name``, ``embed_type``, ``embed_batch_size`` ...), same methods; the Qwen2 forward,
last-token pooling and L2 normalisation run in the CUDA kernels of easyrag_b200/encoder.py instead of
torch/cuBLAS.  Two keyword-only extras exist because this build is offline: ``encoder=`` (a ready
``Qwen2Encoder``) and ``tokenizer=`` (anything callable like a HF tokenizer).  ``precision="fp8"`` builds the encoder
with e4m3 layer GEMMs (Qwen2Encoder); the default "bf16" is the unchanged path.  ``is_causal=True`` runs the model as
``Qwen2Model.forward(is_causal=True)`` does (causal attention in every layer, last-token pooling as before).
"""
from __future__ import annotations

from typing import Any, List

import torch

from ..encoder import PackedBatch, Qwen2Config, Qwen2Encoder, _check_precision
from ..retrievers import get_node_content
from ..schema import BaseEmbedding, PrivateAttr
from . import _loading


class GTEEmbedding(BaseEmbedding):
    # gte_embeddings.py:23-26: private attributes of a (pydantic, when llama_index is installed) BaseEmbedding
    _model: Any = PrivateAttr()
    _tokenizer: Any = PrivateAttr()
    _device: str = PrivateAttr()
    _embed_type: int = PrivateAttr()
    _precision: str = PrivateAttr()
    _is_causal: bool = PrivateAttr()

    def __init__(self, model_name: str = None, embed_type: int = 0, encoder: Qwen2Encoder = None, tokenizer=None,
                 device: str = "cuda", precision: str = "bf16", is_causal: bool = False, **kwargs: Any) -> None:
        _check_precision(precision)
        given = getattr(encoder, "precision", "bf16")
        if encoder is not None and given != precision:
            raise ValueError(f"precision={precision!r} but the given encoder runs {given!r}")
        given_causal = getattr(encoder, "causal", False)
        if encoder is not None and given_causal != bool(is_causal):
            raise ValueError(f"is_causal={is_causal!r} but the given encoder has causal={given_causal!r}")
        if encoder is None:
            cfgd = _loading.load_config(model_name)
            cfg = Qwen2Config(vocab_size=cfgd["vocab_size"], hidden_size=cfgd["hidden_size"],
                              intermediate_size=cfgd["intermediate_size"], num_hidden_layers=cfgd["num_hidden_layers"],
                              num_attention_heads=cfgd["num_attention_heads"],
                              num_key_value_heads=cfgd.get("num_key_value_heads", cfgd["num_attention_heads"]),
                              max_position_embeddings=min(cfgd.get("max_position_embeddings", 8192), 32768),
                              rms_norm_eps=cfgd.get("rms_norm_eps", 1e-6), rope_theta=cfgd.get("rope_theta", 10000.0),
                              sliding_window=cfgd.get("sliding_window"))     # the causal mask applies it (:1050)
            encoder = Qwen2Encoder(cfg, _loading.strip_prefix(_loading.load_state_dict(model_name)), device=device,
                                   precision=precision, causal=is_causal)
        if tokenizer is None:
            tokenizer = _loading.load_tokenizer(model_name)
        kwargs.setdefault("model_name", model_name or "gte-qwen2")
        super().__init__(**kwargs)                 # base fields first, private attributes after (pydantic v1 and v2)
        self._model = encoder
        self._tokenizer = tokenizer
        self._device = str(encoder.device)
        self._embed_type = embed_type
        self._precision = precision
        self._is_causal = bool(is_causal)

    def get_detailed_instruct(self, query: str) -> str:
        """gte_embeddings.py:52-53."""
        return f'Instruct: Given a web search query, retrieve relevant passages that answer the query\nQuery: {query}'

    @classmethod
    def class_name(cls) -> str:
        return "GTEEmbedding"

    def embed_tensor(self, texts: List[str]):
        """-> (bf16 [B, d] on the device, float32 [B, d] on the device); gte_embeddings.py:59-71 without the lists."""
        max_length = min(8192, int(self._model.cfg.max_position_embeddings))     # gte_embeddings.py:60 caps at 8192
        batch_dict = self._tokenizer(texts, max_length=max_length, padding=True, truncation=True, return_tensors='pt')
        batch = PackedBatch.from_padded(torch.as_tensor(batch_dict['input_ids']),
                                        torch.as_tensor(batch_dict['attention_mask']), self._model.device)
        return self._model.embed_packed(batch)

    def _embed(self, texts: List[str]) -> List[List[float]]:
        return self.embed_tensor(texts)[1].cpu().tolist()

    async def _aget_query_embedding(self, query: str) -> List[float]:
        return self._get_query_embedding(query)

    async def _aget_text_embedding(self, text: str) -> List[float]:
        return self._get_text_embedding(text)

    def _get_query_embedding(self, query: str) -> List[float]:
        return self._embed([self.get_detailed_instruct(query)])[0]

    def _get_text_embedding(self, text: str) -> List[float]:
        return self._embed([text])[0]

    def _get_text_embeddings(self, texts: List[str]) -> List[List[float]]:
        return self._embed(texts)

    def __call__(self, nodes, **kwargs: Any):
        embeddings = self.get_text_embedding_batch([get_node_content(node, self._embed_type) for node in nodes], **kwargs)
        for node, embedding in zip(nodes, embeddings):
            node.embedding = embedding
        return nodes

    async def acall(self, nodes, **kwargs: Any):
        embeddings = await self.aget_text_embedding_batch(
            [get_node_content(node, self._embed_type) for node in nodes], **kwargs)
        for node, embedding in zip(nodes, embeddings):
            node.embedding = embedding
        return nodes
