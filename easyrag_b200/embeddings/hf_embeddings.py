"""Drop-in ``HuggingFaceEmbedding`` (reference: src/easyrag/custom/embeddings/hf_embeddings.py:25-165).

The reference wraps ``SentenceTransformer(model_name).encode(..., normalize_embeddings=True)``; here the BERT-shaped
encoder, pooling and normalisation run in easyrag_b200/encoder.py's CUDA kernels.  Same constructor arguments
(including the rejection of the deprecated ones, hf_embeddings.py:67-78) and methods.  ``precision="fp8"`` builds
the encoder with e4m3 layer GEMMs (BertEncoder); the default "bf16" is the unchanged path.
"""
from __future__ import annotations

import json
from pathlib import Path
from typing import Any, List, Optional

import torch

from ..encoder import BertConfig, BertEncoder, PackedBatch, _check_precision
from ..retrievers import get_node_content
from ..schema import BaseEmbedding, Field, PrivateAttr
from . import _loading

DEFAULT_HUGGINGFACE_LENGTH = 512
DEFAULT_EMBED_BATCH_SIZE = 10
DEFAULT_HUGGINGFACE_EMBEDDING_MODEL = "BAAI/bge-small-en"

BGE_QUERY_EN = "Represent this sentence for searching relevant passages: "
BGE_QUERY_ZH = "为这个句子生成表示以用于检索相关文章："


def get_query_instruct_for_model_name(model_name: Optional[str]) -> str:
    """llama_index.embeddings.huggingface.utils: BGE models prepend an instruction to queries only."""
    name = (model_name or "").lower()
    if "bge" in name:
        return BGE_QUERY_ZH if "zh" in name else BGE_QUERY_EN
    return ""


def get_text_instruct_for_model_name(model_name: Optional[str]) -> str:
    return ""


def _pooling_from_dir(model_dir: str) -> str:
    cfg = Path(model_dir) / "1_Pooling" / "config.json"
    if cfg.exists():
        c = json.loads(cfg.read_text())
        if c.get("pooling_mode_mean_tokens"):
            return "mean"
        if c.get("pooling_mode_lasttoken"):
            return "last"
    return "cls"


class HuggingFaceEmbedding(BaseEmbedding):
    # declared like the reference (hf_embeddings.py:26-43): with llama_index installed BaseEmbedding is a pydantic
    # model, which only accepts declared fields / private attributes
    max_length: int = Field(default=DEFAULT_HUGGINGFACE_LENGTH, description="Maximum length of input.", gt=0)
    normalize: bool = Field(default=True, description="Normalize embeddings or not.")
    query_instruction: Optional[str] = Field(default=None, description="Instruction to prepend to query text.")
    text_instruction: Optional[str] = Field(default=None, description="Instruction to prepend to text.")
    cache_folder: Optional[str] = Field(default=None, description="Cache folder for Hugging Face files.")

    _model: Any = PrivateAttr()
    _tok: Any = PrivateAttr()
    _prompts: Any = PrivateAttr()
    _device: str = PrivateAttr()
    _embed_type: int = PrivateAttr()
    _precision: str = PrivateAttr()

    def __init__(self, model_name: str = DEFAULT_HUGGINGFACE_EMBEDDING_MODEL, tokenizer_name: Optional[str] = "deprecated",
                 pooling: str = "deprecated", max_length: Optional[int] = None, query_instruction: Optional[str] = None,
                 text_instruction: Optional[str] = None, normalize: bool = True, model: Optional[Any] = "deprecated",
                 tokenizer: Optional[Any] = "deprecated", embed_batch_size: int = DEFAULT_EMBED_BATCH_SIZE,
                 cache_folder: Optional[str] = None, trust_remote_code: bool = False, device: Optional[str] = None,
                 callback_manager=None, embed_type: int = 0, encoder: BertEncoder = None, hf_tokenizer=None,
                 precision: str = "bf16", **model_kwargs):
        device = device or "cuda"
        _check_precision(precision)
        given = getattr(encoder, "precision", "bf16")
        if encoder is not None and given != precision:
            raise ValueError(f"precision={precision!r} but the given encoder runs {given!r}")
        for variable, value in [("model", model), ("tokenizer", tokenizer), ("pooling", pooling),
                                ("tokenizer_name", tokenizer_name)]:
            if value != "deprecated":
                raise ValueError(f"{variable} is deprecated. Please remove it from the arguments.")
        if model_name is None:
            raise ValueError("The `model_name` argument must be provided.")
        if encoder is None:
            c = _loading.load_config(model_name)
            cfg = BertConfig(vocab_size=c["vocab_size"], hidden_size=c["hidden_size"],
                             intermediate_size=c["intermediate_size"], num_hidden_layers=c["num_hidden_layers"],
                             num_attention_heads=c["num_attention_heads"],
                             max_position_embeddings=c.get("max_position_embeddings", 512),
                             layer_norm_eps=c.get("layer_norm_eps", 1e-12))
            encoder = BertEncoder(cfg, _loading.strip_prefix(_loading.load_state_dict(model_name)),
                                  device=device, pooling=_pooling_from_dir(model_name), precision=precision)
        max_pos = int(encoder.cfg.max_position_embeddings)
        max_length = max_length or min(DEFAULT_HUGGINGFACE_LENGTH, max_pos)
        if max_length > max_pos:
            # the position table has max_pos rows; a longer input would index past it
            raise ValueError(f"max_length={max_length} exceeds the model's max_position_embeddings={max_pos}")
        # public fields go through the base constructor (pydantic validates them), private attributes after it
        super().__init__(embed_batch_size=embed_batch_size, callback_manager=callback_manager, model_name=model_name,
                         max_length=max_length, normalize=normalize, query_instruction=query_instruction,
                         text_instruction=text_instruction, cache_folder=cache_folder)
        self._device = device
        self._embed_type = embed_type
        self._precision = precision
        self._model = encoder
        self._tok = hf_tokenizer if hf_tokenizer is not None else _loading.load_tokenizer(model_name)
        self._prompts = {"query": query_instruction or get_query_instruct_for_model_name(model_name),
                         "text": text_instruction or get_text_instruct_for_model_name(model_name)}

    @classmethod
    def class_name(cls) -> str:
        return "HuggingFaceEmbedding"

    def embed_tensor(self, sentences: List[str], prompt_name: Optional[str] = None):
        prompt = self._prompts.get(prompt_name, "") if prompt_name else ""
        texts = [prompt + s for s in sentences]
        out_b, out_f = [], []
        bs = max(1, int(self.embed_batch_size))
        for i in range(0, len(texts), bs):
            enc = self._tok(texts[i:i + bs], max_length=self.max_length, padding=True, truncation=True,
                            return_tensors='pt')
            batch = PackedBatch.from_padded(torch.as_tensor(enc['input_ids']), torch.as_tensor(enc['attention_mask']),
                                            self._model.device, column_positions=False)
            b, f = self._model.embed_packed(batch, normalize=self.normalize)
            out_b.append(b)
            out_f.append(f)
        return torch.cat(out_b), torch.cat(out_f)

    def _embed(self, sentences, prompt_name: Optional[str] = None):
        """hf_embeddings.py:112-123: a str gives one vector, a list gives a list of vectors (SentenceTransformer.encode)."""
        single = isinstance(sentences, str)
        f = self.embed_tensor([sentences] if single else list(sentences), prompt_name)[1].cpu()
        return f[0].tolist() if single else f.tolist()

    def _get_query_embedding(self, query: str) -> List[float]:
        return self._embed(query, prompt_name="query")

    async def _aget_query_embedding(self, query: str) -> List[float]:
        return self._get_query_embedding(query)

    async def _aget_text_embedding(self, text: str) -> List[float]:
        return self._get_text_embedding(text)

    def _get_text_embedding(self, text: str) -> List[float]:
        return self._embed(text, prompt_name="text")

    def _get_text_embeddings(self, texts: List[str]) -> List[List[float]]:
        return self._embed(texts, prompt_name="text")

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
