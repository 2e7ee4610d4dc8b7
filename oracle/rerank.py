"""Oracle: the cross-encoder reranker of the reference (SentenceTransformerRerank, rerankers.py:15-99).  TEST
INFRASTRUCTURE ONLY.

* ``cross_encoder_inputs`` restates what ``CrossEncoder.predict`` tokenises for one (query, passage) pair: the fast
  tokenizer's pair encoding with ``truncation="longest_first"`` at ``max_length``, on ids tokenised without special
  tokens.  Pinned against a real ``tokenizers`` fast tokenizer in tests/test_rerank_host.py.
* ``cross_encoder_scores`` is transformers' ``BertForSequenceClassification`` / ``XLMRobertaForSequenceClassification``
  (installed library, eager attention) over right-padded batches of 32, followed by the sigmoid of
  ``CrossEncoder.predict`` for one label.  sentence-transformers itself is absent here: PARITY UNPINNED for that
  wrapper, restated from its published behaviour.
* ``rerank_order`` is the literal ``sorted`` of ``_postprocess_nodes`` (rerankers.py:94-96).
"""
from __future__ import annotations

from typing import Dict, List, Sequence, Tuple

import numpy as np
import torch

# family -> (separators between the two segments, token type of the second segment)
TEMPLATES = {"bert": (1, 1), "roberta": (2, 0)}


def truncate_longest_first(a: int, b: int, room: int) -> Tuple[int, int]:
    """Lengths kept of a query of ``a`` and a passage of ``b`` tokens when ``room`` tokens are left for both."""
    if a + b <= room:
        return a, b
    if a > b:
        nb = min(b, room // 2)
        return room - nb, nb
    na = min(a, room // 2)
    return na, room - na


def cross_encoder_inputs(query: Sequence[int], passage: Sequence[int], max_length: int, family: str, cls: int,
                         sep: int, pad_id: int = 1) -> Tuple[List[int], List[int], List[int]]:
    """-> (input_ids, token_type_ids, position_ids) of one pair.  BERT: ``[CLS] q [SEP] p [SEP]``, types 0 | 1,
    positions from 0.  RoBERTa / XLM-R: ``<s> q </s></s> p </s>``, types 0, positions from ``pad_id + 1``."""
    n_mid, type_b = TEMPLATES[family]
    na, nb = truncate_longest_first(len(query), len(passage), max_length - 2 - n_mid)
    head = [cls] + list(query[:na]) + [sep] * n_mid
    tail = list(passage[:nb]) + [sep]
    ids = head + tail
    types = [0] * (na + 2) + [type_b] * (len(ids) - na - 2)
    off = pad_id + 1 if family == "roberta" else 0
    return ids, types, list(range(off, off + len(ids)))


def _hf_model(family: str, cfg, state: Dict[str, torch.Tensor], pad_id: int):
    common = dict(vocab_size=cfg.vocab_size, hidden_size=cfg.hidden_size, num_hidden_layers=cfg.num_hidden_layers,
                  num_attention_heads=cfg.num_attention_heads, intermediate_size=cfg.intermediate_size,
                  max_position_embeddings=cfg.max_position_embeddings, layer_norm_eps=cfg.layer_norm_eps,
                  hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0, num_labels=1,
                  attn_implementation="eager")
    if family == "bert":
        from transformers import BertConfig, BertForSequenceClassification
        model = BertForSequenceClassification(BertConfig(**common))
    else:
        from transformers import XLMRobertaConfig, XLMRobertaForSequenceClassification
        model = XLMRobertaForSequenceClassification(XLMRobertaConfig(pad_token_id=pad_id, type_vocab_size=1, **common))
    missing, unexpected = model.load_state_dict({k: v.float() for k, v in state.items()}, strict=False)
    assert not [m for m in missing if "position_ids" not in m and "token_type_ids" not in m], missing
    assert not unexpected, unexpected
    return model.eval()


def cross_encoder_scores(family: str, cfg, state: Dict[str, torch.Tensor], pairs: Sequence[Tuple[List[int], List[int]]],
                         pad_id: int = 1, dtype=torch.float32, batch_size: int = 32, device="cpu"
                         ) -> Tuple[np.ndarray, np.ndarray]:
    """``pairs`` = (input_ids, token_type_ids) from :func:`cross_encoder_inputs` -> (logits, sigmoid scores), float32
    [N].  ``dtype=torch.bfloat16`` evaluates the same model in bf16: its distance from the fp32 result is the noise
    floor of any bf16 evaluation of these weights.  Padding uses ``pad_id`` (RoBERTa derives positions from it)."""
    model = _hf_model(family, cfg, state, pad_id).to(device=device, dtype=dtype)
    logits = []
    for b0 in range(0, len(pairs), batch_size):
        chunk = pairs[b0:b0 + batch_size]
        width = max(len(ids) for ids, _ in chunk)
        ids = torch.full((len(chunk), width), pad_id, dtype=torch.long)
        types = torch.zeros(len(chunk), width, dtype=torch.long)
        mask = torch.zeros(len(chunk), width, dtype=torch.long)
        for i, (s, t) in enumerate(chunk):
            ids[i, :len(s)] = torch.tensor(s)
            types[i, :len(t)] = torch.tensor(t)
            mask[i, :len(s)] = 1
        with torch.no_grad():
            out = model(input_ids=ids.to(device), attention_mask=mask.to(device),
                        token_type_ids=types.to(device)).logits
        logits.append(out.float().cpu()[:, 0])
    lg = torch.cat(logits) if logits else torch.zeros(0)
    return lg.numpy(), torch.sigmoid(lg).numpy()


def rerank_order(scores: Sequence[float], top_n: int) -> List[int]:
    """Indices of ``sorted(nodes, key=lambda x: -x.score if x.score else 0)[:top_n]`` for nodes scored ``scores``."""
    return sorted(range(len(scores)), key=lambda i: -scores[i] if scores[i] else 0)[:top_n]
