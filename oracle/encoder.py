"""Oracle: the embedding forward pass of the reference in plain PyTorch.  TEST INFRASTRUCTURE ONLY.

* ``qwen2_hidden`` / ``gte_embed`` restate the bidirectional Qwen2 forward of the reference's vendored model
  (src/easyrag/utils/modeling_qwen.py: RMSNorm :82-96, rotary :100-170, MLP :174-186, eager attention with
  ``is_causal=False`` :202-324, decoder layer :729-805, model :956-1116) and the pooling / normalisation of
  GTEEmbedding._embed (gte_embeddings.py:42-50,59-72), in the padded-batch form the reference runs.
  Pinned against tests/golden/qwen2_tiny.npz, which was produced by the reference's own module
  (tests/golden/make_encoder_golden.py) -- see tests/test_oracle_encoder.py.
* ``bert_embed`` is transformers.BertModel (installed library) + CLS/mean pooling + L2 norm: what
  SentenceTransformer.encode(normalize_embeddings=True) computes for bge-*/gte-base checkpoints
  (hf_embeddings.py:118-123).  sentence-transformers itself is absent here: PARITY UNPINNED for that wrapper.
"""
from __future__ import annotations

import math
from typing import Dict

import torch
import torch.nn.functional as F


def _rms(x, w, eps):
    dt = x.dtype
    x = x.to(torch.float32)
    var = x.pow(2).mean(-1, keepdim=True)
    x = x * torch.rsqrt(var + eps)
    return w * x.to(dt)


def _rotate_half(x):
    x1 = x[..., : x.shape[-1] // 2]
    x2 = x[..., x.shape[-1] // 2:]
    return torch.cat((-x2, x1), dim=-1)


def qwen2_hidden(state: Dict[str, torch.Tensor], cfg, input_ids: torch.Tensor, attention_mask: torch.Tensor,
                 dtype=torch.float32, device="cpu") -> torch.Tensor:
    """[B, L] ids + mask -> last_hidden_state [B, L, d] (final norm applied), non-causal, additive padding mask.
    Runs on ``device``: weights, inputs and the position / mask / rotary tensors are all placed there."""
    d, H, KV = cfg.hidden_size, cfg.num_attention_heads, cfg.num_key_value_heads
    hd = d // H
    w = {k: v.to(device=device, dtype=dtype) for k, v in state.items()}
    input_ids, attention_mask = input_ids.to(device), attention_mask.to(device)
    b, l = input_ids.shape
    x = F.embedding(input_ids.long(), w["embed_tokens.weight"])
    pos = torch.arange(l, device=device)
    inv_freq = 1.0 / (cfg.rope_theta ** (torch.arange(0, hd, 2, dtype=torch.int64, device=device).float() / hd))
    freqs = torch.outer(pos.float(), inv_freq)
    emb = torch.cat((freqs, freqs), dim=-1)
    cos, sin = emb.cos().to(dtype)[None, None], emb.sin().to(dtype)[None, None]
    # padding-only additive mask (modeling_qwen.py:1052-1056 with is_causal=False)
    neg = torch.finfo(dtype).min
    add = torch.zeros(b, 1, l, l, dtype=dtype, device=device)
    add = add.masked_fill(attention_mask[:, None, None, :] == 0, neg)
    for i in range(cfg.num_hidden_layers):
        p = f"layers.{i}."
        res = x
        h = _rms(x, w[p + "input_layernorm.weight"], cfg.rms_norm_eps)
        q = F.linear(h, w[p + "self_attn.q_proj.weight"], w[p + "self_attn.q_proj.bias"]).view(b, l, H, hd).transpose(1, 2)
        k = F.linear(h, w[p + "self_attn.k_proj.weight"], w[p + "self_attn.k_proj.bias"]).view(b, l, KV, hd).transpose(1, 2)
        v = F.linear(h, w[p + "self_attn.v_proj.weight"], w[p + "self_attn.v_proj.bias"]).view(b, l, KV, hd).transpose(1, 2)
        q = q * cos + _rotate_half(q) * sin
        k = k * cos + _rotate_half(k) * sin
        k = k.repeat_interleave(H // KV, dim=1)
        v = v.repeat_interleave(H // KV, dim=1)
        att = torch.matmul(q, k.transpose(2, 3)) / math.sqrt(hd) + add
        att = F.softmax(att, dim=-1, dtype=torch.float32).to(dtype)
        o = torch.matmul(att, v).transpose(1, 2).reshape(b, l, H * hd)
        x = res + F.linear(o, w[p + "self_attn.o_proj.weight"])
        res = x
        h = _rms(x, w[p + "post_attention_layernorm.weight"], cfg.rms_norm_eps)
        h = F.linear(F.silu(F.linear(h, w[p + "mlp.gate_proj.weight"])) * F.linear(h, w[p + "mlp.up_proj.weight"]),
                     w[p + "mlp.down_proj.weight"])
        x = res + h
    return _rms(x, w["norm.weight"], cfg.rms_norm_eps)


def last_token_pool(h: torch.Tensor, attention_mask: torch.Tensor) -> torch.Tensor:
    """gte_embeddings.py:42-50."""
    left_padding = (attention_mask[:, -1].sum() == attention_mask.shape[0])
    if left_padding:
        return h[:, -1]
    lens = attention_mask.sum(dim=1) - 1
    return h[torch.arange(h.shape[0]), lens]


def gte_embed(state, cfg, input_ids, attention_mask, dtype=torch.float32, device="cpu") -> torch.Tensor:
    """GTEEmbedding._embed after tokenisation (gte_embeddings.py:65-71) -> float32 [B, d] on ``device``."""
    h = qwen2_hidden(state, cfg, input_ids, attention_mask, dtype, device)
    e = F.normalize(last_token_pool(h, attention_mask.to(device)), p=2, dim=1)
    return e.to(torch.float)


def pad_left(seqs, pad_id=0):
    l = max(len(s) for s in seqs)
    ids = torch.full((len(seqs), l), pad_id, dtype=torch.long)
    mask = torch.zeros(len(seqs), l, dtype=torch.long)
    for i, s in enumerate(seqs):
        ids[i, l - len(s):] = torch.tensor(s, dtype=torch.long)
        mask[i, l - len(s):] = 1
    return ids, mask


def pad_right(seqs, pad_id=0):
    l = max(len(s) for s in seqs)
    ids = torch.full((len(seqs), l), pad_id, dtype=torch.long)
    mask = torch.zeros(len(seqs), l, dtype=torch.long)
    for i, s in enumerate(seqs):
        ids[i, :len(s)] = torch.tensor(s, dtype=torch.long)
        mask[i, :len(s)] = 1
    return ids, mask


def bert_embed(state, cfg, seqs, pooling: str = "cls", normalize: bool = True, device="cpu",
               dtype=torch.float32) -> torch.Tensor:
    """transformers.BertModel (eager; fp32 = what SentenceTransformer.encode runs, hf_embeddings.py:80-92 passes no
    dtype) + pooling + F.normalize -> float32 [B, d].  ``dtype=torch.bfloat16`` evaluates the same model in bf16: its
    distance from the fp32 result is the noise floor of ANY bf16 evaluation of these weights."""
    from transformers import BertConfig as HFBertConfig, BertModel
    hf = HFBertConfig(vocab_size=cfg.vocab_size, hidden_size=cfg.hidden_size, num_hidden_layers=cfg.num_hidden_layers,
                      num_attention_heads=cfg.num_attention_heads, intermediate_size=cfg.intermediate_size,
                      max_position_embeddings=cfg.max_position_embeddings, layer_norm_eps=cfg.layer_norm_eps,
                      hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0, attn_implementation="eager")
    model = BertModel(hf, add_pooling_layer=False).eval()
    missing, unexpected = model.load_state_dict({k: v.float() for k, v in state.items()}, strict=False)
    assert not [m for m in missing if "position_ids" not in m], missing
    model = model.to(device=device, dtype=dtype)
    ids, mask = pad_right(seqs)
    with torch.no_grad():
        h = model(input_ids=ids.to(device), attention_mask=mask.to(device)).last_hidden_state.float()
    m = mask.to(device).unsqueeze(-1).float()
    if pooling == "cls":
        e = h[:, 0]
    elif pooling == "mean":
        e = (h * m).sum(1) / m.sum(1)
    else:
        e = h[torch.arange(h.shape[0]), mask.sum(1) - 1]
    if normalize:
        e = F.normalize(e, p=2, dim=1)
    return e.float().cpu()
