"""Causal form of the Qwen2 oracle (oracle/encoder.py) for the tests: the same plain-PyTorch restatement of the
reference's vendored Qwen2Model, called with ``is_causal=True`` (modeling_qwen.py:968): the additive mask is the
padding mask plus the causal mask (:1043-1051, no sliding window).  Pinned against tests/golden/qwen2_tiny_causal.npz
(tests/golden/make_encoder_causal_golden.py) by tests/test_oracle_encoder_causal.py."""
from __future__ import annotations

import math
from pathlib import Path
from typing import Dict

import numpy as np
import torch
import torch.nn.functional as F

from oracle.encoder import _rms, _rotate_half, last_token_pool
from easyrag_b200.encoder import Qwen2Config

GOLD = Path(__file__).parent / "golden" / "qwen2_tiny_causal.npz"


def causal_mask(attention_mask: torch.Tensor, dtype) -> torch.Tensor:
    """[B, L] 0/1 padding mask -> additive [B, 1, L, L]: the minimum of ``dtype`` where query row i may not see key j
    (j > i, or j a padding column), 0 elsewhere."""
    b, l = attention_mask.shape
    neg = torch.finfo(dtype).min
    future = torch.ones(l, l, dtype=torch.bool, device=attention_mask.device).triu(1)
    blocked = future[None, None] | (attention_mask[:, None, None, :] == 0)
    return torch.zeros(b, 1, l, l, dtype=dtype, device=attention_mask.device).masked_fill(blocked, neg)


def qwen2_hidden_causal(state: Dict[str, torch.Tensor], cfg, input_ids: torch.Tensor, attention_mask: torch.Tensor,
                        dtype=torch.float32, device="cpu") -> torch.Tensor:
    """oracle.encoder.qwen2_hidden with is_causal=True: [B, L] ids + mask -> last_hidden_state [B, L, d]."""
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
    add = causal_mask(attention_mask, dtype)
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
        # the reference's softmax runs in float32; a float64 evaluation keeps float64, where float64's minimum stays
        # finite.  Cast to float32 it is -inf, a padding query row (which sees no real key) turns NaN, and 0 * NaN
        # carries that into every real row of the next layer through the padding keys and values.
        att = F.softmax(att, dim=-1, dtype=torch.float64 if dtype == torch.float64 else torch.float32).to(dtype)
        o = torch.matmul(att, v).transpose(1, 2).reshape(b, l, H * hd)
        x = res + F.linear(o, w[p + "self_attn.o_proj.weight"])
        res = x
        h = _rms(x, w[p + "post_attention_layernorm.weight"], cfg.rms_norm_eps)
        h = F.linear(F.silu(F.linear(h, w[p + "mlp.gate_proj.weight"])) * F.linear(h, w[p + "mlp.up_proj.weight"]),
                     w[p + "mlp.down_proj.weight"])
        x = res + h
    return _rms(x, w["norm.weight"], cfg.rms_norm_eps)


def gte_embed_causal(state, cfg, input_ids, attention_mask, dtype=torch.float32, device="cpu") -> torch.Tensor:
    """oracle.encoder.gte_embed with is_causal=True -> float32 [B, d] on ``device``."""
    h = qwen2_hidden_causal(state, cfg, input_ids, attention_mask, dtype, device)
    e = F.normalize(last_token_pool(h, attention_mask.to(device)), p=2, dim=1)
    return e.to(torch.float)


def load_golden():
    z = np.load(GOLD)
    c = z["cfg"]
    cfg = Qwen2Config(vocab_size=int(c[0]), hidden_size=int(c[1]), intermediate_size=int(c[2]),
                      num_hidden_layers=int(c[3]), num_attention_heads=int(c[4]), num_key_value_heads=int(c[5]),
                      max_position_embeddings=int(c[6]), rms_norm_eps=float(z["rms_norm_eps"][0]),
                      rope_theta=float(z["rope_theta"][0]))
    state = {k[3:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("w::")}
    return z, cfg, state
