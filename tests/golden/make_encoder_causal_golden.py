#!/usr/bin/env python
"""Generates tests/golden/qwen2_tiny_causal.npz from the REFERENCE's own vendored model, run with is_causal=True.

Run in the authoring container only (needs the reference checkout, which the GPU machines do not have):

    python tests/golden/make_encoder_causal_golden.py

The same recipe as make_encoder_golden.py -- ``easyrag.utils.modeling_qwen.Qwen2Model`` imported unmodified, a tiny
random config, a left-padded batch, last_token_pool, F.normalize -- except that the model is called with
``is_causal=True`` (modeling_qwen.py:968; mask = padding mask + causal mask, :1043-1051).  The causal mask also applies
``config.sliding_window`` (:1050); it is set to None here (use_sliding_window=False), so no window is in play.
Recorded:
  * the weights (values already rounded to bf16, stored as float32),
  * input_ids / attention_mask,
  * emb_fp32 / emb_bf16: the pipeline evaluated in float32 / bfloat16,
  * hidden_fp32_packed: the float32 last_hidden_state of every real token, sequences one after another.
The two transformers-5 config shims of make_encoder_golden.py are kept (cfg.rope_theta, use_cache=False).
"""
import sys
from pathlib import Path

import numpy as np
import torch
import torch.nn.functional as F

REF = Path("/root/reference/src")
OUT = Path(__file__).resolve().parent / "qwen2_tiny_causal.npz"


def last_token_pool(h, mask):
    """gte_embeddings.py:42-50."""
    left_padding = (mask[:, -1].sum() == mask.shape[0])
    if left_padding:
        return h[:, -1]
    lens = mask.sum(dim=1) - 1
    return h[torch.arange(h.shape[0]), lens]


def main():
    sys.path.insert(0, str(REF))
    from transformers import Qwen2Config
    from easyrag.utils.modeling_qwen import Qwen2Model

    torch.manual_seed(20241017)
    cfg = Qwen2Config(vocab_size=512, hidden_size=128, intermediate_size=256, num_hidden_layers=2,
                      num_attention_heads=2, num_key_value_heads=1, max_position_embeddings=512, rms_norm_eps=1e-6,
                      use_cache=False, use_sliding_window=False, attn_implementation="eager")
    cfg.rope_theta = 1000000.0
    cfg.use_sliding_window = False
    cfg.sliding_window = None
    model = Qwen2Model(cfg).eval()
    with torch.no_grad():
        for name, p in model.named_parameters():
            if "norm" in name:
                p.copy_(1.0 + 0.1 * torch.randn_like(p))
            elif name.endswith("bias"):
                p.copy_(0.05 * torch.randn_like(p))
            else:
                p.copy_(0.06 * torch.randn_like(p))
            p.copy_(p.to(torch.bfloat16).float())            # bf16-representable weights
    lens = [37, 5, 64, 1, 23, 50]
    L = max(lens)
    ids = torch.zeros(len(lens), L, dtype=torch.long)
    mask = torch.zeros(len(lens), L, dtype=torch.long)
    for i, n in enumerate(lens):                              # tokenizer pads LEFT (tokenization_qwen.py:218)
        ids[i, L - n:] = torch.randint(1, cfg.vocab_size, (n,))
        mask[i, L - n:] = 1
    with torch.no_grad():
        h32 = model(input_ids=ids, attention_mask=mask, is_causal=True).last_hidden_state
        emb32 = F.normalize(last_token_pool(h32, mask), p=2, dim=1)
        mb = Qwen2Model(cfg).eval()
        mb.load_state_dict(model.state_dict())
        mb = mb.to(torch.bfloat16)
        hb = mb(input_ids=ids, attention_mask=mask, is_causal=True).last_hidden_state
        embb = F.normalize(last_token_pool(hb, mask), p=2, dim=1).to(torch.float)
    packed = torch.cat([h32[i, L - n:] for i, n in enumerate(lens)])
    blob = {f"w::{k}": v.detach().numpy().astype(np.float32) for k, v in model.state_dict().items()
            if "rotary_emb" not in k}
    blob.update(input_ids=ids.numpy().astype(np.int32), attention_mask=mask.numpy().astype(np.int32),
                emb_fp32=emb32.numpy(), emb_bf16=embb.numpy(), hidden_fp32_packed=packed.numpy(),
                cfg=np.array([cfg.vocab_size, cfg.hidden_size, cfg.intermediate_size, cfg.num_hidden_layers,
                              cfg.num_attention_heads, cfg.num_key_value_heads, cfg.max_position_embeddings],
                             dtype=np.int64),
                rope_theta=np.array([cfg.rope_theta]), rms_norm_eps=np.array([cfg.rms_norm_eps]))
    np.savez_compressed(OUT, **blob)
    print("wrote", OUT, OUT.stat().st_size, "bytes; cos(fp32,bf16) =",
          F.cosine_similarity(emb32, embb).min().item())


if __name__ == "__main__":
    main()
