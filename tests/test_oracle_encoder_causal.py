"""CPU: pin the causal Qwen2 oracle against vectors produced by the reference's own Qwen2Model run with is_causal=True."""
import numpy as np
import torch

from _oracle_causal import gte_embed_causal, load_golden, qwen2_hidden_causal
from oracle import encoder as oenc
from easyrag_b200.encoder import Qwen2Config, Qwen2Encoder


def _inputs(z):
    return torch.from_numpy(z["input_ids"]), torch.from_numpy(z["attention_mask"])


def test_causal_oracle_reproduces_reference_model_fp32():
    z, cfg, state = load_golden()
    ids, mask = _inputs(z)
    got = gte_embed_causal(state, cfg, ids, mask, torch.float32).numpy()
    assert np.abs(got - z["emb_fp32"]).max() < 2e-6           # same math, same weights: float32 round-off only
    h = qwen2_hidden_causal(state, cfg, ids, mask, torch.float32)
    real = h[mask.bool()].numpy()                              # every real token, sequences in order
    assert np.abs(real - z["hidden_fp32_packed"]).max() < 2e-5


def test_causal_oracle_bf16_tracks_reference_bf16():
    z, cfg, state = load_golden()
    got = gte_embed_causal(state, cfg, *_inputs(z), torch.bfloat16).numpy()
    cos = (got * z["emb_bf16"]).sum(1) / np.linalg.norm(got, axis=1) / np.linalg.norm(z["emb_bf16"], axis=1)
    assert cos.min() > 1 - 1e-3


def test_causal_oracle_fp64_on_left_padded_batches():
    # the float64 evaluation the GPU tests compare against: every sequence but the longest is left-padded, so padding
    # query rows see no real key.  With the softmax in float32 the float64 mask became -inf there and NaN reached every
    # padded sequence's embedding through the second layer.
    z, cfg, state = load_golden()
    assert cfg.num_hidden_layers >= 2 and (z["attention_mask"][:, 0] == 0).sum() >= 2
    got = gte_embed_causal(state, cfg, *_inputs(z), torch.float64).numpy()
    assert np.isfinite(got).all()
    assert np.abs(got - z["emb_fp32"]).max() < 2e-6


def test_causal_golden_differs_from_bidirectional_oracle():
    # the same weights through the bidirectional oracle land far from the causal reference: the file pins the mask
    z, cfg, state = load_golden()
    bidir = oenc.gte_embed(state, cfg, *_inputs(z), torch.float32).numpy()
    lens = z["attention_mask"].sum(1)
    multi = lens > 1                                           # a 1-token sequence is the same either way
    assert np.abs(bidir - z["emb_fp32"]).max(1)[multi].min() > 1e-3
    assert np.abs(bidir - z["emb_fp32"])[~multi].max() < 2e-6


def test_causal_oracle_rows_ignore_later_tokens():
    z, cfg, state = load_golden()
    ids, mask = _inputs(z)
    ids2 = ids.clone()
    ids2[:, -10:] = 7                                          # every sequence is left-padded: its last 10 tokens
    a = qwen2_hidden_causal(state, cfg, ids, mask)
    b = qwen2_hidden_causal(state, cfg, ids2, mask)
    keep = mask.bool().clone()                                 # the real tokens before the change
    keep[:, -10:] = False                                      # (a padding row sees every column: it is not compared)
    assert keep.sum() > 100
    assert torch.equal(a[keep], b[keep])
    assert not torch.allclose(a[0, -10:], b[0, -10:])


def test_causal_encoder_flops_count_visible_keys():
    cfg = Qwen2Config(vocab_size=10, hidden_size=3584, intermediate_size=18944, num_hidden_layers=2,
                      num_attention_heads=28, num_key_value_heads=4)
    models = {}
    for causal in (False, True):                               # flops() reads the config only: no device needed
        m = Qwen2Encoder.__new__(Qwen2Encoder)
        m.cfg, m.causal = cfg, causal
        models[causal] = m
    d, layers = cfg.hidden_size, cfg.num_hidden_layers
    for n in (1, 64, 1024, 8192):
        diff = models[False].flops([n]) - models[True].flops([n])
        assert diff == layers * (4 * n * n * d - 2 * n * (n + 1) * d)
