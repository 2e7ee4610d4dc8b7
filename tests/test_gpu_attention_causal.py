"""GPU: causal attention (ezr_attn_causal, the CAUSAL instances of attention_tc.cuh) and the causal Qwen2 encoder.

* Against fp64 at the head shapes of gte-Qwen2-7B (28 / 4 heads of 128) and MiniCPM-2B (36 heads of 64): a
  per-element bound built from the kernel's rounding points, with row r seeing r + 1 keys, and a per-head rms check
  against an fp64 emulation of those rounding points.  Negative controls (the bidirectional output, a diagonal shifted
  either way, the diagonal tile dropped) must be rejected by the same checks.
* Exact properties that follow from the kernel walking the same key tiles in the same order with the same arithmetic
  as the bidirectional instance, fully masked keys adding exact zeros: causal row i of a sequence equals, bit for bit,
  the last row of ezr_attn_bidir on its prefix of i + 1 tokens; rows 0..i do not move when later positions change.
* The encoder: Qwen2Encoder(causal=True) against the reference's own Qwen2Model run with is_causal=True
  (tests/golden/qwen2_tiny_causal.npz) and against the causal fp32 oracle at gte-Qwen2-7B width; prefix identity of
  the hidden states in bf16 and fp8; the GTEEmbedding flag.
"""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from _attn_ref import _causal_check as _check, _causal_ref as _ref, _kernel_tiles
from _bounds import rejects
from _oracle_causal import gte_embed_causal, load_golden
from oracle import encoder as oenc
from easyrag_b200 import _lib, encoder as enc
from easyrag_b200.encoder import PackedBatch, Qwen2Config, Qwen2Encoder, random_state

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture(scope="module", autouse=True)
def _ready(lib_built):
    _lib.require_cuda()


def _randn(*shape, seed, std=1.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(*shape, generator=g, device=DEV) * std).to(torch.bfloat16)


def _cu(lens):
    return torch.tensor(np.cumsum([0] + list(lens)), dtype=torch.int32, device=DEV)


def _causal(qkv, lens, H, KV, hd):
    out = enc.attention(qkv, _cu(lens), max(lens), H, KV, hd, causal=True)
    torch.cuda.synchronize()
    assert _lib.lib().ezr_attn_last_kernel() == b"wgmma-causal"
    return out


def _bidir(qkv, lens, H, KV, hd):
    out = enc.attention(qkv, _cu(lens), max(lens), H, KV, hd)
    torch.cuda.synchronize()
    return out


LENS = [1, 2, 63, 64, 65, 127, 128, 129, 300, 1024, 4097, 8192]
SHAPES = [(28, 4, 128), (36, 36, 64)]          # gte-Qwen2-7B (GQA group 7), MiniCPM-2B


@pytest.mark.parametrize("H,KV,hd", SHAPES, ids=["gte-qwen2-7b", "minicpm-2b"])
def test_causal_attention_model_shapes_vs_fp64(H, KV, hd):
    lens = LENS
    t = sum(lens)
    qkv = _randn(t, (H + 2 * KV) * hd, seed=60 + H, std=0.8)
    got = _causal(qkv, lens, H, KV, hd).view(t, H, hd)
    scale = 1.0 / math.sqrt(hd)
    offs = np.cumsum([0] + lens)
    worst = 0.0
    for b, n in enumerate(lens):
        rows = qkv[offs[b]:offs[b] + n]
        r = torch.arange(n, device=DEV)
        ref = _ref(rows, H, KV, hd, scale, r + 1)
        worst = max(worst, _check(got[offs[b]:offs[b] + n], ref, r + 1, _kernel_tiles(n), f"seq {b} (len {n})"))
    print(f"\n[bounds] causal attention H={H} KV={KV} hd={hd}: worst_rms_ratio={worst:.4g}, tokens={t}")
    # negative controls on a 300-token sequence, each on the rows where it differs from causal attention
    b = lens.index(300)
    n = 300
    rows = qkv[offs[b]:offs[b] + n]
    g_b = got[offs[b]:offs[b] + n]
    r = torch.arange(n, device=DEV)
    tiles = _kernel_tiles(n)
    bid = _bidir(qkv, lens, H, KV, hd).view(t, H, hd)[offs[b]:offs[b] + n]
    ref = _ref(rows, H, KV, hd, scale, r + 1)
    sel = slice(0, n - 1)                                     # the last row sees every key either way
    assert rejects(_check, bid[sel], tuple(x[sel] for x in ref), (r + 1)[sel], tiles[sel], "control: bidirectional")
    controls = {
        "diagonal excluded": (r, slice(1, n)),                                   # row r sees keys 0 .. r - 1
        "one future key included": (torch.clamp(r + 2, max=n), slice(0, n - 1)),  # keys 0 .. r + 1
        "diagonal tile dropped": ((r // 64) * 64, slice(64, n)),                 # keys of earlier tiles only
    }
    for what, (hi, sel) in controls.items():
        wrong = _ref(rows, H, KV, hd, scale, hi)
        assert rejects(_check, g_b[sel], tuple(x[sel] for x in wrong), hi[sel], tiles[sel], f"control: {what}"), \
            f"accepted a reference with the {what}"


# ------------------------------------------------------------------------------------------ exact properties
PREFIX_CASES = [(64, 4, 4), (64, 6, 2), (128, 4, 1), (128, 2, 2)]     # (hd, H, KV): MHA and GQA at both head dims
PREFIX_LENS = [1, 2, 63, 64, 65, 127, 128, 129, 191, 192, 193, 257, 300]


@pytest.mark.parametrize("hd,H,KV", PREFIX_CASES, ids=[f"hd{c[0]}-H{c[1]}-KV{c[2]}" for c in PREFIX_CASES])
def test_causal_row_equals_bidirectional_last_row_of_its_prefix(hd, H, KV):
    lens = PREFIX_LENS
    t = sum(lens)
    qkv = _randn(t, (H + 2 * KV) * hd, seed=7 * hd + H, std=0.9)
    got = _causal(qkv, lens, H, KV, hd)
    offs = np.cumsum([0] + lens)
    # every prefix S[:i + 1] of every sequence, packed as a sequence of its own, through the bidirectional kernel
    idx, plens = [], []
    for b, n in enumerate(lens):
        for i in range(n):
            idx.append(torch.arange(offs[b], offs[b] + i + 1))
            plens.append(i + 1)
    pre = qkv[torch.cat(idx).to(DEV)]
    bid = _bidir(pre, plens, H, KV, hd)
    assert _lib.lib().ezr_attn_last_kernel() == b"wgmma"
    last = bid[_cu(plens)[1:].long() - 1]                    # the last row of each prefix, in causal row order
    assert (got == last).all(), f"{int((got != last).any(1).sum())} causal rows differ from their prefix's last row"
    whole = _bidir(qkv, lens, H, KV, hd)                     # last row of each sequence: bidirectional on all of it
    ends = torch.tensor(offs[1:] - 1, device=DEV)
    assert (got[ends] == whole[ends]).all()
    assert (got != whole).any(1).sum() > 0.9 * (t - len(lens))    # elsewhere the two differ


def test_causal_rows_ignore_later_positions():
    hd, H, KV = 128, 4, 2
    lens = [300, 129, 64]
    t = sum(lens)
    qkv = _randn(t, (H + 2 * KV) * hd, seed=91, std=0.9)
    base = _causal(qkv, lens, H, KV, hd)
    for i in (0, 1, 63, 64, 127, 128, 191, 200, 298):
        changed = qkv.clone()
        changed[i + 1:300] = _randn(299 - i, (H + 2 * KV) * hd, seed=92 + i, std=0.9)   # Q, K and V after row i
        out = _causal(changed, lens, H, KV, hd)
        assert torch.equal(out[:i + 1], base[:i + 1]), f"rows 0..{i} moved when positions after {i} changed"
        assert not torch.equal(out[i + 1:300], base[i + 1:300])
        assert torch.equal(out[300:], base[300:])            # the other sequences are untouched


def test_causal_entry_point_checks():
    L = _lib.lib()
    qkv = _randn(70, 3 * 64, seed=3)
    out = torch.empty(70, 64, dtype=torch.bfloat16, device=DEV)
    cu = _cu([70])
    args = lambda hd: (_lib.ptr(qkv), 70, qkv.stride(0), _lib.ptr(cu), 1, 70, 1, 1, hd, 0.125, _lib.ptr(out),
                       out.stride(0), _lib.stream_ptr())
    assert L.ezr_attn_causal(*args(96)) != 0                  # the same argument checks as ezr_attn_bidir
    assert b"head_dim" in L.ezr_last_error()
    try:
        _lib.check(L.ezr_attn_set_kernel(1))
        assert L.ezr_attn_causal(*args(64)) != 0
        assert b"bidirectional only" in L.ezr_last_error()
    finally:
        _lib.check(L.ezr_attn_set_kernel(0))
    _lib.check(L.ezr_attn_causal(*args(64)), "ezr_attn_causal")
    torch.cuda.synchronize()
    assert L.ezr_attn_last_kernel() == b"wgmma-causal"


# ------------------------------------------------------------------------------------------ the encoder
def _cos_rows(a, b):
    return F.cosine_similarity(torch.as_tensor(a).float(), torch.as_tensor(b).float(), dim=1)


def test_causal_qwen2_encoder_matches_reference_model_golden():
    """CUDA path vs the reference's own Qwen2Model run with is_causal=True; tolerances of the bidirectional golden test
    (test_gpu_encoder.py::test_qwen2_encoder_matches_reference_model_golden)."""
    z, cfg, state = load_golden()
    model = Qwen2Encoder(cfg, state, device=DEV, causal=True)
    batch = PackedBatch.from_padded(torch.from_numpy(z["input_ids"]), torch.from_numpy(z["attention_mask"]), DEV)
    eb, ef = model.embed_packed(batch)
    ef = ef.cpu()
    assert (_cos_rows(ef, z["emb_fp32"]) > 1 - 1e-3).all()
    assert (_cos_rows(ef, z["emb_bf16"]) > 1 - 1e-3).all()
    assert (ef - torch.from_numpy(z["emb_fp32"])).abs().max() < 2e-2
    ref = torch.from_numpy(z["emb_fp32"])
    refb = F.normalize(torch.from_numpy(z["emb_bf16"]), dim=1)
    floor = ((refb @ refb.T) - (ref @ ref.T)).abs().max().item()
    mine = F.normalize(ef, dim=1)
    err = ((mine @ mine.T) - (ref @ ref.T)).abs().max().item()
    assert err <= floor + 1e-3, (err, floor)
    assert torch.equal(eb.float().cpu(), ef)
    # the bidirectional encoder on the same input lands elsewhere
    _, e_bi = Qwen2Encoder(cfg, state, device=DEV).embed_packed(batch)
    multi = torch.from_numpy(z["attention_mask"]).sum(1) > 1
    assert ((e_bi.cpu() - ef).abs().max(1).values[multi] > 1e-2).all()


def test_causal_qwen2_encoder_gte_qwen2_7b_width_vs_oracle():
    """Two layers of the real width (d 3584, 28 / 4 heads, FFN 18944) against the causal fp32 oracle."""
    cfg = Qwen2Config(vocab_size=1000, hidden_size=3584, intermediate_size=18944, num_hidden_layers=2,
                      num_attention_heads=28, num_key_value_heads=4, max_position_embeddings=8192, rope_theta=1e6)
    state = random_state("qwen2", cfg, 71)
    g = torch.Generator().manual_seed(73)
    lens = [1, 17, 48, 300, 1024]
    seqs = [torch.randint(1, cfg.vocab_size, (n,), generator=g).tolist() for n in lens]
    ids, mask = oenc.pad_left(seqs)
    tf32 = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False                       # a true fp32 oracle
    try:
        ref = gte_embed_causal(state, cfg, ids, mask, device=DEV).cpu()
    finally:
        torch.backends.cuda.matmul.allow_tf32 = tf32
    model = Qwen2Encoder(cfg, state, device=DEV, causal=True)
    _, ef = model.embed_packed(PackedBatch.from_padded(ids, mask, DEV))
    cos = _cos_rows(ef.cpu(), ref)
    print(f"\n[bounds] causal qwen2 encoder d=3584 2 layers: min_cos={cos.min().item():.7f}")
    assert (cos > 1 - 1e-3).all(), cos


@pytest.mark.parametrize("precision", ["bf16", "fp8"])
def test_causal_encoder_hidden_rows_equal_those_of_the_prefix(precision):
    cfg = Qwen2Config(vocab_size=500, hidden_size=512, intermediate_size=1024, num_hidden_layers=2,
                      num_attention_heads=4, num_key_value_heads=2, max_position_embeddings=1024)
    model = Qwen2Encoder(cfg, random_state("qwen2", cfg, 5), device=DEV, precision=precision, causal=True)
    g = torch.Generator().manual_seed(6)
    seq = torch.randint(1, cfg.vocab_size, (300,), generator=g).tolist()
    cuts = [1, 2, 64, 65, 128, 129, 200, 300]
    batch = PackedBatch.from_lists([seq] + [seq[:c] for c in cuts], DEV)      # positions from 0 for every sequence
    h = model.hidden(batch)
    torch.cuda.synchronize()
    o = len(seq)
    for c in cuts:
        assert torch.equal(h[:c], h[o:o + c]), f"{precision}: hidden rows 0..{c - 1} differ from those of the prefix"
        o += c
    bi = Qwen2Encoder(cfg, random_state("qwen2", cfg, 5), device=DEV, precision=precision)
    hb = bi.hidden(PackedBatch.from_lists([seq], DEV))
    assert not torch.equal(hb[:299], h[:299])


def test_gte_embedding_is_causal():
    from easyrag_b200.embeddings import GTEEmbedding

    class Tok:
        def __call__(self, texts, max_length=512, padding=True, truncation=True, return_tensors="pt"):
            seqs = [[3 + (sum(map(ord, w)) * 7919) % 297 for w in t.split()][: max_length - 1] + [2] for t in texts]
            return dict(zip(("input_ids", "attention_mask"), oenc.pad_left(seqs)))

    cfg = Qwen2Config(vocab_size=300, hidden_size=256, intermediate_size=512, num_hidden_layers=2,
                      num_attention_heads=4, num_key_value_heads=2, max_position_embeddings=512, sliding_window=40)
    state = random_state("qwen2", cfg, 7)
    causal = Qwen2Encoder(cfg, state, device=DEV, causal=True)
    gte = GTEEmbedding(model_name="gte-tiny", tokenizer=Tok(), encoder=causal, is_causal=True)
    texts = [" ".join(f"w{(i * 5 + j) % 31}" for j in range(3 + 4 * i)) for i in range(8)]
    eb, ef = gte.embed_tensor(texts)
    batch_dict = Tok()(texts)
    _, want = causal.embed_packed(PackedBatch.from_padded(batch_dict["input_ids"], batch_dict["attention_mask"], DEV))
    assert torch.equal(ef, want)
    _, bi = Qwen2Encoder(cfg, state, device=DEV).embed_packed(
        PackedBatch.from_padded(batch_dict["input_ids"], batch_dict["attention_mask"], DEV))
    assert not torch.equal(bi, want)
    with pytest.raises(ValueError, match="is_causal"):
        GTEEmbedding(model_name="gte-tiny", tokenizer=Tok(), encoder=causal)
    with pytest.raises(ValueError, match="is_causal"):
        GTEEmbedding(model_name="gte-tiny", tokenizer=Tok(), encoder=Qwen2Encoder(cfg, state, device=DEV),
                     is_causal=True)
    with pytest.raises(ValueError, match="sliding window"):
        gte.embed_tensor(["w1 " * 60])                         # 61 tokens: past the window of 40
    Qwen2Encoder(cfg, state, device=DEV).embed_packed(PackedBatch.from_lists([[5] * 61], DEV))   # bidirectional: no window
