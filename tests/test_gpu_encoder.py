"""GPU: embedding forward pass (wgmma GEMMs, attention, norms, pooling) vs PyTorch fp32 and vs the reference model.

Tolerances: the north star allows 1e-3 on cosine scores for the bf16 embedding path; per-op checks compare the
bf16 kernels with an fp32 evaluation of the same bf16 inputs (error budget = bf16 output rounding, 2^-8 relative).
"""
from pathlib import Path

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import encoder as oenc
from easyrag_b200 import _lib, encoder as enc
from easyrag_b200.encoder import BertConfig, BertEncoder, PackedBatch, Qwen2Config, Qwen2Encoder, random_state

pytestmark = pytest.mark.gpu
DEV = "cuda"
GOLD = Path(__file__).parent / "golden" / "qwen2_tiny.npz"


@pytest.fixture(scope="module", autouse=True)
def _ready(lib_built):
    _lib.require_cuda()


def _rand(*shape, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(torch.bfloat16)


def _close(got, ref, rtol=2e-2, atol=2e-2):
    got, ref = got.float().cpu(), ref.float().cpu()
    err = (got - ref).abs()
    tol = atol + rtol * ref.abs()
    assert (err <= tol).all(), f"max err {err.max().item():.4g} (ref scale {ref.abs().max().item():.3g})"


# ----------------------------------------------------------------------------------- GEMM
@pytest.mark.parametrize("m,n,k", [(300, 256, 128), (1000, 768, 768), (4099, 3072, 768), (77, 2304, 768), (128, 128, 64),
                                   (33, 200, 192)])
def test_gemm_bias(m, n, k):
    a, w, b = _rand(m, k, seed=1), _rand(n, k, seed=2, scale=0.05), _rand(n, seed=3)
    got = enc.gemm(a.to(DEV), w.to(DEV), bias=b.to(DEV))
    ref = a.float() @ w.float().T + b.float()
    _close(got, ref)


def test_gemm_store_paths_strided_and_unaligned_outputs():
    # (a) a column slice of a wider buffer (row stride > N, TMA-store path): the neighbours stay untouched, rows past M
    #     and columns past N are clipped; (b) a row stride that is not a multiple of 8 (register-store path)
    m, n, k = 333, 136, 128
    a, w = _rand(m, k, seed=11), _rand(n, k, seed=12, scale=0.05)
    ref = a.float() @ w.float().T
    wide = torch.full((m + 5, 256), 7.0, dtype=torch.bfloat16, device=DEV)
    out = wide[:m, 64:64 + n]
    enc.gemm(a.to(DEV), w.to(DEV), out=out)
    _close(wide[:m, 64:64 + n], ref)
    keep = wide.float().cpu()
    assert (keep[:m, :64] == 7).all() and (keep[:m, 64 + n:] == 7).all() and (keep[m:] == 7).all()
    n2 = 100
    w2 = _rand(n2, k, seed=13, scale=0.05)
    got = enc.gemm(a.to(DEV), w2.to(DEV))                       # ldo = 100: not a multiple of 8
    _close(got, a.float() @ w2.float().T)


def test_gemm_exact_small_integers():
    # integer-valued operands: every partial sum is exact, so the tensor-core result must be bit-exact
    g = torch.Generator().manual_seed(5)
    a = torch.randint(-3, 4, (513, 256), generator=g).to(torch.bfloat16)
    w = torch.randint(-3, 4, (384, 256), generator=g).to(torch.bfloat16)
    got = enc.gemm(a.to(DEV), w.to(DEV)).float().cpu()
    ref = (a.float() @ w.float().T).to(torch.bfloat16).float()
    assert torch.equal(got, ref)


def test_gemm_gelu_and_residual():
    m, n, k = 700, 1024, 256
    a, w, b, r = _rand(m, k, seed=1), _rand(n, k, seed=2, scale=0.05), _rand(n, seed=3), _rand(m, n, seed=4)
    got = enc.gemm(a.to(DEV), w.to(DEV), bias=b.to(DEV), epilogue=enc.EPI_GELU)
    _close(got, F.gelu(a.float() @ w.float().T + b.float()))
    x = r.to(DEV).clone()
    got = enc.gemm(a.to(DEV), w.to(DEV), bias=b.to(DEV), residual=x, out=x)       # in place, as the layers use it
    _close(got, a.float() @ w.float().T + b.float() + r.float())


def test_gemm_swiglu_interleaved():
    m, ffn, d = 500, 512, 256
    x, wg, wu = _rand(m, d, seed=1), _rand(ffn, d, seed=2, scale=0.08), _rand(ffn, d, seed=3, scale=0.08)
    wgu = enc._interleave_gate_up(wg.float(), wu.float()).to(torch.bfloat16)
    got = enc.gemm(x.to(DEV), wgu.to(DEV), epilogue=enc.EPI_SWIGLU)
    assert got.shape == (m, ffn)
    ref = F.silu(x.float() @ wg.float().T) * (x.float() @ wu.float().T)
    _close(got, ref)


# ------------------------------------------------------------------------------ attention
@pytest.mark.parametrize("hd,H,KV", [(64, 4, 4), (64, 6, 2), (128, 2, 1)])
def test_attention_packed_bidirectional(hd, H, KV):
    lens = [1, 5, 64, 65, 200, 37, 128]
    t = sum(lens)
    qkv = _rand(t, (H + 2 * KV) * hd, seed=hd + H, scale=0.7)
    cu = torch.tensor(np.cumsum([0] + lens), dtype=torch.int32, device=DEV)
    got = enc.attention(qkv.to(DEV), cu, max(lens), H, KV, hd).float().cpu()
    q = qkv.float()[:, :H * hd].view(t, H, hd)
    k = qkv.float()[:, H * hd:(H + KV) * hd].view(t, KV, hd).repeat_interleave(H // KV, 1)
    v = qkv.float()[:, (H + KV) * hd:].view(t, KV, hd).repeat_interleave(H // KV, 1)
    o = 0
    for n in lens:
        qq, kk, vv = (z[o:o + n].transpose(0, 1) for z in (q, k, v))
        ref = torch.softmax(qq @ kk.transpose(1, 2) / hd ** 0.5, -1) @ vv             # [H, n, hd], non-causal
        _close(got[o:o + n].view(n, H, hd).transpose(0, 1), ref, rtol=2e-2, atol=1e-2)
        o += n


def _attn_ref(qkv, lens, H, KV, hd):
    t = sum(lens)
    q = qkv.float()[:, :H * hd].view(t, H, hd)
    k = qkv.float()[:, H * hd:(H + KV) * hd].view(t, KV, hd).repeat_interleave(H // KV, 1)
    v = qkv.float()[:, (H + KV) * hd:].view(t, KV, hd).repeat_interleave(H // KV, 1)
    out = torch.empty(t, H, hd)
    o = 0
    for n in lens:
        qq, kk, vv = (z[o:o + n].transpose(0, 1) for z in (q, k, v))
        out[o:o + n] = (torch.softmax(qq @ kk.transpose(1, 2) / hd ** 0.5, -1) @ vv).transpose(0, 1)
        o += n
    return out


# the test names below keep the kernel generation they were written for; the kernel they check is attention_tc.cu
@pytest.mark.parametrize("hd,H,KV", [(64, 3, 3), (64, 4, 2), (128, 2, 2), (128, 4, 1)])
def test_attention_tcgen05_ragged_lengths_and_kernel_name(hd, H, KV):
    """Every tile-boundary case of the 128-row / 128-key tiling (and the 16-key granularity of the last tile), a
    sequence that ends exactly at the last token of the buffer, sequences longer than four key tiles."""
    lens = [1, 15, 16, 17, 127, 128, 129, 255, 256, 257, 300, 512, 700, 3, 31]
    qkv = _rand(sum(lens), (H + 2 * KV) * hd, seed=7 * hd + H, scale=0.8)
    cu = torch.tensor(np.cumsum([0] + lens), dtype=torch.int32, device=DEV)
    got = enc.attention(qkv.to(DEV), cu, max(lens), H, KV, hd).float().cpu()
    assert _lib.lib().ezr_attn_last_kernel() == b"wgmma"
    ref = _attn_ref(qkv, lens, H, KV, hd)
    _close(got.view(-1, H, hd), ref, rtol=2e-2, atol=1e-2)


@pytest.mark.parametrize("hd", [64, 128])
def test_attention_tcgen05_rescales_when_the_row_maximum_grows(hd):
    """Keys are arranged so that every later key tile raises the row maximum by far more than 2^8: the online
    rescaling of O must be right on every tile (and on flat tiles)."""
    H = KV = 2
    lens = [640, 384, 130]
    t = sum(lens)
    g = torch.Generator().manual_seed(11)
    qkv = (torch.randn(t, 3 * H * hd, generator=g) * 0.5)
    o = 0
    for n in lens:                                           # key norm grows with the tile index -> logits grow
        for j in range(0, n, 128):
            qkv[o + j:o + min(n, j + 128), H * hd:2 * H * hd] *= 1.0 + 2.5 * (j // 128)
        o += n
    qkv[:, :H * hd] = qkv[:, :H * hd].abs()                  # same-sign q . k so the growth is systematic
    qkv[:, H * hd:2 * H * hd] = qkv[:, H * hd:2 * H * hd].abs()
    qkv = qkv.to(torch.bfloat16)
    cu = torch.tensor(np.cumsum([0] + lens), dtype=torch.int32, device=DEV)
    got = enc.attention(qkv.to(DEV), cu, max(lens), H, KV, hd).float().cpu()
    ref = _attn_ref(qkv, lens, H, KV, hd)
    assert torch.isfinite(got).all()
    _close(got.view(-1, H, hd), ref, rtol=2e-2, atol=1e-2)


def test_attention_tcgen05_agrees_with_the_mma_sync_kernel():
    """Two independent implementations of the same function (wgmma vs the warp-level mma.sync kernel)."""
    L = _lib.lib()
    hd, H, KV = 64, 12, 12
    g = torch.Generator().manual_seed(5)
    lens = torch.randint(8, 513, (40,), generator=g).tolist()
    qkv = _rand(sum(lens), (H + 2 * KV) * hd, seed=3, scale=0.6).to(DEV)
    cu = torch.tensor(np.cumsum([0] + lens), dtype=torch.int32, device=DEV)
    a = enc.attention(qkv, cu, max(lens), H, KV, hd).float()
    try:
        _lib.check(L.ezr_attn_set_kernel(1))
        b = enc.attention(qkv, cu, max(lens), H, KV, hd).float()
        assert L.ezr_attn_last_kernel() == b"mma.sync"
    finally:
        _lib.check(L.ezr_attn_set_kernel(0))
    assert (a - b).abs().max().item() < 2e-2


# ------------------------------------------------------------------------- norms, rope, pool
def test_rmsnorm_layernorm():
    x, g, b = _rand(333, 768, seed=1, scale=3), 1 + _rand(768, seed=2, scale=0.1), _rand(768, seed=3)
    _close(enc.rmsnorm(x.to(DEV), g.to(DEV), 1e-6), oenc._rms(x.float(), g.float(), 1e-6), rtol=1e-2, atol=1e-2)
    _close(enc.layernorm(x.to(DEV), g.to(DEV), b.to(DEV), 1e-12),
           F.layer_norm(x.float(), (768,), g.float(), b.float(), 1e-12), rtol=1e-2, atol=1e-2)


@pytest.mark.parametrize("hd", [64, 128, 8])        # 16-byte path (two head sizes) and the scalar path
def test_rope_matches_bf16_tensor_ops(hd):
    L = _lib.lib()
    t, h_qk, h_v, max_pos = 77, 5, 2, 64
    half = hd // 2
    qkv = _rand(t, (h_qk + h_v) * hd, seed=hd)
    pos = torch.randint(0, 50, (t,), dtype=torch.int32, generator=torch.Generator().manual_seed(3))
    inv = 1.0 / (10000.0 ** (torch.arange(0, hd, 2).float() / hd))
    fr = torch.arange(max_pos).float()[:, None] * inv[None]
    cos, sin = fr.cos().to(torch.bfloat16).contiguous(), fr.sin().to(torch.bfloat16).contiguous()
    x = qkv.to(DEV).clone()
    d_pos, d_cos, d_sin = pos.to(DEV), cos.to(DEV), sin.to(DEV)         # named: the pointers must outlive the launch
    _lib.check(L.ezr_rope(_lib.ptr(x), x.stride(0), _lib.ptr(d_pos), _lib.ptr(d_cos), _lib.ptr(d_sin),
                          max_pos, h_qk, hd, t, _lib.stream_ptr()), "ezr_rope")
    torch.cuda.synchronize()
    # q * cos + rotate_half(q) * sin on bf16 tensors: every product and the sum are rounded to bf16
    q = qkv[:, :h_qk * hd].view(t, h_qk, hd)
    c, sn = cos[pos.long()][:, None, :], sin[pos.long()][:, None, :]
    x1, x2 = q[..., :half], q[..., half:]
    ref = qkv.clone()
    ref[:, :h_qk * hd] = torch.cat([x1 * c + (-x2) * sn, x2 * c + x1 * sn], -1).reshape(t, -1)
    assert torch.equal(x.cpu(), ref)                        # V columns untouched, Q/K columns bit-exact


def test_pool_normalize_modes():
    L = _lib.lib()
    lens = [3, 1, 17]
    h = _rand(sum(lens), 256, seed=9)
    cu = torch.tensor(np.cumsum([0] + lens), dtype=torch.int32, device=DEV)
    hd = h.to(DEV)
    for pool, pick in ((enc.POOL_LAST, lambda s: s[-1]), (enc.POOL_CLS, lambda s: s[0]), (enc.POOL_MEAN, lambda s: s.mean(0))):
        ob = torch.empty(3, 256, dtype=torch.bfloat16, device=DEV)
        of = torch.empty(3, 256, dtype=torch.float32, device=DEV)
        _lib.check(L.ezr_pool_normalize(_lib.ptr(hd), 256, _lib.ptr(cu), 3, pool, 0, None, 0.0, 2, 256, _lib.ptr(ob),
                                        _lib.ptr(of), _lib.stream_ptr()))
        o = 0
        for i, n in enumerate(lens):
            ref = F.normalize(pick(h.float()[o:o + n]), dim=0)
            assert (of[i].cpu() - ref).abs().max() < 1e-5
            o += n


# ------------------------------------------------------------------------ whole encoders
def _golden():
    z = np.load(GOLD)
    c = z["cfg"]
    cfg = Qwen2Config(vocab_size=int(c[0]), hidden_size=int(c[1]), intermediate_size=int(c[2]),
                      num_hidden_layers=int(c[3]), num_attention_heads=int(c[4]), num_key_value_heads=int(c[5]),
                      max_position_embeddings=int(c[6]), rms_norm_eps=float(z["rms_norm_eps"][0]),
                      rope_theta=float(z["rope_theta"][0]))
    state = {k[3:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("w::")}
    return z, cfg, state


def _cos_rows(a, b):
    a, b = torch.as_tensor(a).float(), torch.as_tensor(b).float()
    return F.cosine_similarity(a, b, dim=1)


def test_qwen2_encoder_matches_reference_model_golden():
    """CUDA path vs vectors produced by the reference's own vendored Qwen2Model (tests/golden/qwen2_tiny.npz)."""
    z, cfg, state = _golden()
    model = Qwen2Encoder(cfg, state, device=DEV)
    batch = PackedBatch.from_padded(torch.from_numpy(z["input_ids"]), torch.from_numpy(z["attention_mask"]), DEV)
    eb, ef = model.embed_packed(batch)
    ef = ef.cpu()
    assert (_cos_rows(ef, z["emb_fp32"]) > 1 - 1e-3).all()          # vs the fp32 evaluation of the reference
    assert (_cos_rows(ef, z["emb_bf16"]) > 1 - 1e-3).all()          # vs the reference run in its own dtype (bf16)
    assert (ef - torch.from_numpy(z["emb_fp32"])).abs().max() < 2e-2
    # Scores a retriever would see (qdrant re-normalises for COSINE): pairwise cosines vs the reference's fp32 run.
    # This fixture is a stress case (weights ~ N(0, 0.06^2)): the reference's OWN bf16 run deviates from its fp32
    # run by 1.9e-3 here (and by 5.1e-3 before re-normalisation: F.normalize divides by a bf16-rounded norm), so
    # that is the noise floor; we must stay within it plus the 1e-3 budget of the north star.
    ref = torch.from_numpy(z["emb_fp32"])
    refb = F.normalize(torch.from_numpy(z["emb_bf16"]), dim=1)
    floor = ((refb @ refb.T) - (ref @ ref.T)).abs().max().item()
    mine = F.normalize(ef, dim=1)
    err = ((mine @ mine.T) - (ref @ ref.T)).abs().max().item()
    assert err <= floor + 1e-3, (err, floor)
    assert torch.equal(eb.float().cpu(), ef)                          # API floats are exactly the bf16 index rows


def test_qwen2_encoder_768d_vs_oracle_ragged():
    cfg = Qwen2Config(vocab_size=2000, hidden_size=768, intermediate_size=3072, num_hidden_layers=3,
                      num_attention_heads=12, num_key_value_heads=4, max_position_embeddings=1024)
    state = random_state("qwen2", cfg, 11, std=0.03)
    g = torch.Generator().manual_seed(12)
    lens = [8, 48, 64, 129, 300, 511, 17, 1]
    seqs = [torch.randint(1, cfg.vocab_size, (n,), generator=g).tolist() for n in lens]
    ids, mask = oenc.pad_left(seqs)
    ref = oenc.gte_embed(state, cfg, ids, mask)
    model = Qwen2Encoder(cfg, state, device=DEV)
    _, ef = model.embed_packed(PackedBatch.from_padded(ids, mask, DEV))
    assert (_cos_rows(ef.cpu(), ref) > 1 - 1e-3).all()
    # pairwise cosines (what a retriever sees).  The reference runs this model in bf16 (gte_embeddings.py:36); its own
    # deviation from the fp32 evaluation is the noise floor (same restatement, dtype=bfloat16, on the CPU); we must
    # stay within that floor plus the north star's 1e-3.
    refb = F.normalize(oenc.gte_embed(state, cfg, ids, mask, torch.bfloat16), dim=1)
    floor = ((refb @ refb.T) - (ref @ ref.T)).abs().max().item()
    mine = F.normalize(ef.cpu(), dim=1)
    err = ((mine @ mine.T) - (ref @ ref.T)).abs().max().item()
    assert err <= floor + 1e-3, f"pairwise cosine error {err:.2e} vs fp32; the reference's own bf16 floor is {floor:.2e}"
    # packed with positions from 0 (right-padding view): RoPE is relative, same vectors
    _, ef0 = model.embed_packed(PackedBatch.from_lists(seqs, DEV))
    assert (_cos_rows(ef0.cpu(), ref) > 1 - 1e-3).all()


@pytest.mark.parametrize("pooling", ["cls", "mean"])
def test_bert_encoder_vs_transformers(pooling):
    cfg = BertConfig(vocab_size=3000, hidden_size=768, intermediate_size=3072, num_hidden_layers=3,
                     num_attention_heads=12, max_position_embeddings=512)
    state = random_state("bert", cfg, 21, std=0.03)
    g = torch.Generator().manual_seed(22)
    lens = [5, 33, 64, 200, 512, 1]
    seqs = [torch.randint(1, cfg.vocab_size, (n,), generator=g).tolist() for n in lens]
    ref = oenc.bert_embed(state, cfg, seqs, pooling=pooling)
    model = BertEncoder(cfg, state, device=DEV, pooling=pooling)
    _, ef = model.embed_packed(PackedBatch.from_lists(seqs, DEV))
    assert (_cos_rows(ef.cpu(), ref) > 1 - 1e-3).all()
    assert (ef.cpu() - ref).abs().max() < 2e-2


# ------------------------------------------------------------ drop-in embedding classes
class _FakeHFTokenizer:
    """Minimal stand-in for a HF tokenizer (no tokenizer files offline): whitespace words -> ids by hash.

    Same call shape GTEEmbedding / HuggingFaceEmbedding use: tokenizer(texts, max_length=, padding=True,
    truncation=True, return_tensors='pt') -> {"input_ids", "attention_mask"}; pads LEFT like Qwen2Tokenizer
    (tokenization_qwen.py:218) or RIGHT like BERT tokenizers.
    """

    def __init__(self, vocab, side="left", eos=2):
        self.vocab, self.side, self.eos = vocab, side, eos

    def __call__(self, texts, max_length=512, padding=True, truncation=True, return_tensors="pt"):
        seqs = []
        for t in texts:
            ids = [3 + (sum(map(ord, w)) * 7919) % (self.vocab - 3) for w in t.split()][: max_length - 1] + [self.eos]
            seqs.append(ids)
        return dict(zip(("input_ids", "attention_mask"), (oenc.pad_left if self.side == "left" else oenc.pad_right)(seqs)))


def test_gte_embedding_dropin_surface():
    from easyrag_b200.embeddings import GTEEmbedding
    from easyrag_b200.schema import TextNode
    z, cfg, state = _golden()
    enc_model = Qwen2Encoder(cfg, state, device=DEV)
    tok = _FakeHFTokenizer(cfg.vocab_size, "left")
    emb = GTEEmbedding(model_name="gte-tiny", embed_batch_size=4, embed_type=1, encoder=enc_model, tokenizer=tok)
    texts = ["alpha beta gamma", "delta", "epsilon zeta eta theta iota kappa"]
    got = emb._get_text_embeddings(texts)
    ids, mask = tok(texts)["input_ids"], tok(texts)["attention_mask"]
    ref = oenc.gte_embed(state, cfg, ids, mask)
    assert len(got) == 3 and len(got[0]) == cfg.hidden_size and isinstance(got[0][0], float)
    assert (_cos_rows(torch.tensor(got), ref) > 1 - 1e-3).all()
    # query path prepends the instruct string (gte_embeddings.py:52-53,80-82)
    q = emb.get_query_embedding("what is alpha")
    iq, mq = tok([emb.get_detailed_instruct("what is alpha")]).values()
    assert _cos_rows(torch.tensor([q]), oenc.gte_embed(state, cfg, iq, mq)).item() > 1 - 1e-3
    # TransformComponent behaviour: __call__(nodes) fills node.embedding from get_node_content(node, embed_type)
    nodes = [TextNode(text="body one", metadata={"file_path": "a/b.txt"}), TextNode(text="body two")]
    out = emb(nodes)
    assert out is nodes and all(len(n.embedding) == cfg.hidden_size for n in nodes)
    want = emb._get_text_embeddings(["###\na/b.txt\n\nbody one", "body two"])
    assert np.allclose(nodes[0].embedding, want[0]) and np.allclose(nodes[1].embedding, want[1])


def test_hf_embedding_dropin_surface():
    from easyrag_b200.embeddings import HuggingFaceEmbedding
    cfg = BertConfig(vocab_size=500, hidden_size=128, intermediate_size=256, num_hidden_layers=2,
                     num_attention_heads=2, max_position_embeddings=64)
    state = random_state("bert", cfg, 31, std=0.05)
    model = BertEncoder(cfg, state, device=DEV, pooling="cls")
    tok = _FakeHFTokenizer(cfg.vocab_size, "right")
    with pytest.raises(ValueError):
        HuggingFaceEmbedding(model_name="x", pooling="mean", encoder=model, hf_tokenizer=tok)   # hf_embeddings.py:67-76
    emb = HuggingFaceEmbedding(model_name="BAAI/bge-small-zh", embed_batch_size=2, encoder=model, hf_tokenizer=tok)
    texts = ["one two three", "four", "five six"]
    got = torch.tensor(emb._get_text_embeddings(texts))
    seqs = [[int(t) for t, m in zip(r, mk) if m] for r, mk in zip(*tok(texts).values())]
    ref = oenc.bert_embed(state, cfg, seqs, pooling="cls")
    assert (_cos_rows(got, ref) > 1 - 1e-3).all()
    assert np.allclose(got.norm(dim=1).numpy(), 1.0, atol=1e-4)
    # a str gives one vector; the query prompt of BGE-zh models is prepended (llama_index get_query_instruct_for_model_name)
    q = emb._get_query_embedding("seven eight")
    assert isinstance(q, list) and len(q) == cfg.hidden_size
    from easyrag_b200.embeddings.hf_embeddings import BGE_QUERY_ZH
    seq = [[int(t) for t, m in zip(r, mk) if m] for r, mk in zip(*tok([BGE_QUERY_ZH + "seven eight"]).values())]
    assert _cos_rows(torch.tensor([q]), oenc.bert_embed(state, cfg, seq, pooling="cls")).item() > 1 - 1e-3
