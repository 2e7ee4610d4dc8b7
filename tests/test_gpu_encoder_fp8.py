"""The FP8 encoder path on the GPU: quantisers, the e4m3 GEMM and the encoders with precision="fp8".

* Quantisers (ezr_quant_rows_fp8 / ezr_quant_weight_fp8 / ezr_rmsnorm_fp8 / ezr_layernorm_fp8) are bit-exact against
  torch's (x / s).to(float8_e4m3fn) with the same power-of-two s, and the fused norms' bf16 rows are bit-exact against
  the bf16 norm kernels.
* The GEMM is checked twice against fp64 (tests/_bounds_fp8.py: fp8_gemm_bound): on the dequantised operands, which
  leaves only the accumulation, epilogue and store terms, and on the original bf16 operands within the full bound.
* The encoders at gte-Qwen2-7B width (2 layers) and BGE-large (24 layers) against the fp64 oracle, next to the bf16
  floor of the same run; a model whose weight scales are dropped must fail the same tolerance.
* precision="bf16" (the default) is bit-identical to not passing it; the drop-in classes run with precision="fp8".
"""
import pytest
import torch
import torch.nn.functional as F

from _bounds import rejects
from _bounds_fp8 import check_fp8, fp8_gemm_bound, pow2_scale
from oracle import encoder as oenc
from easyrag_b200 import _lib, encoder as enc
from easyrag_b200.encoder import BertConfig, BertEncoder, PackedBatch, Qwen2Config, Qwen2Encoder, random_state

pytestmark = pytest.mark.gpu
DEV = "cuda"
W_STD = 0.02
# Tolerance of the FP8 encoders against fp64 on random weights (std 0.02): every GEMM input is rounded to 3 mantissa
# bits (about 2.5 % rms relative error per operand), so per-sequence cosines sit well below the bf16 path's 1e-3.
FP8_COS_TOL = 2e-2
FP8_PAIR_TOL = 3e-2


@pytest.fixture(scope="module", autouse=True)
def _ready(lib_built):
    _lib.require_cuda()


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _randn(*shape, seed, std=1.0):
    return (torch.randn(*shape, generator=_gen(seed), device=DEV) * std).to(torch.bfloat16)


def _report(what, info):
    print(f"\n[fp8] {what}: " + ", ".join(f"{k}={v:.5g}" if isinstance(v, float) else f"{k}={v}"
                                       for k, v in info.items()))


def _torch_quant(x):
    s = pow2_scale(x.double().abs().amax(1)).float()
    return (x.float() / s[:, None]).to(torch.float8_e4m3fn), s


def _assert_same_fp8(q, s, x, what):
    rq, rs = _torch_quant(x)
    assert torch.equal(s, rs), f"{what}: scales differ"
    assert torch.equal(q.view(torch.uint8), rq.view(torch.uint8)), \
        f"{what}: {int((q.view(torch.uint8) != rq.view(torch.uint8)).sum())} bytes differ"


# ------------------------------------------------------------------------------------------------ quantisers
def _quant_input(rows, cols, seed, ld=None):
    ld = ld or cols
    x = torch.randn(rows, ld, generator=_gen(seed), device=DEV)
    x *= torch.exp2(torch.randint(-20, 20, (rows, 1), generator=_gen(seed + 1), device=DEV).float())
    x[0] = 0.0                                                      # zero row: s = 1
    x[1, 3] = 3.0e4                                                 # one huge element: the rest become subnormal e4m3
    x[2] = torch.randn(ld, generator=_gen(seed + 2), device=DEV) * 1e-39   # bf16 subnormals (s below 2^-126)
    x[3] = 448.0 * 2.0 ** torch.randint(-5, 5, (ld,), generator=_gen(seed + 3), device=DEV).float()  # at 448 * 2^k
    return x.to(torch.bfloat16)[:, :cols]


@pytest.mark.parametrize("rows,cols,ld", [(203, 768, None), (77, 3584, 3600), (19, 18944, None), (9, 136, 200)])
def test_quant_rows_bit_exact_vs_torch(rows, cols, ld):
    x = _quant_input(rows, cols, 40 + cols, ld)
    q, s = enc.quant_rows(x)
    _assert_same_fp8(q, s, x, f"quant_rows {rows}x{cols}")
    # strided output: a column slice of a wider e4m3 buffer
    buf = torch.zeros(rows, cols + 24, dtype=torch.float8_e4m3fn, device=DEV)
    q2, s2 = enc.quant_rows(x, out8=buf[:, 8:8 + cols])
    _assert_same_fp8(q2, s2, x, "quant_rows strided out")
    assert (buf[:, :8].view(torch.uint8) == 0).all() and (buf[:, 8 + cols:].view(torch.uint8) == 0).all()
    w8, sw = enc.quant_weight(x.contiguous())
    _assert_same_fp8(w8, sw, x, "quant_weight")


@pytest.mark.parametrize("dim", [768, 1024, 3584])
def test_norm_fp8_bit_exact(dim):
    x = _randn(203, dim, seed=dim)
    x[:, 5] *= 1000
    g = (1 + _randn(dim, seed=dim + 1, std=0.1).float()).to(torch.bfloat16)
    b = _randn(dim, seed=dim + 2, std=0.1)
    ref = enc.rmsnorm(x, g, 1e-6)
    q, s = enc.rmsnorm_fp8(x, g, 1e-6)
    _assert_same_fp8(q, s, ref, f"rmsnorm_fp8 {dim}")
    out = torch.empty_like(x)
    q, s = enc.rmsnorm_fp8(x, g, 1e-6, out=out)
    assert torch.equal(out, ref)
    ref = enc.layernorm(x, g, b, 1e-12)
    out = torch.empty_like(x)
    q, s = enc.layernorm_fp8(x, g, b, 1e-12, out=out)
    assert torch.equal(out, ref)
    _assert_same_fp8(q, s, ref, f"layernorm_fp8 {dim}")


# ------------------------------------------------------------------------------------------------------ GEMM
# (name, M, K, N, bias, epilogue, residual, strided output)
GEMM_CASES = [
    ("qwen2-qkv", 333, 3584, 4608, True, enc.EPI_NONE, False, False),
    ("qwen2-o-proj-inplace", 300, 3584, 3584, False, enc.EPI_NONE, True, False),
    ("qwen2-swiglu", 333, 3584, 2 * 18944, False, enc.EPI_SWIGLU, False, False),
    ("qwen2-down-inplace", 77, 18944, 3584, False, enc.EPI_NONE, True, False),
    ("bert-base-qkv-strided-out", 513, 768, 2304, True, enc.EPI_NONE, False, True),
    ("bert-base-ffn1-gelu", 333, 768, 3072, True, enc.EPI_GELU, False, False),
    ("bert-base-ffn2", 200, 3072, 768, True, enc.EPI_NONE, True, False),
    ("bert-large-ffn1-gelu-strided-out", 129, 1024, 4096, True, enc.EPI_GELU, False, True),
    ("bert-large-ffn2", 200, 4096, 1024, True, enc.EPI_NONE, True, False),
]


def _gemm_case(case):
    name, m, k, n, has_bias, epi, has_res, strided = case
    seed = 3000 + k + n + m
    a = _randn(m, k, seed=seed)
    w = _randn(n, k, seed=seed + 1, std=W_STD)
    bias = _randn(n, seed=seed + 2, std=W_STD) if has_bias else None
    n_out = n // 2 if epi == enc.EPI_SWIGLU else n
    res = _randn(m, n_out, seed=seed + 3) if has_res else None
    qa, sa = enc.quant_rows(a)
    qw, sw = enc.quant_weight(w)
    if has_res:                                     # in place, as the layers call it: out = residual = x
        x = res.clone()
        got = enc.gemm_fp8(qa, sa, qw, sw, bias=bias, residual=x, out=x, epilogue=epi)
        assert got.data_ptr() == x.data_ptr()
    elif strided:                                   # odd row stride, odd start: scalar stores
        buf = torch.zeros(m, n_out + 3, dtype=torch.bfloat16, device=DEV)
        got = enc.gemm_fp8(qa, sa, qw, sw, bias=bias, out=buf[:, 1:1 + n_out], epilogue=epi)
        assert (buf[:, 0] == 0).all() and (buf[:, 1 + n_out:] == 0).all()
    else:
        got = enc.gemm_fp8(qa, sa, qw, sw, bias=bias, epilogue=epi)
    assert got.shape == (m, n_out)
    return a, w, bias, res, qa, sa, qw, sw, got


@pytest.mark.parametrize("case", GEMM_CASES, ids=[c[0] for c in GEMM_CASES])
def test_gemm_fp8_accumulation_vs_dequantised_fp64(case):
    name, epi = case[0], case[5]
    a, w, bias, res, qa, sa, qw, sw, got = _gemm_case(case)
    exact, delta = fp8_gemm_bound(qa.double(), sa, qw.double(), sw, bias, res, epi)
    info = check_fp8(got, exact, delta, name)
    _report(f"gemm {name} vs dequantised operands", info)
    # negative controls: references that are wrong in a small way
    ctl = {"last 128 K columns dropped": fp8_gemm_bound(qa.double()[:, :-128], sa, qw.double()[:, :-128], sw, bias,
                                                       res, epi)[0]}
    if bias is not None:
        ctl["bias shifted by one column"] = fp8_gemm_bound(qa.double(), sa, qw.double(), sw, torch.roll(bias, 1), res,
                                                           epi)[0]
    for what, wrong in ctl.items():
        assert rejects(check_fp8, got, wrong, delta, f"{name} control"), f"{name}: accepted {what}"


@pytest.mark.parametrize("case", [c for c in GEMM_CASES if c[0] in ("qwen2-qkv", "qwen2-swiglu", "qwen2-down-inplace",
                                                                     "bert-large-ffn1-gelu-strided-out")],
                         ids=lambda c: c[0])
def test_gemm_fp8_end_to_end_vs_bf16_operands(case):
    name, epi = case[0], case[5]
    a, w, bias, res, qa, sa, qw, sw, got = _gemm_case(case)
    exact, delta = fp8_gemm_bound(qa.double(), sa, qw.double(), sw, bias, res, epi, a=a, w=w)
    info = check_fp8(got, exact, delta, name)
    _report(f"gemm {name} vs bf16 operands (full bound)", info)
    if epi != enc.EPI_SWIGLU and case[2] <= 4096:
        # the worst-case quantisation term grows with K (sum |a| |w|) and, through SwiGLU or at K = 18944, exceeds the
        # outputs themselves: a factor-2 error cannot fail it there
        wrong = fp8_gemm_bound(qa.double(), sa, qw.double(), sw * 2, bias, res, epi)[0]
        assert rejects(check_fp8, got, wrong, delta, f"{name} control"), f"{name}: accepted weight scales doubled"


# ---------------------------------------------------------------------------------------------- encoders
def _drop_weight_scales(model):
    for ly in model.layers:
        for key, v in ly.items():
            if isinstance(v, tuple):
                ly[key] = (v[0], torch.ones_like(v[1]))


def _compare(ef, ref, refb):
    cos = F.cosine_similarity(ef, ref, dim=1)
    floor = ((refb @ refb.T) - (ref @ ref.T)).abs().max().item()
    mine = F.normalize(ef, dim=1)
    err = ((mine @ mine.T) - (ref @ ref.T)).abs().max().item()
    return cos, err, floor


def _within(cos, err, floor):
    return bool((cos > 1 - FP8_COS_TOL).all()) and err <= floor + FP8_PAIR_TOL


def test_qwen2_encoder_fp8_gte_qwen2_7b_width_vs_oracle():
    cfg = Qwen2Config(vocab_size=1000, hidden_size=3584, intermediate_size=18944, num_hidden_layers=2,
                      num_attention_heads=28, num_key_value_heads=4, max_position_embeddings=8192, rope_theta=1e6)
    state = random_state("qwen2", cfg, 71)
    g = torch.Generator().manual_seed(72)
    lens = [1, 17, 48, 300, 1024]
    seqs = [torch.randint(1, cfg.vocab_size, (n,), generator=g).tolist() for n in lens]
    ids, mask = oenc.pad_left(seqs)
    tf32 = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        ref = oenc.gte_embed(state, cfg, ids, mask, device=DEV).cpu().double()        # fp32, tf32 off
    finally:
        torch.backends.cuda.matmul.allow_tf32 = tf32
    refb = F.normalize(oenc.gte_embed(state, cfg, ids, mask, torch.bfloat16, device=DEV).cpu().double(), dim=1)
    batch = PackedBatch.from_padded(ids, mask, DEV)
    eb = Qwen2Encoder(cfg, state, device=DEV).embed_packed(batch)[1].cpu().double()
    model = Qwen2Encoder(cfg, state, device=DEV, precision="fp8")
    ef = model.embed_packed(batch)[1].cpu().double()
    cos, err, floor = _compare(ef, ref, refb)
    cos_b, err_b, _ = _compare(eb, ref, refb)
    _drop_weight_scales(model)
    cos_c, err_c, _ = _compare(model.embed_packed(batch)[1].cpu().double(), ref, refb)
    _report("qwen2 d=3584 2 layers fp8", dict(min_cos=cos.min().item(), pairwise_err=err, bf16_floor=floor,
                                              bf16_kernels_min_cos=cos_b.min().item(), bf16_kernels_pairwise=err_b,
                                              control_min_cos=cos_c.min().item()))
    assert _within(cos, err, floor), (cos, err, floor)
    assert not _within(cos_c, err_c, floor), "weight scales dropped accepted"


def test_bge_large_fp8_24_layers_vs_fp64():
    cfg = BertConfig(vocab_size=21128, hidden_size=1024, intermediate_size=4096, num_hidden_layers=24,
                     num_attention_heads=16, max_position_embeddings=512, layer_norm_eps=1e-12)
    state = random_state("bert", cfg, 401)
    g = torch.Generator().manual_seed(402)
    lens = [1, 2, 64, 65, 200, 511, 512]
    seqs = [torch.randint(1, cfg.vocab_size, (n,), generator=g).tolist() for n in lens]
    ref = oenc.bert_embed(state, cfg, seqs, device=DEV, dtype=torch.float64).double()
    refb = oenc.bert_embed(state, cfg, seqs, device=DEV, dtype=torch.bfloat16).double()
    batch = PackedBatch.from_lists(seqs, DEV)
    eb = BertEncoder(cfg, state, device=DEV, pooling="cls").embed_packed(batch)[1].cpu().double()
    model = BertEncoder(cfg, state, device=DEV, pooling="cls", precision="fp8")
    ef = model.embed_packed(batch)[1].cpu().double()
    cos, err, floor = _compare(ef, ref, refb)
    cos_b, err_b, _ = _compare(eb, ref, refb)
    _drop_weight_scales(model)
    cos_c, err_c, _ = _compare(model.embed_packed(batch)[1].cpu().double(), ref, refb)
    _report("bge-large 24 layers fp8", dict(min_cos=cos.min().item(), pairwise_err=err, bf16_floor=floor,
                                            bf16_kernels_min_cos=cos_b.min().item(), bf16_kernels_pairwise=err_b,
                                            control_min_cos=cos_c.min().item()))
    assert _within(cos, err, floor), (cos, err, floor)
    assert not _within(cos_c, err_c, floor), "weight scales dropped accepted"


# ------------------------------------------------------------------------------------- default path, drop-ins
def test_default_precision_is_bf16_bit_identical():
    qc = Qwen2Config(vocab_size=300, hidden_size=256, intermediate_size=512, num_hidden_layers=2,
                     num_attention_heads=4, num_key_value_heads=2, max_position_embeddings=512)
    qs = random_state("qwen2", qc, 5)
    batch = PackedBatch.from_lists([[1, 2, 3], list(range(5, 200)), [7] * 64], DEV)
    a = Qwen2Encoder(qc, qs, device=DEV).embed_packed(batch)
    b = Qwen2Encoder(qc, qs, device=DEV, precision="bf16").embed_packed(batch)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    bc = BertConfig(vocab_size=300, hidden_size=256, intermediate_size=1024, num_hidden_layers=2,
                    num_attention_heads=4, max_position_embeddings=256)
    bs = random_state("bert", bc, 6)
    a = BertEncoder(bc, bs, device=DEV).embed_packed(batch)
    b = BertEncoder(bc, bs, device=DEV, precision="bf16").embed_packed(batch)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    assert all(isinstance(v, torch.Tensor) for ly in Qwen2Encoder(qc, qs, device=DEV).layers for v in ly.values())
    f8 = Qwen2Encoder(qc, qs, device=DEV, precision="fp8")
    assert f8.layers[0]["wqkv"][0].dtype == torch.float8_e4m3fn and f8.embed.dtype == torch.bfloat16


class _Tok:
    """Whitespace words -> ids by hash, padded like a HF tokenizer (left for Qwen2, right for BERT)."""

    def __init__(self, vocab, side):
        self.vocab, self.side = vocab, side

    def __call__(self, texts, max_length=512, padding=True, truncation=True, return_tensors="pt"):
        seqs = [[3 + (sum(map(ord, w)) * 7919) % (self.vocab - 3) for w in t.split()][: max_length - 1] + [2]
                for t in texts]
        pad = oenc.pad_left if self.side == "left" else oenc.pad_right
        return dict(zip(("input_ids", "attention_mask"), pad(seqs)))


def test_dropin_classes_fp8_fill_vector_store():
    from easyrag_b200.embeddings import GTEEmbedding, HuggingFaceEmbedding
    from easyrag_b200.retrievers import B200VectorStore
    from easyrag_b200.schema import TextNode
    nodes = [TextNode(text=f"chunk {i} " + " ".join(f"w{(i * 7 + j) % 97}" for j in range(5 + i % 40)))
             for i in range(37)]
    qc = Qwen2Config(vocab_size=300, hidden_size=256, intermediate_size=512, num_hidden_layers=2,
                     num_attention_heads=4, num_key_value_heads=2, max_position_embeddings=512)
    qs = random_state("qwen2", qc, 7)
    bc = BertConfig(vocab_size=300, hidden_size=256, intermediate_size=1024, num_hidden_layers=2,
                    num_attention_heads=4, max_position_embeddings=256)
    bs = random_state("bert", bc, 8)
    gte8 = GTEEmbedding(model_name="gte-tiny", embed_batch_size=8, tokenizer=_Tok(300, "left"), precision="fp8",
                        encoder=Qwen2Encoder(qc, qs, device=DEV, precision="fp8"))
    gte = GTEEmbedding(model_name="gte-tiny", embed_batch_size=8, tokenizer=_Tok(300, "left"),
                       encoder=Qwen2Encoder(qc, qs, device=DEV))
    hf8 = HuggingFaceEmbedding(model_name="bge-tiny", embed_batch_size=8, hf_tokenizer=_Tok(300, "right"),
                               precision="fp8", encoder=BertEncoder(bc, bs, device=DEV, precision="fp8"))
    hf = HuggingFaceEmbedding(model_name="bge-tiny", embed_batch_size=8, hf_tokenizer=_Tok(300, "right"),
                              encoder=BertEncoder(bc, bs, device=DEV))
    with pytest.raises(ValueError, match="precision"):
        GTEEmbedding(model_name="gte-tiny", tokenizer=_Tok(300, "left"), encoder=gte._model, precision="fp8")
    with pytest.raises(ValueError, match="precision"):
        HuggingFaceEmbedding(model_name="bge-tiny", hf_tokenizer=_Tok(300, "right"), encoder=hf._model,
                             precision="bf8")
    for e8, e16 in ((gte8, gte), (hf8, hf)):
        store = B200VectorStore.from_embed_model(nodes, e8)
        ref = B200VectorStore.from_embed_model(nodes, e16)
        assert store.index.n_rows == len(nodes) and len(store.nodes) == len(nodes)
        v8, v = store.index.vectors.float().cpu(), ref.index.vectors.float().cpu()
        cos = F.cosine_similarity(v8, v, dim=1)
        _report(f"{type(e8).__name__} fp8 vs bf16 rows", dict(min_cos=cos.min().item()))
        assert ((v8.norm(dim=1) - 1).abs() < 5e-3).all()
        assert (cos > 1 - FP8_COS_TOL).all(), cos
        q = e8.get_query_embedding("w3 w5 w7")
        assert len(q) == v8.shape[1]
