"""GPU: the BERT-family encoder path and the cross-encoder head at the shapes of the models the pipeline runs, against
fp64 references.

Shapes: BGE-large (24 layers, d 1024, 16 heads, FFN 4096, CLS pooling + normalize), XLM-R large (bge-reranker-large /
-v2-m3: the same stack, a 250002-row vocabulary, one token type, positions from ``pad_id + 1``, 514 or 8194 position
rows) and a BERT-base cross-encoder (12 layers, d 768, two token types).  Every reference is computed in float64 on
the same bf16 inputs.  Kernel outputs rounded once to bf16 go through ``_bounds.check_bf16``; the head's fp32 sigmoid
goes through ``_bounds.check_sigmoid``; both bounds are derived from the kernels' rounding points, every term
commented with the step it covers (tests/_bounds.py).  The 24-layer forwards compare with transformers' models run in
float64, within a tolerance taken from the same models run in bf16 (the noise floor of any bf16 evaluation).  Each
check also runs negative controls -- references that are wrong in a small, specific way -- and asserts that the
check rejects them.  The figures each check measures are printed (``pytest -s``).
"""
import time

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from _bounds import (U32, Z_ONE, Z_SUB, Z_ZERO, F32_MIN_NORMAL, check_bf16, check_sigmoid, cross_head_bound,
                     cross_head_case, cross_head_logit, ln_exact_and_delta, rejects, round_bf16)
from oracle import encoder as oenc
from oracle import rerank as orr
from easyrag_b200 import _lib
from easyrag_b200.batched import TopK
from easyrag_b200.encoder import POOL_CLS, BertConfig, BertEncoder, PackedBatch, random_state
from easyrag_b200.rerank import CrossEncoderModel, CrossEncoderReranker, random_cross_encoder_state

pytestmark = pytest.mark.gpu
DEV = "cuda"
HEAD_MEDIAN_ULPS = 128     # the head bound's median over |z| < 1, in fp32 ulps of the score (about 45 at d = 768 in
                           # the CPU emulation of tests/test_bounds_cpu.py, which holds it to the same figure)
COS_TOL = 1e-3             # cosine scores of the bf16 dense route
# cross-encoder logits: within FLOOR_FACTOR x the bf16 noise floor + FLOOR_ABS, the tolerance of test_gpu_rerank.py
FLOOR_FACTOR, FLOOR_ABS = 1.5, 0.02
# special ids of the two families: BERT [CLS]=2 [SEP]=3; RoBERTa <s>=0 <pad>=1 </s>=2
SPECIAL = {"bert": dict(cls_id=2, sep_id=3, pad_id=0), "roberta": dict(cls_id=0, sep_id=2, pad_id=1)}


@pytest.fixture(scope="module", autouse=True)
def _ready(lib_built):
    _lib.require_cuda()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    yield
    torch.cuda.synchronize()
    print(f"\n[bounds] test_gpu_bert_shapes.py: {time.perf_counter() - t0:.1f} s, peak "
          f"{torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB allocated on {torch.cuda.get_device_name()}")


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _randn(*shape, seed, std=1.0):
    return (torch.randn(*shape, generator=_gen(seed), device=DEV) * std).to(torch.bfloat16)


def _report(what, info):
    print(f"\n[bounds] {what}: " + ", ".join(f"{k}={v:.5g}" if isinstance(v, float) else f"{k}={v}"
                                          for k, v in info.items()))


# ------------------------------------------------------------------------------------ embedding + LayerNorm
# (name, vocab, dim, position rows, type rows (0: the untyped kernel, which adds type row 0), first position, eps)
EMBED_CASES = [
    ("bge-large-zh", 21128, 1024, 512, 0, 0, 1e-12),
    ("xlmr-large", 250002, 1024, 514, 1, 2, 1e-5),           # bge-reranker-large
    ("xlmr-large-8194", 250002, 1024, 8194, 1, 2, 1e-5),     # bge-reranker-v2-m3
    ("bert-base-typed", 30522, 768, 512, 2, 0, 1e-12),       # 128-thread block below d = 1024
]
EMBED_TOKENS = 512


def _embed_exact(word, posw, tt, ids, pos, types, gamma, beta, eps, rounded=True):
    """BertEmbeddings in fp64: x = bf16(bf16(word + type) + position) (each sum of two bf16 values is exact in fp64,
    so round_bf16 is the kernel's rounding), then LayerNorm.  ``rounded=False`` skips both roundings (a control)."""
    w, t, p = word[ids.long()].double(), tt[types.long()].double(), posw[pos.long()].double()
    x = round_bf16(round_bf16(w + t) + p) if rounded else w + t + p
    return ln_exact_and_delta(x, gamma, beta, eps)


@pytest.mark.parametrize("case", EMBED_CASES, ids=[c[0] for c in EMBED_CASES])
def test_bert_embedding_layernorm_vs_fp64(case):
    name, vocab, dim, max_pos, n_types, lo, eps = case
    L = _lib.lib()
    seed = 200 + dim + max_pos + n_types
    word = _randn(vocab, dim, seed=seed, std=0.05)
    posw = _randn(max_pos, dim, seed=seed + 1, std=0.02)
    tt = _randn(max(n_types, 2), dim, seed=seed + 2, std=0.02)[:max(n_types, 1)].contiguous()
    gamma = (1 + 0.1 * torch.randn(dim, generator=_gen(seed + 3), device=DEV)).to(torch.bfloat16)
    beta = _randn(dim, seed=seed + 4, std=0.05)
    g = _gen(seed + 5)
    ids = torch.randint(0, vocab, (EMBED_TOKENS,), generator=g, device=DEV, dtype=torch.int32)
    pos = torch.randint(lo, max_pos, (EMBED_TOKENS,), generator=g, device=DEV, dtype=torch.int32)
    types = torch.randint(0, max(n_types, 1), (EMBED_TOKENS,), generator=g, device=DEV, dtype=torch.int32)
    ids[0], ids[1] = 0, vocab - 1                    # both ends of the word table
    pos[2], pos[3] = max_pos - 1, lo                 # the last position row, and the first one the model uses
    out = torch.empty(EMBED_TOKENS, dim, dtype=torch.bfloat16, device=DEV)
    st = _lib.stream_ptr()
    if n_types:
        _lib.check(L.ezr_bert_embed_typed(_lib.ptr(ids), _lib.ptr(pos), _lib.ptr(types), EMBED_TOKENS, _lib.ptr(word),
                                          _lib.ptr(posw), _lib.ptr(tt), n_types, _lib.ptr(gamma), _lib.ptr(beta), eps,
                                          vocab, max_pos, dim, _lib.ptr(out), st), "ezr_bert_embed_typed")
    else:
        _lib.check(L.ezr_bert_embed(_lib.ptr(ids), _lib.ptr(pos), EMBED_TOKENS, _lib.ptr(word), _lib.ptr(posw),
                                    _lib.ptr(tt[0]), _lib.ptr(gamma), _lib.ptr(beta), eps, vocab, max_pos, dim,
                                    _lib.ptr(out), st), "ezr_bert_embed")
    torch.cuda.synchronize()
    # the LayerNorm bound's chain term covers the kernel's block sums: dim / 128 (or / 256 from d = 1024) serial adds
    # per thread, 5 shuffle levels, 5 block levels
    exact, delta = _embed_exact(word, posw, tt, ids, pos, types, gamma, beta, eps)
    info = check_bf16(out, exact, delta, name, median_ulps=0.1)
    _report(f"bert embed+ln {name} vocab={vocab} d={dim} positions={max_pos} types={n_types}", info)
    ctl = {"position rows shifted by one": _embed_exact(word, posw, tt, ids, pos - 1, types, gamma, beta, eps)[0],
           "sum without the intermediate bf16 roundings":
               _embed_exact(word, posw, tt, ids, pos, types, gamma, beta, eps, rounded=False)[0]}
    if n_types == 2:
        ctl["type rows swapped"] = _embed_exact(word, posw, tt, ids, pos, 1 - types, gamma, beta, eps)[0]
    for what, wrong in ctl.items():
        assert rejects(check_bf16, out, wrong, delta, f"{name} control", median_ulps=0.1), f"{name}: accepted {what}"


# -------------------------------------------------------------------------------------------------- pooling
def _pool(h, cu, pool, l2):
    L = _lib.lib()
    n_seq, dim = cu.numel() - 1, h.shape[1]
    ob = torch.empty(n_seq, dim, dtype=torch.bfloat16, device=DEV)
    of = torch.empty(n_seq, dim, dtype=torch.float32, device=DEV)
    _lib.check(L.ezr_pool_normalize(_lib.ptr(h), h.stride(0), _lib.ptr(cu), n_seq, pool, 0, None, 0.0, l2, dim,
                                    _lib.ptr(ob), _lib.ptr(of), _lib.stream_ptr()), "ezr_pool_normalize")
    torch.cuda.synchronize()
    return ob, of


def _check_rows(got, exact, bound, what):
    err = (got.double() - exact).abs()
    worst = int(torch.argmax((err / bound).reshape(-1)))
    assert (err <= bound).all(), (f"{what}: worst element {worst}: |err| {err.reshape(-1)[worst].item():.3g} vs bound "
                                  f"{bound.reshape(-1)[worst].item():.3g}")
    return (err / bound).max().item()


def test_pool_cls_1024_fp32_l2_and_no_norm():
    """BGE-large's pooling (CLS, normalize_embeddings: fp32 L2) and the cross-encoder's (CLS, no norm) at d = 1024."""
    dim = 1024
    g = torch.Generator().manual_seed(7)
    lens = [1, 512] + torch.randint(1, 600, (198,), generator=g).tolist()
    h = (torch.randn(sum(lens), dim, generator=_gen(70), device=DEV)
         + torch.randn(dim, generator=_gen(71), device=DEV)).to(torch.bfloat16)      # per-channel offsets
    cu = torch.tensor(np.cumsum([0] + lens), dtype=torch.int32, device=DEV)
    cls = h[cu[:-1].long()]
    ob, of = _pool(h, cu, POOL_CLS, 2)
    assert torch.equal(ob, of.to(torch.bfloat16))                       # the bf16 row is the rounded float row
    H = cls.double()
    nrm = H.norm(dim=1, keepdim=True)
    exact = H / nrm
    chain = dim / 256 + 10                        # sum of squares: 4 serial adds per thread (256 threads), 5 shuffle
                                                  # levels, 5 block levels
    bound = exact.abs() * (chain + 3) * U32       # + the squares' roundings, sqrtf (halves the relative error of the
                                                  # sum, then rounds once) and the division
    worst = _check_rows(of, exact, bound, "cls + fp32 l2")
    _report("pool cls + fp32 l2 d=1024", dict(worst=worst, median_bound=(bound / exact.abs()).median().item(),
                                                seqs=len(lens)))
    # control: the norm rounded to bf16 first (F.normalize on a bf16 tensor, the l2 = 1 semantics)
    assert rejects(_check_rows, of, H / round_bf16(nrm), bound, "control: bf16 norm")
    ob0, of0 = _pool(h, cu, POOL_CLS, 0)
    assert torch.equal(ob0, cls) and torch.equal(of0, cls.float())      # no norm: the CLS rows, bit for bit
    assert not torch.equal(ob0, h[cu[1:].long() - 1])                    # control: the last token's rows differ


# ------------------------------------------------------------------------------------- cross-encoder head
HEAD_Q, HEAD_K, HEAD_TOP = 528, 192, 100      # 101376 pairs


@pytest.mark.parametrize("dim", [1024, 768])
def test_cross_head_vs_fp64(dim):
    L = _lib.lib()
    n = HEAD_Q * HEAD_K
    rows, w, b = cross_head_case(n, dim, 300 + dim, device=DEV)
    z, s, ds = cross_head_bound(rows, w, b)
    bands = {"|z|<1": z.abs() < 1, f"z>={Z_ONE}": z >= Z_ONE, "subnormal": (z > Z_SUB[0]) & (z < Z_SUB[1]),
             f"z<{Z_ZERO}": z < Z_ZERO}
    counts = {k: int(v.sum()) for k, v in bands.items()}
    assert min(counts.values()) >= 10_000, counts
    st = _lib.stream_ptr()
    sig = torch.empty(n, dtype=torch.float32, device=DEV)
    _lib.check(L.ezr_cross_pair_scores(_lib.ptr(rows), dim, n, _lib.ptr(w), b, _lib.ptr(sig), st),
               "ezr_cross_pair_scores")
    pair_off = torch.arange(HEAD_Q + 1, dtype=torch.int32, device=DEV) * HEAD_K
    cand = (torch.arange(n, dtype=torch.int32, device=DEV) + 5000).view(HEAD_Q, HEAD_K)   # coarse order = column
    all_s = torch.empty(HEAD_Q, HEAD_K, dtype=torch.float32, device=DEV)
    top_s = torch.empty(HEAD_Q, HEAD_TOP, dtype=torch.float32, device=DEV)
    top_i = torch.empty(HEAD_Q, HEAD_TOP, dtype=torch.int32, device=DEV)
    cnt = torch.empty(HEAD_Q, dtype=torch.int32, device=DEV)
    _lib.check(L.ezr_cross_score_topk(_lib.ptr(rows), dim, _lib.ptr(pair_off), HEAD_Q, HEAD_K, _lib.ptr(cand), HEAD_K,
                                      _lib.ptr(w), b, dim, HEAD_TOP, _lib.ptr(all_s), _lib.ptr(top_s), _lib.ptr(top_i),
                                      _lib.ptr(cnt), st), "ezr_cross_score_topk")
    torch.cuda.synchronize()
    # both forms score a pair with the same device function: the same bits
    assert torch.equal(all_s.view(-1).view(torch.int32), sig.view(torch.int32))
    info = check_sigmoid(sig, z, s, ds, f"head d={dim}", median_ulps=HEAD_MEDIAN_ULPS)
    _report(f"cross head d={dim}", dict(**info, **counts))
    # the bands are what torch.sigmoid returns on the CPU for the same logits in fp32
    zc, tc = z.float().cpu(), torch.sigmoid(z.float().cpu())
    assert (tc[zc >= Z_ONE] == 1).all()
    assert (tc[zc < Z_ZERO] == 0).all() and not torch.signbit(tc[zc < Z_ZERO]).any()
    sub = (zc > Z_SUB[0]) & (zc < Z_SUB[1])
    assert ((tc[sub] > 0) & (tc[sub] < F32_MIN_NORMAL)).all()
    # order: score descending, exact ties (the saturated 1.0 and 0.0 scores) in coarse order
    assert (cnt == HEAD_TOP).all()
    order = torch.sort(-all_s, dim=1, stable=True).indices
    assert torch.equal(top_i, cand.gather(1, order[:, :HEAD_TOP]))
    assert torch.equal(top_s, all_s.gather(1, order[:, :HEAD_TOP]))
    # ... which is the order of the fp64 scores, except between pairs closer than the sum of their bounds (past the
    # overflow of expf the kernel returns 0, off by s itself)
    tol = torch.where(z > Z_SUB[0], ds, s).view(HEAD_Q, HEAD_K).gather(1, order)
    se = s.view(HEAD_Q, HEAD_K).gather(1, order)
    ahead = torch.triu(torch.ones(HEAD_K, HEAD_K, dtype=torch.bool, device=DEV), 1)      # [i, j]: i ranked before j
    inverted = ((se[:, None, :] - se[:, :, None]) > (tol[:, :, None] + tol[:, None, :])) & ahead
    assert not inverted.any(), f"{int(inverted.sum())} pairs ranked against their fp64 scores"
    # controls
    ctl = {"bias dropped": cross_head_logit(rows, w, 0.0),
           "tanh rounded to bf16": cross_head_logit(rows, w, b, tanh=lambda x: round_bf16(torch.tanh(x))),
           "tanh omitted": cross_head_logit(rows, w, b, tanh=lambda x: x),
           "w_out shifted by one": cross_head_logit(rows, torch.roll(w, 1), b)}
    for what, zw in ctl.items():
        assert rejects(check_sigmoid, sig, zw, torch.sigmoid(zw), ds, f"head d={dim} control",
                       median_ulps=HEAD_MEDIAN_ULPS), f"head d={dim}: accepted {what}"


# ------------------------------------------------------------------------------------ 24-layer forwards
def test_bge_large_24_layers_vs_fp64():
    """BGE-large: BertEncoder, CLS pooling, normalize_embeddings; random weights (std 0.02)."""
    cfg = BertConfig(vocab_size=21128, hidden_size=1024, intermediate_size=4096, num_hidden_layers=24,
                     num_attention_heads=16, max_position_embeddings=512, layer_norm_eps=1e-12)
    state = random_state("bert", cfg, 401)
    g = torch.Generator().manual_seed(402)
    lens = [1, 2, 64, 65, 200, 511, 512]
    seqs = [torch.randint(1, cfg.vocab_size, (n,), generator=g).tolist() for n in lens]
    ref = oenc.bert_embed(state, cfg, seqs, device=DEV, dtype=torch.float64)
    refb = oenc.bert_embed(state, cfg, seqs, device=DEV, dtype=torch.bfloat16)
    model = BertEncoder(cfg, state, device=DEV, pooling="cls")
    _, ef = model.embed_packed(PackedBatch.from_lists(seqs, DEV))
    ef = ef.cpu()
    cos = F.cosine_similarity(ef, ref, dim=1)
    cos_b = F.cosine_similarity(refb, ref, dim=1)
    floor = ((refb @ refb.T) - (ref @ ref.T)).abs().max().item()
    mine = F.normalize(ef, dim=1)
    err = ((mine @ mine.T) - (ref @ ref.T)).abs().max().item()
    # control: every sequence but the 512-token one read with positions from 1 (an off-by-one position offset)
    _, ec = model.embed_packed(PackedBatch.from_lists(seqs, DEV, pos_offset=[1] * (len(lens) - 1) + [0]))
    cos_c = F.cosine_similarity(ec.cpu(), ref, dim=1)[:-1]
    _report("bge-large 24 layers d=1024", dict(min_cos=cos.min().item(), min_cos_bf16_floor=cos_b.min().item(),
                                               pairwise_err=err, bf16_floor=floor,
                                               control_max_cos=cos_c.max().item()))
    assert (cos > 1 - COS_TOL).all(), cos
    assert err <= floor + COS_TOL, f"pairwise cosine error {err:.2e} vs fp64; the bf16 floor is {floor:.2e}"
    assert (cos_c < 1 - COS_TOL).all(), f"position offset off by one accepted: cosines {cos_c.tolist()}"


def _csr(queries):
    ptr = torch.tensor(np.cumsum([0] + [len(q) for q in queries]), dtype=torch.int32)
    tok = torch.tensor([t for q in queries for t in q], dtype=torch.int32)
    return ptr.to(DEV), tok.to(DEV)


def _logit(s):
    s = np.asarray(s, np.float64)
    return np.log(s) - np.log1p(-s)


# (family, layers, d, eps, position rows, control: the model attribute set off by one, its wrong value)
CE_CASES = [
    ("roberta", 24, 1024, 1e-5, 514, "pos_offset", 1),     # bge-reranker-large: positions from pad_id + 1 = 2
    ("bert", 12, 768, 1e-12, 512, "type_b", 0),            # BERT-base cross-encoder: segment B is token type 1
]


@pytest.mark.parametrize("case", CE_CASES, ids=["xlmr-large-24L", "bert-base-12L"])
def test_cross_encoder_deep_vs_fp64(case):
    family, layers, d, eps, max_pos, attr, wrong = case
    cfg = BertConfig(vocab_size=8000, hidden_size=d, intermediate_size=4 * d, num_hidden_layers=layers,
                     num_attention_heads=d // 64, max_position_embeddings=max_pos, layer_norm_eps=eps)
    state = random_cross_encoder_state(family, cfg, 500 + layers)
    model = CrossEncoderModel(family, cfg, state, device=DEV, **SPECIAL[family])
    rng = np.random.default_rng(501 + layers)
    n_docs, nq, k, top_n, max_length = 500, 2, 192, 6, 512
    passages = [rng.integers(4, cfg.vocab_size, int(rng.integers(64, 601))).tolist() for _ in range(n_docs)]
    queries = [rng.integers(4, cfg.vocab_size, int(rng.integers(8, 41))).tolist() for _ in range(nq)]
    c_ids = np.stack([rng.choice(n_docs, k, replace=False) for _ in range(nq)]).astype(np.int32)
    cand = TopK(torch.zeros(nq, k, device=DEV), torch.from_numpy(c_ids).to(DEV),
                torch.full((nq,), k, dtype=torch.int32, device=DEV))
    rr = CrossEncoderReranker(model, passages, max_length=max_length)
    top, all_scores = rr.rerank(cand, *_csr(queries), top_n=top_n)
    pairs = [orr.cross_encoder_inputs(queries[q], passages[c_ids[q, r]], max_length, family, model.cls_id,
                                      model.sep_id, pad_id=model.pad_id)[:2] for q in range(nq) for r in range(k)]
    assert max(len(p[0]) for p in pairs) == max_length                  # truncation happened
    logits, _ = orr.cross_encoder_scores(family, cfg, state, pairs, pad_id=model.pad_id, dtype=torch.float64,
                                         device=DEV)
    logits_b, _ = orr.cross_encoder_scores(family, cfg, state, pairs, pad_id=model.pad_id, dtype=torch.bfloat16,
                                           device=DEV)
    floor = float(np.abs(logits_b - logits).max())
    tol = FLOOR_FACTOR * floor + FLOOR_ABS
    got = all_scores.cpu().numpy()
    assert np.all((got > 0) & (got < 1)), "scores should not saturate here: their logits are compared"
    err = float(np.abs(_logit(got.reshape(-1)) - logits).max())
    right = getattr(model, attr)
    setattr(model, attr, wrong)
    try:
        _, ctl_scores = rr.rerank(cand, *_csr(queries), top_n=top_n)
    finally:
        setattr(model, attr, right)
    err_c = float(np.abs(_logit(ctl_scores.cpu().numpy().reshape(-1)) - logits).max())
    _report(f"cross-encoder {family} {layers} layers d={d}", dict(logit_err=err, bf16_floor=floor, tol=tol,
                                                                  control_err=err_c,
                                                                  logit_spread=float(logits.std())))
    # Random weights keep these logits close together (measured on an H100: std 0.10 at 24 layers, 0.06 at 12, against
    # bf16 floors of 0.07 / 0.06), so the order is checked against the GPU's own scores; the controls below move the
    # logits by 0.6 / 0.3, outside the tolerance.
    assert err <= tol, f"logit error {err:.3g}; bf16 noise floor {floor:.3g}"
    t_ids, t_sc = top.ids.cpu().numpy(), top.scores.cpu().numpy()
    assert top.counts.cpu().tolist() == [top_n] * nq
    for q in range(nq):
        want = orr.rerank_order(got[q].tolist(), top_n)                  # the reference's sort of the GPU's scores
        assert t_ids[q].tolist() == [int(c_ids[q, i]) for i in want]
        assert t_sc[q].tolist() == [float(got[q, i]) for i in want]
    assert err_c > tol, f"{attr} = {wrong} accepted: logit error {err_c:.3g} within {tol:.3g}"
