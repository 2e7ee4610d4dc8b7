"""GPU: cross-encoder reranking (SentenceTransformerRerank) -- pair packing, the typed embedding, scores against
transformers' sequence classifiers, the reference's order, chunking under a token budget, coarse-ranker input and the
drop-in postprocessor."""
import numpy as np
import pytest
import torch

from oracle import rerank as orr
from easyrag_b200 import _lib, batched, synth
from easyrag_b200.batched import TopK
from easyrag_b200.encoder import BertConfig
from easyrag_b200.rerank import (CrossEncoderModel, CrossEncoderReranker, SentenceTransformerRerank,
                                 random_cross_encoder_state)
from easyrag_b200.schema import NodeWithScore, QueryBundle, TextNode

pytestmark = pytest.mark.gpu
DEV = "cuda"
# special ids of the two families: BERT [CLS]=2 [SEP]=3; RoBERTa <s>=0 <pad>=1 </s>=2
SPECIAL = {"bert": dict(cls_id=2, sep_id=3, pad_id=0), "roberta": dict(cls_id=0, sep_id=2, pad_id=1)}
# Tolerance on the logits, from the noise floor: the largest |logit| error of the bf16 evaluation of the same model
# (transformers, bf16) against its fp32 evaluation.  The GPU path is a bf16 encoder with an fp32 head, so it must
# stay within this multiple of the floor (plus a small absolute term for cases where the floor happens to be tiny).
FLOOR_FACTOR, FLOOR_ABS = 1.5, 0.02
# end-to-end tests compare sigmoid scores directly: a bf16 encoder moves these logits by a few 1e-2 at most, and the
# sigmoid's slope is at most 1/4
SCORE_TOL = 2e-2


@pytest.fixture(scope="module", autouse=True)
def _ready(lib_built):
    _lib.require_cuda()


def _cfg(family, d=768, layers=2, vocab=3000):
    return BertConfig(vocab_size=vocab, hidden_size=d, intermediate_size=4 * d, num_hidden_layers=layers,
                      num_attention_heads=d // 64, max_position_embeddings=514 if family == "roberta" else 512,
                      layer_norm_eps=1e-5 if family == "roberta" else 1e-12)


def _model(family, d=768, layers=2, seed=7, vocab=3000):
    cfg = _cfg(family, d, layers, vocab)
    state = random_cross_encoder_state(family, cfg, seed, std=0.03)
    return cfg, state, CrossEncoderModel(family, cfg, state, device=DEV, **SPECIAL[family])


def _tokens(rng, n, lo, hi, vocab):
    return [rng.integers(4, vocab, int(rng.integers(lo, hi + 1))).tolist() for _ in range(n)]


def _csr(queries):
    ptr = torch.tensor(np.cumsum([0] + [len(q) for q in queries]), dtype=torch.int32)
    tok = torch.tensor([t for q in queries for t in q], dtype=torch.int32)
    return ptr.to(DEV), tok.to(DEV)


def _cand(rng, nq, k, n_docs, id_base=0, counts=None, dup=False):
    cnt = rng.integers(1, k + 1, nq).astype(np.int32) if counts is None else np.asarray(counts, np.int32)
    ids = np.full((nq, k), -1, np.int32)
    for q in range(nq):
        ids[q, :cnt[q]] = rng.choice(n_docs, cnt[q], replace=False) + id_base
        if dup and cnt[q] >= 4:
            ids[q, 3] = ids[q, 1]                          # the same passage twice: an exact tie
    return TopK(torch.zeros(nq, k, device=DEV), torch.from_numpy(ids).to(DEV), torch.from_numpy(cnt).to(DEV))


# ------------------------------------------------------------------------------------------ packing
@pytest.mark.parametrize("family", ["bert", "roberta"])
def test_pack_matches_the_tokenizer_restatement(family):
    _, _, model = _model(family, d=128, layers=1, vocab=500)
    rng = np.random.default_rng(11)
    max_length, n_docs, nq, k, id_base = 64, 200, 9, 30, 1000
    passages = _tokens(rng, n_docs, 0, 150, 500)                       # empty ones and ones longer than max_length
    queries = _tokens(rng, nq, 0, 90, 500)                             # beyond T/2 and beyond T
    queries[2] = []
    counts = rng.integers(0, k + 1, nq)
    counts[0], counts[1] = k, 0
    rr = CrossEncoderReranker(model, passages, max_length=max_length, id_base=id_base)
    cand = _cand(rng, nq, k, n_docs, id_base=id_base, counts=counts)
    pairs = rr.pack(cand.ids, cand.counts, *_csr(queries))
    ids, types, pos = (x.cpu().numpy() for x in (pairs.ids, pairs.types, pairs.positions))
    cu = pairs.cu_h
    assert pairs.pair_off.cpu().tolist() == np.concatenate([[0], np.cumsum(counts)]).tolist()
    assert cu[0] == 0 and cu[-1] == ids.size and pairs.n_pairs == counts.sum()
    c_ids = cand.ids.cpu().numpy()
    p = 0
    for q in range(nq):
        for r in range(counts[q]):
            want = orr.cross_encoder_inputs(queries[q], passages[c_ids[q, r] - id_base], max_length, family,
                                            model.cls_id, model.sep_id, pad_id=model.pad_id)
            s = slice(cu[p], cu[p + 1])
            assert (ids[s].tolist(), types[s].tolist(), pos[s].tolist()) == want, (q, r)
            assert len(want[0]) <= max_length
            p += 1
    # an id outside the passage range is an error, not a silent empty pair
    bad = TopK(cand.scores, cand.ids.clone(), cand.counts)
    bad.ids[0, 0] = id_base + n_docs
    with pytest.raises(_lib.EzrError, match="outside"):
        rr.pack(bad.ids, bad.counts, *_csr(queries))


# ----------------------------------------------------------------------------------------- embedding
def test_typed_embedding_is_bit_exact():
    """Per-token types select exactly the type row the untyped kernel adds (same rounding order: word + type, then
    + position, then LayerNorm), and agree with a torch bf16 restatement of BertEmbeddings."""
    L = _lib.lib()
    d, vocab, max_pos, t = 768, 1000, 512, 700
    g = torch.Generator().manual_seed(3)
    bf = lambda *s, sc=0.05: (torch.randn(*s, generator=g) * sc).to(torch.bfloat16).to(DEV)
    word, posw, tt, gamma, beta = bf(vocab, d), bf(max_pos, d), bf(2, d), 1 + bf(d, sc=0.1), bf(d)
    ids = torch.randint(0, vocab, (t,), generator=g, dtype=torch.int32).to(DEV)
    pos = torch.randint(0, max_pos, (t,), generator=g, dtype=torch.int32).to(DEV)
    types = torch.randint(0, 2, (t,), generator=g, dtype=torch.int32).to(DEV)
    st = _lib.stream_ptr()

    def typed(ty):
        out = torch.empty(t, d, dtype=torch.bfloat16, device=DEV)
        _lib.check(L.ezr_bert_embed_typed(_lib.ptr(ids), _lib.ptr(pos), _lib.ptr(ty), t, _lib.ptr(word), _lib.ptr(posw),
                                          _lib.ptr(tt), 2, _lib.ptr(gamma), _lib.ptr(beta), 1e-12, vocab, max_pos, d,
                                          _lib.ptr(out), st))
        return out

    def untyped(row):
        out = torch.empty(t, d, dtype=torch.bfloat16, device=DEV)
        _lib.check(L.ezr_bert_embed(_lib.ptr(ids), _lib.ptr(pos), t, _lib.ptr(word), _lib.ptr(posw), _lib.ptr(row),
                                    _lib.ptr(gamma), _lib.ptr(beta), 1e-12, vocab, max_pos, d, _lib.ptr(out), st))
        return out

    got = typed(types)
    u0, u1 = untyped(tt[0].contiguous()), untyped(tt[1].contiguous())
    m = (types == 1)[:, None]
    assert torch.equal(got, torch.where(m, u1, u0))
    assert torch.equal(typed(torch.zeros_like(types)), u0)
    # torch bf16 restatement: the sums rounded exactly as the kernel rounds them; LayerNorm statistics are fp32
    # reductions in a different order, so its bf16 output may differ by one rounding step
    x = (word[ids.long()] + tt[types.long()]) + posw[pos.long()]
    ref = torch.nn.functional.layer_norm(x.float(), (d,), gamma.float(), beta.float(), 1e-12).to(torch.bfloat16)
    diff = (got.float() - ref.float()).abs()
    assert (diff <= ref.float().abs() * 2 ** -7 + 1e-6).all()
    assert (diff == 0).float().mean().item() > 0.95


# ------------------------------------------------------------------------------------- scores + order
def _oracle_scores(family, cfg, state, model, queries, passages, cand, max_length, id_base=0, dtype=torch.float32):
    c_ids, cnt = cand.ids.cpu().numpy(), cand.counts.cpu().numpy()
    pairs, where = [], []
    for q in range(len(queries)):
        for r in range(cnt[q]):
            ids, types, _ = orr.cross_encoder_inputs(queries[q], passages[c_ids[q, r] - id_base], max_length, family,
                                                     model.cls_id, model.sep_id, pad_id=model.pad_id)
            pairs.append((ids, types))
            where.append((q, r))
    logits, scores = orr.cross_encoder_scores(family, cfg, state, pairs, pad_id=model.pad_id, dtype=dtype, device=DEV)
    return logits, scores, where


def _logit(s):
    s = np.asarray(s, np.float64)
    return np.log(s) - np.log1p(-s)


@pytest.mark.parametrize("family", ["bert", "roberta"])
def test_scores_match_transformers_and_order_is_the_reference_sort(family):
    cfg, state, model = _model(family)
    rng = np.random.default_rng(21 if family == "bert" else 22)
    n_docs, nq, k, top_n, max_length = 120, 4, 24, 6, 512
    passages = _tokens(rng, n_docs, 20, 520, cfg.vocab_size)
    queries = _tokens(rng, nq, 4, 300, cfg.vocab_size)
    cand = _cand(rng, nq, k, n_docs, counts=[k, 7, 1, 19], dup=True)
    rr = CrossEncoderReranker(model, passages, max_length=max_length)
    top, all_scores = rr.rerank(cand, *_csr(queries), top_n=top_n)
    all_h = all_scores.cpu().numpy()
    logits, scores, where = _oracle_scores(family, cfg, state, model, queries, passages, cand, max_length)
    logits_b, _, _ = _oracle_scores(family, cfg, state, model, queries, passages, cand, max_length,
                                    dtype=torch.bfloat16)
    floor = float(np.abs(logits_b - logits).max())
    got = np.array([all_h[q, r] for q, r in where])
    assert np.all(np.isfinite(got)) and np.all((got > 0) & (got < 1)), "scores should not saturate in this test"
    err = float(np.abs(_logit(got) - logits).max())
    assert err <= FLOOR_FACTOR * floor + FLOOR_ABS, f"logit error {err:.3g}; bf16 noise floor {floor:.3g}"
    tol_s = float(np.abs(got - scores).max())
    cnt = cand.counts.cpu().numpy()
    c_ids = cand.ids.cpu().numpy()
    t_ids, t_sc, t_cnt = top.ids.cpu().numpy(), top.scores.cpu().numpy(), top.counts.cpu().numpy()
    for q in range(nq):
        row = all_h[q, :cnt[q]].tolist()
        assert np.all(np.isneginf(all_h[q, cnt[q]:]))
        # bit-exact to the reference sort applied to the GPU's own scores
        want = orr.rerank_order(row, top_n)
        assert t_cnt[q] == len(want)
        assert t_ids[q, :t_cnt[q]].tolist() == [int(c_ids[q, i]) for i in want]
        assert t_sc[q, :t_cnt[q]].tolist() == [row[i] for i in want]
        assert np.all(t_ids[q, t_cnt[q]:] == -1) and np.all(np.isneginf(t_sc[q, t_cnt[q]:]))
        # and to the fp32 oracle's order outside near-ties
        ref = [s for (qq, _), s in zip(where, scores) if qq == q]
        ref_top = orr.rerank_order(ref, top_n)
        for i, r in enumerate(want):
            assert abs(ref[r] - ref[ref_top[i]]) <= 2 * tol_s, (q, i)
    # the duplicated candidate scores exactly like its twin, and the earlier one ranks first
    for q in range(nq):
        if cnt[q] >= 4:
            assert all_h[q, 3] == all_h[q, 1]
            order = orr.rerank_order(all_h[q, :cnt[q]].tolist(), cnt[q])
            assert order.index(1) < order.index(3)


@pytest.mark.parametrize("family", ["bert", "roberta"])
def test_scores_do_not_depend_on_the_token_budget(family):
    cfg, state, model = _model(family, layers=2)
    rng = np.random.default_rng(31)
    n_docs, nq, k = 150, 5, 40
    passages = _tokens(rng, n_docs, 0, 600, cfg.vocab_size)
    queries = _tokens(rng, nq, 1, 60, cfg.vocab_size)
    cand = _cand(rng, nq, k, n_docs, counts=[40, 0, 13, 40, 1])
    one = CrossEncoderReranker(model, passages, max_tokens=10 ** 7)
    many = CrossEncoderReranker(model, passages, max_tokens=512)
    pairs = many.pack(cand.ids, cand.counts, *_csr(queries))
    assert len(one.chunks(pairs.cu_h)) == 1 and len(many.chunks(pairs.cu_h)) > 20
    a_top, a = one.rerank(cand, *_csr(queries), top_n=6)
    b_top, b = many.rerank(cand, *_csr(queries), top_n=6)
    assert torch.equal(a, b)
    assert torch.equal(a_top.ids, b_top.ids) and torch.equal(a_top.scores, b_top.scores)
    assert b_top.counts.cpu().tolist() == [6, 0, 6, 6, 1]


def test_reranks_a_coarse_ranker_result_with_short_lists():
    """End to end from CoarseRanker.hybrid: a 40-document corpus asked for k = 64, so every list is short."""
    from easyrag_b200.index import Bm25Index, Bm25Stats, DenseIndex
    n, vocab, dim, nq, k = 40, 300, 128, 6, 64
    corpus = synth.make_sparse_corpus(n, vocab, 1)
    qs = synth.make_queries(corpus, nq, 2)
    g = torch.Generator().manual_seed(4)
    c = torch.randn(n, dim, generator=g).to(torch.bfloat16)
    qv = torch.randn(nq, dim, generator=g).to(torch.bfloat16)
    ranker = batched.CoarseRanker(DenseIndex(c, device=DEV),
                                  Bm25Index(Bm25Stats.from_tokens(corpus.tokens, corpus.doc_ptr, vocab), device=DEV))
    fused, _, _ = ranker.hybrid(qv.to(DEV), qs.term_ptr.to(DEV), qs.terms.to(DEV), k, k, k)
    cnt = fused.counts.cpu().numpy()
    assert np.all((cnt > 0) & (cnt < k))
    cfg, state, model = _model("roberta", layers=2)
    rng = np.random.default_rng(41)
    passages = _tokens(rng, n, 5, 300, cfg.vocab_size)
    queries = _tokens(rng, nq, 3, 30, cfg.vocab_size)
    rr = CrossEncoderReranker(model, passages)
    top, all_scores = rr.rerank(fused, *_csr(queries), top_n=6)
    all_h = all_scores.cpu().numpy()
    _, scores, where = _oracle_scores("roberta", cfg, state, model, queries, passages, fused, 512)
    got = np.array([all_h[q, r] for q, r in where])
    assert np.abs(got - scores).max() < SCORE_TOL
    assert top.counts.cpu().tolist() == [min(6, int(x)) for x in cnt]
    f_ids = fused.ids.cpu().numpy()
    for q in range(nq):
        assert np.all(np.isneginf(all_h[q, cnt[q]:]))
        want = orr.rerank_order(all_h[q, :cnt[q]].tolist(), 6)
        assert top.ids[q, :len(want)].cpu().tolist() == [int(f_ids[q, i]) for i in want]


# -------------------------------------------------------------------------------------------- drop-in
class _WordTokenizer:
    """Whitespace words -> ids by hash, HF call shape: tok(texts, add_special_tokens=False)["input_ids"]."""

    def __init__(self, vocab):
        self.vocab = vocab

    def __call__(self, texts, add_special_tokens=True):
        assert add_special_tokens is False
        return {"input_ids": [[4 + (sum(map(ord, w)) * 7919) % (self.vocab - 4) for w in t.split()] for t in texts]}


def test_sentence_transformer_rerank_dropin():
    cfg, state, model = _model("roberta", d=256, layers=2, vocab=800)
    tok = _WordTokenizer(cfg.vocab_size)
    rr = SentenceTransformerRerank(top_n=3, model="local-ce", keep_retrieval_score=True, encoder=model, tokenizer=tok)
    assert rr.top_n == 3 and rr.class_name() == "SentenceTransformerRerank"
    words = "alpha beta gamma delta epsilon zeta eta theta iota kappa lambda mu".split()
    rng = np.random.default_rng(2)
    texts = [" ".join(rng.choice(words, int(rng.integers(1, 30)))) for _ in range(9)]
    texts[5] = texts[2]                                               # an exact tie
    nodes = [NodeWithScore(TextNode(t, id_=str(i), metadata={"file_path": f"d/{i}.txt"}), 1.0 / (i + 1))
             for i, t in enumerate(texts)]
    with pytest.raises(ValueError):
        rr.postprocess_nodes(nodes)
    assert rr.postprocess_nodes([], QueryBundle("q")) == []
    out = rr.postprocess_nodes(nodes, QueryBundle("alpha kappa mu"))
    # scores: the model on (query, raw node text) pairs; order: the reference's sorted(...)[:top_n]
    q_ids = tok(["alpha kappa mu"], add_special_tokens=False)["input_ids"][0]
    pairs = [orr.cross_encoder_inputs(q_ids, p, 512, "roberta", model.cls_id, model.sep_id, model.pad_id)[:2]
             for p in tok(texts, add_special_tokens=False)["input_ids"]]
    _, ref = orr.cross_encoder_scores("roberta", cfg, state, pairs, pad_id=model.pad_id, device=DEV)
    got = [n.score for n in nodes]
    assert all(isinstance(s, float) for s in got)
    assert np.abs(np.array(got) - ref).max() < SCORE_TOL
    assert got[5] == got[2]
    assert [n.node.node_id for n in out] == [str(i) for i in orr.rerank_order(got, 3)]
    assert [n.node.metadata["retrieval_score"] for n in nodes] == [1.0 / (i + 1) for i in range(9)]
    rr.top_n = 20
    again = rr.postprocess_nodes(nodes, query_str="alpha kappa mu")
    assert len(again) == 9 and [n.node.node_id for n in again] == [str(i) for i in orr.rerank_order(got, 9)]
