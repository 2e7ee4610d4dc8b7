"""GPU: the reranker pair packers (csrc/handoff.cu) and the cross-encoder order (csrc/rerank.cu) at pipeline scale.

Every packer output is compared bit for bit, as whole arrays, with the torch restatement in tests/_pack_ref.py
(pinned to the per-pair oracles on the CPU by test_pack_ref_cpu.py):

* the offset scan across its 1024-element blocks (slot and query counts on both sides of each multiple of 1024);
* pipeline-sized batches (10 000 x 192 cross-encoder slots, ~4 000 x 288 LLM slots) with duplicates, a [Q, k] view
  of a wider top-k and global ids near 2^31, and a real ``CoarseRanker.hybrid`` result;
* k = 1023 and 1024 (``MAX_CANDIDATES``) through the packers and both forms of the ordering kernel;
* ``CrossEncoderReranker.rerank`` end to end under token budgets from one pair to a few chunks;
* the int32 ``cu_seqlens`` limit (totals of exactly 2^31 - 1 and 2^31) and candidate ids outside the passage range.
"""
import ctypes

import numpy as np
import pytest
import torch

import _pack_ref as pr
from oracle import rerank as orr
from easyrag_b200 import _lib, batched, synth
from easyrag_b200.batched import TopK
from easyrag_b200.encoder import BertConfig
from easyrag_b200.handoff import RerankPacker
from easyrag_b200.rerank import MAX_CANDIDATES, CrossEncoderModel, CrossEncoderReranker, random_cross_encoder_state

pytestmark = pytest.mark.gpu
DEV = "cuda"
SPECIAL = {"bert": dict(cls_id=2, sep_id=3, pad_id=0), "roberta": dict(cls_id=0, sep_id=2, pad_id=1)}
N_DOCS = 10_000
TOP_ID_BASE = 2 ** 31 - 1 - N_DOCS          # global ids of the last shard of a sharded coarse ranker
SEP, PROMPT, BOS = [13, 14], [31, 32, 33, 34, 35, 36, 37], 1
CHUNK_TOKENS = 1 << 26                      # token comparisons walk the pack in pieces of about this size
FLOOR_FACTOR, FLOOR_ABS = 1.5, 0.02         # as test_gpu_rerank.py: logits within 1.5x the bf16 floor + 0.02


@pytest.fixture(scope="module", autouse=True)
def _ready(lib_built):
    _lib.require_cuda()


def _rng(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _csr(lens, g, vocab=30000):
    ptr = torch.zeros(lens.numel() + 1, dtype=torch.int64, device=DEV)
    torch.cumsum(lens.to(torch.int64), 0, out=ptr[1:])
    tok = torch.randint(4, vocab, (max(int(ptr[-1]), 1),), generator=g, device=DEV, dtype=torch.int32)
    return ptr, tok[:int(ptr[-1])]


def _queries(nq, hi, seed):
    g = _rng(seed)
    ptr, tok = _csr(torch.randint(0, hi + 1, (nq,), generator=g, device=DEV), g)
    return ptr.to(torch.int32), tok


def _cands(nq, k, seed, width=None, id_base=0, n_docs=N_DOCS, counts=None):
    """[Q, k] candidates drawn with replacement (duplicates in most lists), -1 past each count, and junk in columns k..
    of a wider buffer when ``width`` > k (the view a caller slices from a larger top-k)."""
    g = _rng(seed)
    width = width or k
    buf = torch.randint(-3, 2 ** 31 - 1, (nq, width), generator=g, device=DEV, dtype=torch.int32)
    if counts is None:
        counts = torch.randint(0, k + 1, (nq,), generator=g, device=DEV, dtype=torch.int32)
        counts[:3] = torch.tensor([k, 0, k], dtype=torch.int32)[:nq]
    ids = torch.randint(0, n_docs, (nq, k), generator=g, device=DEV, dtype=torch.int32) + id_base
    if k >= 3:
        ids[:, 2] = ids[:, 0]                                          # the same document twice in every list
    r = torch.arange(k, device=DEV)
    buf[:, :k] = torch.where(r[None, :] < counts[:, None].long(), ids, torch.full_like(ids, -1))
    return buf[:, :k], counts


@pytest.fixture(scope="module")
def corpus():
    """Passages of U[0, 700] tokens: device CSR and the per-passage lists the packers' constructors take."""
    g = _rng(1)
    p_ptr, p_tok = _csr(torch.randint(0, 701, (N_DOCS,), generator=g, device=DEV), g)
    ptr_h, tok_h = p_ptr.cpu().numpy(), p_tok.cpu().numpy()
    return p_ptr, p_tok, np.split(tok_h, ptr_h[1:-1])


def _model(family, d=128, layers=1, seed=7, vocab=30000):
    cfg = BertConfig(vocab_size=vocab, hidden_size=d, intermediate_size=4 * d, num_hidden_layers=layers,
                     num_attention_heads=d // 64, max_position_embeddings=514 if family == "roberta" else 512,
                     layer_norm_eps=1e-5 if family == "roberta" else 1e-12)
    state = random_cross_encoder_state(family, cfg, seed, std=0.03)
    return cfg, state, CrossEncoderModel(family, cfg, state, device=DEV, **SPECIAL[family])


_CACHE = {}


def _cross(corpus, family, max_length=512, id_base=0):
    key = ("cross", family, max_length, id_base)
    if key not in _CACHE:
        _CACHE[key] = CrossEncoderReranker(_model(family)[2], corpus[2], max_length=max_length, id_base=id_base)
    return _CACHE[key]


def _llm(corpus, max_length=1024, id_base=0):
    key = ("llm", max_length, id_base)
    if key not in _CACHE:
        _CACHE[key] = RerankPacker(corpus[2], SEP, PROMPT, BOS, max_length=max_length, id_base=id_base)
    return _CACHE[key]


def _chunks(cu, tokens=CHUNK_TOKENS):
    """Pair ranges [p0, p1) of about ``tokens`` tokens each, from an int64 host cu."""
    n, out, p0 = cu.size - 1, [], 0
    while p0 < n:
        p1 = min(max(int(np.searchsorted(cu, cu[p0] + tokens, side="right")) - 1, p0 + 1), n)
        out.append((p0, p1))
        p0 = p1
    return out


def _cross_plan_abi(rr, cand, counts, q_ptr):
    """ezr_cross_pack_plan alone -> (rc, pair_off, cu int32 [Q*k + 1], totals)."""
    L = _lib.lib()
    nq, k = cand.shape
    m = rr.model
    ws = torch.empty(L.ezr_cross_pack_workspace(nq, k), dtype=torch.uint8, device=DEV)
    pair_off = torch.empty(nq + 1, dtype=torch.int32, device=DEV)
    cu = torch.empty(nq * k + 1, dtype=torch.int32, device=DEV)
    totals = (ctypes.c_int64 * 2)()
    rc = L.ezr_cross_pack_plan(_lib.ptr(cand), _lib.ptr(counts), nq, k, cand.stride(0), rr.id_base, rr.n_docs,
                               _lib.ptr(q_ptr), _lib.ptr(rr.p_ptr), m.n_mid, rr.max_length, _lib.ptr(pair_off),
                               _lib.ptr(cu), totals, _lib.ptr(ws), ws.numel(), _lib.stream_ptr())
    return rc, pair_off, cu, (int(totals[0]), int(totals[1]))


def _llm_plan_abi(pk, cand, counts, q_ptr):
    """ezr_rerank_pack_plan alone -> (rc, cu int64 [Q*k + 1], query_len, total)."""
    L = _lib.lib()
    nq, k = cand.shape
    n = nq * k
    ln = torch.empty(n, dtype=torch.int64, device=DEV)
    cu = torch.empty(n + 1, dtype=torch.int64, device=DEV)
    qlen = torch.empty(n, dtype=torch.int32, device=DEV)
    total = ctypes.c_int64(-1)
    rc = L.ezr_rerank_pack_plan(_lib.ptr(cand), _lib.ptr(counts), nq, k, cand.stride(0), pk.id_base, pk.n_docs,
                                _lib.ptr(q_ptr), _lib.ptr(pk.p_ptr), pk.n_sep, pk.n_prompt, pk.max_length,
                                _lib.ptr(ln), _lib.ptr(cu), _lib.ptr(qlen), ctypes.byref(total), _lib.stream_ptr())
    return rc, cu, qlen, int(total.value)


def check_cross(rr, cand, counts, q_ptr, q_tok):
    """rr.pack and the plan's device arrays == the restatement, bit for bit on every array."""
    m, k = rr.model, cand.shape[1]
    ref = pr.cross_plan(q_ptr, rr.p_ptr, cand, counts, k, rr.id_base, m.n_mid, rr.max_length)
    rc, pair_off, cu, totals = _cross_plan_abi(rr, cand, counts, q_ptr)
    assert rc == 0
    assert totals == (ref["T"], ref["P"])
    assert torch.equal(pair_off.long(), ref["pair_off"])
    assert torch.equal(cu[:ref["P"] + 1].long(), ref["cu"])
    pairs = rr.pack(cand, counts, q_ptr, q_tok)
    cu_h = ref["cu"].cpu().numpy()
    assert np.array_equal(pairs.cu_h, cu_h) and pairs.n_pairs == ref["P"]
    assert torch.equal(pairs.pair_off.long(), ref["pair_off"])
    assert pairs.ids.numel() == pairs.types.numel() == pairs.positions.numel() == ref["T"]
    for p0, p1 in _chunks(cu_h):
        ids, types, pos = pr.cross_tokens(ref, q_ptr, q_tok, rr.p_ptr, rr.p_tok, m.cls_id, m.sep_id, m.type_b,
                                          m.pos_offset, p0, p1)
        s = slice(int(cu_h[p0]), int(cu_h[p1]))
        assert torch.equal(pairs.ids[s], ids), (p0, p1)
        assert torch.equal(pairs.types[s], types), (p0, p1)
        assert torch.equal(pairs.positions[s], pos), (p0, p1)
    return pairs, ref


def check_llm(pk, cand, counts, q_ptr, q_tok):
    k = cand.shape[1]
    sep, prompt = pk.sep[:pk.n_sep], pk.prompt[:pk.n_prompt]
    ref = pr.llm_plan(q_ptr, pk.p_ptr, cand, counts, k, pk.id_base, pk.n_sep, pk.n_prompt, pk.max_length)
    rc, cu64, qlen64, total = _llm_plan_abi(pk, cand, counts, q_ptr)
    assert rc == 0 and total == ref["T"]
    assert torch.equal(cu64, ref["cu"]) and torch.equal(qlen64, ref["query_len"])
    out = pk.pack(cand, counts, q_ptr, q_tok)
    assert out.ids.numel() == ref["T"] and out.prompt_len == pk.n_sep + pk.n_prompt
    assert torch.equal(out.cu.long(), ref["cu"])
    assert torch.equal(out.query_len, ref["query_len"])
    cu_h = ref["cu"].cpu().numpy()
    for p0, p1 in _chunks(cu_h):
        want = pr.llm_tokens(ref, q_ptr, q_tok, pk.p_ptr, pk.p_tok, sep, prompt, pk.bos, p0, p1)
        assert torch.equal(out.ids[int(cu_h[p0]):int(cu_h[p1])], want), (p0, p1)
    assert list(out.slices(32)) == pr.llm_slices(cand.shape[0], k)
    return out, ref


# ------------------------------------------------------------------------------------------ scan boundaries
# (Q, k): Q * k slots on both sides of one and two scan blocks and well past them; then Q itself past 1024 (pair_off)
SLOTS = [(3, 341), (4, 256), (5, 205), (23, 89), (2, 1024), (3, 683), (51, 743)]
QUERIES = [(1023, 2), (1024, 2), (1025, 2), (4097, 2)]


@pytest.mark.parametrize("nq,k", SLOTS + QUERIES)
def test_scan_boundaries(corpus, nq, k):
    q_ptr, q_tok = _queries(nq, 900, seed=nq * 7 + k)
    cand, counts = _cands(nq, k, seed=nq + 3 * k)
    for family in ("bert", "roberta"):
        check_cross(_cross(corpus, family), cand, counts, q_ptr, q_tok)
    check_llm(_llm(corpus), cand, counts, q_ptr, q_tok)


# ------------------------------------------------------------------------------------------ pipeline scale
@pytest.mark.parametrize("family,width,id_base", [("bert", 256, 0), ("roberta", 192, TOP_ID_BASE)])
def test_cross_pack_at_pipeline_scale(corpus, family, width, id_base):
    nq, k = 10_000, 192
    q_ptr, q_tok = _queries(nq, 900, seed=11)
    cand, counts = _cands(nq, k, seed=12, width=width, id_base=id_base)
    assert cand.stride(0) == width
    pairs, ref = check_cross(_cross(corpus, family, id_base=id_base), cand, counts, q_ptr, q_tok)
    assert ref["P"] > 900_000 and ref["T"] > 4e8 and int(ref["slot_len"].max()) == 512


@pytest.mark.parametrize("width,id_base", [(300, TOP_ID_BASE), (288, 0)])
def test_llm_pack_at_pipeline_scale(corpus, width, id_base):
    nq, k = 4_000, 288
    q_ptr, q_tok = _queries(nq, 900, seed=21)
    cand, counts = _cands(nq, k, seed=22, width=width, id_base=id_base)
    out, ref = check_llm(_llm(corpus, id_base=id_base), cand, counts, q_ptr, q_tok)
    assert int(ref["len"].max()) == 1024 + len(SEP) + len(PROMPT) and ref["T"] > 3e8


def test_packs_a_coarse_ranker_result_with_short_lists(corpus):
    """CoarseRanker.hybrid over a 100-document corpus asked for k = 192: every fused list is short, and -1 padded."""
    from easyrag_b200.index import Bm25Index, Bm25Stats, DenseIndex
    n, vocab, dim, nq, k = 100, 500, 128, 40, 192
    sparse = synth.make_sparse_corpus(n, vocab, 1)
    qs = synth.make_queries(sparse, nq, 2)
    g = torch.Generator().manual_seed(4)
    c = torch.randn(n, dim, generator=g).to(torch.bfloat16)
    qv = torch.randn(nq, dim, generator=g).to(torch.bfloat16)
    ranker = batched.CoarseRanker(DenseIndex(c, device=DEV),
                                  Bm25Index(Bm25Stats.from_tokens(sparse.tokens, sparse.doc_ptr, vocab), device=DEV))
    fused, _, _ = ranker.hybrid(qv.to(DEV), qs.term_ptr.to(DEV), qs.terms.to(DEV), k, k, k)
    cnt = fused.counts
    assert bool(((cnt > 0) & (cnt < k)).all()) and bool((fused.ids[:, -1] == -1).all())
    passages = corpus[2][:n]
    q_ptr, q_tok = _queries(nq, 900, seed=31)
    for family in ("bert", "roberta"):
        rr = CrossEncoderReranker(_model(family)[2], passages, max_length=512)
        check_cross(rr, fused.ids, fused.counts, q_ptr, q_tok)
    check_llm(RerankPacker(passages, SEP, PROMPT, BOS, max_length=1024), fused.ids, fused.counts, q_ptr, q_tok)


# ------------------------------------------------------------------------------- k = 1023 and 1024: pack + order
def _order_both_forms(dense, pair_off, cand, w_out, b_out, top_n):
    """ezr_cross_score_topk (one launch) and ezr_cross_pair_scores + ezr_cross_order_topk -> two result tuples."""
    L = _lib.lib()
    nq, k = cand.shape
    d = dense.shape[1]
    st = _lib.stream_ptr()
    res = []
    for fused in (True, False):
        out = (torch.full((nq, k), 7.0, device=DEV), torch.full((nq, top_n), 7.0, device=DEV),
               torch.full((nq, top_n), 7, dtype=torch.int32, device=DEV),
               torch.full((nq,), 7, dtype=torch.int32, device=DEV))
        ptrs = [_lib.ptr(x) for x in out]
        if fused:
            _lib.check(L.ezr_cross_score_topk(_lib.ptr(dense), d, _lib.ptr(pair_off), nq, k, _lib.ptr(cand),
                                              cand.stride(0), _lib.ptr(w_out), b_out, d, top_n, *ptrs, st))
        else:
            sig = torch.empty(dense.shape[0], device=DEV)
            _lib.check(L.ezr_cross_pair_scores(_lib.ptr(dense), d, dense.shape[0], _lib.ptr(w_out), b_out,
                                               _lib.ptr(sig), st))
            _lib.check(L.ezr_cross_order_topk(_lib.ptr(sig), _lib.ptr(pair_off), nq, k, _lib.ptr(cand),
                                              cand.stride(0), top_n, *ptrs, st))
        res.append(out)
    return res


@pytest.mark.parametrize("k", [MAX_CANDIDATES - 1, MAX_CANDIDATES])
def test_max_candidates_pack_and_order(corpus, k):
    nq, d = 2_000, 256
    q_ptr, q_tok = _queries(nq, 200, seed=k)
    cand, counts = _cands(nq, k, seed=k + 1, width=k + 3)
    check_llm(_llm(corpus, max_length=128), cand, counts, q_ptr, q_tok)
    pairs, ref = check_cross(_cross(corpus, "bert", max_length=128), cand, counts, q_ptr, q_tok)
    # The head on random CLS rows: some rows repeated (exact ties), some saturated so the sigmoid is exactly 1.0f
    g = _rng(k + 2)
    P = ref["P"]
    w_out = torch.randn(d, generator=g, device=DEV) * 0.3
    dense = (torch.randn(P, d, generator=g, device=DEV) * 0.5).to(torch.bfloat16)
    sat = torch.rand(P, generator=g, device=DEV) < 0.05
    dense[sat] = (torch.sign(w_out) * 8).to(torch.bfloat16)
    dup = torch.nonzero(torch.rand(P, generator=g, device=DEV) < 0.1).squeeze(1)
    dup = dup[dup > 0]
    dense[dup] = dense[dup - 1]
    cnt_h, c_ids = counts.cpu().numpy(), cand.cpu().numpy()
    orders, all_h = None, None
    for top_n in (1, 6, 192, 1024, 1500):
        a, b = _order_both_forms(dense, pairs.pair_off, pairs.cand_ids, w_out, 0.25, top_n)
        for x, y in zip(a, b):
            assert torch.equal(x, y), top_n                    # the fused and two-launch forms agree bit for bit
        all_scores, t_sc, t_ids, t_cnt = (x.cpu().numpy() for x in a)
        if orders is None:
            all_h = all_scores
            assert (all_h == 1.0).sum() > 1000
            orders = [orr.rerank_order(all_h[q, :cnt_h[q]].tolist(), k) for q in range(nq)]
        assert np.array_equal(all_scores, all_h)
        assert np.array_equal(t_cnt, np.minimum(cnt_h, top_n))
        for q in range(nq):
            n = int(cnt_h[q])
            assert np.all(np.isneginf(all_h[q, n:]))
            want = orders[q][:top_n]
            c = len(want)
            assert t_ids[q, :c].tolist() == [int(c_ids[q, i]) for i in want], (top_n, q)
            assert t_sc[q, :c].tolist() == [float(all_h[q, i]) for i in want], (top_n, q)
            assert np.all(t_ids[q, c:] == -1) and np.all(np.isneginf(t_sc[q, c:])), (top_n, q)
    # ties were exercised: duplicate rows inside one list score alike and keep their coarse order
    off = pairs.pair_off.cpu().numpy()
    q = int(np.argmax(cnt_h))
    row = all_h[q, :cnt_h[q]]
    assert len(set(row.tolist())) < row.size
    assert 1.0 in row.tolist()
    assert off[-1] == P


# ------------------------------------------------------------------------------- CrossEncoderReranker.rerank
def test_rerank_end_to_end_does_not_depend_on_chunking():
    """2 000 queries x up to 192 candidates through a 2-layer d = 256 model: the budget of one max_length pair
    (thousands of chunks), 65 536 tokens and 2^22 tokens (a few) give the same bits, as does one query at a time; a
    sample of pairs agrees with transformers' classifier within the bf16 noise-floor criterion."""
    family, max_length = "bert", 512
    cfg, state, model = _model(family, d=256, layers=2, seed=5, vocab=3000)
    g = _rng(41)
    n_docs, nq, k = 4_000, 2_000, 192
    p_ptr, p_tok = _csr(torch.randint(0, 25, (n_docs,), generator=g, device=DEV), g, vocab=3000)
    passages = np.split(p_tok.cpu().numpy(), p_ptr.cpu().numpy()[1:-1])
    q_ptr, q_tok = _csr(torch.randint(0, 9, (nq,), generator=g, device=DEV), g, vocab=3000)
    q_ptr = q_ptr.to(torch.int32)
    ids, counts = _cands(nq, k, seed=42, n_docs=n_docs)
    cand = TopK(torch.zeros(nq, k, device=DEV), ids, counts)
    results, n_chunks = [], []
    for budget in (max_length, 65536, 1 << 22):
        rr = CrossEncoderReranker(model, passages, max_length=max_length, max_tokens=budget)
        n_chunks.append(len(rr.chunks(rr.pack(ids, counts, q_ptr, q_tok).cu_h)))
        results.append(rr.rerank(cand, q_ptr, q_tok, top_n=10))
    assert n_chunks[0] > 1000 and n_chunks[2] <= 4, n_chunks
    (top, all_s) = results[0]
    for t, a in results[1:]:
        assert torch.equal(a, all_s)
        assert torch.equal(t.ids, top.ids) and torch.equal(t.scores, top.scores) and torch.equal(t.counts, top.counts)
    cnt_h = counts.cpu().numpy()
    qp_h = q_ptr.cpu().numpy()
    for q in (0, 2, 5, 17, 999, nq - 1):
        one = TopK(cand.scores[q:q + 1], ids[q:q + 1], counts[q:q + 1])
        t1, a1 = rr.rerank(one, q_ptr[q:q + 2] - q_ptr[q], q_tok[int(qp_h[q]):int(qp_h[q + 1])], top_n=10)
        assert torch.equal(a1[0], all_s[q]), q
        assert torch.equal(t1.ids[0], top.ids[q]) and torch.equal(t1.scores[0], top.scores[q]), q
    # ~64 pairs against transformers (fp32), within 1.5x the bf16 evaluation's distance + 0.02 on the logits
    all_h, ids_h, q_tok_h = all_s.cpu().numpy(), ids.cpu().numpy(), q_tok.cpu().numpy()
    sample, got = [], []
    for q in range(3, 3 + 40):
        for r in range(min(int(cnt_h[q]), 2)):
            query = q_tok_h[qp_h[q]:qp_h[q + 1]].tolist()
            ids_, types, _ = orr.cross_encoder_inputs(query, passages[ids_h[q, r]].tolist(), max_length, family,
                                                      model.cls_id, model.sep_id, pad_id=model.pad_id)
            sample.append((ids_, types))
            got.append(float(all_h[q, r]))
    assert 48 <= len(sample) <= 80
    logits, _ = orr.cross_encoder_scores(family, cfg, state, sample, pad_id=model.pad_id, device=DEV)
    logits_b, _ = orr.cross_encoder_scores(family, cfg, state, sample, pad_id=model.pad_id, dtype=torch.bfloat16,
                                           device=DEV)
    floor = float(np.abs(logits_b - logits).max())
    got = np.asarray(got, np.float64)
    err = float(np.abs(np.log(got) - np.log1p(-got) - logits).max())
    assert err <= FLOOR_FACTOR * floor + FLOOR_ABS, f"logit error {err:.3g}; bf16 noise floor {floor:.3g}"


# --------------------------------------------------------------------------------------------- the int32 limit
def _limit_inputs(nq, k, short_len, long_len):
    """Every query empty, every slot filled with passage 0 (``long_len`` tokens) except slot (0, 0), passage 1
    (``short_len`` tokens): the plan's lengths alone decide the totals."""
    p_ptr = torch.tensor([0, long_len, long_len + short_len], dtype=torch.int64, device=DEV)
    q_ptr = torch.zeros(nq + 1, dtype=torch.int32, device=DEV)
    cand = torch.zeros(nq, k, dtype=torch.int32, device=DEV)
    cand[0, 0] = 1
    counts = torch.full((nq,), k, dtype=torch.int32, device=DEV)
    return p_ptr, q_ptr, cand, counts


def _peak_during(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


@pytest.mark.parametrize("family", ["bert", "roberta"])
def test_cross_pack_refuses_two_to_the_31_tokens(family):
    """4096 x 1024 pairs of max_length = 512 tokens are 2^31: one token less is accepted, 2^31 is refused."""
    model = _model(family)[2]
    nq, k, max_length = 4096, 1024, 512
    room = max_length - 2 - model.n_mid
    for short, want_t in ((room - 1, 2 ** 31 - 1), (room, 2 ** 31)):
        p_ptr, q_ptr, cand, counts = _limit_inputs(nq, k, short, 1000)
        rr = CrossEncoderReranker(model, [[5] * 1000, [6] * short], max_length=max_length)
        assert torch.equal(rr.p_ptr, p_ptr)
        ref = pr.cross_plan(q_ptr, p_ptr, cand, counts, k, 0, model.n_mid, max_length)
        assert ref["T"] == want_t and ref["P"] == nq * k
        rc, pair_off, cu, totals = _cross_plan_abi(rr, cand, counts, q_ptr)
        if want_t < 2 ** 31:
            assert rc == 0 and totals == (want_t, nq * k)
            assert int(cu[-1]) == want_t == 2 ** 31 - 1
            assert torch.equal(cu.long(), ref["cu"]) and torch.equal(pair_off.long(), ref["pair_off"])
        else:
            assert rc == -1                                             # EZR_ERR_INVALID
            assert "T=2147483648" in _lib.lib().ezr_last_error().decode()

            def pack():
                with pytest.raises(_lib.EzrError, match="T=2147483648"):
                    rr.pack(cand, counts, q_ptr, torch.zeros(0, dtype=torch.int32))
            # the plan's own buffers are ~0.1 GB; the refused token buffers would be 3 x 8 GB
            assert _peak_during(pack) < 2 ** 30


def test_llm_pack_refuses_two_to_the_31_tokens():
    """2048 x 1024 pairs of 1 + 1 + 998 + 1 + 23 = 1024 tokens are 2^31 (max_length 1000, one sep id, a 23-id
    prompt): one token less is accepted, 2^31 is refused."""
    nq, k, max_length, sep, prompt = 2048, 1024, 1000, [13], list(range(40, 63))
    room = max_length - 1 - len(sep)
    for short, want_t in ((room - 1, 2 ** 31 - 1), (room, 2 ** 31)):
        p_ptr, q_ptr, cand, counts = _limit_inputs(nq, k, short, 1000)
        pk = RerankPacker([[5] * 1000, [6] * short], sep, prompt, BOS, max_length=max_length)
        ref = pr.llm_plan(q_ptr, p_ptr, cand, counts, k, 0, len(sep), len(prompt), max_length)
        assert ref["T"] == want_t
        rc, cu, qlen, total = _llm_plan_abi(pk, cand, counts, q_ptr)
        if want_t < 2 ** 31:
            assert rc == 0 and total == want_t and int(cu[-1]) == want_t
            assert torch.equal(cu, ref["cu"]) and torch.equal(qlen, ref["query_len"])
        else:
            assert rc == -1
            assert "T=2147483648" in _lib.lib().ezr_last_error().decode()

            def pack():
                with pytest.raises(_lib.EzrError, match="T=2147483648"):
                    pk.pack(cand, counts, q_ptr, torch.zeros(0, dtype=torch.int32))
            assert _peak_during(pack) < 2 ** 30


# ------------------------------------------------------------------------------------------ out-of-range ids
@pytest.mark.parametrize("id_base", [0, TOP_ID_BASE])
def test_llm_pack_refuses_ids_outside_the_passages(corpus, id_base):
    """As the cross-encoder pack does: an id below id_base or at id_base + n_docs and above, among a query's first
    count candidates, is refused by the plan; the same ids past the count are padding and ignored."""
    pk = _llm(corpus, id_base=id_base)
    rr = _cross(corpus, "roberta", id_base=id_base)
    nq, k = 50, 40
    q_ptr, q_tok = _queries(nq, 900, seed=51)
    cand, counts = _cands(nq, k, seed=52, id_base=id_base)
    counts[:] = torch.clamp(counts, max=k - 1)
    counts[0] = 5
    bad_ids = sorted(b for b in {id_base + N_DOCS, id_base + N_DOCS + 1, 2 ** 31 - 1, id_base - 1, -1} if b < 2 ** 31)
    for bad in bad_ids:
        for r in (0, 4):                                                 # inside query 0's count of 5
            c = cand.clone()
            c[0, r] = bad
            for plan in (_llm_plan_abi(pk, c, counts, q_ptr), _cross_plan_abi(rr, c, counts, q_ptr)):
                assert plan[0] == -1, (bad, r)
                assert "outside [id_base, id_base + n_docs)" in _lib.lib().ezr_last_error().decode()
            with pytest.raises(_lib.EzrError, match="outside"):
                pk.pack(c, counts, q_ptr, q_tok)
        # past the count (slot 5 of query 0, and the last slot of every query) it is padding
        c = cand.clone()
        c[0, 5] = bad
        c[:, k - 1] = bad
        check_llm(pk, c, counts, q_ptr, q_tok)
        check_cross(rr, c, counts, q_ptr, q_tok)
