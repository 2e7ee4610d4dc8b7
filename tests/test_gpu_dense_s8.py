"""Dense top-k over a quantized index (csrc/dense_s8.cu) against its definition, bit for bit.

The expected lists come from ``rescore`` over EVERY row that passes the filter: the fp32 dot product of the bf16
query and bf16 row, ``acc = acc + q[:, i] * r[:, i]`` for i = 0 .. dim-1, evaluated here with eager torch float32
multiplies and adds on the device (separate IEEE-rounded kernels, no fused op), then the canonical order (score
descending, id descending) through one int64 key per (score, id).
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
I64_MIN = torch.iinfo(torch.int64).min


def _lib():
    from easyrag_b200 import _lib
    return _lib


def rescore_all(q: torch.Tensor, c: torch.Tensor, q_chunk: int = 64, row_chunk: int = 0) -> torch.Tensor:
    """[Q, N] float32 rescore values (``-0.0`` as ``+0.0``).  ``row_chunk`` > 0 converts the corpus to float32 that
    many rows at a time (the same operations per element, so the same bits; a 4M x 1024 float copy would be 16 GB)."""
    n = c.shape[0]
    row_chunk = row_chunk if row_chunk > 0 else max(n, 1)
    qf = q.float()
    out = torch.empty(q.shape[0], n, dtype=torch.float32, device=q.device)
    for r0 in range(0, n, row_chunk):
        r1 = min(n, r0 + row_chunk)
        ct = c[r0:r1].float().T.contiguous()            # [dim, rows]
        for q0 in range(0, q.shape[0], q_chunk):
            qq = qf[q0:q0 + q_chunk]
            acc = torch.zeros(qq.shape[0], r1 - r0, dtype=torch.float32, device=q.device)
            for i in range(c.shape[1]):
                acc = acc + qq[:, i:i + 1] * ct[i][None, :]
            out[q0:q0 + q_chunk, r0:r1] = acc + 0.0
        del ct
    return out


def canonical_topk(s: torch.Tensor, k: int, allowed=None, id_base: int = 0):
    """(ids + id_base, scores, counts) of the canonical top-k of float32 scores [Q, N]."""
    b = s.view(torch.int32).long()
    ordered = torch.where(b >= 0, b, b ^ 0x7fffffff)               # float order as integers
    n = s.shape[1]
    key = ordered * (1 << 32) + torch.arange(n, device=s.device)
    if allowed is not None:
        key = torch.where(allowed, key, torch.full_like(key, I64_MIN))
    kk = min(k, n)
    kv, ki = key.topk(kk, dim=1)
    valid = kv != I64_MIN
    counts = valid.sum(1).to(torch.int32)
    ids = torch.where(valid, ki + id_base, torch.full_like(ki, -1)).to(torch.int32)
    sc = torch.where(valid, s.gather(1, ki), torch.full_like(s.gather(1, ki), -float("inf")))
    return ids, sc, counts


def run_s8(index, q, k, q_group=None, id_base=None, cap=0):
    """One search; ``cap`` = candidate capacity per query for this call (0: the default)."""
    from easyrag_b200 import batched
    L = _lib().lib()
    cc = torch.empty(q.shape[0], dtype=torch.int32, device=DEV)
    _lib().check(L.ezr_dense_s8_set_capacity(cap))
    try:
        out = batched.dense_topk(index, q, k, q_group=q_group, id_base=id_base, cand_counts=cc)
        torch.cuda.synchronize()
    finally:
        _lib().check(L.ezr_dense_s8_set_capacity(0))
    return out, cc


def run_certified(index, q, k, q_group=None, id_base=None):
    """A search whose every query is answered by the int8 pass + rescoring: the capacity is the number of rows, and
    no query may have overflowed (k <= 16; larger k always takes the full scan)."""
    cap = max(index.n_rows, 1)
    out, cc = run_s8(index, q, k, q_group=q_group, id_base=id_base, cap=cap)
    assert k > 16 or (cc <= cap).all(), "a query overflowed a buffer as large as the corpus"
    return out, cc


def assert_same(out, ids, sc, counts, what=""):
    assert torch.equal(out.counts, counts), what
    k = ids.shape[1]
    mask = torch.arange(k, device=DEV)[None, :] < counts[:, None].long()
    assert torch.equal(torch.where(mask, out.ids, -1), torch.where(mask, ids, -1)), what
    a = torch.where(mask, out.scores, 0.0).view(torch.int32)
    b = torch.where(mask, sc, 0.0).view(torch.int32)
    assert torch.equal(a, b), what


def make_index(c, **kw):
    from easyrag_b200.index import DenseIndex
    return DenseIndex(c, device=DEV, quantized=True, **kw)


def np_quantize(x: np.ndarray):
    """The quantizer's definition in numpy (float32 division, round half to even)."""
    x = x.astype(np.float32)
    m = np.abs(x).max(1)
    scale = (m / np.float32(127)).astype(np.float32)
    safe = np.where(scale > 0, scale, np.float32(1))
    r = np.clip(np.rint((x / safe[:, None]).astype(np.float32)), -127, 127)
    r = np.where(scale[:, None] > 0, r, 0).astype(np.int8)
    a = scale[:, None].astype(np.float64) * r.astype(np.float64)
    e = np.sqrt(((x.astype(np.float64) - a) ** 2).sum(1))
    n = np.sqrt((a ** 2).sum(1))
    return r, scale, e, n


def test_quantizer_matches_numpy(lib_built):
    from easyrag_b200 import synth
    dim = 768
    c = synth.make_dense_corpus(3000, dim, 11)
    c[5] = 0                                                    # zero row
    c[6] = 0.001
    c[6, 17] = 0.999                                            # one dominant coordinate
    idx = make_index(c)
    r, scale, e, n = np_quantize(c.float().numpy())
    assert np.array_equal(idx.rows_s8.cpu().numpy(), r)
    assert idx.row_scale.cpu().numpy().tobytes() == scale.tobytes()
    for got, ref in ((idx.row_err, e), (idx.row_norm, n)):
        g = got.cpu().numpy().astype(np.float64)
        assert (g >= ref * (1 - 2.0 ** -40)).all()             # fp64 sums in another order: 2^-40 slack
        ulp = np.spacing(got.cpu().numpy()).astype(np.float64)
        assert (g - ref <= ulp).all()
    mx = idx.maxima.cpu().numpy()
    assert mx[0] == idx.row_err.max().item() and mx[1] == idx.row_norm.max().item()


@pytest.mark.parametrize("dim", [128, 768, 1024])
def test_topk_bit_exact(lib_built, dim):
    from easyrag_b200 import synth
    c = synth.make_dense_corpus(40_000, dim, 21 + dim).to(DEV)
    q = synth.make_dense_queries(c, 150, 22 + dim)
    idx = make_index(c)
    ref = rescore_all(q, c)
    for k in list(range(1, 18)) + [288]:
        ids, sc, counts = canonical_topk(ref, k)
        out, cc = run_s8(idx, q, k)
        assert_same(out, ids, sc, counts, f"dim={dim} k={k}")
        out, cc = run_certified(idx, q, k)
        assert_same(out, ids, sc, counts, f"dim={dim} k={k}, int8 pass + rescoring")
        if k <= 16:
            assert (cc >= k).all()


def test_filters_and_id_base(lib_built):
    from easyrag_b200 import synth
    n, dim = 30_000, 768
    c = synth.make_dense_corpus(n, dim, 31).to(DEV)
    q = synth.make_dense_queries(c, 130, 32)
    g = torch.Generator().manual_seed(33)
    dg = torch.randint(0, 4, (n,), generator=g, dtype=torch.int32)
    qg = torch.randint(-1, 4, (130,), generator=g, dtype=torch.int32)
    qg[0] = 7                                                   # matches no row
    idx = make_index(c, doc_group=dg)
    base = 2 ** 31 - 1 - n
    ref = rescore_all(q, c)
    allowed = (qg.to(DEV)[:, None] == -1) | (dg.to(DEV)[None, :] == qg.to(DEV)[:, None])
    for k in (1, 10, 16, 17, 288):
        ids, sc, counts = canonical_topk(ref, k, allowed, id_base=base)
        for run in (run_s8, run_certified):
            out, _ = run(idx, q, k, q_group=qg, id_base=base)
            assert_same(out, ids, sc, counts, f"k={k} {run.__name__}")
            assert int(out.counts[0]) == 0


def test_ties_zero_query_negative_scores(lib_built):
    from easyrag_b200 import synth
    n, dim = 50_000, 256
    c = synth.make_dense_corpus(n, dim, 41)
    c[::997] = c[3]                                             # one row repeated across every split
    c = c.to(DEV)
    q = synth.make_dense_queries(c, 70, 42)
    q[0] = c[3]                                                 # ties among all the copies
    q[1] = 0                                                    # all-zero query: every score is 0
    cpos = c.abs().to(torch.bfloat16)                           # all-negative scores against -|q|
    q_neg = -q.abs()
    q_neg[1] = 0
    for corpus, queries in ((c, q), (cpos, q_neg)):
        idx = make_index(corpus)
        ref = rescore_all(queries, corpus)
        for k in (1, 10, 16, 40):
            ids, sc, counts = canonical_topk(ref, k)
            for run in (run_s8, run_certified):
                out, _ = run(idx, queries, k)
                assert_same(out, ids, sc, counts, f"k={k} {run.__name__}")
    assert (ref[2:] < 0).all()


def test_constructed_worst_case(lib_built):
    """The negative-control corpus of test_dense_s8_bound_cpu.py: the answer row's s^ sits nearly 2 D_q below the
    top s^; the kernel keeps it and returns it."""
    from test_dense_s8_bound_cpu import constructed_case
    q, c = constructed_case()
    qd = torch.from_numpy(q).to(DEV, torch.bfloat16)
    cd = torch.from_numpy(c).to(DEV, torch.bfloat16)
    idx = make_index(cd)
    ids, sc, counts = canonical_topk(rescore_all(qd, cd), 1)
    assert int(ids[0, 0]) == 0
    out, cc = run_certified(idx, qd, 1)
    assert_same(out, ids, sc, counts, "constructed case")
    assert int(cc[0]) == 2


@pytest.mark.parametrize("k", [10, 16])
def test_capacity_does_not_change_results(lib_built, k):
    from easyrag_b200 import synth
    c = synth.make_dense_corpus(60_000, 768, 51).to(DEV)
    q = synth.make_dense_queries(c, 200, 52)
    idx = make_index(c)
    ref = rescore_all(q, c)
    ids, sc, counts = canonical_topk(ref, k)
    out, cc = run_certified(idx, q, k)                         # every query through the int8 pass + rescoring
    assert_same(out, ids, sc, counts, "capacity = rows")
    print(f"[s8] k={k}: candidates per query mean {cc.float().mean().item():.1f} max {int(cc.max())}")
    out1, cc1 = run_s8(idx, q, k, cap=1)
    assert (cc1 > 1).all()                                      # every query overflowed and took the full scan
    assert_same(out1, ids, sc, counts, "capacity 1")
    out_d, _ = run_s8(idx, q, k)
    assert_same(out_d, ids, sc, counts, "default capacity")


def test_scale_1m(lib_built):
    from easyrag_b200 import synth
    c = synth.make_dense_corpus(1_000_000, 768, 61, device=DEV)
    q = synth.make_dense_queries(c, 1000, 62)
    idx = make_index(c)
    ref = rescore_all(q, c, q_chunk=32)
    for k in (10, 16):
        ids, sc, counts = canonical_topk(ref, k)
        out, cc = run_certified(idx, q, k)                     # many work units per CTA, shared bound across them
        assert_same(out, ids, sc, counts, f"1M x 768 k={k}, int8 pass + rescoring")
        print(f"[s8] 1M x 768, 1000 queries, k={k}: candidates mean {cc.float().mean().item():.1f} "
              f"max {int(cc.max())}")
        out, _ = run_s8(idx, q, k, cap=1)
        assert_same(out, ids, sc, counts, f"1M x 768 k={k}, full scan")


def test_mirror_maintenance(lib_built, tmp_path):
    from easyrag_b200 import synth
    from easyrag_b200.index import DenseIndex
    n, dim = 20_000, 512
    c = synth.make_dense_corpus(n, dim, 71).to(DEV)
    q = synth.make_dense_queries(c, 64, 72)
    whole = make_index(c)
    ids, sc, counts = canonical_topk(rescore_all(q, c), 10)
    out, _ = run_certified(whole, q, 10)
    assert_same(out, ids, sc, counts, "built in one go")
    mirror = lambda ix: (ix.rows_s8, ix.row_scale, ix.row_err, ix.row_norm, ix.maxima)
    # append + in-place commit after a search
    grown = DenseIndex(c[:5000], device=DEV, quantized=True)
    run_certified(grown, q, 10)
    grown.append(c[5000:12000])
    dst = grown.rows_for_append(n - 12000)
    dst.copy_(c[12000:])
    grown.commit(n - 12000)
    assert all(torch.equal(a, b) for a, b in zip(mirror(grown), mirror(whole)))
    out, _ = run_certified(grown, q, 10)
    assert_same(out, ids, sc, counts, "append / commit")
    # save / load round trip keeps the mirror
    whole.save(str(tmp_path / "q"))
    loaded = DenseIndex.load(str(tmp_path / "q"), device=DEV)
    assert loaded.quantized and all(torch.equal(a, b) for a, b in zip(mirror(loaded), mirror(whole)))
    out, _ = run_certified(loaded, q, 10)
    assert_same(out, ids, sc, counts, "save / load")
    # a directory saved without the mirror loads as a bf16 index
    DenseIndex(c, device=DEV).save(str(tmp_path / "b"))
    plain = DenseIndex.load(str(tmp_path / "b"), device=DEV)
    assert not plain.quantized
    with pytest.raises(ValueError):
        DenseIndex(None, device=DEV, dim=700, quantized=True)
    with pytest.raises(ValueError):
        DenseIndex(None, device=DEV, quantized=True)


def test_vector_store_and_hybrid(lib_built):
    import asyncio
    from easyrag_b200 import batched, synth
    from easyrag_b200.index import Bm25Index, Bm25Stats
    from easyrag_b200.retrievers import B200VectorStore, QdrantRetriever
    from easyrag_b200.schema import BaseEmbedding, QueryBundle, TextNode, build_qdrant_filters
    from oracle import bm25 as obm, retrieve as ort

    n, dim = 3000, 256
    dirs = ["d0", "d1", "d2"]
    c = synth.make_dense_corpus(n, dim, 81)
    nodes = [TextNode(text=f"doc {i}", id_=f"node-{i}", metadata={"dir": dirs[i % 3]},
                      embedding=c[i].float().tolist()) for i in range(n)]
    store = B200VectorStore(nodes, device=DEV, quantize=True)
    assert store.index.quantized
    qv = synth.make_dense_queries(c, 4, 82)

    class Emb(BaseEmbedding):
        def __init__(self, vecs):
            super().__init__(model_name="fixed", embed_batch_size=8)
            self._vecs = vecs

        def _get_query_embedding(self, query):
            return self._vecs[int(query)]

        _get_text_embedding = _get_query_embedding

    vecs = [qv[i].float().tolist() for i in range(4)]
    stored = store.index.vectors
    for i in range(4):
        qn = torch.nn.functional.normalize(torch.tensor([vecs[i]], device=DEV), dim=1).to(torch.bfloat16)
        ref = rescore_all(qn, stored)
        for filt in (None, "d1"):
            r = QdrantRetriever(store, Emb(vecs), similarity_top_k=7)
            r.filters = build_qdrant_filters(filt) if filt else None
            allowed = None
            if filt:
                allowed = torch.tensor([i % 3 == 1 for i in range(n)], device=DEV)[None, :]
            got = asyncio.run(r.aretrieve(QueryBundle(str(i))))
            ids, sc, counts = canonical_topk(ref, 7, allowed)
            assert [int(g.node.node_id.split("-")[1]) for g in got] == ids[0, :int(counts[0])].tolist()
            assert [g.score for g in got] == sc[0, :int(counts[0])].tolist()

    # CoarseRanker.hybrid on a quantized index = RRF of the definition's dense lists and the BM25 lists
    vocab, nq, k = 2000, 48, 10
    corpus = synth.make_sparse_corpus(n, vocab, 83)
    queries = synth.make_queries(corpus, nq, 84)
    cd = c.to(DEV)
    qd = synth.make_dense_queries(cd, nq, 85)
    ranker = batched.CoarseRanker(make_index(cd),
                                  Bm25Index(Bm25Stats.from_tokens(corpus.tokens, corpus.doc_ptr, vocab), device=DEV))
    fused, sparse, dense = ranker.hybrid(qd, queries.term_ptr.to(DEV), queries.terms.to(DEV), k, k, k)
    torch.cuda.synchronize()
    d_ids, d_sc, d_cnt = canonical_topk(rescore_all(qd, cd), k)
    assert_same(dense, d_ids, d_sc, d_cnt, "hybrid dense route")
    oracle = obm.OkapiCSR(corpus.doc_lists(), vocab)
    f_ids, f_sc = fused.ids.cpu().numpy(), fused.scores.cpu().numpy()
    for i, terms in enumerate(queries.term_lists()):
        s_ref, _ = ort.bm25_topk_ids(oracle.get_scores([int(t) for t in terms]), k)
        r_ids, r_sc = ort.rrf_ids([s_ref, d_ids[i].cpu().numpy()], None, K=60, topk=k)
        assert np.array_equal(f_ids[i, :r_ids.size], r_ids) and f_sc[i, :r_ids.size].tobytes() == r_sc.tobytes()
