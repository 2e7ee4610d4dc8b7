"""GPU: the candidate form of dense top-k (csrc/dense_cand.cu, ``ezr_dense_cand_topk`` / ``batched.dense_topk_cand``).

The candidate form computes the same fp32 scores as form 6 (one accumulator chain per score, same k16 order) and
returns the canonical top-k of them, so every case compares against form 6 on the same inputs: counts and ids in full,
score bytes wherever a result is listed.  On integer vectors (exact in fp32) it is also checked against the fp64
canonical top-k of tests/_topk_ref.py.  ``cand_counts`` tells which queries the form-6 fallback answered (-1) and
which the candidate pass did (>= 0); the threshold cases assert which one ran.

1. Shapes: dims 64 / 768 / 1024 / 3584 / 4096, k from 1 to 1024, Q from 1 to 10 001 (several query blocks at 4096),
   n_rows of 1, k - 1, k and the chunk boundaries +- 1.
2. Exactness at the threshold: duplicates of the k-th row in the first and last chunks, mass ties that overflow, and
   scores that rise with the row index (every query overflows); capacities 1, k, the default and n_rows.
3. Filters, id_base near 2^31, row strides larger than dim, all-zero queries, all-negative scores, refusals, the
   empty corpus and the empty batch.
4. Scale: 1M x 768 x 10 000 queries at k 288 and 4M x 1024 x 64 queries at k 288, bit-identical to form 6.
5. The drop-in store (``dense_cand=True``) and ``pipeline_hybrid(dense_cand=True)`` over G = 1, 3, 8 simulated ranks.

What each case ran is printed (``pytest -s``).
"""
import asyncio
import time

import pytest
import torch

import _loopback
from _topk_ref import canonical_topk
from test_gpu_dense_wide import _TableEmbedding, _plus_minus_rows
from test_gpu_sharded import _assert_same, _clone
from test_gpu_sharded_deep import _rankers, _sharded
from easyrag_b200 import _lib, batched, synth
from easyrag_b200.index import Bm25Index, Bm25Stats, DenseIndex
from easyrag_b200.retrievers import B200VectorStore, QdrantRetriever
from easyrag_b200.schema import QueryBundle, TextNode, build_qdrant_filters

pytestmark = pytest.mark.gpu
DEV = "cuda"
EZR_ERR_WORKSPACE, EZR_ERR_UNSUPPORTED = -3, -4


@pytest.fixture(scope="module", autouse=True)
def _ready(lib_built):
    _lib.require_cuda()
    _lib.lib()


@pytest.fixture(autouse=True)
def _loop(monkeypatch):
    _loopback.install(monkeypatch)


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _ints(n, d, seed, lo=-2, hi=2):
    return torch.randint(lo, hi + 1, (n, d), generator=_gen(seed), device=DEV).to(torch.bfloat16)


def _report(what, info):
    print(f"\n[dense cand] {what}: " + ", ".join(f"{k}={v:.4g}" if isinstance(v, float) else f"{k}={v}"
                                               for k, v in info.items()))


def _raw(c, q, k, doc_group=None, q_group=None, id_base=0, cand=False, ws_bytes=None):
    """ezr_dense_cand_topk (cand) or form 6 of ezr_dense_topk on any (possibly strided) views, outputs poisoned first.
    -> (status, TopK, cand_counts)."""
    L = _lib.lib()
    n, d = c.shape
    nq = q.shape[0]
    out = batched.TopK(torch.full((nq, k), 7.0, device=DEV), torch.full((nq, k), 7, dtype=torch.int32, device=DEV),
                       torch.full((nq,), 7, dtype=torch.int32, device=DEV))
    cc = torch.full((nq,), 7, dtype=torch.int32, device=DEV)
    if ws_bytes is None:
        ws_bytes = (L.ezr_dense_cand_topk_workspace if cand else L.ezr_dense_topk_workspace)(n, d, nq, k)
    buf = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=DEV)
    args = (_lib.ptr(c), n, d, c.stride(0), _lib.ptr(q), nq, q.stride(0), k, _lib.ptr(doc_group), _lib.ptr(q_group),
            id_base, _lib.ptr(out.scores), _lib.ptr(out.ids), _lib.ptr(out.counts))
    if cand:
        rc = L.ezr_dense_cand_topk(*args, _lib.ptr(cc), _lib.ptr(buf), ws_bytes, _lib.stream_ptr())
    else:
        _lib.check(L.ezr_dense_set_kernel(6))
        try:
            rc = L.ezr_dense_topk(*args, _lib.ptr(buf), ws_bytes, _lib.stream_ptr())
        finally:
            L.ezr_dense_set_kernel(0)
    torch.cuda.synchronize()
    return rc, out, cc


def _both(c, q, k, **kw):
    """(candidate form, form 6, cand_counts) on the same inputs, both successful, compared."""
    rc, got, cc = _raw(c, q, k, cand=True, **kw)
    assert rc == 0, _lib.lib().ezr_last_error()
    rc, want, _ = _raw(c, q, k, **kw)
    assert rc == 0, _lib.lib().ezr_last_error()
    _assert_same(got, want, f"candidate form vs form 6, n={c.shape[0]} d={c.shape[1]} Q={q.shape[0]} k={k}")
    past = torch.arange(k, device=DEV)[None, :] >= got.counts[:, None].long()
    assert bool((got.ids[past] == -1).all()) and bool((got.scores[past] == float("-inf")).all())
    return got, want, cc


def _fp64(c, q, k, got, allowed=None, id_base=0):
    """The integer-vector result equals the fp64 canonical top-k (n >= k and every query has >= k allowed rows)."""
    sims = q.double() @ c.double().T
    top, s = canonical_topk(sims, k, allowed)
    assert torch.equal(got.ids.long(), top + id_base)
    assert torch.equal(got.scores.double(), s)


def _with_capacity(cap, fn):
    L = _lib.lib()
    _lib.check(L.ezr_dense_cand_set_capacity(cap))
    try:
        return fn()
    finally:
        L.ezr_dense_cand_set_capacity(0)


# ============================================================================ 1. shapes
@pytest.mark.parametrize("d", [64, 768, 1024, 3584, 4096])
def test_dims_and_depths(d):
    n, nq = 3000, 129
    c, q = _ints(n, d, 10 + d), _ints(nq, d, 20 + d)
    over = {}
    for k in (1, 16, 17, 192, 256, 288, 1023, 1024):
        got, _, cc = _both(c, q, k)
        _fp64(c, q, k, got)
        over[k] = int((cc < 0).sum())
    _report(f"dims d={d}", dict(overflowed_by_k=over))


@pytest.mark.parametrize("nq", [1, 127, 128, 129, 10_001])
def test_query_counts(nq):
    n, d, k = 2000, 768, 288
    c, q = _ints(n, d, 30), _ints(nq, d, 31 + nq)
    got, _, cc = _both(c, q, k)
    if nq <= 129:
        _fp64(c, q, k, got)
    _report(f"Q={nq}", dict(cand_mean=float(cc.float().mean()), overflowed=int((cc < 0).sum())))


def test_several_query_blocks():
    # dim 4096: query blocks of 2048 rows (16 MB of bf16), so 10 001 queries run in five blocks
    n, d, k = 1500, 4096, 16
    c, q = _ints(n, d, 40), _ints(10_001, d, 41)
    got, _, cc = _both(c, q, k)
    _fp64(c[:, :], q[:300], k, batched.TopK(got.scores[:300], got.ids[:300], got.counts[:300]))
    assert bool((cc >= 0).all())


@pytest.mark.parametrize("k", [1, 288, 1024])
def test_row_counts_and_chunk_boundaries(k):
    d, nq = 256, 64
    c0 = (k + 255) // 256 * 256
    edges = [c0, 3 * c0, 7 * c0]                                   # chunks of c0, 2 c0, 4 c0 rows
    ns = sorted({1, max(1, k - 1), k} | {e + o for e in edges for o in (-1, 0, 1)})
    for n in ns:
        c, q = _ints(n, d, 50 + n), _ints(nq, d, 51)
        got, _, cc = _both(c, q, k)
        assert bool((got.counts == min(n, k)).all())
        if n >= k:
            _fp64(c, q, k, got)
    _report(f"row counts k={k}", dict(n=ns))


# ============================================================================ 2. the threshold
def _axis_rows(values, d):
    """rows whose only nonzero is values[i] in dimension 0 (every score = values[i] * q[0])"""
    x = torch.zeros(len(values), d, device=DEV)
    x[:, 0] = torch.as_tensor(values, dtype=torch.float32, device=DEV)
    return x.to(torch.bfloat16)


def test_tied_kth_row_in_first_and_last_chunk():
    n, d, k = 20_000, 128, 288
    vals = torch.full((n,), -1.0)
    vals[10:10 + k - 1] = 3.0                                      # k - 1 rows above the k-th
    vals[5] = vals[n - 1] = 2.0                                    # the k-th row, in the first and the last chunk
    c = _axis_rows(vals, d)
    q = torch.zeros(4, d, device=DEV, dtype=torch.bfloat16)
    q[:, 0] = 1.0
    got, _, cc = _both(c, q, k)
    assert bool((cc >= 0).all()), "the tie must not need the fallback"
    assert bool((got.ids[:, k - 1] == n - 1).all()) and not bool((got.ids == 5).any())
    _fp64(c, q, k, got)


def test_mass_ties_overflow():
    n, d, k = 20_000, 128, 288
    c = _axis_rows(torch.ones(n), d)                               # every row ties
    q = torch.zeros(3, d, device=DEV, dtype=torch.bfloat16)
    q[:, 0] = torch.tensor([1.0, 0.5, -2.0])
    got, _, cc = _both(c, q, k)
    assert bool((cc == -1).all()), f"mass ties must overflow: {cc.tolist()}"
    assert got.ids[0].tolist() == list(range(n - 1, n - 1 - k, -1))


def test_rising_scores_every_query_overflows():
    # score of row i = i exactly: rows (i // 256, i % 256), queries (256, 1, noise in dims the rows leave zero)
    n, d, k = 30_000, 128, 192
    i = torch.arange(n, device=DEV)
    c = torch.zeros(n, d, device=DEV)
    c[:, 0], c[:, 1] = (i // 256).float(), (i % 256).float()
    c = c.to(torch.bfloat16)
    q = _ints(5, d, 60).float()
    q[:, 0], q[:, 1] = 256.0, 1.0
    q = q.to(torch.bfloat16)
    got, _, cc = _both(c, q, k)
    assert bool((cc == -1).all())
    assert got.ids[0].tolist() == list(range(n - 1, n - 1 - k, -1))
    got, _, cc = _with_capacity(n, lambda: _both(c, q, k))        # a buffer of n slots never overflows
    assert bool((cc >= 0).all())


def test_capacity_never_changes_the_result():
    n, d, k, nq = 20_000, 256, 288, 129
    c, q = _ints(n, d, 70, -1, 1), _ints(nq, d, 71)
    base, _, cc0 = _both(c, q, k)
    seen = {}
    for cap in (1, k, 0, n):
        got, _, cc = _with_capacity(cap, lambda: _both(c, q, k))
        _assert_same(got, base, f"capacity {cap}", full_scores=True)
        seen[cap] = int((cc < 0).sum())
    assert seen[1] == nq and seen[n] == 0
    _fp64(c, q, k, base)
    _report("capacities", dict(overflowed=seen))


# ============================================================================ 3. filters, edges, refusals
def test_filters_and_id_base():
    n, d, k = 20_000, 256, 288
    c, q = _ints(n, d, 80), _ints(8, d, 81)
    g = torch.randint(0, 4, (n,), generator=_gen(82), device=DEV, dtype=torch.int32)
    g[5000:5100] = 7                                               # class 7: 100 rows (fewer than k)
    qg = torch.tensor([-1, 0, 7, 9, 3, -1, 7, 2], dtype=torch.int32, device=DEV)
    for base in (0, 2 ** 31 - n - 1):
        got, _, cc = _both(c, q, k, doc_group=g, q_group=qg, id_base=base)
        assert got.counts.tolist() == [k, k, 100, 0, k, k, 100, k]
        assert int(cc[3]) == 0
        full = [i for i in range(8) if int(got.counts[i]) == k]
        allowed = (qg[:, None] == -1) | (qg[:, None] == g[None, :])
        _fp64(c, q[full], k, batched.TopK(got.scores[full], got.ids[full], got.counts[full]), allowed[full], base)


def test_row_strides_larger_than_dim():
    n, d, k = 5000, 768, 288
    c = _ints(n, 832, 90)[:, :d]
    q = _ints(33, 896, 91)[:, :d]
    got, _, _ = _both(c, q, k)
    _fp64(c, q, k, got)


def test_zero_queries_and_negative_scores():
    n, d, k = 4000, 256, 288
    c = _ints(n, d, 100, 1, 2)                                     # positive rows
    q = torch.cat([torch.zeros(2, d, device=DEV), -_ints(3, d, 101, 1, 2).float()]).to(torch.bfloat16)
    got, _, cc = _both(c, q, k)
    assert bool((got.scores[:2] == 0).all()) and not bool(torch.signbit(got.scores[:2]).any())   # +0.0
    assert bool((got.scores[2:] < 0).all())
    assert got.ids[0].tolist() == list(range(n - 1, n - 1 - k, -1))
    _fp64(c, q, k, got)


def test_refusals():
    L = _lib.lib()
    n, k = 1000, 10
    assert _raw(_ints(n, 96, 110), _ints(4, 96, 111), k, cand=True)[0] == EZR_ERR_UNSUPPORTED
    assert b"dim % 64" in L.ezr_last_error()
    assert _raw(_ints(n, 772, 112)[:, :768], _ints(4, 768, 113), k, cand=True)[0] == EZR_ERR_UNSUPPORTED
    assert _raw(_ints(n, 768, 114), _ints(4, 772, 115)[:, :768], k, cand=True)[0] == EZR_ERR_UNSUPPORTED
    flat = _ints(1, n * 768 + 8, 116)[0]
    assert _raw(flat[4:4 + n * 768].view(n, 768), _ints(4, 768, 117), k, cand=True)[0] == EZR_ERR_UNSUPPORTED
    need = L.ezr_dense_cand_topk_workspace(n, 768, 4, k)
    assert _raw(_ints(n, 768, 118), _ints(4, 768, 119), k, cand=True, ws_bytes=need - 1)[0] == EZR_ERR_WORKSPACE
    idx = DenseIndex(_ints(n, 768, 120), device=DEV)
    with pytest.raises(_lib.EzrError, match="workspace|unsupported"):
        batched.dense_topk_cand(DenseIndex(_ints(n, 96, 121), device=DEV), _ints(4, 96, 122), k)
    with pytest.raises(ValueError, match="cand_counts"):
        batched.dense_topk_cand(idx, _ints(4, 768, 123), k, cand_counts=torch.zeros(3, dtype=torch.int32, device=DEV))


def test_empty_corpus_and_empty_batch():
    k = 288
    rc, out, cc = _raw(torch.empty(0, 256, dtype=torch.bfloat16, device=DEV), _ints(5, 256, 130), k, cand=True,
                       ws_bytes=0)
    assert rc == 0 and out.counts.tolist() == [0] * 5 and bool((out.ids == -1).all()) and cc.tolist() == [0] * 5
    rc, out, cc = _raw(_ints(100, 256, 131), torch.empty(0, 256, dtype=torch.bfloat16, device=DEV), k, cand=True,
                       ws_bytes=0)
    assert rc == 0
    idx = DenseIndex(None, device=DEV, dim=256)
    res = batched.dense_topk_cand(idx, _ints(3, 256, 132), k)
    assert res.counts.tolist() == [0, 0, 0]


# ============================================================================ 4. scale
def _scale_case(n, d, nq, k, seed):
    t0 = time.perf_counter()
    c = synth.make_dense_corpus(n, d, seed, device=DEV)
    q = synth.make_dense_queries(c, nq, seed + 1)
    index = DenseIndex(c, device=DEV)
    cc = torch.empty(nq, dtype=torch.int32, device=DEV)
    got = _clone(batched.dense_topk_cand(index, q, k, cand_counts=cc))
    want = batched.dense_topk(index, q, k, form=6)
    torch.cuda.synchronize()
    _assert_same(got, want, f"scale {n} x {d} x {nq} k={k}")
    assert bool((got.counts == k).all())
    _report(f"scale {n} x {d}, Q={nq}, k={k}", dict(cand_mean=float(cc.float().mean()), cand_max=int(cc.max()),
                                                  overflowed=int((cc < 0).sum()), seconds=time.perf_counter() - t0))


def test_scale_1m_768_10k_queries():
    _scale_case(1_000_000, 768, 10_000, 288, 140)


def test_scale_configs4_shape():
    _scale_case(4_000_000, 1024, 64, 288, 150)


# ============================================================================ 5. store and sharded pipeline
def test_vector_store_dense_cand_matches_form_6():
    n, d, k, dirs = 3000, 256, 288, ["director", "emsplus", "rcp", "umac"]
    emb = _plus_minus_rows(n, d, 16, 900)
    g = torch.Generator().manual_seed(901)
    nodes = [TextNode(text=f"chunk {i}", id_=f"node-{i}", metadata={"dir": dirs[int(torch.randint(4, (1,), generator=g))]},
                      embedding=emb[i].tolist()) for i in range(n)]
    queries = _TableEmbedding(_plus_minus_rows(8, d, 16, 902))
    wide, cand = B200VectorStore(nodes, dense_form=6), B200VectorStore(nodes, dense_cand=True)
    for qi in range(8):
        lists = []
        for store in (wide, cand):
            r = QdrantRetriever(store, queries, similarity_top_k=k)
            r.filters = build_qdrant_filters(dirs[qi % 4]) if qi % 2 else None
            lists.append([(x.node.node_id, x.score) for x in asyncio.run(r.aretrieve(QueryBundle(str(qi))))])
        assert lists[0] == lists[1]
        assert len(lists[0]) == (k if qi % 2 == 0 else min(k, sum(nd.metadata["dir"] == dirs[qi % 4] for nd in nodes)))


def test_pipeline_hybrid_dense_cand_sharded():
    # bench_sharded_deep's shapes scaled down: 200k x 768, 20k vocabulary, 512 queries, 288 / 192 / 256
    t0 = time.perf_counter()
    n, vocab, d, nq = 200_000, 20_000, 768, 512
    corpus = synth.make_sparse_corpus(n, vocab, 160, device=DEV)
    qs = synth.make_queries(corpus, nq, 161)
    stats = Bm25Stats.from_tokens(corpus.tokens, corpus.doc_ptr, vocab)
    del corpus
    vec = synth.make_dense_corpus(n, d, 162, device=DEV)
    qv = synth.make_dense_queries(vec, nq, 163).contiguous()
    qp, qt = qs.term_ptr.to(DEV), qs.terms.to(DEV)
    groups = synth.make_groups(n, 4, 164, device=DEV)
    qg = torch.tensor([(-1, 0, 2, 3)[i % 4] for i in range(nq)], dtype=torch.int32, device=DEV)
    kd, ks, ko = 288, 192, 256
    dense_full = DenseIndex(vec, device=DEV, doc_group=groups)
    sparse_full = Bm25Index(stats, device=DEV, doc_group=groups)
    info = {}
    for q_group in (None, qg):
        d = _clone(batched.dense_topk_cand(dense_full, qv, kd, q_group=q_group))
        d6 = batched.dense_topk(dense_full, qv, kd, q_group=q_group, form=6)
        _assert_same(d, d6, "unsharded candidate form vs form 6")
        s = batched.bm25_topk(sparse_full, qp, qt, ks, q_group=q_group)
        w = max(kd, ks)
        pad = lambda ids: torch.nn.functional.pad(ids, (0, w - ids.shape[1]), value=-1)
        f = batched.fuse_lists([pad(s.ids), pad(d.ids)], [s.counts, d.counts], ko, rrf=True, K=60)
        torch.cuda.synchronize()
        want = (_clone(f), _clone(s), d)
        for world, align in ((1, 1), (3, 1), (8, 64)):
            t1 = time.perf_counter()
            rankers = _rankers(vec, stats, groups, None, world, align)
            call = dict(queries=qv, q_ptr=qp, q_terms=qt, k_dense=kd, k_sparse=ks, k_out=ko, q_group=q_group,
                        dense_cand=True)
            got = _sharded(rankers, [call])[0]
            del rankers
            for name, a, b in zip(("fused", "sparse", "dense"), got, want):
                _assert_same(a, b, f"G={world} filtered={q_group is not None} {name}", full_scores=name == "fused")
            _assert_same(got[2], d6, f"G={world} dense vs form 6")
            info[f"G{world}_{'f' if q_group is not None else 'u'}_s"] = time.perf_counter() - t1
    info["seconds"] = time.perf_counter() - t0
    _report("pipeline_hybrid(dense_cand=True)", info)
