"""GPU: BM25 top-k on bm25s (float32) indexes with packed postings (``Bm25Index(stats, packed=True)``), which run the
two-phase path (csrc/bm25_pk.cuh: integer candidate pass, float32 bracket with slack e(m), exact float32 rescoring)
for 1 <= k <= 1024.  Every result must equal, byte for byte, the ordered kernel's on the same arrays
(``ordered_view()``) and the canonical top-k of the float32 reference rows of tests/_bm25_ref.py (``bm25s_row``).

The main corpus is test_gpu_bm25_scale.py's (bench.py's 1M documents and 200k vocabulary, 123 ranges of 8192, with
3000 copies of D spread over every range and 600 copies of E inside one range), with bm25s statistics, so the range
chunks, the bound steps, both overflow routes and the token limits all run.  What each case ran is printed
(``pytest -s``).
"""
import time

import numpy as np
import pytest
import torch

import _loopback
from _bm25_ref import bm25s_row, bm25s_weights
from test_gpu_bm25_scale import (DEFAULT_PLAN, DEFAULT_SKIP, DEFAULT_SPAN, N_DOCS, SEED, VOCAB, _assert_topk, _chunks,
                                 _pack, _ref_topk, _term_of)
from test_gpu_bm25_scale import corp  # noqa: F401  (module fixture: the 1M-document corpus)
from test_gpu_dropin import DIRS
from test_gpu_dropin import world  # noqa: F401  (module fixture: nodes, tokenizer and queries of the drop-in tests)
from test_gpu_sharded import _assert_same, _clone
from test_gpu_sharded_deep import _compare, _sharded, _unsharded
from test_gpu_sharded_deep import mid  # noqa: F401  (module fixture: 60k documents with ties across shards)
from easyrag_b200 import _lib, batched, synth
from easyrag_b200 import dist as ezdist
from easyrag_b200.index import Bm25Index, Bm25Stats, DenseIndex
from easyrag_b200.retrievers import BM25Retriever

pytestmark = pytest.mark.gpu
DEV = "cuda"
KS = (1, 10, 32, 33, 192, 288, 1023, 1024)
WBITS, KPK_MAX_TERMS = 19, 4096           # csrc/bm25_pk.cuh for 8192-document ranges


@pytest.fixture(scope="module", autouse=True)
def _ready(lib_built):
    _lib.require_cuda()


@pytest.fixture(autouse=True)
def _loop(monkeypatch):
    _loopback.install(monkeypatch)


def _report(what, info):
    info = dict(info, peak_gb=torch.cuda.max_memory_allocated() / 2 ** 30)
    print(f"\n[bm25s-packed] {what}: " + ", ".join(f"{k}={v:.4g}" if isinstance(v, float) else f"{k}={v}"
                                                 for k, v in info.items()))


def _bm25s_stats(st, n_docs):
    """bm25s statistics over the counted postings of ``st`` (its idf does not depend on the first-seen order)."""
    return Bm25Stats.from_counts(n_docs, st.vocab, int(st.doc_len.long().sum()), st.doc_len, st.df, st.indptr,
                                 st.post_doc, st.post_tf, np.zeros(st.vocab, np.uint64), bm25_type=1)


def _ref_weights(st1):
    """float32 bm25s weight of every posting of ``st1`` from tests/_bm25_ref.py."""
    idf32 = torch.from_numpy(st1.idf.astype(np.float32)).to(DEV)
    n = int(st1.post_doc.numel())
    w32 = torch.empty(n, dtype=torch.float32, device=DEV)
    for s, e in _chunks(n):
        w32[s:e] = bm25s_weights(st1.post_tf[s:e], st1.doc_len[st1.post_doc[s:e].long()],
                                 idf32[_term_of(st1.indptr, s, e)], st1.avgdl)
    return w32


def _rows_fn(w32, st1, n_docs):
    ih, df = st1.indptr.cpu().numpy(), st1.df.cpu().numpy()
    return lambda c, qidx: torch.stack([bm25s_row(c["lists"][i], ih, st1.post_doc, w32, df, n_docs) for i in qidx])


def _check_pack(ix):
    """The packed words and term maxima against their definition (ezr_bm25_pack_f32)."""
    wmax = float(ix.post_w.max())
    _, ex = np.frexp(wmax)
    assert ix.pk_scale_log2 == WBITS - 1 - int(ex)
    mask = (1 << WBITS) - 1
    tmax = torch.zeros(ix.vocab, dtype=torch.int64, device=DEV)
    for s, e in _chunks(ix.n_postings):
        w = ix.post_w[s:e].double()                                    # widening is exact
        wq = torch.ceil(w * 2.0 ** ix.pk_scale_log2).long()
        assert int(wq.max()) <= 1 << (WBITS - 1) and bool((wq[w > 0] >= 1).all())
        pk = ix.post_pk[s:e].long() & 0xffffffff
        assert torch.equal(pk >> WBITS, (ix.post_doc[s:e] % 8192).long())
        assert torch.equal(pk & mask, wq)
        tmax.scatter_reduce_(0, _term_of(ix.indptr, s, e), wq, reduce="amax")
    assert torch.equal(ix.term_max.long(), tmax)


def _overflowed(ws, nq, k, n_ranges):
    """Queries the two-phase path handed on, read from the call's workspace (``ovf_n`` / ``ovf_list`` of ``pk_carve``
    in csrc/bm25.cu: after the k <= 32 path's float32 candidate scores and ids, at offset 0 in the deep form)."""
    align = lambda x: (x + 255) // 256 * 256
    n = nq * n_ranges * k
    base = align(n * 4) + align(n * 4) if k <= 32 else 0
    buf = ws.buf
    n_ovf = int(buf[base + 24 * nq:base + 24 * nq + 4].view(torch.int32))
    assert 0 <= n_ovf <= nq, f"k={k}: {n_ovf} overflowed queries of {nq}: the workspace layout changed"
    lst = buf[base + align((6 * nq + 1) * 4):].narrow(0, 0, 4 * n_ovf).view(torch.int32).tolist()
    assert len(set(lst)) == n_ovf and all(0 <= q < nq for q in lst), f"k={k}: overflow list {lst}"
    return sorted(lst)


def _profiled(fn):
    """-> (result, candidate launches, rescoring launches) of one call."""
    L = _lib.lib()
    L.ezr_profile_enable(1)
    try:
        L.ezr_profile_reset()
        r = fn()
        torch.cuda.synchronize()
        return r, _lib.profile_read("bm25_cand")[1], _lib.profile_read("bm25_rescore")[1]
    finally:
        L.ezr_profile_enable(0)


# --------------------------------------------------------------------------------------------- the 1M corpus
@pytest.fixture(scope="module")
def bs(corp):
    t0 = time.perf_counter()
    st1 = _bm25s_stats(corp["stats"], N_DOCS)
    ix = Bm25Index(st1, device=DEV, doc_group=corp["groups"], packed=True)
    assert ix.post_w.dtype == torch.float32 and ix.post_pk is not None and ix.term_max is not None
    w32 = _ref_weights(st1)
    assert torch.equal(ix.post_w.view(torch.int32), w32.view(torch.int32))
    present = np.nonzero(st1.df.cpu().numpy())[0]
    rng = np.random.default_rng(12)
    lists = list(corp["lists"])
    names = dict(corp["names"])
    for nm, q in dict(at4096=[int(t) for t in rng.choice(present, KPK_MAX_TERMS)],
                      past4097=[int(t) for t in rng.choice(present, KPK_MAX_TERMS + 1)],
                      dup_oov=[int(present[3])] * 20 + [-7, VOCAB + 1] + [int(present[3])] * 5).items():
        names[nm] = len(lists)
        lists.append(q)
    qp, qt = _pack(lists)
    out = dict(stats=st1, index=ix, ordered=ix.ordered_view(), w32=w32, lists=lists, names=names, qp=qp, qt=qt,
               groups=corp["groups"], cache={})
    out["rows_fn"] = _rows_fn(w32, st1, N_DOCS)
    _report("bm25s index", dict(queries=len(lists), index_gb=ix.index_bytes() / 2 ** 30,
                                pk_scale_log2=ix.pk_scale_log2, seconds=time.perf_counter() - t0))
    return out


def _ref1024(bs):
    if "ref" not in bs["cache"]:
        bs["cache"]["ref"] = _ref_topk(bs, list(range(len(bs["lists"]))), 1024, rows_fn=bs["rows_fn"])
    return bs["cache"]["ref"]


def test_packed_words_match_definition(bs):
    _check_pack(bs["index"])


def test_topk_bit_exact_at_every_depth(bs):
    t0 = time.perf_counter()
    ref = _ref1024(bs)
    info = {}
    for k in KS:
        a, n_cand, n_rs = _profiled(lambda: batched.bm25_topk(bs["index"], bs["qp"], bs["qt"], k))
        assert n_cand >= 1 and n_rs == 1, f"k={k}: the two-phase path did not run ({n_cand}, {n_rs})"
        _assert_topk(a, ref, k, f"packed bm25s k={k}", bs)
        b, n_cand_o, _ = _profiled(lambda: batched.bm25_topk(bs["ordered"], bs["qp"], bs["qt"], k))
        assert n_cand_o == 0
        _assert_same(a, b, f"packed vs ordered k={k}")
        info[f"cand_launches_k{k}"] = n_cand
    _report("top-k at every depth", dict(queries=len(bs["lists"]), **info, seconds=time.perf_counter() - t0))


def test_overflow_routes_and_token_limits(bs):
    ref = _ref1024(bs)
    nm, nq, ix = bs["names"], len(bs["lists"]), bs["index"]
    rows = bs["rows_fn"](bs, [nm["tieD"], nm["tieE"]])
    n_tie = (rows == rows.max(1, keepdim=True).values).sum(1).tolist()
    assert n_tie[0] > 4 * 192 + 1024 and n_tie[1] == 600 > 512     # past the query lists / one CTA's list (k <= 32)
    del rows
    info = {}
    for k in (10, 192):
        ws = batched.Workspace(DEV)
        r = batched.bm25_topk(ix, bs["qp"], bs["qt"], k, ws=ws)
        torch.cuda.synchronize()
        ovf = _overflowed(ws, nq, k, ix.n_ranges)
        names = sorted(n for n, j in nm.items() if j in ovf)
        for must in ("tieD", "huge4200", "past4097") + (("tieE",) if k == 10 else ()):
            assert nm[must] in ovf, f"k={k}: {must} not handed on ({names})"
        _assert_topk(r, ref, k, f"overflow k={k}", bs)
        info[f"overflowed_k{k}"] = names + [f"{len(ovf) - len(names)} others"]
    _report("overflow", info)


def test_filters_and_id_base(bs):
    nq = len(bs["lists"])
    pattern = torch.tensor([-1, 0, 1, 2, 3, 9], dtype=torch.int32, device=DEV)
    want = pattern[torch.arange(nq, device=DEV) % pattern.numel()]
    base = 2 ** 31 - 1 - N_DOCS
    ref = _ref_topk(bs, list(range(nq)), 192, want=want, rows_fn=bs["rows_fn"])
    for k in (10, 192):
        r = batched.bm25_topk(bs["index"], bs["qp"], bs["qt"], k, q_group=want, id_base=base)
        _assert_topk(r, ref, k, f"filtered k={k}", bs, id_base=base)
        assert (r.counts[want == 9] == 0).all()
        o = batched.bm25_topk(bs["ordered"], bs["qp"], bs["qt"], k, q_group=want, id_base=base)
        _assert_same(r, o, f"ordered view, filtered k={k}")


def test_switch_matrix(bs):
    t0 = time.perf_counter()
    L = _lib.lib()
    ref = _ref1024(bs)
    ix, qp, qt = bs["index"], bs["qp"], bs["qt"]
    base = {k: batched.bm25_topk(ix, qp, qt, k) for k in (10, 192)}
    n = 0
    try:
        for plan in (0, 1):
            for skip in (0, 1):
                for span in (1, 4, 8, 32):
                    _lib.check(L.ezr_bm25_set_plan(plan))
                    _lib.check(L.ezr_bm25_set_skipping(skip))
                    _lib.check(L.ezr_bm25_set_span(span))
                    for k in (10, 192):
                        r = batched.bm25_topk(ix, qp, qt, k)
                        what = f"plan={plan} skip={skip} span={span} k={k}"
                        _assert_topk(r, ref, k, what, bs)
                        _assert_same(r, base[k], what)
                        n += 1
    finally:
        L.ezr_bm25_set_plan(DEFAULT_PLAN)
        L.ezr_bm25_set_skipping(DEFAULT_SKIP)
        L.ezr_bm25_set_span(DEFAULT_SPAN)
    _report("switch matrix", dict(runs=n, seconds=time.perf_counter() - t0))


def test_batch_of_10k_queries(bs, corp):
    """bench.py's batch size: 10 000 queries drawn like bench.py's (seed SEED + 1) from the corpus."""
    t0 = time.perf_counter()
    c = synth.SparseCorpus(tokens=corp["tokens"], doc_ptr=corp["doc_ptr"], vocab=VOCAB)
    qs = synth.make_queries(c, 10_000, SEED + 1)
    qp, qt = qs.term_ptr.to(DEV), qs.terms.to(DEV)
    lists = [[int(t) for t in q] for q in qs.term_lists()]
    sample = list(range(0, 10_000, 211))
    sub = dict(bs, lists=[lists[i] for i in sample], names={})
    ref = _ref_topk(sub, list(range(len(sample))), 1024, rows_fn=bs["rows_fn"])
    sel = torch.tensor(sample, device=DEV)
    info = {}
    for k in (10, 192, 1024):
        a, n_cand, _ = _profiled(lambda: batched.bm25_topk(bs["index"], qp, qt, k))
        b = batched.bm25_topk(bs["ordered"], qp, qt, k)
        _assert_same(a, b, f"10k queries k={k}")
        _assert_topk(batched.TopK(a.scores[sel], a.ids[sel], a.counts[sel]), ref, k, f"10k sample k={k}", sub)
        info[f"cand_launches_k{k}"] = n_cand
        del a, b
    _report("10k queries", dict(sampled=len(sample), **info, seconds=time.perf_counter() - t0))


# ------------------------------------------------------------------------------------------ small corpora
def _small(n, seed):
    c = synth.make_sparse_corpus(n, 3000, seed, device=DEV, mean_len=40, min_len=1, max_len=120)
    st = _bm25s_stats(Bm25Stats.from_tokens(c.tokens, c.doc_ptr, 3000), n)
    qs = synth.make_queries(c, 150, seed + 1)
    present = np.nonzero(st.df.cpu().numpy())[0]
    rng = np.random.default_rng(seed)
    lists = [[int(t) for t in q] for q in qs.term_lists()] + [
        [], [-1, 5000], [int(present[1])] * 9, [int(t) for t in rng.choice(present, 300)],
        [int(t) for t in rng.choice(present, KPK_MAX_TERMS + 3)]]
    return st, lists


@pytest.mark.parametrize("n", [8193, 20_011, 3 * 8192 - 1])
def test_small_corpora(n):
    st, lists = _small(n, 500 + n % 97)
    ix = Bm25Index(st, device=DEV, packed=True)
    assert ix.post_pk is not None and ix.n_ranges == -(-n // 8192)
    _check_pack(ix)
    w32 = _ref_weights(st)
    assert torch.equal(ix.post_w.view(torch.int32), w32.view(torch.int32))
    c = dict(lists=lists, names={}, groups=None)
    ref = _ref_topk(c, list(range(len(lists))), 1024, rows_fn=_rows_fn(w32, st, n))
    qp, qt = _pack(lists)
    ordered = ix.ordered_view()
    for k in KS:
        a = batched.bm25_topk(ix, qp, qt, k)
        _assert_topk(a, ref, k, f"n={n} k={k}", c)
        _assert_same(a, batched.bm25_topk(ordered, qp, qt, k), f"n={n} k={k} vs ordered")


def test_save_load_equals_a_fresh_build(tmp_path):
    st, lists = _small(20_011, 77)
    ix = Bm25Index(st, device=DEV, packed=True)
    ix.save(str(tmp_path / "ix"))
    ld = Bm25Index.load(str(tmp_path / "ix"), packed=True)
    assert ld.pk_scale_log2 == ix.pk_scale_log2
    assert torch.equal(ld.post_pk, ix.post_pk) and torch.equal(ld.term_max, ix.term_max)
    assert Bm25Index.load(str(tmp_path / "ix")).post_pk is None          # the default stays unpacked for bm25s
    qp, qt = _pack(lists)
    for k in (10, 192):
        _assert_same(batched.bm25_topk(ld, qp, qt, k), batched.bm25_topk(ix, qp, qt, k), f"loaded k={k}")


# ------------------------------------------------------------------------------- sharded and fused routes
def _packed_rankers(mid, world, align):
    n = mid["n"]
    out = []
    for r in range(world):
        lo, hi = ezdist.shard_bounds(n, world, r, align=align)
        sparse = Bm25Index(mid["stats_s"], device=DEV, doc_lo=lo, doc_hi=hi, doc_group=mid["groups"], packed=True)
        assert sparse.post_pk is not None or sparse.n_postings == 0
        dense = DenseIndex(mid["vec"][lo:hi], device=DEV, row_lo=lo, doc_group=mid["groups"][lo:hi])
        out.append(batched.CoarseRanker(dense, sparse, canon=mid["canon"]))
    return out


def test_pipeline_hybrid_with_packed_bm25s_shards(mid):
    t0 = time.perf_counter()
    g, canon = mid["groups"], mid["canon"]
    dense_full = DenseIndex(mid["vec"], device=DEV, doc_group=g)
    sparse_full = Bm25Index(mid["stats_s"], device=DEV, doc_group=g)                 # one unpacked index
    assert sparse_full.post_pk is None
    runs = 0
    for world, align in ((1, 1), (3, 1), (8, 64)):
        rankers = _packed_rankers(mid, world, align)
        calls, shapes = [], []
        for kd, ks, ko in ((288, 192, 256), (33, 1024, 100), (10, 10, 10)):
            for qg in (None, mid["want"]):
                calls.append(dict(queries=mid["q"], q_ptr=mid["qp"], q_terms=mid["qt"], k_dense=kd, k_sparse=ks,
                                  k_out=ko, q_group=qg))
                shapes.append((kd, ks, ko, qg))
        got = _sharded(rankers, calls, form=1)
        for (kd, ks, ko, qg), res in zip(shapes, got):
            what = f"packed bm25s G={world} {kd}/{ks}/{ko} filtered={qg is not None}"
            _compare(res, _unsharded(dense_full, sparse_full, mid["q"], mid["qp"], mid["qt"], kd, ks, ko, qg, canon,
                                     form=1), what)
            runs += 1
        del rankers
    _report("pipeline_hybrid, packed bm25s shards", dict(runs=runs, seconds=time.perf_counter() - t0))


def test_dual_sparse_fusion_with_packed_bm25s(mid):
    t0 = time.perf_counter()
    n, g, canon = mid["n"], mid["groups"], mid["canon"]
    pc = synth.make_sparse_corpus(n, 500, 91, device=DEV, mean_len=12, min_len=1, max_len=30)
    p_stats = _bm25s_stats(Bm25Stats.from_tokens(pc.tokens, pc.doc_ptr, 500), n)
    pq = synth.make_queries(pc, mid["nq"], 92, min_terms=1, max_terms=5)
    pqp, pqt = pq.term_ptr.to(DEV), pq.terms.to(DEV)
    c_stats = mid["stats_s"]
    chunk_full = Bm25Index(c_stats, device=DEV, doc_group=g)
    path_full = Bm25Index(p_stats, device=DEV, doc_group=g)
    assert chunk_full.post_pk is None and path_full.post_pk is None
    chunk_pk = Bm25Index(c_stats, device=DEV, doc_group=g, packed=True)
    path_pk = Bm25Index(p_stats, device=DEV, doc_group=g, packed=True)
    calls = [(kc, kp, ko, qg) for kc, kp, ko in ((192, 6, 256), (33, 1024, 1024)) for qg in (None, mid["want"])]
    wants = [batched.dual_sparse_fusion(chunk_full, path_full, mid["qp"], mid["qt"], pqp, pqt, kc, kp, ko,
                                        canon=canon, q_group=qg) for kc, kp, ko, qg in calls]
    for (kc, kp, ko, qg), want in zip(calls, wants):
        got = batched.dual_sparse_fusion(chunk_pk, path_pk, mid["qp"], mid["qt"], pqp, pqt, kc, kp, ko, canon=canon,
                                         q_group=qg)
        _assert_same(got, want, f"dual packed {kc}/{kp}/{ko} filtered={qg is not None}", full_scores=True)
    runs = 0
    for world, align in ((1, 1), (3, 1), (8, 64)):
        bounds = [ezdist.shard_bounds(n, world, r, align=align) for r in range(world)]

        def fn(h):
            lo, hi = bounds[h.rank]
            sh = ezdist.ShardedDualSparseRanker(
                Bm25Index(c_stats, device=DEV, doc_lo=lo, doc_hi=hi, doc_group=g, packed=True),
                Bm25Index(p_stats, device=DEV, doc_lo=lo, doc_hi=hi, doc_group=g, packed=True), canon=canon, group=h)
            res = []
            for kc, kp, ko, qg in calls:
                res.append(_clone(sh.fuse(mid["qp"], mid["qt"], pqp, pqt, k_chunk=kc, k_path=kp, k_out=ko,
                                          q_group=qg)))
                torch.cuda.current_stream().synchronize()
            return res
        outs = _loopback.run_ranks(world, fn)
        for (kc, kp, ko, qg), want, *per_rank in zip(calls, wants, *outs):
            for r, got in enumerate(per_rank):
                _assert_same(got, want, f"dual G={world} rank {r} {kc}/{kp}/{ko} filtered={qg is not None}",
                             full_scores=True)
            runs += 1
    _report("dual sparse fusion, packed bm25s", dict(runs=runs, seconds=time.perf_counter() - t0))


# ------------------------------------------------------------------------------------------ drop-in retriever
def test_dropin_retriever_packed_bm25s(world):
    kw = dict(nodes=world["nodes"], tokenizer=world["tk"], stopwords=world["stop"], embed_type=0, bm25_type=1)
    for top_k in (6, 32, 192):
        plain = BM25Retriever.from_defaults(similarity_top_k=top_k, **kw)
        packed = BM25Retriever.from_defaults(similarity_top_k=top_k, packed=True, **kw)
        assert plain.bm25.post_pk is None and packed.bm25.post_pk is not None
        for qi, query in enumerate(world["queries"][:10]):
            fd = {"dir": DIRS[qi % 4]} if qi % 2 else None
            plain.filter_dict = packed.filter_dict = fd
            a = plain.retrieve(query)
            b, n_cand, _ = _profiled(lambda: packed.retrieve(query))
            assert n_cand >= 1
            assert [x.node.node_id for x in a] == [x.node.node_id for x in b], (top_k, qi)
            assert [x.score for x in a] == [x.score for x in b], (top_k, qi)
        q = world["queries"][3]
        assert packed.get_scores(q).tobytes() == plain.get_scores(q).tobytes()
