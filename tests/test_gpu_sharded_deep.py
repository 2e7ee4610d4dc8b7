"""GPU: row-sharded coarse ranking at the pipeline's depths (k up to 1024 per route), on one GPU with simulated ranks.

``ShardedCoarseRanker.pipeline_hybrid`` (dense top-288 + BM25 top-192 + RRF to 256) and ``ShardedDualSparseRanker``
(chunk BM25 top-192 + path BM25 top-6 + ``HybridRetriever.fusion``) run G ranks of one process, each in its own host
thread, their one all-gather through tests/_loopback.py; the per-route merge is ``ezr_merge_sorted_parts``.

1. ``ezr_merge_sorted_parts`` against a numpy ``lexsort`` of the gathered candidates: G in {1, 2, 3, 8}, k and n_cand
   in {1, 33, 192, 288, 1023, 1024}, per-part counts from 0 to full, ties within and across parts, +-0.0, f32 and
   f64, poisoned slots past each count (id -1 with +inf or NaN), rows wider than k, 10k rows; argument errors.
2. What the merge relies on: every route the sharded path runs, at k in {33, 192, 288, 1024}, writes a canonical
   sorted prefix of length ``count`` into a poisoned record and id -1 after it (dense forms 1 and 6, an int8 shard's
   full scan, the deep two-phase BM25 with a mass tie that overflows to score rows, bm25s, a negative-idf index).
3. ``pipeline_hybrid`` on the benchmark corpus (1M x 768, 200k vocabulary, 1024 queries) at 288 / 192 / 256 and at
   1024 on both routes, G = 2, 8 (align 64) and G = 3 (align 1), bit-identical to one GPU's
   ``dense_topk`` (same forced form) + ``bm25_topk`` + ``fuse_lists``; constructed cases (filters, duplicates across
   shards, bm25s and int8 shards, empty ranks, equal k <= 32 against ``hybrid``).
4. ``ShardedDualSparseRanker`` against ``batched.dual_sparse_fusion`` for G = 2, 3, 8, with and without filters.
5. Two GPUs over NCCL (skipped on one GPU).

What each case ran is printed (``pytest -s``).  Peak device memory of the whole file was 23.0 GB on an H100 80GB HBM3
(700 W power limit), and the file ran in about 41 s there (the two-GPU case skipped).
"""
import os
import time
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import _loopback
from test_gpu_sharded import _assert_padded, _assert_same, _clone, _dup_tokens, _ints, _pack, _poisoned_record
from easyrag_b200 import _lib, batched, synth
from easyrag_b200 import dist as ezdist
from easyrag_b200.index import Bm25Index, Bm25Stats, DenseIndex

pytestmark = pytest.mark.gpu
DEV = "cuda"
INF = float("inf")
KS = (1, 33, 192, 288, 1023, 1024)


@pytest.fixture(scope="module", autouse=True)
def _ready(lib_built):
    _lib.require_cuda()
    _lib.lib()


@pytest.fixture(autouse=True)
def _loop(monkeypatch):
    _loopback.install(monkeypatch)


def _report(what, info):
    info = dict(info, peak_gb=torch.cuda.max_memory_allocated() / 2 ** 30)
    print(f"\n[sharded-deep] {what}: " + ", ".join(f"{k}={v:.4g}" if isinstance(v, float) else f"{k}={v}"
                                                 for k, v in info.items()))


# ============================================================================ 1. ezr_merge_sorted_parts
SCORE_SET = np.array([-1.5, -0.0, 0.0, 0.25, 1.0, 3.0])


def _sorted_parts(rng, G, Q, n, dtype, full=False):
    """G canonical lists [G, Q, n] with distinct ids across parts, random counts in [0, n] (``full``: n), and id -1
    with a +inf or NaN score past each count."""
    span = 2 * n + 3
    s = SCORE_SET[rng.integers(0, SCORE_SET.size, (G, Q, n))].astype(dtype)
    ids = np.argsort(rng.random((G, Q, span)), -1)[..., :n].astype(np.int32) + (np.arange(G) * span)[:, None, None]
    order = np.lexsort((-ids, -s), axis=-1)
    s, ids = np.take_along_axis(s, order, -1), np.take_along_axis(ids, order, -1).astype(np.int32)
    cnt = np.full((G, Q), n) if full else rng.integers(0, n + 1, (G, Q))
    if Q >= 3:
        cnt[:, 0], cnt[:, 1], cnt[:, 2] = 0, n, n // 2                # an empty, a full and a half list in every part
    past = np.arange(n)[None, None, :] >= cnt[..., None]
    poison = np.where(rng.random((G, Q, n)) < 0.5, np.inf, np.nan).astype(dtype)
    return np.where(past, poison, s), np.where(past, -1, ids).astype(np.int32)


def _ref(s, ids, k):
    """(ids [Q, k] -1 padded, scores [Q, k], counts [Q]) of the canonical top-k over the valid slots of all parts."""
    G, Q, n = s.shape
    s = np.transpose(s, (1, 0, 2)).reshape(Q, G * n)
    i = np.transpose(ids, (1, 0, 2)).reshape(Q, G * n)
    valid = i >= 0
    order = np.lexsort((-i, -np.where(valid, s, 0), (~valid).astype(np.int8)), axis=-1)[:, :k]
    cnt = np.minimum(valid.sum(1), k)
    keep = np.arange(order.shape[1])[None, :] < cnt[:, None]
    oi = np.full((Q, k), -1, np.int32)
    os_ = np.zeros((Q, k), s.dtype)
    oi[:, :order.shape[1]] = np.where(keep, np.take_along_axis(i, order, -1), -1)
    os_[:, :order.shape[1]] = np.take_along_axis(s, order, -1)
    return oi, os_, cnt


def _check(got, ref, k, what):
    """ids and counts equal, score bytes equal before each count, and id -1 / -inf in every slot from the count to the
    end of the (possibly wider) output row."""
    ri, rs, rc = ref
    gi, gs, gc = got.ids.cpu().numpy(), got.scores.cpu().numpy(), got.counts.cpu().numpy()
    w = gi.shape[1]
    bits = np.int64 if gs.dtype == np.float64 else np.int32
    keep = np.arange(k)[None, :] < rc[:, None]
    bad = (gc != rc) | (gi[:, :k] != ri).any(1) | ((gs[:, :k].view(bits) != rs.view(bits)) & keep).any(1)
    past = np.arange(w)[None, :] >= gc[:, None]
    bad |= (past & ((gi != -1) | ~np.isneginf(gs))).any(1)
    if bad.any():
        q = int(np.nonzero(bad)[0][0])
        raise AssertionError(f"{what}: {int(bad.sum())} rows differ; first row {q}: count {gc[q]} vs {rc[q]}\n"
                             f"  got  {gi[q][:40].tolist()}\n  want {ri[q][:40].tolist()}")


def _gathered(layout, parts):
    nb = layout.nbytes
    buf = torch.zeros(len(parts) * nb, dtype=torch.uint8, device=DEV)
    for p, arrs in enumerate(parts):
        for view, a in zip(ezdist.record_views(layout, buf[p * nb:(p + 1) * nb]), arrs):
            view.copy_(torch.from_numpy(np.ascontiguousarray(a)))
    return buf


def _merge_case(rng, G, Q, n, ks, sb, pad=0, full=False):
    sdt = np.float64 if sb == 8 else np.float32
    ds, di = _sorted_parts(rng, G, Q, n, np.float32, full)
    ss, si = _sorted_parts(rng, G, Q, n, sdt, full)
    layout = ezdist.RecordLayout(Q, n, sb)
    buf = _gathered(layout, [(ds[p], di[p], ss[p], si[p]) for p in range(G)])
    g_ds, g_di, g_ss, g_si = ezdist.record_views(layout, buf[:layout.nbytes])
    for k in ks:
        for (s, i, gs, gi, dt) in ((ds, di, g_ds, g_di, torch.float32), (ss, si, g_ss, g_si, g_ss.dtype)):
            out = batched.TopK(torch.full((Q, k + pad), 7.0, dtype=dt, device=DEV),
                               torch.full((Q, k + pad), 12345, dtype=torch.int32, device=DEV),
                               torch.full((Q,), -5, dtype=torch.int32, device=DEV))
            got = batched.merge_sorted_parts(gs, gi, G, layout.nbytes, k, out=out)
            _check(got, _ref(s, i, k), k, f"G={G} n_cand={n} k={k} Q={Q} {dt} pad={pad}")


def test_merge_sorted_parts_against_lexsort():
    t0 = time.perf_counter()
    rng = np.random.default_rng(23)
    runs = 0
    for G in (1, 2, 3, 8):
        for n in KS:
            for sb in (8, 4):
                _merge_case(rng, G, 7, n, KS, sb, pad=3 if n % 2 else 0)
                runs += 2 * len(KS)
    # every part full: the total exceeds k for every k < G * n
    for G, n in ((2, 1024), (8, 1024), (3, 288)):
        _merge_case(rng, G, 5, n, (1, 192, 288, 1024), 8, full=True)
    # 10k rows at the pipeline's shapes
    _merge_case(rng, 8, 10_003, 288, (288, 256), 8, pad=0)
    _merge_case(rng, 8, 10_003, 192, (192,), 4, pad=96)
    _report("merge_sorted_parts", dict(merges=runs, seconds=time.perf_counter() - t0))


def test_merge_sorted_parts_argument_errors():
    layout = ezdist.RecordLayout(9, 1024, 8)
    buf = torch.full((9 * layout.nbytes,), 0xff, dtype=torch.uint8, device=DEV)      # ids -1 everywhere
    _, _, g_ss, g_si = ezdist.record_views(layout, buf[:layout.nbytes])
    m = batched.merge_sorted_parts(g_ss, g_si, 8, layout.nbytes, 1024)
    assert m.counts.sum().item() == 0 and bool((m.ids == -1).all()) and bool(torch.isneginf(m.scores).all())
    for k in (0, 1025):
        with pytest.raises(_lib.EzrError, match=f"k={k}"):
            batched.merge_sorted_parts(g_ss, g_si, 8, layout.nbytes, k)
    with pytest.raises(_lib.EzrError, match="n_parts \\* n_cand"):
        batched.merge_sorted_parts(g_ss, g_si, 9, layout.nbytes, 32)
    for stride in (layout.nbytes + 4, -layout.nbytes):
        with pytest.raises(_lib.EzrError, match="part_stride_bytes"):
            batched.merge_sorted_parts(g_ss, g_si, 2, stride, 32)
    narrow = batched.TopK(torch.empty(9, 31, dtype=torch.float64, device=DEV),
                          torch.empty(9, 31, dtype=torch.int32, device=DEV), torch.empty(9, dtype=torch.int32, device=DEV))
    with pytest.raises(_lib.EzrError, match="out_stride"):
        batched.merge_sorted_parts(g_ss, g_si, 2, layout.nbytes, 32, out=narrow)


# ============================================================================ 2. the route-output precondition
DEEP_KS = (33, 192, 288, 1024)


def _assert_canonical(scores, ids, counts, what):
    """The prefix of each row is strictly decreasing in (score, id): better(slot j, slot j + 1) for j + 1 < count."""
    s, i = scores[:, :-1], ids[:, :-1]
    s1, i1 = scores[:, 1:], ids[:, 1:]
    both = torch.arange(1, ids.shape[1], device=DEV)[None, :] < counts[:, None].long()
    ok = (s > s1) | ((s == s1) & (i > i1))
    bad = both & ~ok
    if bad.any():
        q = int(torch.nonzero(bad.any(1))[0])
        raise AssertionError(f"{what}: query {q} is not in canonical order: {ids[q][:40].tolist()}")


def _precondition(layout, views, which, out, what):
    s, i = views[which], views[which + 1]
    assert out.ids.data_ptr() == i.data_ptr() and out.scores.data_ptr() == s.data_ptr()
    torch.cuda.synchronize()
    _assert_padded(i, out.counts, what)
    _assert_canonical(s, i, out.counts, what)
    return int(out.counts.sum())


@pytest.fixture(scope="module")
def small():
    """20k documents (3 BM25 ranges): 6000 copies of D spread over the corpus, so [T_D] ties more documents than the
    deep path's per-query list holds at any k <= 1024 (4k + 1024) and overflows to its score row; integer dense
    vectors (dim 256), 77 queries."""
    n, v0, dim = 20_000, 4_000, 256
    c = synth.make_sparse_corpus(n, v0, 61, device=DEV)
    qs = synth.make_queries(c, 70, 62)
    tokens, doc_ptr, a_ids, d_tok = _dup_tokens(c, n, v0, 6000, 600, 8192 + 1000, 4242, 15_000)
    stats = Bm25Stats.from_tokens(tokens, doc_ptr, v0 + 2)
    groups = synth.make_groups(n, 4, 63, device=DEV)
    lists = [[int(t) for t in q] for q in qs.term_lists()]
    lists += [[v0], [v0 + 1], d_tok + [v0], [], [-1, v0 + 9], [v0, v0 + 1], [v0 + 1] * 3]
    qp, qt = _pack(lists)
    want = torch.tensor([(-1, 0, 1, 9)[i % 4] for i in range(len(lists))], dtype=torch.int32, device=DEV)
    assert len(a_ids) > 4 * 1024 + 1024
    return dict(n=n, stats=stats, groups=groups, lists=lists, qp=qp, qt=qt, vec=_ints(n, dim, 64),
                q=_ints(len(lists), dim, 65), want=want)


def test_route_precondition_dense(small):
    t0 = time.perf_counter()
    L = _lib.lib()
    vec, q, g, n = small["vec"], small["q"], small["groups"], small["n"]
    idx = dict(shard=DenseIndex(vec[5000:13001], device=DEV, row_lo=5000, doc_group=g[5000:13001]),
               few=DenseIndex(vec[100:105], device=DEV, row_lo=100, doc_group=g[100:105]),
               empty=DenseIndex(vec[n:], device=DEV, row_lo=n, doc_group=g[n:]),
               s8=DenseIndex(vec[5000:13001], device=DEV, row_lo=5000, doc_group=g[5000:13001], quantized=True),
               s8_few=DenseIndex(vec[100:105], device=DEV, row_lo=100, doc_group=g[100:105], quantized=True))
    runs, results, kernels = 0, 0, set()
    for name, ix in idx.items():
        for form in ((0,) if getattr(ix, "quantized", False) else (1, 6)):
            for k in DEEP_KS:
                for qg in (None, small["want"]):
                    layout, _, views = _poisoned_record(q.shape[0], k, 8)
                    out = batched.TopK(views[0], views[1], torch.empty(q.shape[0], dtype=torch.int32, device=DEV))
                    batched.dense_topk(ix, q, k, q_group=qg, out=out, form=form or None)
                    torch.cuda.synchronize()
                    kernels.add(L.ezr_dense_last_kernel().decode())
                    what = f"dense {name} form {form} k={k} filtered={qg is not None}"
                    results += _precondition(layout, views, 0, out, what)
                    runs += 1
    _report("route precondition, dense", dict(runs=runs, results=results, kernels=sorted(kernels),
                                              seconds=time.perf_counter() - t0))


def test_route_precondition_bm25(small):
    t0 = time.perf_counter()
    L = _lib.lib()
    st, n, g = small["stats"], small["n"], small["groups"]
    st1 = Bm25Stats.from_counts(n, st.vocab, int(st.doc_len.long().sum()), st.doc_len, st.df, st.indptr, st.post_doc,
                                st.post_tf, np.zeros(st.vocab, np.uint64), bm25_type=1)
    rng = np.random.default_rng(17)
    docs = []
    for _ in range(20_000):                                          # mean idf < 0 (as tests/test_gpu_bm25_deep.py)
        d = [t for t in range(5) if rng.random() < 0.9] * int(rng.integers(1, 3))
        if rng.random() < 0.3:
            d += [5] * int(rng.integers(1, 4))
        docs.append(np.array(d if d else [0], dtype=np.int32))
    neg = Bm25Index(Bm25Stats.from_tokens(torch.from_numpy(np.concatenate(docs)).to(torch.int32),
                                          torch.tensor(np.cumsum([0] + [len(d) for d in docs]), dtype=torch.int64), 6),
                    device=DEV, doc_lo=3000, doc_hi=17001)
    assert not neg.monotone
    neg_lists = [[int(t) for t in rng.integers(0, 6, int(rng.integers(1, 7)))] for _ in range(len(small["lists"]))]
    nqp, nqt = _pack(neg_lists)
    shard = Bm25Index(st, device=DEV, doc_lo=5000, doc_hi=13001, doc_group=g)
    idx = dict(full=(Bm25Index(st, device=DEV, doc_group=g), small["qp"], small["qt"]),
               shard=(shard, small["qp"], small["qt"]),
               few=(Bm25Index(st, device=DEV, doc_lo=100, doc_hi=105, doc_group=g), small["qp"], small["qt"]),
               empty=(Bm25Index(st, device=DEV, doc_lo=n, doc_hi=n, doc_group=g), small["qp"], small["qt"]),
               bm25s=(Bm25Index(st1, device=DEV, doc_lo=5000, doc_hi=13001, doc_group=g), small["qp"], small["qt"]),
               negative_idf=(neg, nqp, nqt))
    assert idx["full"][0].post_pk is not None and shard.post_pk is not None
    runs, results, overflowed = 0, 0, 0
    L.ezr_profile_enable(1)
    try:
        for name, (ix, qp, qt) in idx.items():
            for k in DEEP_KS:
                for qg in ((None, small["want"]) if ix.doc_group is not None else (None,)):
                    sb = 8 if ix.score_dtype == torch.float64 else 4
                    layout, _, views = _poisoned_record(len(small["lists"]), k, sb)
                    out = batched.TopK(views[2], views[3], torch.empty(len(small["lists"]), dtype=torch.int32,
                                                                       device=DEV))
                    L.ezr_profile_reset()
                    batched.bm25_topk(ix, qp, qt, k, q_group=qg, out=out)
                    torch.cuda.synchronize()
                    if name == "full" and qg is None:
                        # the deep two-phase path ran and the mass tie [T_D] went to its score row
                        assert _lib.profile_read("bm25_cand")[1] == 1, f"k={k}: the deep path did not run"
                        assert _lib.profile_read("bm25_score")[1] >= 1, f"k={k}: no query overflowed"
                        overflowed += 1
                    results += _precondition(layout, views, 2, out, f"bm25 {name} k={k} filtered={qg is not None}")
                    runs += 1
    finally:
        L.ezr_profile_enable(0)
    _report("route precondition, bm25", dict(runs=runs, results=results, overflow_runs=overflowed,
                                             seconds=time.perf_counter() - t0))


# ============================================================================ 3. pipeline_hybrid
def _unsharded(dense, sparse, q, qp, qt, kd, ks, ko, qg=None, canon=None, form=0):
    """One GPU: dense_topk(kd) + bm25_topk(ks) + fuse_lists over lists padded to one width."""
    d = batched.dense_topk(dense, q, kd, q_group=qg, form=form or None)
    s = batched.bm25_topk(sparse, qp, qt, ks, q_group=qg)
    w = max(kd, ks)
    pad = lambda ids: torch.nn.functional.pad(ids, (0, w - ids.shape[1]), value=-1)
    f = batched.fuse_lists([pad(s.ids), pad(d.ids)], [s.counts, d.counts], ko, rrf=True, K=60, canon=canon)
    torch.cuda.synchronize()
    return f, s, d


def _rankers(vec, stats, groups, canon, world, align, quantized=False):
    n = vec.shape[0]
    out = []
    for r in range(world):
        lo, hi = ezdist.shard_bounds(n, world, r, align=align)
        dense = DenseIndex(vec[lo:hi], device=DEV, row_lo=lo, quantized=quantized,
                           doc_group=None if groups is None else groups[lo:hi])
        out.append(batched.CoarseRanker(dense, Bm25Index(stats, device=DEV, doc_lo=lo, doc_hi=hi, doc_group=groups),
                                        canon=canon))
    return out


def _sharded(rankers, calls, form=0, method="pipeline_hybrid"):
    """Every rank runs ``method(**c)`` for each ``c`` of ``calls`` with the dense form ``form`` forced in its thread;
    all ranks must return the same bytes.  -> rank 0's [(fused, sparse, dense)]."""
    L = _lib.lib()

    def fn(h):
        _lib.check(L.ezr_dense_set_kernel(form))
        try:
            sh = ezdist.ShardedCoarseRanker(rankers[h.rank], group=h)
            res = []
            for c in calls:
                out = getattr(sh, method)(**c)
                torch.cuda.current_stream().synchronize()
                res.append(tuple(_clone(t) for t in out))
            return res
        finally:
            L.ezr_dense_set_kernel(0)
    outs = _loopback.run_ranks(len(rankers), fn)
    for r, o in enumerate(outs[1:], 1):
        for i, (a, b) in enumerate(zip(outs[0], o)):
            for name, x, y in zip(("fused", "sparse", "dense"), a, b):
                _assert_same(x, y, f"rank {r} vs rank 0, call {i}, {name}", full_scores=True)
    return outs[0]


def _compare(got, want, what):
    for name, a, b in zip(("fused", "sparse", "dense"), got, want):
        assert a.ids.shape == b.ids.shape, f"{what} {name}: shape {tuple(a.ids.shape)} vs {tuple(b.ids.shape)}"
        _assert_same(a, b, f"{what} {name}", full_scores=name == "fused")


BENCH = SimpleNamespace(rows=1_000_000, dim=768, vocab=200_000, queries=1024)


def test_pipeline_hybrid_at_bench_scale():
    import bench
    t0 = time.perf_counter()
    torch.cuda.reset_peak_memory_stats()
    data = bench.make_data(BENCH, torch.device(DEV))
    stats, vec, qv = data["stats"], data["vec"], data["qvec"].contiguous()
    qp, qt = data["queries"].term_ptr.to(DEV), data["queries"].terms.to(DEV)
    form = 6
    shapes = [(288, 192, 256), (1024, 1024, 1024)]
    dense_full, sparse_full = DenseIndex(vec, device=DEV), Bm25Index(stats, device=DEV)
    want = [tuple(_clone(t) for t in _unsharded(dense_full, sparse_full, qv, qp, qt, *s, form=form)) for s in shapes]
    del dense_full, sparse_full
    info = dict(gen_s=data["gen_s"])
    for world, align in ((2, 64), (8, 64), (3, 1)):
        t1 = time.perf_counter()
        rankers = _rankers(vec, stats, None, None, world, align)
        calls = [dict(queries=qv, q_ptr=qp, q_terms=qt, k_dense=kd, k_sparse=ks, k_out=ko) for kd, ks, ko in shapes]
        got = _sharded(rankers, calls if world == 8 else calls[:1], form=form)
        del rankers
        for s, g, w in zip(shapes, got, want):
            _compare(g, w, f"G={world} align={align} {s}")
        info[f"G{world}_s"] = time.perf_counter() - t1
    f, s, d = want[0]
    info.update(full_dense=int((d.counts == 288).sum()), full_sparse=int((s.counts == 192).sum()),
                fused_256=int((f.counts == 256).sum()), seconds=time.perf_counter() - t0)
    _report("pipeline_hybrid at bench scale", info)


@pytest.fixture(scope="module")
def mid():
    """60k documents (8 BM25 ranges): 1500 copies of D and 200 copies of dense row R spread over the corpus (ties at
    every depth straddle shard boundaries); groups 5 and 6 only in the first / last 1000 rows; the D and R copies are
    duplicates of one text each (``canon``)."""
    n, v0, dim, nq = 60_000, 8_000, 256, 260
    c = synth.make_sparse_corpus(n, v0, 71, device=DEV)
    qs = synth.make_queries(c, nq - 6, 72)
    tokens, doc_ptr, a_ids, d_tok = _dup_tokens(c, n, v0, 1500, 600, 3 * 8192 + 77, 4242, 45_000)
    stats = Bm25Stats.from_tokens(tokens, doc_ptr, v0 + 2)
    lists = [[int(t) for t in q] for q in qs.term_lists()] + [[v0], [v0 + 1], d_tok + [v0], [], [-1, v0 + 9], d_tok]
    qp, qt = _pack(lists)
    vec = _ints(n, dim, 73)
    r_pos = torch.arange(200, device=DEV) * (n - 1) // 199
    vec[r_pos] = vec[1234].clone()
    q = _ints(nq, dim, 74)
    q[-6:] = vec[1234].clone()
    groups = synth.make_groups(n, 4, 75, device=DEV)
    groups[:1000], groups[-1000:] = 5, 6
    canon = synth.make_duplicates(n, 0.03, 76, device=DEV)
    canon[torch.tensor(a_ids, device=DEV)] = min(a_ids)
    canon[r_pos] = int(r_pos.min())
    want = torch.tensor([(-1, 0, 5, 6, 9, 2)[i % 6] for i in range(nq)], dtype=torch.int32, device=DEV)
    st1 = Bm25Stats.from_counts(n, stats.vocab, int(stats.doc_len.long().sum()), stats.doc_len, stats.df, stats.indptr,
                                stats.post_doc, stats.post_tf, np.zeros(stats.vocab, np.uint64), bm25_type=1)
    return dict(n=n, stats=stats, stats_s=st1, lists=lists, qp=qp, qt=qt, vec=vec, q=q, groups=groups, canon=canon,
                want=want, nq=nq)


def test_pipeline_hybrid_constructed_cases(mid):
    t0 = time.perf_counter()
    vec, g, canon = mid["vec"], mid["groups"], mid["canon"]
    runs = 0
    for sname, stats in (("okapi", mid["stats"]), ("bm25s", mid["stats_s"])):
        dense_full = DenseIndex(vec, device=DEV, doc_group=g)
        sparse_full = Bm25Index(stats, device=DEV, doc_group=g)
        for world, align, quantized in ((3, 1, False), (8, 64, False), (3, 1, True), (8, 8192, True)):
            if sname == "bm25s" and not quantized:
                continue
            rankers = _rankers(vec, stats, g, canon, world, align, quantized=quantized)
            calls, shapes = [], []
            for kd, ks, ko in ((288, 192, 256), (33, 1024, 100), (1024, 6, 1024)):
                for qg in (None, mid["want"]):
                    calls.append(dict(queries=mid["q"], q_ptr=mid["qp"], q_terms=mid["qt"], k_dense=kd, k_sparse=ks,
                                      k_out=ko, q_group=qg))
                    shapes.append((kd, ks, ko, qg))
            got = _sharded(rankers, calls, form=1)
            for (kd, ks, ko, qg), res in zip(shapes, got):
                what = f"{sname} G={world} align={align} int8={quantized} {kd}/{ks}/{ko} filtered={qg is not None}"
                _compare(res, _unsharded(dense_full, sparse_full, mid["q"], mid["qp"], mid["qt"], kd, ks, ko, qg, canon,
                                         form=1), what)
                if qg is not None:
                    assert bool((res[0].counts[mid["want"] == 9] == 0).all()), what
                runs += 1
            del rankers
    _report("pipeline_hybrid constructed cases", dict(runs=runs, seconds=time.perf_counter() - t0))


def test_pipeline_hybrid_equal_small_k_matches_hybrid(mid):
    rankers = _rankers(mid["vec"], mid["stats"], mid["groups"], mid["canon"], 3, 1)
    for k in (1, 10, 32):
        for qg in (None, mid["want"]):
            c = dict(queries=mid["q"], q_ptr=mid["qp"], q_terms=mid["qt"], q_group=qg)
            a = _sharded(rankers, [dict(c, k_dense=k, k_sparse=k, k_out=k)])[0]
            b = _sharded(rankers, [dict(c, k=k, k_out=k)], method="hybrid")[0]
            _compare(a, b, f"k={k} filtered={qg is not None}")


def test_pipeline_hybrid_empty_ranks_and_argument_errors():
    """100 documents over G = 8 with align 64: ranks 2..7 hold no row and no document."""
    n, vocab, dim, nq = 100, 300, 256, 19
    c = synth.make_sparse_corpus(n, vocab, 81, mean_len=20, min_len=1, max_len=40)
    qs = synth.make_queries(c, nq, 82, min_terms=1, max_terms=6)
    stats = Bm25Stats.from_tokens(c.tokens, c.doc_ptr, vocab)
    vec = _ints(n, dim, 83)
    vec[60:70] = vec[3].clone()
    q = _ints(nq, dim, 84)
    groups = synth.make_groups(n, 3, 85, device=DEV)
    want = torch.tensor([(-1, 0, 1, 2, 7)[i % 5] for i in range(nq)], dtype=torch.int32, device=DEV)
    qp, qt = qs.term_ptr.to(DEV), qs.terms.to(DEV)
    dense_full, sparse_full = DenseIndex(vec, device=DEV, doc_group=groups), Bm25Index(stats, device=DEV,
                                                                                     doc_group=groups)
    for quantized in (False, True):
        rankers = _rankers(vec, stats, groups, None, 8, 64, quantized=quantized)
        assert rankers[5].dense.n_rows == 0 and rankers[5].sparse.n_docs == 0
        shapes = [(kd, ks, ko, qg) for kd, ks, ko in ((288, 192, 256), (1024, 1024, 1024), (33, 1, 5))
                  for qg in (None, want)]
        calls = [dict(queries=q, q_ptr=qp, q_terms=qt, k_dense=kd, k_sparse=ks, k_out=ko, q_group=qg)
                 for kd, ks, ko, qg in shapes]
        for (kd, ks, ko, qg), res in zip(shapes, _sharded(rankers, calls, form=1)):
            _compare(res, _unsharded(dense_full, sparse_full, q, qp, qt, kd, ks, ko, qg, form=1),
                     f"tiny int8={quantized} {kd}/{ks}/{ko} filtered={qg is not None}")
    sh = ezdist.ShardedCoarseRanker(rankers[0], group=_loopback.Loopback(1).handles()[0])
    for kw in (dict(k_dense=0), dict(k_dense=1025), dict(k_sparse=0), dict(k_sparse=1025), dict(k_out=0)):
        with pytest.raises(ValueError, match="out of|k_out"):
            sh.pipeline_hybrid(q, qp, qt, **kw)


# ============================================================================ 4. sharded dual sparse fusion
def test_sharded_dual_sparse_fusion(mid):
    t0 = time.perf_counter()
    n, g, canon = mid["n"], mid["groups"], mid["canon"]
    pc = synth.make_sparse_corpus(n, 500, 91, device=DEV, mean_len=12, min_len=1, max_len=30)
    p_stats = Bm25Stats.from_tokens(pc.tokens, pc.doc_ptr, 500)
    pq = synth.make_queries(pc, mid["nq"], 92, min_terms=1, max_terms=5)
    pqp, pqt = pq.term_ptr.to(DEV), pq.terms.to(DEV)
    runs = 0
    for c_stats in (mid["stats"], mid["stats_s"]):
        chunk_full = Bm25Index(c_stats, device=DEV, doc_group=g)
        path_full = Bm25Index(p_stats, device=DEV, doc_group=g)
        for world, align in ((2, 64), (3, 1), (8, 64)):
            bounds = [ezdist.shard_bounds(n, world, r, align=align) for r in range(world)]
            calls = [(kc, kp, ko, qg) for kc, kp, ko in ((192, 6, 256), (33, 1024, 1024)) for qg in (None, mid["want"])]

            def fn(h):
                lo, hi = bounds[h.rank]
                sh = ezdist.ShardedDualSparseRanker(Bm25Index(c_stats, device=DEV, doc_lo=lo, doc_hi=hi, doc_group=g),
                                                    Bm25Index(p_stats, device=DEV, doc_lo=lo, doc_hi=hi, doc_group=g),
                                                    canon=canon, group=h)
                res = []
                for kc, kp, ko, qg in calls:
                    res.append(_clone(sh.fuse(mid["qp"], mid["qt"], pqp, pqt, k_chunk=kc, k_path=kp, k_out=ko,
                                              q_group=qg)))
                    torch.cuda.current_stream().synchronize()
                return res
            outs = _loopback.run_ranks(world, fn)
            for (kc, kp, ko, qg), *per_rank in zip(calls, *outs):
                want = batched.dual_sparse_fusion(chunk_full, path_full, mid["qp"], mid["qt"], pqp, pqt, kc, kp, ko,
                                                  canon=canon, q_group=qg)
                torch.cuda.synchronize()
                for r, got in enumerate(per_rank):
                    _assert_same(got, want, f"dual G={world} rank {r} {kc}/{kp}/{ko} filtered={qg is not None}",
                                 full_scores=True)
                runs += 1
    _report("sharded dual sparse fusion", dict(runs=runs, seconds=time.perf_counter() - t0))


# ============================================================================ 5. two GPUs, NCCL
def _nccl_worker(rank, world, port, ret):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    try:
        n, vocab, dim, nq = 40_000, 8_000, 256, 300
        corpus = synth.make_sparse_corpus(n, vocab, 5)
        queries = synth.make_queries(corpus, nq, 6)
        stats = Bm25Stats.from_tokens(corpus.tokens, corpus.doc_ptr, vocab)
        g = torch.Generator().manual_seed(7)
        vec = torch.randint(-2, 3, (n, dim), generator=g).to(torch.bfloat16)       # exact dot products
        qv = torch.randint(-2, 3, (nq, dim), generator=g).to(torch.bfloat16).to(dev)
        canon = synth.make_duplicates(n, 0.03, 8)
        lo, hi = ezdist.shard_bounds(n, world, rank, align=64)
        ranker = batched.CoarseRanker(DenseIndex(vec[lo:hi], device=dev, row_lo=lo),
                                      Bm25Index(stats, device=dev, doc_lo=lo, doc_hi=hi), canon=canon)
        qp, qt = queries.term_ptr.to(dev), queries.terms.to(dev)
        f, s, d = ezdist.ShardedCoarseRanker(ranker).pipeline_hybrid(qv, qp, qt, 288, 192, 256)
        dual = ezdist.ShardedDualSparseRanker(ranker.sparse, ranker.sparse, canon=canon).fuse(qp, qt, qp, qt, 192, 6,
                                                                                              256)
        torch.cuda.synchronize()
        ok = True
        if rank == 0:
            full_s = Bm25Index(stats, device=dev)
            want = _unsharded(DenseIndex(vec, device=dev), full_s, qv, qp, qt, 288, 192, 256, canon=canon.to(dev))
            for a, b in zip((f, s, d), want):
                ok &= torch.equal(a.ids, b.ids) and torch.equal(a.counts, b.counts)
                keep = torch.arange(a.ids.shape[1], device=dev)[None, :] < a.counts[:, None]
                ok &= bool(((a.scores == b.scores) | ~keep).all())
            w = batched.dual_sparse_fusion(full_s, full_s, qp, qt, qp, qt, 192, 6, 256, canon=canon)
            ok &= torch.equal(dual.ids, w.ids) and torch.equal(dual.scores.view(torch.int64), w.scores.view(torch.int64))
        ret[rank] = bool(ok)
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpu_nccl():
    import socket
    import torch.multiprocessing as mp
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    mgr = mp.get_context("spawn").Manager()
    ret = mgr.dict()
    mp.spawn(_nccl_worker, args=(2, port, ret), nprocs=2, join=True)
    assert dict(ret) == {0: True, 1: True}
