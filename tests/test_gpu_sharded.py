"""GPU: the row-sharded coarse ranker (easyrag_b200/dist.py, bench.py configs[3]) on one GPU, with simulated ranks.

``ShardedCoarseRanker`` runs G ranks of one process here, each in its own host thread with its own shard-local
``CoarseRanker``; their one all-gather goes through a loopback collective (tests/_loopback.py).  So the N > 1 path --
route kernels writing straight into the exchange record, the gathered buffer, ``ezr_merge_topk_parts`` reading G
records in place (``merge_warp_kernel`` with ``n_parts > 1``) and the RRF over the merged lists -- runs on a machine
with one GPU, where tests/test_gpu_dist.py (NCCL, two GPUs) skips.

1. ``ezr_merge_topk_parts`` against a numpy ``lexsort`` of the gathered candidates, with ties across parts, both
   zeros, poisoned padding and both sparse record widths.
2. The contract the merge relies on: it takes every slot with ``id >= 0`` and ignores the per-shard counts, so every
   route must write id -1 to every slot of the record past its count, in every kernel form and fallback.
3. configs[3] at benchmark scale (1M x 768, 200k vocabulary, 10k queries): G = 2, 8 (align 64, as bench.py) and
   G = 3 (align 1) equal the unsharded ranker bit for bit, and the first 512 queries equal independent references.
4. Constructed cases at 200k rows with ties that straddle shard boundaries, filters, duplicates, bm25s, quantized
   shards and empty ranks.
5. The pipelined path (``submit``, ``HostPipeline``) over the sharded ranker.

Two faults these tests found are fixed with them: the int8 rescoring of a quantized dense index left the slots past
the count unwritten when a query had fewer than k candidates (the merge then took whatever the record held, id 0 of a
fresh record), and the routes refused a ``q_group`` filter on an empty shard, whose empty ``doc_group`` has no address.

What each case ran is printed (``pytest -s``).  Peak device memory of the whole file was 13.9 GB on an H100 80GB HBM3
(power limit not recorded), and the file ran in about 26 s there.
"""
import hashlib
import json
import sys
import time
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import _loopback
from _bm25_ref import canonical_topk as bm25_canonical_topk
from _bm25_ref import okapi_row, okapi_weights
from _bounds import check_dense_topk, dense_delta_max, dense_score_bound
from _topk_ref import fp64_top
from easyrag_b200 import _lib, batched, synth
from easyrag_b200 import dist as ezdist
from easyrag_b200.index import Bm25Index, Bm25Stats, DenseIndex
from oracle import retrieve as ort

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import bench                                   # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
POISON_ID = 0x7ffffff0                         # a valid id (>= 0) that no corpus here has
INF = float("inf")


@pytest.fixture(scope="module", autouse=True)
def _ready(lib_built):
    _lib.require_cuda()
    _lib.lib()


@pytest.fixture(autouse=True)
def _loop(monkeypatch):
    _loopback.install(monkeypatch)


def _report(what, info):
    info = dict(info, peak_gb=torch.cuda.max_memory_allocated() / 2 ** 30)
    print(f"\n[sharded] {what}: " + ", ".join(f"{k}={v:.4g}" if isinstance(v, float) else f"{k}={v}"
                                            for k, v in info.items()))


def _clone(t: batched.TopK) -> batched.TopK:
    return batched.TopK(t.scores.clone(), t.ids.clone(), t.counts.clone())


def _bits(x: torch.Tensor) -> torch.Tensor:
    return x.view(torch.int64 if x.element_size() == 8 else torch.int32)


def _assert_same(a: batched.TopK, b: batched.TopK, what: str, full_scores: bool = False):
    """counts, ids (the -1 padding included) and score bytes of every listed result equal; ``full_scores``: every
    score slot (the fused lists, which bench.py's digest hashes whole)."""
    k = a.ids.shape[1]
    valid = torch.arange(k, device=a.ids.device)[None, :] < a.counts[:, None].long()
    diff = (_bits(a.scores) != _bits(b.scores))
    if not full_scores:
        diff &= valid
    bad = (a.counts != b.counts) | (a.ids != b.ids).any(1) | diff.any(1)
    if bad.any():
        q = int(torch.nonzero(bad)[0])
        raise AssertionError(f"{what}: {int(bad.sum())} queries differ; first: query {q}, counts {int(a.counts[q])} vs "
                             f"{int(b.counts[q])}\n  ids {a.ids[q].tolist()}\n  vs  {b.ids[q].tolist()}\n  scores "
                             f"{a.scores[q].tolist()}\n  vs     {b.scores[q].tolist()}")


def _pack(lists):
    ptr = torch.tensor(np.cumsum([0] + [len(q) for q in lists]), dtype=torch.int32, device=DEV)
    terms = torch.tensor([t for q in lists for t in q] or [0], dtype=torch.int32, device=DEV)
    return ptr, terms


def _rankers(vec, stats, groups, canon, world, align, quantized=False, overlap=False, serial=False):
    """One shard-local CoarseRanker per rank, cut as bench.py's run_ours cuts (global statistics, global ids)."""
    n = vec.shape[0]
    out = []
    for r in range(world):
        lo, hi = ezdist.shard_bounds(n, world, r, align=align)
        dense = DenseIndex(vec[lo:hi], device=DEV, row_lo=lo, quantized=quantized,
                           doc_group=None if groups is None else groups[lo:hi])
        sparse = Bm25Index(stats, device=DEV, doc_lo=lo, doc_hi=hi, doc_group=groups)
        out.append(batched.CoarseRanker(dense, sparse, canon=canon, overlap=overlap, serial_routes=serial))
    return out


def _sharded_hybrid(rankers, calls, form=0):
    """Every rank runs ``ShardedCoarseRanker.hybrid(**c)`` for each ``c`` of ``calls`` (with the dense kernel form
    ``form`` forced in its thread); all ranks must return the same lists.  -> [(fused, sparse, dense)] of rank 0."""
    L = _lib.lib()

    def fn(h):
        _lib.check(L.ezr_dense_set_kernel(form))
        try:
            sh = ezdist.ShardedCoarseRanker(rankers[h.rank], group=h)
            res = []
            for c in calls:
                out = sh.hybrid(**c)
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


# ============================================================================ 1. the loopback collective itself
def test_loopback_all_gather_orders_ranks_and_propagates_errors():
    def fn(h):
        rec = torch.full((5,), h.rank + 1, dtype=torch.int32, device=DEV)
        out = torch.zeros(5 * 3, dtype=torch.int32, device=DEV)
        torch.distributed.all_gather_into_tensor(out, rec, group=h)
        assert torch.distributed.get_world_size(h) == 3 and torch.distributed.get_rank(h) == h.rank
        return out.cpu()
    outs = _loopback.run_ranks(3, fn)
    want = torch.arange(1, 4, dtype=torch.int32).repeat_interleave(5)
    assert all(torch.equal(o, want) for o in outs)

    def bad(h):
        if h.rank == 1:
            raise KeyError("rank 1 fails")
        torch.distributed.all_gather_into_tensor(torch.zeros(2, device=DEV), torch.zeros(1, device=DEV), group=h)
    with pytest.raises(KeyError, match="rank 1 fails"):
        _loopback.run_ranks(2, bad, timeout=60)


# ============================================================================ 2. ezr_merge_topk_parts
SCORE_SET = np.array([-1.5, -0.0, 0.0, 0.25, 1.0, 3.0])          # few values: ties across parts are common


def _random_parts(rng, G, Q, k, dtype):
    """G shards' canonical lists [G, Q, k]: distinct ids per shard (shard p owns [p * span, (p + 1) * span)), a
    random count in [0, k] per list, id -1 and a +inf score past it."""
    span = 2 * k + 3
    s = SCORE_SET[rng.integers(0, SCORE_SET.size, (G, Q, k))].astype(dtype)
    ids = np.argsort(rng.random((G, Q, span)), -1)[..., :k].astype(np.int32) + (np.arange(G) * span)[:, None, None]
    order = np.lexsort((-ids, -s), axis=-1)
    s, ids = np.take_along_axis(s, order, -1), np.take_along_axis(ids, order, -1).astype(np.int32)
    cnt = rng.integers(0, k + 1, (G, Q))
    past = np.arange(k)[None, None, :] >= cnt[..., None]
    return np.where(past, np.array(INF, dtype), s), np.where(past, -1, ids).astype(np.int32)


def _ref_merge(s, ids, k, ids_asc=False):
    """Plain reference: (score desc, id desc) over the valid candidates of all parts -> (ids [Q, k] -1 padded,
    scores [Q, k], counts [Q]).  ``ids_asc``: the opposite tie order (a negative control)."""
    G, Q, kin = s.shape
    s = np.transpose(s, (1, 0, 2)).reshape(Q, G * kin)
    i = np.transpose(ids, (1, 0, 2)).reshape(Q, G * kin)
    valid = i >= 0
    order = np.lexsort((i if ids_asc else -i, -np.where(valid, s, 0), (~valid).astype(np.int8)), axis=-1)[:, :k]
    cnt = np.minimum(valid.sum(1), k)
    keep = np.arange(k)[None, :] < cnt[:, None]
    return (np.where(keep, np.take_along_axis(i, order, -1), -1), np.take_along_axis(s, order, -1), cnt)


def _check_merge(got, ref, what):
    ri, rs, rc = ref
    gi, gs, gc = got.ids.cpu().numpy(), got.scores.cpu().numpy(), got.counts.cpu().numpy()
    keep = np.arange(ri.shape[1])[None, :] < rc[:, None]
    bits = np.int64 if gs.dtype == np.float64 else np.int32
    bad = (gc != rc) | (gi != ri).any(1) | ((gs.view(bits) != rs.view(bits)) & keep).any(1)
    if bad.any():
        q = int(np.nonzero(bad)[0][0])
        raise AssertionError(f"{what}: {int(bad.sum())} rows differ; first: row {q}, count {gc[q]} vs {rc[q]}\n  got ids "
                             f"{gi[q].tolist()}\n  want    {ri[q].tolist()}\n  got scores {gs[q].tolist()}\n  want "
                             f"{rs[q].tolist()}")


def _gathered(layout, parts):
    """The all-gathered buffer of G records whose four views hold ``parts[p]`` = (ds, di, ss, si) numpy arrays."""
    nb = layout.nbytes
    buf = torch.zeros(len(parts) * nb, dtype=torch.uint8, device=DEV)
    for p, arrs in enumerate(parts):
        for view, a in zip(ezdist.record_views(layout, buf[p * nb:(p + 1) * nb]), arrs):
            view.copy_(torch.from_numpy(np.ascontiguousarray(a)))
    return buf


def test_merge_topk_parts_against_lexsort():
    t0 = time.perf_counter()
    rng = np.random.default_rng(11)
    n, ties, zeros = 0, 0, 0
    for sb in (8, 4):
        sdt = np.float64 if sb == 8 else np.float32
        for G in (1, 2, 3, 8):
            for k in (1, 2, 10, 16, 17, 31, 32):
                for Q in (1, 7, 8, 9, 10003):
                    ds, di = _random_parts(rng, G, Q, k, np.float32)
                    ss, si = _random_parts(rng, G, Q, k, sdt)
                    layout = ezdist.RecordLayout(Q, k, sb)
                    buf = _gathered(layout, [(ds[p], di[p], ss[p], si[p]) for p in range(G)])
                    g_ds, g_di, g_ss, g_si = ezdist.record_views(layout, buf[:layout.nbytes])
                    md = batched.merge_topk_parts(g_ds, g_di, G, layout.nbytes, k)
                    ms = batched.merge_topk_parts(g_ss, g_si, G, layout.nbytes, k)
                    torch.cuda.synchronize()
                    what = f"G={G} k={k} Q={Q} sparse_bytes={sb}"
                    rd, rs_ = _ref_merge(ds, di, k), _ref_merge(ss, si, k)
                    _check_merge(md, rd, what + " dense")
                    _check_merge(ms, rs_, what + " sparse")
                    n += 2
                    for ref in (rd, rs_):
                        c = ref[2]
                        ties += int(((ref[1][:, :-1] == ref[1][:, 1:]) &
                                     (np.arange(1, k)[None, :] < c[:, None])).sum()) if k > 1 else 0
                        zeros += int(((ref[1] == 0) & (np.arange(k)[None, :] < c[:, None])).sum())
    # the negative control: the same check rejects the id-ascending tie order on these inputs
    G, k, Q = 8, 10, 10003
    ss, si = _random_parts(rng, G, Q, k, np.float64)
    layout = ezdist.RecordLayout(Q, k, 8)
    buf = _gathered(layout, [(np.zeros((Q, k), np.float32), np.full((Q, k), -1, np.int32), ss[p], si[p])
                             for p in range(G)])
    _, _, g_ss, g_si = ezdist.record_views(layout, buf[:layout.nbytes])
    ms = batched.merge_topk_parts(g_ss, g_si, G, layout.nbytes, k)
    _check_merge(ms, _ref_merge(ss, si, k), "control base")
    with pytest.raises(AssertionError, match="rows differ"):
        _check_merge(ms, _ref_merge(ss, si, k, ids_asc=True), "id-ascending tie order")
    _report("merge_topk_parts", dict(merges=n, equal_adjacent_scores=ties, zero_scores=zeros,
                                     seconds=time.perf_counter() - t0))


def test_merge_topk_parts_argument_errors():
    layout = ezdist.RecordLayout(9, 32, 8)
    buf = torch.full((3 * layout.nbytes,), 0xff, dtype=torch.uint8, device=DEV)      # ids -1 everywhere
    _, _, g_ss, g_si = ezdist.record_views(layout, buf[:layout.nbytes])
    assert batched.merge_topk_parts(g_ss, g_si, 3, layout.nbytes, 32).counts.sum().item() == 0
    with pytest.raises(_lib.EzrError, match="k=33"):
        batched.merge_topk_parts(g_ss, g_si, 3, layout.nbytes, 33)
    for stride in (layout.nbytes + 4, -layout.nbytes):
        with pytest.raises(_lib.EzrError, match="part_stride_bytes"):
            batched.merge_topk_parts(g_ss, g_si, 3, stride, 32)
    with pytest.raises(_lib.EzrError, match="n_parts"):
        batched.merge_topk_parts(g_ss, g_si, 0, layout.nbytes, 32)


# ============================================================================ BM25 duplicate documents
def _dup_tokens(c, n_docs, v0, n_dup, e_run, e_lo, D, E, f_ids=()):
    """``c`` (a synth corpus on the device) with (a) ``n_dup`` documents spread over the whole corpus replaced by
    copies of document D with term v0 appended three times, and (b) ``e_run`` consecutive documents from ``e_lo``
    replaced by copies of document E with term v0 + 1 appended (as tests/test_gpu_bm25_scale.py's ``corp``).
    ``f_ids``: documents replaced by copies of document D with term v0 + 2 appended once (a few copies, placed by the
    caller).  -> (tokens, doc_ptr, ids of the D copies, D's tokens)."""
    ptr_h = c.doc_ptr.cpu()
    tok = c.tokens
    a_ids = [int(x) for x in (torch.arange(n_dup) * (n_docs - 20) // (n_dup - 1) + 10)]
    a_ids = [d for d in a_ids if d not in (D, E) and d not in f_ids and not e_lo <= d < e_lo + e_run]
    d_new = torch.cat([tok[ptr_h[D]:ptr_h[D + 1]], torch.full((3,), v0, dtype=torch.int32, device=DEV)])
    e_new = torch.cat([tok[ptr_h[E]:ptr_h[E + 1]], torch.full((1,), v0 + 1, dtype=torch.int32, device=DEV)])
    f_new = torch.cat([tok[ptr_h[D]:ptr_h[D + 1]], torch.full((1,), v0 + 2, dtype=torch.int32, device=DEV)])
    runs = sorted([(d, d + 1, d_new) for d in a_ids] + [(d, d + 1, f_new) for d in f_ids] +
                  [(e_lo, e_lo + e_run, e_new.repeat(e_run))], key=lambda r: r[0])
    pieces, prev = [], 0
    for lo, hi, new in runs:
        pieces += [tok[ptr_h[prev]:ptr_h[lo]], new]
        prev = hi
    pieces.append(tok[ptr_h[prev]:])
    lens = ptr_h[1:] - ptr_h[:-1]
    lens[a_ids] = d_new.numel()
    lens[list(f_ids)] = f_new.numel()
    lens[e_lo:e_lo + e_run] = e_new.numel()
    doc_ptr = torch.zeros(n_docs + 1, dtype=torch.int64)
    torch.cumsum(lens, 0, out=doc_ptr[1:])
    tokens = torch.cat(pieces)
    assert tokens.numel() == int(doc_ptr[-1])
    return tokens, doc_ptr.to(DEV), a_ids, [int(t) for t in d_new[:-3].cpu()]


def _ints(rows, dim, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randint(-2, 3, (rows, dim), generator=g, device=DEV, dtype=torch.int8).to(torch.bfloat16)


# ============================================================================ 3. the route-output contract
@pytest.fixture(scope="module")
def small():
    """20k documents (3 BM25 ranges): 1300 copies of D over all ranges (the query [T_D] overflows a query's candidate
    list of 1024), 600 consecutive copies of E in range 1 (the query [T_E] overflows one CTA's local list of 512);
    integer dense vectors (dim 256), 77 queries."""
    n, v0, dim = 20_000, 4_000, 256
    c = synth.make_sparse_corpus(n, v0, 31, device=DEV)
    qs = synth.make_queries(c, 70, 32)
    tokens, doc_ptr, a_ids, d_tok = _dup_tokens(c, n, v0, 1300, 600, 8192 + 1000, 4242, 15_000)
    stats = Bm25Stats.from_tokens(tokens, doc_ptr, v0 + 2)
    groups = synth.make_groups(n, 4, 33, device=DEV)
    lists = [[int(t) for t in q] for q in qs.term_lists()]
    lists += [[v0], [v0 + 1], d_tok + [v0], [], [-1, v0 + 9], [v0, v0 + 1], [v0 + 1] * 3]
    qp, qt = _pack(lists)
    vec = _ints(n, dim, 34)
    q = _ints(len(lists), dim, 35)
    want = torch.tensor([(-1, 0, 1, 9)[i % 4] for i in range(len(lists))], dtype=torch.int32, device=DEV)
    index = Bm25Index(stats, device=DEV, doc_group=groups)
    assert index.post_pk is not None, "the two-phase BM25 path needs packed postings"
    return dict(n=n, v0=v0, stats=stats, groups=groups, lists=lists, qp=qp, qt=qt, vec=vec, q=q, want=want,
                index=index, a_ids=a_ids)


def _poisoned_record(nq, k, sparse_bytes):
    layout = ezdist.RecordLayout(nq, k, sparse_bytes)
    rec = torch.empty(layout.nbytes, dtype=torch.uint8, device=DEV)
    ds, di, ss, si = ezdist.record_views(layout, rec)
    ds.fill_(INF), ss.fill_(INF), di.fill_(POISON_ID), si.fill_(POISON_ID)
    return layout, rec, (ds, di, ss, si)


def _assert_padded(ids, counts, what):
    """The merge's precondition: id -1 in every slot past ``counts[q]``, a real id (>= 0, not the poison) before."""
    k = ids.shape[1]
    past = torch.arange(k, device=ids.device)[None, :] >= counts[:, None].long()
    assert bool(((counts >= 0) & (counts <= k)).all()), f"{what}: count out of [0, {k}]"
    bad = (past & (ids != -1)) | (~past & ((ids < 0) | (ids == POISON_ID)))
    if bad.any():
        q = int(torch.nonzero(bad.any(1))[0])
        raise AssertionError(f"{what}: a slot past the count is not -1 (or one before it is); query {q}, count "
                             f"{int(counts[q])}, ids {ids[q].tolist()}")


def _contract(layout, views, which, out, what):
    """``out``: the route's TopK, whose scores / ids are views ``which`` (0 dense, 2 sparse) of the record.  Checks the
    padding, then merges the record as a one-part gathered buffer: the merge must reproduce the route's list and no
    poison value may come out of it."""
    s, i = views[which], views[which + 1]
    assert out.ids.data_ptr() == i.data_ptr() and out.scores.data_ptr() == s.data_ptr()
    torch.cuda.synchronize()
    _assert_padded(i, out.counts, what)
    m = batched.merge_topk_parts(s, i, 1, layout.nbytes, layout.k)
    torch.cuda.synchronize()
    assert not bool((m.ids == POISON_ID).any()) and not bool(torch.isposinf(m.scores).any()), f"{what}: poison merged"
    _assert_same(m, batched.TopK(s, i, out.counts), f"{what}: merge of the record")
    return int(out.counts.sum())


def _dense_into(index, q, k, views, form=0, q_group=None, s8_cap=0):
    L = _lib.lib()
    out = batched.TopK(views[0], views[1], torch.empty(q.shape[0], dtype=torch.int32, device=DEV))
    _lib.check(L.ezr_dense_set_kernel(form))
    _lib.check(L.ezr_dense_s8_set_capacity(s8_cap))
    try:
        batched.dense_topk(index, q, k, q_group=q_group, out=out)
        torch.cuda.synchronize()
        ran = L.ezr_dense_last_kernel().decode()
    finally:
        L.ezr_dense_set_kernel(0)
        L.ezr_dense_s8_set_capacity(0)
    return out, ran


def test_route_contract_dense_forms(small):
    t0 = time.perf_counter()
    vec, q, g, n = small["vec"], small["q"], small["groups"], small["n"]
    idx = dict(full=DenseIndex(vec, device=DEV, row_lo=0, doc_group=g),
               shard=DenseIndex(vec[5000:13001], device=DEV, row_lo=5000, doc_group=g[5000:13001]),
               few=DenseIndex(vec[100:105], device=DEV, row_lo=100, doc_group=g[100:105]),
               empty=DenseIndex(vec[n:], device=DEV, row_lo=n, doc_group=g[n:]),
               s8=DenseIndex(vec[5000:13001], device=DEV, row_lo=5000, doc_group=g[5000:13001], quantized=True),
               s8_few=DenseIndex(vec[100:105], device=DEV, row_lo=100, doc_group=g[100:105], quantized=True),
               s8_empty=DenseIndex(vec[n:], device=DEV, row_lo=n, doc_group=g[n:], quantized=True))
    runs, kernels = 0, set()
    plan = [(1, (1, 10, 17, 32))] + [(f, (1, 10, 16)) for f in (2, 3, 4, 5)] + [(0, (17, 31, 32))]
    for form, ks in plan:
        for k in ks:
            for name in ("full", "shard", "few", "empty"):
                for qg in (None, small["want"]):
                    layout, _, views = _poisoned_record(q.shape[0], k, 8)
                    out, ran = _dense_into(idx[name], q, k, views, form, qg)
                    kernels.add(ran)
                    what = f"dense form {form} ({ran}) k={k} {name} filtered={qg is not None}"
                    _contract(layout, views, 0, out, what)
                    if qg is not None and idx[name].n_rows:
                        assert bool((out.counts[small["want"] == 9] == 0).all())
                    runs += 1
    for k in (1, 10, 16, 17, 32):
        for name in ("s8", "s8_few", "s8_empty"):
            for cap in (0, 1):                        # cap 1: every query overflows to the full scan
                for qg in (None, small["want"]):
                    layout, _, views = _poisoned_record(q.shape[0], k, 8)
                    out, ran = _dense_into(idx[name], q, k, views, q_group=qg, s8_cap=cap)
                    _contract(layout, views, 0, out, f"dense int8 k={k} {name} cap={cap} filtered={qg is not None}")
                    runs += 1
    assert {"simt", "wgmma", "wgmma-q64", "wgmma-q64-n128", "wgmma-q64-n128-mc2"} <= kernels, kernels
    _report("route contract, dense", dict(runs=runs, kernels=sorted(kernels), seconds=time.perf_counter() - t0))


def test_route_contract_bm25(small):
    t0 = time.perf_counter()
    st, n, g = small["stats"], small["n"], small["groups"]
    st1 = Bm25Stats.from_counts(n, st.vocab, int(st.doc_len.long().sum()), st.doc_len, st.df, st.indptr, st.post_doc,
                                st.post_tf, np.zeros(st.vocab, np.uint64), bm25_type=1)
    shard = Bm25Index(st, device=DEV, doc_lo=5000, doc_hi=13001, doc_group=g)
    idx = dict(full=small["index"], full_ordered=small["index"].ordered_view(), shard=shard,
               shard_ordered=shard.ordered_view(),
               few=Bm25Index(st, device=DEV, doc_lo=100, doc_hi=105, doc_group=g),
               empty=Bm25Index(st, device=DEV, doc_lo=n, doc_hi=n, doc_group=g),
               empty_mid=Bm25Index(st, device=DEV, doc_lo=7000, doc_hi=7000, doc_group=g),
               bm25s=Bm25Index(st1, device=DEV, doc_group=g),
               bm25s_shard=Bm25Index(st1, device=DEV, doc_lo=5000, doc_hi=13001, doc_group=g),
               bm25s_empty=Bm25Index(st1, device=DEV, doc_lo=n, doc_hi=n, doc_group=g))
    assert idx["empty"].n_ranges == 0 and idx["shard"].post_pk is not None
    runs, results = 0, 0
    for name, ix in idx.items():
        for k in (1, 10, 32):
            for qg in (None, small["want"]):
                sb = 8 if ix.score_dtype == torch.float64 else 4
                layout, _, views = _poisoned_record(len(small["lists"]), k, sb)
                out = batched.TopK(views[2], views[3], torch.empty(len(small["lists"]), dtype=torch.int32, device=DEV))
                batched.bm25_topk(ix, small["qp"], small["qt"], k, q_group=qg, out=out)
                results += _contract(layout, views, 2, out, f"bm25 {name} k={k} filtered={qg is not None}")
                runs += 1
    # the overflowed queries did produce full lists through the fallback
    full = batched.bm25_topk(small["index"], small["qp"], small["qt"], 32)
    tie_d, tie_e = len(small["lists"]) - 7, len(small["lists"]) - 6
    assert int(full.counts[tie_d]) == 32 and int(full.counts[tie_e]) == 32
    _report("route contract, bm25", dict(runs=runs, results=results, seconds=time.perf_counter() - t0))


def test_route_contract_negative_control(small):
    """A slot past the count written by hand is caught by the padding check, and the merge would take it."""
    layout, _, views = _poisoned_record(small["q"].shape[0], 10, 8)
    out, _ = _dense_into(DenseIndex(small["vec"][100:105], device=DEV, row_lo=100), small["q"], 10, views)
    torch.cuda.synchronize()
    _assert_padded(views[1], out.counts, "control base")
    assert int(out.counts[0]) == 5
    views[1][0, 7] = 4242
    with pytest.raises(AssertionError, match="past the count is not -1"):
        _assert_padded(views[1], out.counts, "one slot written past the count")
    m = batched.merge_topk_parts(views[0], views[1], 1, layout.nbytes, 10)
    assert 4242 in m.ids[0].tolist() and int(m.counts[0]) == 6


# ============================================================================ 4. configs[3] at benchmark scale
BENCH = SimpleNamespace(rows=1_000_000, dim=768, vocab=200_000, queries=10_000, k=10)
M_REF = 512


def _inputs_sha(data):
    """bench.py run_ours: what the committed digest was computed from."""
    q = data["queries"]
    h = hashlib.sha256()
    for t in (q.term_ptr, q.terms, data["qvec"].contiguous().view(torch.int16)):
        h.update(np.ascontiguousarray(t.cpu().numpy()).tobytes())
    h.update(str((int(data["vec"].view(torch.int16).to(torch.int64).sum()), data["n_tokens"],
                  int(data["stats"].post_doc.to(torch.int64).sum()))).encode())
    return h.hexdigest()


def test_configs3_at_bench_scale():
    t0 = time.perf_counter()
    torch.cuda.reset_peak_memory_stats()
    data = bench.make_data(BENCH, torch.device(DEV))
    stats, vec, qv = data["stats"], data["vec"], data["qvec"].contiguous()
    qs = data["queries"]
    qp, qt = qs.term_ptr.to(DEV), qs.terms.to(DEV)
    k = BENCH.k
    full = batched.CoarseRanker(DenseIndex(vec, device=DEV), Bm25Index(stats, device=DEV), canon=None, overlap=True)
    want = tuple(_clone(t) for t in full.hybrid(qv, qp, qt, k, k, k))
    torch.cuda.synchronize()
    del full
    info = dict(gen_s=data["gen_s"])
    results = {}
    for world, align in ((2, 64), (8, 64), (3, 1)):
        t1 = time.perf_counter()
        rankers = _rankers(vec, stats, None, None, world, align, overlap=True)
        bounds = [ezdist.shard_bounds(BENCH.rows, world, r, align=align) for r in range(world)]
        got = _sharded_hybrid(rankers, [dict(queries=qv, q_ptr=qp, q_terms=qt, k=k, k_out=k)])[0]
        del rankers
        for name, a, b in zip(("fused", "sparse", "dense"), got, want):
            _assert_same(a, b, f"G={world} align={align} {name}", full_scores=name == "fused")
        results[world] = got
        info[f"G{world}_s"] = time.perf_counter() - t1
        if world == 3:
            info["G3_cuts"] = [lo for lo, _ in bounds[1:]]
    assert all(int(b) % 64 != 0 for b in info["G3_cuts"]), "align 1 must cut through wgmma tiles and BM25 ranges"
    # the committed digest of the unsharded bench run
    with open(ROOT / "tests" / "golden" / "bench_digest.json") as f:
        entry = json.load(f).get(bench.digest_key(BENCH))
    sha = _inputs_sha(data)
    if entry is not None and entry["inputs_sha256"] == sha:
        assert bench.fused_digest(results[8][0]) == entry["fused_sha256"], "G=8 fused lists vs the committed digest"
        info["digest"] = "compared, equal"
    else:
        info["digest"] = "skipped: " + ("no committed entry" if entry is None else
                                        f"inputs_sha256 {sha[:12]} differs from the committed {entry['inputs_sha256'][:12]}")
        print(f"\n[sharded] committed digest NOT compared ({info['digest']})")
    fused, sparse, dense = results[8]
    # ---- independent references for the first 512 queries
    m = M_REF
    lists = [[int(t) for t in x] for x in qs.term_lists()[:m]]
    idf_dev = torch.from_numpy(stats.idf).to(DEV)
    P = stats.post_doc.numel()
    ref_w = torch.empty(P, dtype=torch.float64, device=DEV)
    for s in range(0, P, 1 << 25):
        e = min(P, s + (1 << 25))
        t = torch.searchsorted(stats.indptr[1:], torch.arange(s, e, device=DEV), right=True)
        ref_w[s:e] = okapi_weights(stats.post_tf[s:e], stats.doc_len[stats.post_doc[s:e].long()], idf_dev[t],
                                   stats.avgdl)
    ih = stats.indptr.cpu().numpy()
    ids_l, sc_l, cnt_l = [], [], []
    for b in range(0, m, 32):
        rows = torch.stack([okapi_row(x, ih, stats.post_doc, ref_w, stats.idf, BENCH.rows) for x in lists[b:b + 32]])
        i, s_, c_ = bm25_canonical_topk(rows, k)
        ids_l.append(i), sc_l.append(s_), cnt_l.append(c_)
    del ref_w
    r_ids, r_sc, r_cnt = torch.cat(ids_l), torch.cat(sc_l), torch.cat(cnt_l)
    assert torch.equal(sparse.counts[:m].long(), r_cnt) and torch.equal(sparse.ids[:m].long(), r_ids)
    keep = torch.arange(k, device=DEV)[None, :] < r_cnt[:, None]
    assert bool(((_bits(sparse.scores[:m]) == _bits(r_sc)) | ~keep).all()), "BM25 score bytes vs the reference"
    top_i, top_s, _ = fp64_top(qv[:m], vec, 16, integer=False)
    exact, delta = dense_score_bound(qv[:m], vec, dense.ids[:m].long())
    c_max = max(vec[i:i + 131072].double().norm(dim=1).max().item() for i in range(0, BENCH.rows, 131072))
    assert (dense.counts[:m] == k).all()
    dinfo = check_dense_topk(dense.scores[:m], dense.ids[:m], exact, delta, top_s, top_i, dense_delta_max(qv[:m], c_max),
                             BENCH.rows, "G=8 dense")
    f_ids, f_sc, f_cnt = fused.ids.cpu().numpy(), fused.scores.cpu().numpy(), fused.counts.cpu().numpy()
    s_ids, s_cnt, d_ids = sparse.ids.cpu().numpy(), sparse.counts.cpu().numpy(), dense.ids.cpu().numpy()
    for i in range(m):
        ri, rs = ort.rrf_ids([s_ids[i, :s_cnt[i]], d_ids[i, :k]], None, K=60, topk=k)
        assert f_cnt[i] == ri.size and np.array_equal(f_ids[i, :ri.size], ri), f"RRF ids, query {i}"
        assert f_sc[i, :ri.size].tobytes() == rs.tobytes(), f"RRF scores, query {i}"
    info.update(queries=BENCH.queries, ref_queries=m, dense_worst=dinfo["worst"], dense_ambiguous=dinfo["ambiguous"],
                seconds=time.perf_counter() - t0)
    _report("configs[3] at bench scale", info)


# ============================================================================ 5. constructed cases, 200k rows
N_MID, V_MID, DIM_MID = 200_000, 30_000, 256
NQ_MID, N_RCOPY = 300, 200


@pytest.fixture(scope="module")
def mid():
    """200k documents (25 BM25 ranges): 1500 copies of D and 200 copies of dense row R spread over the whole corpus
    (every shard of every split holds some, so the top-k ties straddle shard boundaries), 16 copies of F (D with
    another term), one per sixteenth of the corpus, so that the ten tied F copies of the query [T_F] come from two
    shards even at G = 2, and 600 consecutive copies of E;
    groups 5 and 6 only in the first / last 1000 rows (whole shards without a row of the group); the D copies and
    the R copies are duplicates of one text each (``canon``)."""
    t0 = time.perf_counter()
    n, v0 = N_MID, V_MID
    c = synth.make_sparse_corpus(n, v0, 41, device=DEV)
    qs = synth.make_queries(c, NQ_MID - 10, 42)
    f_ids = [j * (n // 16) + 5 for j in range(16)]
    tokens, doc_ptr, a_ids, d_tok = _dup_tokens(c, n, v0, 1500, 600, 10 * 8192 + 77, 4242, 150_000, f_ids)
    stats = Bm25Stats.from_tokens(tokens, doc_ptr, v0 + 3)
    del tokens, c
    lists = [[int(t) for t in q] for q in qs.term_lists()]
    lists += [[v0], [v0 + 1], d_tok + [v0], [], [-1, v0 + 9], [v0, v0 + 1], [v0 + 1] * 3, [v0 + 2], d_tok, [v0 + 2, 5]]
    qp, qt = _pack(lists)
    vec = _ints(n, DIM_MID, 43)
    r_pos = torch.arange(N_RCOPY, device=DEV) * (n - 1) // (N_RCOPY - 1)
    vec[r_pos] = vec[1234].clone()
    q = _ints(NQ_MID, DIM_MID, 44)
    q[-10:] = vec[1234].clone()
    groups = synth.make_groups(n, 4, 45, device=DEV)
    groups[:1000], groups[-1000:] = 5, 6
    canon = synth.make_duplicates(n, 0.03, 46, device=DEV)
    canon[torch.tensor(a_ids, device=DEV)] = min(a_ids)
    canon[r_pos] = int(r_pos.min())
    want = torch.tensor([(-1, 0, 5, 6, 9, 2)[i % 6] for i in range(NQ_MID)], dtype=torch.int32, device=DEV)
    # reference BM25 weights (float64 Okapi) of every posting
    idf_dev = torch.from_numpy(stats.idf).to(DEV)
    t = torch.searchsorted(stats.indptr[1:], torch.arange(stats.post_doc.numel(), device=DEV), right=True)
    ref_w = okapi_weights(stats.post_tf, stats.doc_len[stats.post_doc.long()], idf_dev[t], stats.avgdl)
    out = dict(stats=stats, lists=lists, qp=qp, qt=qt, vec=vec, q=q, groups=groups, canon=canon, want=want,
               ref_w=ref_w, a_ids=a_ids, r_pos=r_pos, cache={})
    _report("200k corpus", dict(docs=n, postings=stats.post_doc.numel(), copies_of_D=len(a_ids), copies_of_R=N_RCOPY,
                                queries=NQ_MID, seconds=time.perf_counter() - t0))
    return out


def _mid_ref(mid, k, filtered):
    """Canonical reference top-k of both routes (BM25 from tests/_bm25_ref.py, dense from tests/_topk_ref.py)."""
    key = (k, filtered)
    if key in mid["cache"]:
        return mid["cache"][key]
    st, g = mid["stats"], mid["groups"]
    want = mid["want"] if filtered else None
    ih = st.indptr.cpu().numpy()
    ids, sc, cnt = [], [], []
    for b in range(0, NQ_MID, 64):
        rows = torch.stack([okapi_row(x, ih, st.post_doc, mid["ref_w"], st.idf, N_MID) for x in mid["lists"][b:b + 64]])
        al = None
        if want is not None:
            w = want[b:b + 64]
            al = (w[:, None] == -1) | (g[None, :] == w[:, None])
        i, s, c = bm25_canonical_topk(rows, k, al)
        ids.append(i), sc.append(s), cnt.append(c)
    allowed = None
    if want is not None:
        allowed = lambda q0, q1, c0, c1: (want[q0:q1, None] == -1) | (g[None, c0:c1] == want[q0:q1, None])
    di, ds, dv = fp64_top(mid["q"], mid["vec"], k, integer=True, allowed=allowed)
    mid["cache"][key] = ((torch.cat(ids), torch.cat(sc), torch.cat(cnt)), (di, ds, dv))
    return mid["cache"][key]


def _assert_ref(res_s, res_d, ref, k, what):
    (si, ss, sc), (di, ds, dv) = ref
    s_cnt = sc.clamp(max=k)
    keep = torch.arange(k, device=DEV)[None, :] < s_cnt[:, None]
    want_s = batched.TopK(ss[:, :k].to(res_s.scores.dtype), torch.where(keep, si[:, :k], -1).int(), s_cnt.int())
    _assert_same(res_s, want_s, f"{what}: BM25 vs the reference")
    d_cnt = dv[:, :k].sum(1)
    want_d = batched.TopK(ds[:, :k].float(), torch.where(dv[:, :k], di[:, :k], -1).int(), d_cnt.int())
    _assert_same(res_d, want_d, f"{what}: dense vs the reference")


def _straddles(ref, k, world, align, n):
    """Queries whose k-th reference result ties the (k+1)-th and whose tied results among the top k + 1 come from more
    than one shard: the merge decides between shards at the cut.  -> [BM25, dense]."""
    cuts = torch.tensor([ezdist.shard_bounds(n, world, r, align=align)[1] for r in range(world)], device=DEV)
    out = []
    pos = torch.arange(k + 1, device=DEV)[None, :]
    for ids, sc, valid in ((ref[0][0], ref[0][1], pos < ref[0][2][:, None]), (ref[1][0], ref[1][1], ref[1][2])):
        ids, sc, valid = ids[:, :k + 1], sc[:, :k + 1], valid[:, :k + 1]
        shard = torch.searchsorted(cuts, ids.contiguous(), right=True)
        tied = valid & (sc == sc[:, k - 1:k]) & valid[:, k:k + 1]
        lo = torch.where(tied, shard, torch.full_like(shard, world)).min(1).values
        hi = torch.where(tied, shard, torch.full_like(shard, -1)).max(1).values
        out.append(int((tied[:, k] & (lo < hi)).sum()))
    return out


def test_constructed_cases_against_unsharded_and_references(mid):
    t0 = time.perf_counter()
    stats, vec, g, canon = mid["stats"], mid["vec"], mid["groups"], mid["canon"]
    full = batched.CoarseRanker(DenseIndex(vec, device=DEV, doc_group=g), Bm25Index(stats, device=DEV, doc_group=g),
                                canon=canon)
    ks = (1, 10, 16, 17, 32)
    runs, straddle = 0, {}
    for filtered in (False, True):
        ref = _mid_ref(mid, 33, filtered)
        for world, align in ((2, 64), (3, 1), (8, 64), (8, 8192)):
            straddle[f"G{world}a{align}{'f' if filtered else ''}"] = _straddles(ref, 10, world, align, N_MID)
    assert all(v[0] >= 1 for k_, v in straddle.items() if "f" not in k_), f"no BM25 tie at the 10th place: {straddle}"
    assert all(v[1] >= 1 for k_, v in straddle.items() if "f" not in k_), f"no dense tie at the 10th place: {straddle}"
    for world, align in ((2, 64), (3, 1), (8, 64), (8, 8192)):
        rankers = _rankers(vec, stats, g, canon, world, align)
        for filtered in (False, True):
            qg = mid["want"] if filtered else None
            calls, keys = [], []
            for k in ks:
                for k_out in sorted({1, k, 2 * k}):
                    calls.append(dict(queries=mid["q"], q_ptr=mid["qp"], q_terms=mid["qt"], k=k, k_out=k_out,
                                      q_group=qg))
                    keys.append((k, k_out))
            got = _sharded_hybrid(rankers, calls)
            ref = _mid_ref(mid, 33, filtered)
            for (k, k_out), res in zip(keys, got):
                what = f"G={world} align={align} k={k} k_out={k_out} filtered={filtered}"
                want = full.hybrid(mid["q"], mid["qp"], mid["qt"], k, k, k_out, q_group=qg)
                torch.cuda.synchronize()
                for name, a, b in zip(("fused", "sparse", "dense"), res, want):
                    _assert_same(a, b, f"{what} {name}", full_scores=name == "fused")
                _assert_ref(res[1], res[2], ref, k, what)
                if filtered:
                    assert bool((res[0].counts[mid["want"] == 9] == 0).all())
                runs += 1
        del rankers
    _report("constructed cases", dict(runs=runs, ties_at_10th_straddling_shards_bm25_dense=straddle,
                                      seconds=time.perf_counter() - t0))


def test_constructed_rrf_with_cross_shard_duplicates(mid):
    """``canon`` maps the D copies and the R copies (in every shard) to one text each: the fused lists of the G = 8
    ranker equal the oracle's ``rrf_ids`` over the merged lists, float64 bytes included."""
    rankers = _rankers(mid["vec"], mid["stats"], mid["groups"], mid["canon"], 8, 64)
    f, s, d = _sharded_hybrid(rankers, [dict(queries=mid["q"], q_ptr=mid["qp"], q_terms=mid["qt"], k=32, k_out=32)])[0]
    canon = mid["canon"].cpu().numpy()
    f_ids, f_sc, f_cnt = f.ids.cpu().numpy(), f.scores.cpu().numpy(), f.counts.cpu().numpy()
    s_ids, s_cnt, d_ids, d_cnt = s.ids.cpu().numpy(), s.counts.cpu().numpy(), d.ids.cpu().numpy(), d.counts.cpu().numpy()
    folded = 0
    for i in range(NQ_MID):
        ri, rs = ort.rrf_ids([s_ids[i, :s_cnt[i]], d_ids[i, :d_cnt[i]]], canon, K=60, topk=32)
        assert f_cnt[i] == ri.size and np.array_equal(f_ids[i, :ri.size], ri), f"RRF ids, query {i}"
        assert f_sc[i, :ri.size].tobytes() == rs.tobytes(), f"RRF scores, query {i}"
        folded += int(s_cnt[i] + d_cnt[i] - ri.size)
    assert folded > 0
    _report("RRF with duplicates across shards", dict(queries=NQ_MID, candidates_folded_by_canon=folded))


def test_constructed_bm25s_and_quantized_shards(mid):
    """bm25s (float32 sparse records) and int8-quantized dense shards, whose per-shard ``maxima`` differ from the
    corpus-wide ones, against the unsharded bf16 / bm25s ranker."""
    t0 = time.perf_counter()
    st, vec, g = mid["stats"], mid["vec"], mid["groups"]
    st1 = Bm25Stats.from_counts(N_MID, st.vocab, int(st.doc_len.long().sum()), st.doc_len, st.df, st.indptr,
                                st.post_doc, st.post_tf, np.zeros(st.vocab, np.uint64), bm25_type=1)
    full = batched.CoarseRanker(DenseIndex(vec, device=DEV, doc_group=g), Bm25Index(st1, device=DEV, doc_group=g),
                                canon=mid["canon"])
    maxima = []
    runs = 0
    for world, align in ((3, 1), (8, 64)):
        rankers = _rankers(vec, st1, g, mid["canon"], world, align, quantized=True)
        assert all(r.sparse.score_dtype == torch.float32 for r in rankers)
        maxima.append([tuple(round(x, 4) for x in r.dense.maxima.tolist()) for r in rankers])
        calls = [dict(queries=mid["q"], q_ptr=mid["qp"], q_terms=mid["qt"], k=k, k_out=k, q_group=qg)
                 for k in (1, 10, 16, 17, 32) for qg in (None, mid["want"])]
        got = _sharded_hybrid(rankers, calls)
        for c, res in zip(calls, got):
            want = full.hybrid(mid["q"], mid["qp"], mid["qt"], c["k"], c["k"], c["k"], q_group=c["q_group"])
            torch.cuda.synchronize()
            for name, a, b in zip(("fused", "sparse", "dense"), res, want):
                _assert_same(a, b, f"bm25s + int8 G={world} k={c['k']} {name}", full_scores=name == "fused")
            runs += 1
        del rankers
    assert len(set(maxima[1])) > 1, "the shards' maxima should differ"
    _report("bm25s + quantized shards", dict(runs=runs, shard_maxima_G8=maxima[1][:3], seconds=time.perf_counter() - t0))


def test_k_above_32_is_refused(mid):
    r = _rankers(mid["vec"][:1000], mid["stats"], None, None, 1, 1)[0]
    h = _loopback.Loopback(1).handles()[0]
    sh = ezdist.ShardedCoarseRanker(r, group=h)
    with pytest.raises(ValueError, match="k <= 32"):
        sh.hybrid(mid["q"], mid["qp"], mid["qt"], k=33, k_out=10)
    ro = batched.CoarseRanker(r.dense, r.sparse, overlap=True)
    with pytest.raises(ValueError, match="k <= 32"):
        ezdist.ShardedCoarseRanker(ro, group=h).submit(mid["q"], mid["qp"], mid["qt"], k=33, k_out=10)


def test_tiny_corpus_with_empty_ranks():
    """100 documents over G = 8 with align 64: ranks 2..7 hold no row and no document."""
    n, vocab, dim, nq = 100, 300, 256, 19
    c = synth.make_sparse_corpus(n, vocab, 51, mean_len=20, min_len=1, max_len=40)
    qs = synth.make_queries(c, nq, 52, min_terms=1, max_terms=6)
    stats = Bm25Stats.from_tokens(c.tokens, c.doc_ptr, vocab)
    vec = _ints(n, dim, 53)
    vec[60:70] = vec[3].clone()
    q = _ints(nq, dim, 54)
    q[0] = vec[3]
    groups = synth.make_groups(n, 3, 55, device=DEV)
    want = torch.tensor([(-1, 0, 1, 2, 7)[i % 5] for i in range(nq)], dtype=torch.int32, device=DEV)
    qp, qt = qs.term_ptr.to(DEV), qs.terms.to(DEV)
    bounds = [ezdist.shard_bounds(n, 8, r, align=64) for r in range(8)]
    assert bounds[:2] == [(0, 64), (64, 100)] and all(lo == hi == 100 for lo, hi in bounds[2:])
    full = batched.CoarseRanker(DenseIndex(vec, device=DEV, doc_group=groups),
                                Bm25Index(stats, device=DEV, doc_group=groups))
    runs = 0
    for quantized in (False, True):
        rankers = _rankers(vec, stats, groups, None, 8, 64, quantized=quantized)
        assert rankers[5].dense.n_rows == 0 and rankers[5].sparse.n_docs == 0 and rankers[5].sparse.n_ranges == 0
        calls = [dict(queries=q, q_ptr=qp, q_terms=qt, k=k, k_out=ko, q_group=qg)
                 for k in (1, 10, 32) for ko in (1, k) for qg in (None, want)]
        for c_, res in zip(calls, _sharded_hybrid(rankers, calls)):
            w = full.hybrid(q, qp, qt, c_["k"], c_["k"], c_["k_out"], q_group=c_["q_group"])
            torch.cuda.synchronize()
            for name, a, b in zip(("fused", "sparse", "dense"), res, w):
                _assert_same(a, b, f"tiny quantized={quantized} k={c_['k']} {name}", full_scores=name == "fused")
            if c_["k"] == 32 and c_["q_group"] is None:
                # every row is listed (k < 100 rows), in the canonical fp64 order
                di, ds, dv = fp64_top(q, vec, 32, integer=True)
                assert bool(dv.all()) and torch.equal(res[2].ids.long(), di)
                assert torch.equal(res[2].scores, ds.float())
            runs += 1
    _report("tiny corpus, empty ranks", dict(bounds=bounds[:3], runs=runs))


# ============================================================================ 6. the pipelined path
def _batches(mid):
    """Six batches of two sizes (300 and 150 queries), each a rotation of the query set (dense and sparse)."""
    out = []
    for i in range(6):
        nq = NQ_MID if i % 2 == 0 else NQ_MID // 2
        perm = [(j + 7 * i) % NQ_MID for j in range(nq)]
        qp, qt = _pack([mid["lists"][j] for j in perm])
        out.append((mid["q"][torch.tensor(perm, device=DEV)].contiguous(), qp, qt))
    return out


@pytest.mark.parametrize("serial", [False, True])
def test_submit_over_two_slots_equals_hybrid(mid, serial):
    world, k = 3, 10
    batches = _batches(mid)
    rankers = _rankers(mid["vec"], mid["stats"], mid["groups"], mid["canon"], world, 1)
    want = _sharded_hybrid(rankers, [dict(queries=b[0], q_ptr=b[1], q_terms=b[2], k=k, k_out=k) for b in batches])
    assert not torch.equal(want[0][0].ids, want[2][0].ids) and not torch.equal(want[1][0].ids, want[3][0].ids)
    r_o = [batched.CoarseRanker(r.dense, r.sparse, canon=mid["canon"], overlap=True, depth=2, serial_routes=serial)
           for r in rankers]

    def fn(h):
        sh = ezdist.ShardedCoarseRanker(r_o[h.rank], group=h)
        side = torch.cuda.Stream()
        got = []
        for b in batches:
            t = sh.submit(b[0], b[1], b[2], k=k, k_out=k)
            with torch.cuda.stream(side):
                t.wait(side)
                got.append(tuple(_clone(x) for x in (t.fused, t.sparse, t.dense)))
                t.release(side)
        sh.join()
        torch.cuda.synchronize()
        return got
    outs = _loopback.run_ranks(world, fn)
    for r, got in enumerate(outs):
        for i, (a, b) in enumerate(zip(got, want)):
            for name, x, y in zip(("fused", "sparse", "dense"), a, b):
                _assert_same(x, y, f"rank {r} batch {i} serial_routes={serial} {name}", full_scores=name == "fused")
    _report("submit", dict(ranks=world, batches=len(batches), serial_routes=serial,
                           slot_keys=len(r_o[0]._slots), submits=r_o[0]._n_submit))


def test_host_pipeline_over_the_sharded_ranker(mid):
    world, k = 3, 10
    batches = [b for b in _batches(mid) if b[0].shape[0] == NQ_MID]
    rankers = _rankers(mid["vec"], mid["stats"], mid["groups"], mid["canon"], world, 64)
    want = _sharded_hybrid(rankers, [dict(queries=b[0], q_ptr=b[1], q_terms=b[2], k=k, k_out=k) for b in batches])
    r_o = [batched.CoarseRanker(r.dense, r.sparse, canon=mid["canon"], overlap=True) for r in rankers]
    max_terms = max(int(b[2].numel()) for b in batches)

    def fn(h):
        sh = ezdist.ShardedCoarseRanker(r_o[h.rank], group=h)
        pipe = batched.HostPipeline(sh, NQ_MID, DIM_MID, max_terms, k, k)
        assert pipe.pipelined and pipe.sharded
        outs, keep = [], []
        for b in batches:
            ids = torch.empty(NQ_MID, k, dtype=torch.int32).pin_memory()
            sc = torch.empty(NQ_MID, k, dtype=torch.float64).pin_memory()
            keep.append([x.cpu().pin_memory() for x in b])
            pipe.step(*keep[-1], ids, sc)
            outs.append((ids, sc))
        pipe.drain()
        torch.cuda.synchronize()
        return outs
    for r, outs in enumerate(_loopback.run_ranks(world, fn)):
        for i, ((ids, sc), w) in enumerate(zip(outs, want)):
            assert torch.equal(ids, w[0].ids.cpu()), f"rank {r} step {i}: fused ids"
            assert torch.equal(sc.view(torch.int64), w[0].scores.cpu().view(torch.int64)), f"rank {r} step {i}: scores"
    _report("HostPipeline", dict(ranks=world, steps=len(batches)))
