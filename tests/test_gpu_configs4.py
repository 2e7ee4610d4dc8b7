"""GPU: coarse ranking at the shape of BASELINE.json configs[4] -- 4M chunks, BGE-large's 1024 dims, BM25 and RRF,
batch-64 queries (``bench.py --rows 4000000 --dim 1024 --queries 64``) -- on one GPU and in simulated shards.

The 1M-row files (test_gpu_bm25_scale.py, test_gpu_dense_scale.py, test_gpu_sharded*.py) never reach what only a 4M
corpus reaches: 1.2e9 tokens (over 2^32 bytes), 1.14e9 postings (past 2^30; ``(int)indptr`` in csrc/bm25.cu holds
while P < 2^31, printed with its margin), 489 BM25 ranges (19 candidate launches per top-k call: 4, 4, 8, 16, then 32
at a time, the last 9), score rows of 4M float64 (16 queries per 1 GiB block:
``rows_carve`` gives a block query two rows), a bf16 corpus whose rows 2^20 and 2^21
start at bytes 2^31 and 2^32, an int8 mirror whose row 2^21 starts at byte 2^31, and G = 8 shards of 62 ranges.

1. ``test_dense_unit_vectors_and_int8``: the benchmark's unit vectors (make_dense_corpus(4M, 1024, SEED + 2), 64
   queries) through the wgmma top-10 within the derived error bound (tests/_bounds.py), the int8 quantizer against
   numpy on rows sampled over the whole mirror, and ``dense_s8_topk`` at the default capacity (every query overflows
   to the full scan) and at 2^20 against ``rescore_all``'s definition computed over row chunks, bit for bit.
2. ``test_index_build``: bench.py's sparse corpus with two rewritten document groups (see ``bm``) against
   tests/_bm25_ref.py: counts, postings, tf, lengths and first positions in 8 passes of 64 placement blocks, the host
   statistics, the float64 weights, ``range_off``, the packed postings and term maxima, and the G = 8 shard slices.
3. ``test_bm25_topk``: bench's 64 queries and constructed ones (the D and E ties, the plan, skip and kPkMaxTerms token
   limits) at k = 10, 32 (two-phase and ``ordered_view``) and 192, 1024 (deep), one filtered run, full score rows.
4. ``test_dense_integer_corpus``: integers in [-2, 2] (every fp32 sum exact) with 1500 and 300 copies of two rows
   spread up to row 4M - 1, 64 and 640 queries, forms 3, 4 and auto at k = 1, 10, 16, auto (SIMT) and form 6 at
   k = 288, 1024, a filtered run with id_base = 2^31 - 1 - 4M: all equal to the fp64 canonical top-k.
5. ``test_hybrid_and_shards``: ``CoarseRanker.hybrid`` (k = 10) and the pipeline depths (288 / 192 -> 256) on one GPU
   against the references of 3 and 4 and ``rrf_ids``; then ``ShardedCoarseRanker`` with G = 8 (align 64) and G = 3
   (align 1), simulated ranks through tests/_loopback.py, equal to the one-GPU lists bit for bit.  Both G ran.
6. ``test_bench_digest``: ``bench.make_data`` at 4M x 1024, 64 queries (the unmodified corpus), the one-GPU fused
   lists of all 64 queries against the references, and ``bench.fused_digest`` against the committed entry of
   tests/golden/bench_digest.json when the inputs match (said so when they do not).

Each comparison names the first differing query, and each is shown to reject a copy of a result with one score bit
flipped or two ids swapped.  What each part ran is printed (``pytest -s``): P = 1,141,097,135 postings (a margin of
1.0e9 to 2^31), 1,190,434,062 tokens, 489 ranges and placement blocks, 19 candidate launches at k = 10 and 192, D tied
2999 times and E 600 times, the queries the two-phase path handed on (read from its workspace: tieD and tieE at
k = 10 and 32, tieD at 192, asserted), and every one of the 64 queries over the int8 default capacity (none at 2^20).

The parts run in file order: they share the module fixtures and free what later parts no longer need (``_alive``
fails with that explanation when a part runs out of order).

Measured on an H100 80GB HBM3 (700 W power limit), each part's seconds read after a device synchronisation: unit
vectors and int8 3.6 s, corpus 1.0 s, build check 1.7 s, BM25 top-k 1.0 s, integer corpus 0.3 s, integer dense 2.6 s,
hybrid and shards 1.2 s, digest 1.0 s; the file 12.8 s from its first fixture (23 s with the start-up).  The fp64
references are small next to that: the largest, the top-1024 of 640 integer queries, is 2 x 640 x 4e6 x 1024 =
5.2e12 flop.  Peak device memory of the whole file (``torch.cuda.max_memory_allocated``) was 40.7 GiB, reached with
the G = 8 shard indexes.  Reference rows go in blocks of 32 queries and per-posting arithmetic in chunks of 2^25
postings to keep that peak low.  The file skips, saying so, when the GPU has less than NEED_GIB free: the peak plus
room for the CUDA context, the allocator's cache and the kernels' workspaces.
"""
import gc
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
from _bm25_ref import FIRST_ABSENT, counts, okapi_row, okapi_weights, postings_of_docs
from _bounds import check_dense_topk, dense_delta_max, dense_score_bound, rejects
from _topk_ref import fp64_top
from test_gpu_bm25_scale import _assert_topk, _chunks, _chunks_of, _pack, _ref_topk, _same_bytes, _term_of
from test_gpu_dense_s8 import canonical_topk as s8_topk
from test_gpu_dense_s8 import np_quantize, rescore_all, run_s8
from test_gpu_dense_scale import _assert_exact, _ints, _schedule
from test_gpu_sharded import _assert_same, _clone, _rankers, _sharded_hybrid
from test_gpu_sharded_deep import _sharded, _unsharded
from easyrag_b200 import _lib, batched, synth
from easyrag_b200 import dist as ezdist
from easyrag_b200.index import Bm25Index, Bm25Stats, DenseIndex
from oracle import retrieve as ort

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import bench                                   # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
SEED = bench.SEED
N, DIM, NQ, V0 = 4_000_000, 1024, 64, 200_000
T_D, T_E = V0, V0 + 1                          # terms only the rewritten documents hold
VOCAB = V0 + 2
RANGE = 8192
N_RANGES = 489
N_D, E_RUN, E_RANGE = 3000, 600, 480           # copies of D (spread over every range), of E (inside range 480)
KPK_LIST_CAP, KPK_LOCAL_CAP, KPK_MAX_TERMS = 1024, 512, 4096     # csrc/bm25_pk.cuh
GROUP_DOCS = 64 * RANGE                        # documents per counting pass of the build check (8 passes)
S8_DEFAULT_CAP, S8_MAX_CAP = 4096, 1 << 20     # csrc/dense_s8.cu
NEED_GIB = 48
BENCH4 = SimpleNamespace(rows=N, dim=DIM, vocab=V0, queries=NQ, k=10)
_LIVE = []                                     # the module's large fixtures, emptied before the digest part
_T0 = [0.0]


def _alive(d, *keys):
    """The parts share module fixtures and free them as they go (``tokens`` after the build check, the global BM25
    index before the shards, everything before the digest part), so they must run in file order."""
    gone = [k for k in keys if k not in d]
    if gone:
        pytest.fail(f"{gone} already freed: the parts of this file run in file order and free what later parts do not "
                    f"need (run the whole file, without reordering)", pytrace=False)


def _overflowed(ws, nq, k, n_ranges):
    """Queries the two-phase path handed on (to the ordered kernel at k <= 32, to their score rows in the deep form),
    read from the call's workspace: ``ovf_n`` and ``ovf_list`` of ``pk_carve`` (csrc/bm25.cu), which starts after
    the k <= 32 path's candidate scores and ids and at offset 0 in the deep form."""
    align = lambda x: (x + 255) // 256 * 256
    n = nq * n_ranges * k
    base = align(n * 8) + align(n * 4) if k <= 32 else 0
    buf = ws.buf
    n_ovf = int(buf[base + 24 * nq:base + 24 * nq + 4].view(torch.int32))
    assert 0 <= n_ovf <= nq, f"k={k}: {n_ovf} overflowed queries of {nq}: the workspace layout changed"
    lst = buf[base + align((6 * nq + 1) * 4):].narrow(0, 0, 4 * n_ovf).view(torch.int32).tolist()
    assert len(set(lst)) == n_ovf and all(0 <= q < nq for q in lst), f"k={k}: overflow list {lst}"
    return sorted(lst)


def deep_list_cap(k):
    return 4 * k + 1024                        # csrc/bm25_pk.cuh pk_deep_list_cap


def _report(what, info):
    """Prints a part's figures; the caller's seconds are read after this synchronises, so they include its kernels."""
    torch.cuda.synchronize()
    info = {k: (v() if callable(v) else v) for k, v in info.items()}
    info = dict(info, peak_gb=torch.cuda.max_memory_allocated() / 2 ** 30)
    print(f"\n[configs4] {what}: " + ", ".join(f"{k}={v:.4g}" if isinstance(v, float) else f"{k}={v}"
                                             for k, v in info.items()))


@pytest.fixture(scope="module", autouse=True)
def _ready(lib_built):
    _lib.require_cuda()
    free, _ = torch.cuda.mem_get_info()
    if free < NEED_GIB * 2 ** 30:
        pytest.skip(f"configs[4] at full size (4M x 1024, 1.1e9 postings) needs {NEED_GIB} GiB of free device memory; "
                    f"{free / 2 ** 30:.1f} GiB are free")
    torch.cuda.reset_peak_memory_stats()
    _T0[0] = time.perf_counter()


@pytest.fixture(autouse=True)
def _loop(monkeypatch):
    _loopback.install(monkeypatch)


# ------------------------------------------------------------------------------------------------ controls
def _flip(t, q, j, bit):
    """A copy of ``t`` with bit ``bit`` of score [q, j] flipped."""
    s = t.scores.clone()
    v = s.view(torch.int64 if s.element_size() == 8 else torch.int32)
    v[q, j] ^= 1 << bit
    return batched.TopK(s, t.ids.clone(), t.counts.clone())


def _swap(t, q, a, b):
    ids = t.ids.clone()
    ids[q, a], ids[q, b] = t.ids[q, b], t.ids[q, a]
    return batched.TopK(t.scores.clone(), ids, t.counts.clone())


def _fails(fn, *args, **kw):
    """True when the exact comparison ``fn`` rejects (a negative control)."""
    try:
        fn(*args, **kw)
    except AssertionError as e:
        assert "differ" in str(e), e
        return True
    return False


def _controls(check, res, what, bit=0):
    """``check(result)`` must reject a copy of ``res`` with the lowest (or ``bit``) score bit of the first result of
    a query flipped, and one with its first two ids swapped."""
    q = int(torch.nonzero((res.counts >= 2) & (res.ids[:, 0] != res.ids[:, 1]))[0])
    assert check(_flip(res, q, 0, bit)), f"{what}: a flipped score bit passed"
    assert check(_swap(res, q, 0, 1)), f"{what}: two swapped ids passed"


def _assert_rrf(fused, s_ids, s_cnt, d_ids, d_cnt, k_out, what):
    """``fused`` [Q, >= k_out] equal to ``rrf_ids([sparse, dense])`` of the given lists (host arrays) of every query:
    count, ids and score bytes; the first differing query is named."""
    f_ids, f_sc, f_cnt = fused.ids.cpu().numpy(), fused.scores.cpu().numpy(), fused.counts.cpu().numpy()
    bad = []
    for i in range(f_ids.shape[0]):
        ri, rs = ort.rrf_ids([s_ids[i, :s_cnt[i]], d_ids[i, :d_cnt[i]]], None, K=60, topk=k_out)
        if not (f_cnt[i] == ri.size and np.array_equal(f_ids[i, :ri.size], ri)
                and f_sc[i, :ri.size].tobytes() == rs.tobytes()):
            bad.append((i, ri, rs))
    if bad:
        i, ri, rs = bad[0]
        raise AssertionError(f"{what}: {len(bad)} queries differ; first: query {i}, count {f_cnt[i]} vs {ri.size}\n"
                             f"  got ids {f_ids[i, :f_cnt[i]].tolist()}\n  want ids {ri.tolist()}\n"
                             f"  got scores {f_sc[i, :f_cnt[i]].tolist()}\n  want scores {rs.tolist()}")


def _ref_lists(ref, k, id_base=0):
    """(ids, counts) host arrays of the first k places of a reference (ids, scores, counts) of tests/_bm25_ref.py."""
    ids, _, cnt = ref
    return (ids[:, :k] + id_base).cpu().numpy(), cnt.clamp(max=k).cpu().numpy()


def _dense_lists(ref, k):
    """The same of an fp64_top reference (ids, scores, valid)."""
    return ref[0][:, :k].cpu().numpy(), ref[2][:, :k].sum(1).cpu().numpy()


# =============================================================== 1. unit vectors and the int8 mirror at 4M x 1024
def _run_dense(index, q, k, form, name, q_group=None):
    L = _lib.lib()
    res = batched.dense_topk(index, q, k, q_group=q_group, form=form or None)
    torch.cuda.synchronize()
    ran = L.ezr_dense_last_kernel()
    assert ran == name, f"k={k} form {form}: {ran} ran, not {name}"
    return res


def _c_max(c):
    return max(c[i:i + 131072].double().norm(dim=1).max().item() for i in range(0, c.shape[0], 131072))


def _assert_s8(out, ref, k, what):
    """ids, counts and score bits of an int8-path result equal to ``s8_topk`` of the rescore rows."""
    ids, sc, cnt = ref
    valid = torch.arange(k, device=DEV)[None, :] < cnt[:, None].long()
    bad = (out.counts != cnt) | (torch.where(valid, out.ids, -1) != torch.where(valid, ids, -1)).any(1) | \
          ((torch.where(valid, out.scores, 0.0).view(torch.int32) != torch.where(valid, sc, 0.0).view(torch.int32))
           .any(1))
    if bad.any():
        qi = int(torch.nonzero(bad)[0])
        raise AssertionError(f"{what}: {int(bad.sum())} queries differ; first: query {qi}, count {int(out.counts[qi])} "
                             f"vs {int(cnt[qi])}\n  got ids {out.ids[qi].tolist()}\n  want ids {ids[qi].tolist()}\n"
                             f"  got scores {out.scores[qi].tolist()}\n  want scores {sc[qi].tolist()}")


def test_dense_unit_vectors_and_int8():
    t0 = time.perf_counter()
    c = synth.make_dense_corpus(N, DIM, SEED + 2, device=DEV)
    q = synth.make_dense_queries(c, NQ, SEED + 3)
    info = {}
    # bf16 wgmma top-10 within the derived bound
    sch = _schedule(4, N, DIM, NQ)
    res = _run_dense(DenseIndex(c, device=DEV), q, 10, 0, b"wgmma-q64-n128")
    assert (res.counts == 10).all()
    top_i, top_s, _ = fp64_top(q, c, 16, integer=False)
    exact, delta = dense_score_bound(q, c, res.ids.long())
    dmax = dense_delta_max(q, _c_max(c))
    chk = lambda r, e, dl: check_dense_topk(r.scores, r.ids, e, dl, top_s, top_i, dmax, N, "unit vectors")
    d_info = chk(res, exact, delta)
    assert rejects(chk, _flip(res, 0, 0, 22), exact, delta)    # a flipped high mantissa bit leaves the bound
    sw = _swap(res, 0, 0, 9)
    assert rejects(chk, sw, *dense_score_bound(q, c, sw.ids.long()))
    info.update(splits=sch["splits"], units_per_cta=sch["units_per_cta"], worst=d_info["worst"],
                ambiguous=d_info["ambiguous"])
    del exact, delta, top_i, top_s
    # the int8 mirror: quantizer on rows sampled over the whole mirror (rows 2^21 +- 1 start at byte 2^31), the last
    # rows included
    ix8 = DenseIndex(c, device=DEV, quantized=True)
    rng = np.random.default_rng(12)
    rows = np.unique(np.concatenate([rng.choice(N, 4000, replace=False), [0, 1, (1 << 20) - 1, 1 << 20, (1 << 21) - 1,
                                                                           1 << 21, (1 << 21) + 1],
                                     np.arange(N - 16, N)]))
    sel = torch.from_numpy(rows).to(DEV)
    r8, scale, e, nrm = np_quantize(c[sel].float().cpu().numpy())
    assert np.array_equal(ix8.rows_s8[sel].cpu().numpy(), r8)
    assert ix8.row_scale[sel].cpu().numpy().tobytes() == scale.tobytes()
    for got, ref in ((ix8.row_err[sel], e), (ix8.row_norm[sel], nrm)):
        g = got.cpu().numpy().astype(np.float64)
        assert (g >= ref * (1 - 2.0 ** -40)).all()               # fp64 sums in another order: 2^-40 slack
        assert (g - ref <= np.spacing(got.cpu().numpy()).astype(np.float64)).all()
    mx = ix8.maxima.cpu().numpy()
    assert mx[0] == ix8.row_err.max().item() and mx[1] == ix8.row_norm.max().item()
    # dense_s8_topk against rescore_all's definition
    ref = rescore_all(q, c, q_chunk=NQ, row_chunk=1 << 19)
    for k, cap in ((10, 0), (16, 0), (288, 0), (10, S8_MAX_CAP), (16, S8_MAX_CAP)):
        out, cc = run_s8(ix8, q, k, cap=cap)
        want = s8_topk(ref, k)
        what = f"int8 k={k} capacity {cap or S8_DEFAULT_CAP}"
        _assert_s8(out, want, k, what)
        if k == 10 and cap == 0:
            assert _fails(_assert_s8, _flip(out, 0, 0, 0), want, k, "control")
            assert _fails(_assert_s8, _swap(out, 0, 0, 1), want, k, "control")
        info[f"s8_k{k}_cap{cap or S8_DEFAULT_CAP}_overflowed"] = int((cc > (cap or S8_DEFAULT_CAP)).sum())
        info[f"s8_k{k}_cap{cap or S8_DEFAULT_CAP}_cand_mean"] = cc.float().mean().item()
    assert info[f"s8_k10_cap{S8_DEFAULT_CAP}_overflowed"] == NQ, "the default capacity no longer overflows (README)"
    del ref, ix8, res, c
    _report("unit vectors + int8", dict(info, queries=NQ, seconds=lambda: time.perf_counter() - t0))


# ====================================================================== 2-3. the BM25 corpus at 4M documents
@pytest.fixture(scope="module")
def bm():
    """bench.py's corpus and 64 queries, with two groups of documents rewritten on the device:

    (a) 3000 documents spread over all 489 ranges (up to document 4M - 101) become copies of document D with term T_D
        appended three times.  [T_D] ties all of them: more than a query's candidate list holds (kPkListCap = 1024)
        and than the deep list at k = 192 (pk_deep_list_cap = 1792), so the query overflows in both paths.
    (b) 600 consecutive documents of range 480 become copies of document E with T_E appended: the (query, range) CTA
        of [T_E] sees more crossing documents than its local list holds (kPkLocalCap = 512).

    The index weights are checked against ``okapi_weights`` here, chunk by chunk, so the reference rows below read
    ``index.post_w`` instead of a second 9 GB array."""
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    c = synth.make_sparse_corpus(N, V0, SEED, device=DEV)
    qs = synth.make_queries(c, NQ, SEED + 1)
    ptr_h = c.doc_ptr.cpu()
    tok = c.tokens
    D, E = 4242, 2_500_000
    e0 = E_RANGE * RANGE + 1000
    a_ids = [int(x) for x in (torch.arange(N_D) * (N - 200) // (N_D - 1) + 100)]
    a_ids = [d for d in a_ids if d not in (D, E) and not e0 <= d < e0 + E_RUN]
    d_new = torch.cat([tok[ptr_h[D]:ptr_h[D + 1]], torch.full((3,), T_D, dtype=torch.int32, device=DEV)])
    e_new = torch.cat([tok[ptr_h[E]:ptr_h[E + 1]], torch.full((1,), T_E, dtype=torch.int32, device=DEV)])
    runs = sorted([(d, d + 1, d_new) for d in a_ids] + [(e0, e0 + E_RUN, e_new.repeat(E_RUN))], key=lambda r: r[0])
    pieces, prev = [], 0
    for lo, hi, new in runs:
        pieces += [tok[ptr_h[prev]:ptr_h[lo]], new]
        prev = hi
    pieces.append(tok[ptr_h[prev]:])
    lens = ptr_h[1:] - ptr_h[:-1]
    lens[a_ids] = d_new.numel()
    lens[e0:e0 + E_RUN] = e_new.numel()
    doc_ptr = torch.zeros(N + 1, dtype=torch.int64)
    torch.cumsum(lens, 0, out=doc_ptr[1:])
    doc_ptr = doc_ptr.to(DEV)
    del c, tok
    tokens = torch.cat(pieces)
    del pieces
    assert tokens.numel() == int(doc_ptr[-1]) and tokens.numel() * 4 > 2 ** 32
    t_gen = time.perf_counter() - t0

    stats = Bm25Stats.from_tokens(tokens, doc_ptr, VOCAB)
    groups = synth.make_groups(N, 4, SEED + 7, device=DEV)
    index = Bm25Index(stats, device=DEV, doc_group=groups, packed=True)
    assert index.post_pk is not None and index.n_ranges == N_RANGES
    P = index.n_postings
    assert 2 ** 30 < P < 2 ** 31, P
    t_build = time.perf_counter() - t0 - t_gen
    _check_weights(stats, index)

    df = stats.df.cpu().numpy()
    present = np.nonzero(df)[0]
    top = np.argsort(df, kind="stable")[-300:]                 # the longest posting lists
    rng = np.random.default_rng(8)
    mix = lambda m: [int(t) for t in rng.permutation(np.concatenate([rng.choice(top, m // 2),
                                                                       rng.choice(present, m - m // 2)]))]
    d_tokens = [int(t) for t in d_new[:-3].cpu()]
    lists = [[int(t) for t in x] for x in qs.term_lists()]
    named = dict(plan17=mix(17), plan20=mix(20), batch40=mix(40), rescore100=mix(100),
                 huge4200=[int(t) for t in rng.choice(present, 4200)],
                 dup=[int(top[-1])] * 7 + [int(present[5])] + [int(top[-2])] * 3,
                 oov=[-1, -1, VOCAB + 5], empty=[], tieD=[T_D], tieE=[T_E], mixD=d_tokens + [T_D])
    names = {}
    for nm, x in named.items():
        names[nm] = len(lists)
        lists.append(x)
    qp, qt = _pack(lists)
    out = dict(tokens=tokens, doc_ptr=doc_ptr, stats=stats, index=index, groups=groups, lists=lists, names=names,
               qp=qp, qt=qt, a_ids=a_ids, indptr_h=stats.indptr.cpu().numpy(), cache={})
    _LIVE.append(out)
    _report("corpus", dict(docs=N, vocab=VOCAB, tokens=int(doc_ptr[-1]), token_bytes=int(doc_ptr[-1]) * 4,
                           postings=P, postings_margin_to_2_31=2 ** 31 - P, ranges=index.n_ranges,
                           longest_list=int(df.max()), copies_of_D=len(a_ids), copies_of_E=E_RUN, queries=len(lists),
                           generate_s=t_gen, build_s=t_build, seconds=lambda: time.perf_counter() - t0))
    return out


def _check_weights(stats, index):
    """``index.post_w`` bytes equal to ``okapi_weights`` of every posting, 2^25 postings at a time."""
    idf_dev = torch.from_numpy(stats.idf).to(DEV)
    for s, e in _chunks(index.n_postings):
        t = _term_of(stats.indptr, s, e)
        w = okapi_weights(stats.post_tf[s:e], stats.doc_len[stats.post_doc[s:e].long()], idf_dev[t], stats.avgdl)
        assert torch.equal(index.post_w[s:e].view(torch.int64), w.view(torch.int64)), f"post_w of postings [{s}, {e})"


def _inputs_sha(data):
    """bench.py run_ours's inputs_sha256, with its two int64 sums taken a chunk at a time (one int64 copy of the 4M x
    1024 corpus would take 33.5 GB; an int64 sum does not depend on the order)."""
    q = data["queries"]
    h = hashlib.sha256()
    for t in (q.term_ptr, q.terms, data["qvec"].contiguous().view(torch.int16)):
        h.update(np.ascontiguousarray(t.cpu().numpy()).tobytes())
    vec, pd = data["vec"].view(torch.int16), data["stats"].post_doc
    vsum = sum(int(vec[i:i + 131072].to(torch.int64).sum()) for i in range(0, vec.shape[0], 131072))
    psum = sum(int(pd[i:i + (1 << 26)].to(torch.int64).sum()) for i in range(0, pd.numel(), 1 << 26))
    h.update(str((vsum, data["n_tokens"], psum)).encode())
    return h.hexdigest()


def _rows(corp, qidx):
    st, ix = corp["stats"], corp["index"]
    return torch.stack([okapi_row(corp["lists"][i], corp["indptr_h"], st.post_doc, ix.post_w, st.idf, N)
                        for i in qidx])


def _ref1025(corp):
    """The unfiltered reference top-1025 of every query."""
    if "ref" not in corp["cache"]:
        corp["cache"]["ref"] = _ref_topk(corp, list(range(len(corp["lists"]))), 1025, rows_fn=_rows)
    return corp["cache"]["ref"]


def test_index_build(bm):
    t0 = time.perf_counter()
    _alive(bm, "tokens", "index")
    st, ix = bm["stats"], bm["index"]
    tokens, doc_ptr = bm["tokens"], bm["doc_ptr"]
    # counts and postings, GROUP_DOCS documents (64 placement blocks) per pass over the postings
    df = torch.zeros(VOCAB, dtype=torch.int64, device=DEV)
    first = torch.full((VOCAB,), FIRST_ABSENT, dtype=torch.int64, device=DEV)
    passes = blocks = 0
    for lo in range(0, N, GROUP_DOCS):
        hi = min(N, lo + GROUP_DOCS)
        r = counts(tokens, doc_ptr, VOCAB, lo, hi)
        g = postings_of_docs(st.indptr, st.post_doc, lo, hi)
        what = f"documents [{lo}, {hi})"
        assert torch.equal(g["term"], r["term"]) and torch.equal(g["doc"], r["doc"]), f"postings of {what}"
        assert torch.equal(st.post_tf[g["pos"]].long(), r["tf"]), f"tf of {what}"
        assert torch.equal(st.doc_len[lo:hi].long(), r["doc_len"]), f"doc_len of {what}"
        df += r["df"]
        torch.minimum(first, r["first_pos"], out=first)
        passes += 1
        blocks += -(-(hi - lo) // RANGE)
        del r, g
    assert passes == 8 and blocks == N_RANGES
    assert torch.equal(st.df, df)
    indptr = torch.zeros(VOCAB + 1, dtype=torch.int64, device=DEV)
    torch.cumsum(df, 0, out=indptr[1:])
    assert torch.equal(st.indptr, indptr)
    # term-major with documents ascending across the whole array (each document range above matched on its own)
    P = ix.n_postings
    for s, e in _chunks(P):
        a = max(s - 1, 0)
        key = _term_of(st.indptr, a, e) * N + st.post_doc[a:e].long()
        assert bool((key[1:] > key[:-1]).all()), f"postings [{a}, {e}) not term-major with documents ascending"
    del key
    bm.pop("tokens")                                           # the raw corpus is not needed past this point
    ref = Bm25Stats.from_counts(N, VOCAB, int(doc_ptr[-1]), st.doc_len, df, indptr, st.post_doc[:0], st.post_tf[:0],
                                first.cpu().numpy().astype(np.uint64))
    assert st.avgdl == ref.avgdl and st.average_idf == ref.average_idf and st.idf.tobytes() == ref.idf.tobytes()
    # range offsets of a sample of terms (the weights were checked in ``bm``)
    dfh = df.cpu().numpy()
    rng = np.random.default_rng(9)
    sample = np.unique(np.concatenate([np.argsort(dfh, kind="stable")[-40:], rng.choice(np.nonzero(dfh)[0], 300),
                                       [T_D, T_E], rng.choice(VOCAB, 20)]))
    ro = ix.range_off.view(VOCAB, ix.n_ranges + 1)
    starts = torch.arange(ix.n_ranges + 1, device=DEV, dtype=torch.int32) * RANGE
    for t in sample.tolist():
        s, e = int(indptr[t]), int(indptr[t + 1])
        assert torch.equal(ro[int(t)], torch.searchsorted(st.post_doc[s:e], starts).to(torch.int32)), \
            f"range_off of term {t}"
    # packed postings and per-term maxima (definition as in test_gpu_bm25_scale.py)
    wbits = 32 - 13
    mask = (1 << wbits) - 1
    tmax = torch.zeros(VOCAB, dtype=torch.int64, device=DEV)
    for s, e in _chunks(P):
        w = ix.post_w[s:e]
        wq = torch.ceil(w * 2.0 ** ix.pk_scale_log2).long()
        assert int(wq.max()) < (1 << (wbits - 1)) and bool((wq[w > 0] >= 1).all())
        pk = ix.post_pk[s:e].long() & 0xffffffff
        assert torch.equal(pk >> wbits, (st.post_doc[s:e] % RANGE).long()), f"packed documents of [{s}, {e})"
        assert torch.equal(pk & mask, wq), f"packed weights of [{s}, {e})"
        tmax.scatter_reduce_(0, _term_of(st.indptr, s, e), wq, reduce="amax")
    assert torch.equal(ix.term_max.long(), tmax)
    del w, wq, pk
    t_shards = time.perf_counter()
    # the G = 8 shard slices (bm25_shard_bounds / bm25_shard_copy) against the global postings filtered by document
    shard_ranges = []
    for r in range(8):
        lo, hi = ezdist.shard_bounds(N, 8, r, align=64)
        six = Bm25Index(st, device=DEV, doc_lo=lo, doc_hi=hi)
        g = postings_of_docs(st.indptr, st.post_doc, lo, hi)
        want_ptr = torch.zeros(VOCAB + 1, dtype=torch.int64, device=DEV)
        torch.cumsum(torch.bincount(g["term"], minlength=VOCAB), 0, out=want_ptr[1:])
        assert torch.equal(six.indptr, want_ptr), f"shard {r} [{lo}, {hi}): indptr"
        assert torch.equal(six.post_doc.long(), g["doc"] - lo), f"shard {r} [{lo}, {hi}): postings"
        assert torch.equal(six.post_w.view(torch.int64), ix.post_w[g["pos"]].view(torch.int64)), f"shard {r}: weights"
        shard_ranges.append(six.n_ranges)
        del six, g
    _report("build", dict(blocks=blocks, passes=passes, postings=P, terms_range_checked=sample.size,
                          shard_ranges=shard_ranges, shards_s=time.perf_counter() - t_shards,
                          seconds=lambda: time.perf_counter() - t0))


def test_bm25_topk(bm):
    t0 = time.perf_counter()
    _alive(bm, "index")
    ix, qp, qt, nm = bm["index"], bm["qp"], bm["qt"], bm["names"]
    ref = _ref1025(bm)
    info = {}
    # the constructed regimes are there: mass ties beyond the list capacities, 0 elsewhere
    rows = _rows(bm, [nm["tieD"], nm["tieE"]])
    n_tie = (rows == rows.max(1, keepdim=True).values).sum(1).tolist()
    assert n_tie[0] == len(bm["a_ids"]) > deep_list_cap(192) > KPK_LIST_CAP and n_tie[1] == E_RUN > KPK_LOCAL_CAP
    assert int((rows > 0).sum()) == n_tie[0] + n_tie[1]
    del rows
    assert len(bm["lists"][nm["huge4200"]]) > KPK_MAX_TERMS
    L = _lib.lib()
    L.ezr_profile_enable(1)
    try:
        for k in (10, 32, 192, 1024):
            L.ezr_profile_reset()
            ws = batched.Workspace(DEV)
            a = batched.bm25_topk(ix, qp, qt, k, ws=ws)
            torch.cuda.synchronize()
            assert _lib.profile_read("bm25_cand")[1] == 1 and _lib.profile_read("bm25_rescore")[1] == 1, \
                f"k={k}: the two-phase path did not run"
            ovf = _overflowed(ws, len(bm["lists"]), k, ix.n_ranges)
            names = sorted(n_ for n_, j in nm.items() if j in ovf)
            # [T_D] ties 2999 documents, more than the list holds (1024; 1792 at k = 192); [T_E] ties 600 in one range,
            # fewer than the list holds but more than one CTA's local list (512): only its local overflow hands it on
            if k <= 32:
                assert nm["tieD"] in ovf and nm["tieE"] in ovf, f"k={k}: overflowed {names}, not tieD and tieE"
            if k == 192:
                assert nm["tieD"] in ovf, f"k=192: overflowed {names}, not tieD"
                assert _lib.profile_read("bm25_score")[1] >= 1, "k=192: the overflowed queries got no score rows"
            info[f"overflowed_k{k}"] = names + [f"{len(ovf) - len(names)} bench queries"]
            info[f"score_row_launches_k{k}"] = _lib.profile_read("bm25_score")[1]
            _assert_topk(a, ref, k, f"two-phase k={k}", bm)
            b = batched.bm25_topk(bm["index"].ordered_view(), qp, qt, k)
            assert _same_bytes(a, b), f"ordered view k={k}"
            if k == 10:
                _controls(lambda r: _fails(_assert_topk, r, ref, k, "control", bm), a, "bm25")
    finally:
        L.ezr_profile_enable(0)
    # the chunk schedule over 489 ranges: one plan launch per range chunk
    assert _chunks_of(N_RANGES, 4) == [4, 4, 8, 16] + [32] * 14 + [9]
    sub_p, sub_t = _pack(bm["lists"][:16])

    def launches(k):
        torch.cuda.synchronize()
        n0 = L.ezr_launch_count()
        batched.bm25_topk(ix, sub_p, sub_t, k)
        torch.cuda.synchronize()
        return L.ezr_launch_count() - n0
    try:
        for k in (10, 192):
            _lib.check(L.ezr_bm25_set_plan(1))
            on = launches(k)
            _lib.check(L.ezr_bm25_set_plan(0))
            off = launches(k)
            assert on - off == 19, f"k={k}: {on - off} candidate launches, not 19"
            info[f"candidate_launches_k{k}"] = on - off
    finally:
        L.ezr_bm25_set_plan(1)
    # full score rows of 4M float64, byte for byte
    sel = list(range(4)) + [nm[x] for x in ("batch40", "huge4200", "dup", "oov", "empty", "tieD", "tieE", "mixD")]
    sp, st_ = _pack([bm["lists"][i] for i in sel])
    got = batched.bm25_scores(ix, sp, st_)
    want = _rows(bm, sel)
    assert torch.equal(got.view(torch.int64), want.view(torch.int64))
    del got, want
    # one filtered run with ids next to 2^31
    nq = len(bm["lists"])
    pattern = torch.tensor([-1, 0, 1, 2, 3, 9], dtype=torch.int32, device=DEV)      # 9: no document has it
    want_g = pattern[torch.arange(nq, device=DEV) % pattern.numel()]
    base = 2 ** 31 - 1 - N
    fref = _ref_topk(bm, list(range(nq)), 10, want=want_g, rows_fn=_rows)
    r = batched.bm25_topk(ix, qp, qt, 10, q_group=want_g, id_base=base)
    _assert_topk(r, fref, 10, "filtered k=10", bm, id_base=base)
    assert (r.counts[want_g == 9] == 0).all()
    assert _same_bytes(r, batched.bm25_topk(ix.ordered_view(), qp, qt, 10, q_group=want_g, id_base=base))
    _report("bm25 top-k", dict(info, queries=nq, D_ties=n_tie[0], list_cap=KPK_LIST_CAP,
                                deep_list_cap_192=deep_list_cap(192), E_ties=n_tie[1], local_cap=KPK_LOCAL_CAP,
                                seconds=lambda: time.perf_counter() - t0))


# =============================================================== 4. integer dense corpus at 4M x 1024, exact
N_R, N_S, NQ_BIG = 1500, 300, 640


@pytest.fixture(scope="module")
def dn():
    """Integers in [-2, 2]; rows R and S (entries +-2, so that no other row reaches R.R or S.S) copied 1500 and 300
    times over the whole corpus, the last row a copy of R.  Query 0 is R (1500 ties at the top, across every split and
    past row 2^21), query 1 is S (300 ties: the 288th place lies inside them), query 2 is zero (every score 0)."""
    t0 = time.perf_counter()
    c = _ints(N, DIM, -2, 2, 401)
    g = torch.Generator(device=DEV).manual_seed(402)
    pm2 = lambda: (torch.randint(0, 2, (DIM,), generator=g, device=DEV) * 4 - 2).to(torch.bfloat16)
    R, S = pm2(), pm2()
    r_pos = torch.arange(N_R, device=DEV) * (N - 1) // (N_R - 1)
    s_pos = torch.arange(N_S, device=DEV) * (N // N_S) + 7
    assert not torch.isin(s_pos, r_pos).any() and int(r_pos[-1]) == N - 1
    c[r_pos] = R
    c[s_pos] = S
    q = _ints(NQ_BIG, DIM, -2, 2, 403)
    q[0], q[1], q[2] = R, S, 0
    q[70] = R                                               # inside the 75 queries of the hybrid part too
    ref = fp64_top(q, c, 1024, integer=True)
    out = dict(c=c, q=q, ref=ref)
    _LIVE.append(out)
    _report("integer corpus", dict(rows=N, dim=DIM, queries=NQ_BIG, copies_of_R=N_R, copies_of_S=N_S,
                                   seconds=lambda: time.perf_counter() - t0))
    return out


def test_dense_integer_corpus(dn):
    t0 = time.perf_counter()
    _alive(dn, "c", "q", "ref")
    c, q, ref = dn["c"], dn["q"], dn["ref"]
    index = DenseIndex(c, device=DEV)
    assert index.vectors.data_ptr() == c.data_ptr()
    ids, sc, _ = ref
    assert (ids[0, :1024] >= 0).all() and int(ids[0, 0]) == N - 1 and (sc[0] == 4 * DIM).all()
    assert (sc[1, :N_S] == 4 * DIM).all() and (sc[1, N_S] < 4 * DIM)
    info, runs = {}, 0
    for nq in (NQ, NQ_BIG):
        sub = tuple(t[:nq] for t in ref)
        for form, name in ((3, b"wgmma-q64"), (4, b"wgmma-q64-n128"), (0, b"wgmma-q64-n128")):
            sch = _schedule(form or 4, N, DIM, nq)
            info[f"form{form or 4}_q{nq}"] = f"{sch['splits']}x{sch['rows_per_slice']}"
            for k in (1, 10, 16):
                res = _run_dense(index, q[:nq], k, form, name)
                _assert_exact(res, sub, k, f"{nq} queries form {form} k={k}", sch, qw=64)
                runs += 1
                if nq == NQ and form == 0 and k == 10:
                    _controls(lambda r: _fails(_assert_exact, r, sub, k, "control", sch), res, "dense")
        whole = dict(rows_per_slice=N)
        for form, name in ((0, b"simt"), (6, b"wgmma-scores")):
            for k in (288, 1024):
                res = _run_dense(index, q[:nq], k, form, name)
                _assert_exact(res, sub, k, f"{nq} queries form {form} k={k}", whole, qw=64)
                runs += 1
    # a filter, a class of three rows at the end of the corpus, ids next to 2^31
    groups = synth.make_groups(N, 4, 404, device=DEV)
    groups[-3:] = 7
    pattern = torch.tensor([-1, -2, 7, 0, 3], dtype=torch.int32, device=DEV)         # -2: no such class
    want = pattern[torch.arange(NQ, device=DEV) % 5]
    base = 2 ** 31 - 1 - N
    allowed = lambda q0, q1, c0, c1: (want[q0:q1, None] == -1) | (groups[None, c0:c1] == want[q0:q1, None])
    fref = fp64_top(q[:NQ], c, 288, integer=True, allowed=allowed)
    findex = DenseIndex(c, device=DEV, doc_group=groups, row_lo=base)
    for k, name in ((10, b"wgmma-q64-n128"), (288, b"simt")):
        res = _run_dense(findex, q[:NQ], k, 0, name, q_group=want)
        _assert_exact(res, fref, k, f"filtered k={k}", dict(rows_per_slice=N), id_base=base, qw=64)
        cnt = res.counts.long()
        assert (cnt[want == -2] == 0).all() and (cnt[want == 7] == 3).all() and (cnt[want == 0] == k).all()
        assert (res.ids[want == 7][:, :3].long() >= base + N - 3).all()
        runs += 1
    _report("dense integers", dict(info, runs=runs, seconds=lambda: time.perf_counter() - t0))


# =============================================================================== 5. hybrid, pipeline, shards
def test_hybrid_and_shards(bm, dn):
    t0 = time.perf_counter()
    _alive(bm, "index")
    _alive(dn, "c", "q", "ref")
    nq = len(bm["lists"])
    qp, qt = bm["qp"], bm["qt"]
    qv = dn["q"][:nq].contiguous()
    dref = tuple(t[:nq] for t in dn["ref"])
    sref = _ref1025(bm)
    dense = DenseIndex(dn["c"], device=DEV)
    # one GPU: hybrid at k = 10
    ranker = batched.CoarseRanker(dense, bm["index"], canon=None)
    f, s, d = (_clone(t) for t in ranker.hybrid(qv, qp, qt, 10, 10, 10))
    torch.cuda.synchronize()
    _assert_topk(s, sref, 10, "hybrid sparse", bm)
    _assert_exact(d, dref, 10, "hybrid dense", dict(rows_per_slice=N), qw=64)
    s_ids, s_cnt = _ref_lists(sref, 10)
    d_ids, d_cnt = _dense_lists(dref, 10)
    _assert_rrf(f, s_ids, s_cnt, d_ids, d_cnt, 10, "hybrid fused")
    _controls(lambda r: _fails(_assert_rrf, r, s_ids, s_cnt, d_ids, d_cnt, 10, "control"), f, "rrf")
    one_hybrid = (f, s, d)
    # one GPU at the pipeline's depths: dense_topk(288) + bm25_topk(192) + fuse_lists to 256
    one_pipe = tuple(_clone(t) for t in _unsharded(dense, bm["index"], qv, qp, qt, 288, 192, 256))
    pf, ps, pd = one_pipe
    _assert_topk(ps, sref, 192, "pipeline sparse", bm)
    _assert_exact(pd, dref, 288, "pipeline dense", dict(rows_per_slice=N), qw=64)
    s_ids, s_cnt = _ref_lists(sref, 192)
    d_ids, d_cnt = _dense_lists(dref, 288)
    _assert_rrf(pf, s_ids, s_cnt, d_ids, d_cnt, 256, "pipeline fused")
    info = dict(full_fused_256=int((pf.counts == 256).sum()))
    del ranker
    bm.pop("index")                                            # the shards below hold the whole index again
    gc.collect()
    torch.cuda.empty_cache()
    for world, align in ((8, 64), (3, 1)):
        t1 = time.perf_counter()
        rankers = _rankers(dn["c"], bm["stats"], None, None, world, align)
        bounds = [ezdist.shard_bounds(N, world, r, align=align) for r in range(world)]
        info[f"G{world}_ranges"] = [rk.sparse.n_ranges for rk in rankers]
        got = _sharded_hybrid(rankers, [dict(queries=qv, q_ptr=qp, q_terms=qt, k=10, k_out=10)])[0]
        for name, a, b in zip(("fused", "sparse", "dense"), got, one_hybrid):
            _assert_same(a, b, f"G={world} align={align} hybrid {name}", full_scores=name == "fused")
        if world == 8:
            _controls(lambda r: _fails(_assert_same, r, one_hybrid[0], "control", full_scores=True), got[0], "shards")
        got = _sharded(rankers, [dict(queries=qv, q_ptr=qp, q_terms=qt, k_dense=288, k_sparse=192, k_out=256)])[0]
        for name, a, b in zip(("fused", "sparse", "dense"), got, one_pipe):
            assert a.ids.shape == b.ids.shape, f"G={world} {name}: shape {tuple(a.ids.shape)} vs {tuple(b.ids.shape)}"
            _assert_same(a, b, f"G={world} align={align} pipeline {name}", full_scores=name == "fused")
        del rankers, got
        gc.collect()
        info[f"G{world}_s"] = time.perf_counter() - t1
        if world == 3:
            info["G3_cuts"] = [lo for lo, _ in bounds[1:]]
            assert all(b % 64 != 0 for b in info["G3_cuts"])
    _report("hybrid + shards", dict(info, queries=nq, seconds=lambda: time.perf_counter() - t0))


# ======================================================================== 6. the configs[4] bench digest
def test_bench_digest():
    for d in _LIVE:
        d.clear()
    gc.collect()
    torch.cuda.empty_cache()
    t0 = time.perf_counter()
    data = bench.make_data(BENCH4, torch.device(DEV))
    stats, vec, qv = data["stats"], data["vec"], data["qvec"].contiguous()
    qs = data["queries"]
    qp, qt = qs.term_ptr.to(DEV), qs.terms.to(DEV)
    k = BENCH4.k
    sparse_ix = Bm25Index(stats, device=DEV)
    full = batched.CoarseRanker(DenseIndex(vec, device=DEV), sparse_ix, canon=None, overlap=True)   # as bench.py N = 1
    f, s, d = (_clone(t) for t in full.hybrid(qv, qp, qt, k, k, k))
    torch.cuda.synchronize()
    del full
    digest, sha = bench.fused_digest(f), _inputs_sha(data)
    # BM25: the weights against okapi_weights, then the reference rows of all 64 queries
    _check_weights(stats, sparse_ix)
    lists = [[int(t) for t in x] for x in qs.term_lists()]
    corp = dict(stats=stats, index=sparse_ix, lists=lists, names={}, indptr_h=stats.indptr.cpu().numpy())
    sref = _ref_topk(corp, list(range(NQ)), k, rows_fn=_rows)
    _assert_topk(s, sref, k, "bench sparse", corp)
    # dense: fp64 within the derived bound
    top_i, top_s, _ = fp64_top(qv, vec, 16, integer=False)
    exact, delta = dense_score_bound(qv, vec, d.ids.long())
    assert (d.counts == k).all()
    dinfo = check_dense_topk(d.scores, d.ids, exact, delta, top_s, top_i, dense_delta_max(qv, _c_max(vec)), N,
                             "bench dense")
    # RRF over the lists the GPU produced
    s_ids, s_cnt = s.ids.cpu().numpy(), s.counts.cpu().numpy()
    d_ids, d_cnt = d.ids.cpu().numpy(), d.counts.cpu().numpy()
    _assert_rrf(f, s_ids, s_cnt, d_ids, d_cnt, k, "bench fused")
    with open(ROOT / "tests" / "golden" / "bench_digest.json") as fh:
        entry = json.load(fh).get(bench.digest_key(BENCH4))
    if entry is not None and entry["inputs_sha256"] == sha:
        assert digest == entry["fused_sha256"], "fused lists vs the committed configs[4] digest"
        state = "compared, equal"
    else:
        state = "NOT compared: " + ("no committed entry" if entry is None else
                                    f"inputs_sha256 {sha[:12]} differs from the committed "
                                    f"{entry['inputs_sha256'][:12]}")
        print(f"\n[configs4] committed digest {state}")
    _report("bench digest", dict(key=bench.digest_key(BENCH4), fused_sha256=digest, inputs_sha256=sha, digest=state,
                                 dense_worst=dinfo["worst"], dense_ambiguous=dinfo["ambiguous"],
                                 gen_s=data["gen_s"], seconds=lambda: time.perf_counter() - t0,
                                 file_seconds=lambda: time.perf_counter() - _T0[0]))
