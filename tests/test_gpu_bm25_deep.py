"""GPU: the deep form of the two-phase BM25 top-k (32 < k <= 1024, csrc/bm25_pk.cuh) on the benchmark corpus
(bench.py's 1M chunks, 200k vocabulary and seeds, 123 document ranges of 8192), bit for bit against the torch
restatement in tests/_bm25_ref.py, and the blocked score rows of every other k > 32 case.

Three groups of documents are rewritten (see ``corp``), each sized from the deep path's capacities
(pk_deep_local_cap(k) = 2k + 512 per (query, range), pk_deep_list_cap(k) = 4k + 1024 per query):

* D: 6000 copies spread over all ranges.  [T_D] ties 6000 documents, more than the per-query list holds at k = 1024
  (5120) and every smaller k: the query overflows to its score row.
* E: 3000 consecutive copies inside range 50.  [T_E] puts 3000 documents into one (query, range) CTA, more than its
  list holds at k = 1024 (2560) and every smaller k: that CTA overflows.
* F: 400 copies spread over all ranges.  [T_F] ties 400 documents across the ranges, straddling the 192nd place and
  below both capacities at k = 192, so the deep path itself must order the tie (ids descending).

What each case ran is printed (``pytest -s``).
"""
import time

import numpy as np
import pytest
import torch

from _bm25_ref import bm25s_row, bm25s_weights, canonical_topk, okapi_weights
from test_gpu_bm25_scale import _assert_topk, _chunks, _okapi_rows, _pack, _ref_topk, _same_bytes, _term_of
from easyrag_b200 import _lib, batched, synth
from easyrag_b200.index import Bm25Index, Bm25Stats

pytestmark = pytest.mark.gpu
DEV = "cuda"
SEED = 20240922 + 3            # bench.py's SEED: make_sparse_corpus(SEED), make_queries(SEED + 1)
N_DOCS, V0 = 1_000_000, 200_000
T_D, T_E, T_F = V0, V0 + 1, V0 + 2
VOCAB = V0 + 3
N_D, E_RUN, N_F = 6000, 3000, 400
KS = (33, 64, 192, 256, 288, 1023, 1024)
N_BATCH = 10_000               # bench.py's query batch
QB_ROWS = 256                  # queries per block of the Python-blocked score-row route


def local_cap(k):
    return 2 * k + 512         # csrc/bm25_pk.cuh pk_deep_local_cap


def list_cap(k):
    return 4 * k + 1024        # csrc/bm25_pk.cuh pk_deep_list_cap


def _report(what, info):
    info = dict(info, peak_gb=torch.cuda.max_memory_allocated() / 2 ** 30)
    print(f"\n[bm25-deep] {what}: " + ", ".join(f"{k}={v:.4g}" if isinstance(v, float) else f"{k}={v}"
                                              for k, v in info.items()))


@pytest.fixture(scope="module", autouse=True)
def _ready(lib_built):
    _lib.require_cuda()


@pytest.fixture(scope="module")
def corp():
    assert N_D > list_cap(1024) and E_RUN > local_cap(1024) and E_RUN < 8192 - 1000
    assert 192 < N_F < min(local_cap(192), list_cap(192))
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    c = synth.make_sparse_corpus(N_DOCS, V0, SEED, device=DEV)
    qs = synth.make_queries(c, 512, SEED + 1)
    batch = synth.make_queries(c, N_BATCH, SEED + 1)
    ptr_h = c.doc_ptr.cpu()
    tok = c.tokens
    D, E, F = 4242, 777_777, 31_337
    e0 = 50 * 8192 + 1000

    def spread(n, off):
        return [int(x) for x in (torch.arange(n) * (N_DOCS - 300) // (n - 1) + off)]
    a_ids = [d for d in spread(N_D, 100) if d not in (D, E, F) and not e0 <= d < e0 + E_RUN]
    f_ids = [d for d in spread(N_F, 150) if d not in (D, E, F) and d not in set(a_ids) and not e0 <= d < e0 + E_RUN]
    own = lambda d, t, n: torch.cat([tok[ptr_h[d]:ptr_h[d + 1]], torch.full((n,), t, dtype=torch.int32, device=DEV)])
    d_new, e_new, f_new = own(D, T_D, 3), own(E, T_E, 1), own(F, T_F, 2)
    runs = sorted([(d, d + 1, d_new) for d in a_ids] + [(d, d + 1, f_new) for d in f_ids] +
                  [(e0, e0 + E_RUN, e_new.repeat(E_RUN))], key=lambda r: r[0])
    pieces, prev = [], 0
    for lo, hi, new in runs:
        pieces += [tok[ptr_h[prev]:ptr_h[lo]], new]
        prev = hi
    pieces.append(tok[ptr_h[prev]:])
    lens = ptr_h[1:] - ptr_h[:-1]
    lens[a_ids] = d_new.numel()
    lens[f_ids] = f_new.numel()
    lens[e0:e0 + E_RUN] = e_new.numel()
    doc_ptr = torch.zeros(N_DOCS + 1, dtype=torch.int64)
    torch.cumsum(lens, 0, out=doc_ptr[1:])
    doc_ptr = doc_ptr.to(DEV)
    tokens = torch.cat(pieces)
    del pieces, tok, c
    assert tokens.numel() == int(doc_ptr[-1])

    stats = Bm25Stats.from_tokens(tokens, doc_ptr, VOCAB)
    groups = synth.make_groups(N_DOCS, 4, SEED + 7, device=DEV)
    index = Bm25Index(stats, device=DEV, doc_group=groups, packed=True)
    assert index.post_pk is not None and index.n_ranges == 123
    P = index.n_postings
    idf_dev = torch.from_numpy(stats.idf).to(DEV)
    ref_w = torch.empty(P, dtype=torch.float64, device=DEV)
    for s, e in _chunks(P):
        t = _term_of(stats.indptr, s, e)
        ref_w[s:e] = okapi_weights(stats.post_tf[s:e], stats.doc_len[stats.post_doc[s:e].long()], idf_dev[t],
                                   stats.avgdl)
    assert torch.equal(index.post_w.view(torch.int64), ref_w.view(torch.int64))

    df = stats.df.cpu().numpy()
    present = np.nonzero(df)[0]
    top = np.argsort(df, kind="stable")[-300:]
    rng = np.random.default_rng(8)
    mix = lambda m: [int(t) for t in rng.permutation(np.concatenate([rng.choice(top, m // 2),
                                                                       rng.choice(present, m - m // 2)]))]
    lists = [[int(t) for t in q] for q in qs.term_lists()]
    named = dict(plan17=mix(17), plan20=mix(20), batch40=mix(40), rescore100=mix(100),
                 huge4200=[int(t) for t in rng.choice(present, 4200)],
                 dup=[int(top[-1])] * 7 + [int(present[5])] + [int(top[-2])] * 3,
                 oov=[-1, -1, VOCAB + 5], empty=[], tieD=[T_D], tieE=[T_E], tieF=[T_F],
                 mixD=[int(t) for t in d_new[:-3].cpu()] + [T_D], mixF=[int(top[-3]), T_F])
    names = {}
    for nm, q in named.items():
        names[nm] = len(lists)
        lists.append(q)
    qp, qt = _pack(lists)
    bp = batch.term_ptr.to(device=DEV, dtype=torch.int32)
    bt = batch.terms.to(device=DEV, dtype=torch.int32)
    out = dict(stats=stats, index=index, groups=groups, ref_w=ref_w, indptr_h=stats.indptr.cpu().numpy(),
               lists=lists, names=names, qp=qp, qt=qt, a_ids=a_ids, f_ids=f_ids, doc_ptr=doc_ptr, batch=(bp, bt),
               batch_lists=[[int(t) for t in q] for q in batch.term_lists()], cache={})
    _report("corpus", dict(docs=N_DOCS, postings=P, queries=len(lists), copies_of_D=len(a_ids), copies_of_E=E_RUN,
                           copies_of_F=len(f_ids), batch=N_BATCH, seconds=time.perf_counter() - t0))
    return out


def _ref1024(corp):
    if "ref" not in corp["cache"]:
        corp["cache"]["ref"] = _ref_topk(corp, list(range(len(corp["lists"]))), 1024)
    return corp["cache"]["ref"]


def _blocked_rows_topk(index, qp, qt, k, q_group=None, id_base=0):
    """The score-row route in Python blocks: bm25_scores + select_rows(positive_only=True)."""
    parts = []
    nq = qp.numel() - 1
    for b in range(0, nq, QB_ROWS):
        e = min(nq, b + QB_ROWS)
        sub_p = qp[b:e + 1] - qp[b]
        sub_t = qt[int(qp[b]):int(qp[e])] if int(qp[e]) > int(qp[b]) else qt[:1]
        rows = batched.bm25_scores(index, sub_p, sub_t)
        parts.append(batched.select_rows(rows, k, positive_only=True, doc_group=index.doc_group if q_group is not None
                                         else None, q_group=None if q_group is None else q_group[b:e],
                                         id_base=id_base))
        del rows
    return batched.TopK(torch.cat([p.scores for p in parts]), torch.cat([p.ids for p in parts]),
                        torch.cat([p.counts for p in parts]))


# ------------------------------------------------------------------------------- 1. every k, bit exact
def test_deep_topk_bit_exact(corp):
    t0 = time.perf_counter()
    ref = _ref1024(corp)
    ids, sc, cnt = ref
    nm = corp["names"]
    rows = _okapi_rows(corp, [nm["tieD"], nm["tieE"], nm["tieF"]])
    n_tie = (rows == rows.max(1, keepdim=True).values).sum(1).tolist()
    assert n_tie == [len(corp["a_ids"]), E_RUN, len(corp["f_ids"])]
    assert n_tie[0] > list_cap(1024) and n_tie[1] > local_cap(1024) and 192 < n_tie[2] < list_cap(192)
    del rows
    L = _lib.lib()
    runs = {}
    L.ezr_profile_enable(1)
    try:
        for k in KS:
            L.ezr_profile_reset()
            a = batched.bm25_topk(corp["index"], corp["qp"], corp["qt"], k)
            torch.cuda.synchronize()
            n_cand, n_rescore = _lib.profile_read("bm25_cand")[1], _lib.profile_read("bm25_rescore")[1]
            n_rows = _lib.profile_read("bm25_score")[1]
            assert n_cand == 1 and n_rescore == 1, f"k={k}: the deep path did not run"
            assert n_rows >= 1, f"k={k}: the overflowed queries were not answered from score rows"
            _assert_topk(a, ref, k, f"deep k={k}", corp)
            b = batched.bm25_topk(corp["index"], corp["qp"], corp["qt"], k)
            assert _same_bytes(a, b), f"two calls differ at k={k}"
            runs[f"rows_blocks_k{k}"] = n_rows
    finally:
        L.ezr_profile_enable(0)
    straddle = int(((cnt > 192) & (sc[:, 191] == sc[:, 192])).sum())
    assert bool(cnt[nm["tieF"]] > 192) and bool(sc[nm["tieF"], 191] == sc[nm["tieF"], 192])
    _report("deep top-k", dict(queries=len(corp["lists"]), tie_at_192=straddle, **runs,
                               seconds=time.perf_counter() - t0))


# ------------------------------------------------------------------------- 2. filters, id_base, shards
def test_deep_filters_and_id_base(corp):
    nq = len(corp["lists"])
    pattern = torch.tensor([-1, 0, 1, 2, 3, 9], dtype=torch.int32, device=DEV)
    want = pattern[torch.arange(nq, device=DEV) % pattern.numel()]
    base = 2 ** 31 - 1 - N_DOCS
    ref = _ref_topk(corp, list(range(nq)), 192, want=want)
    r = batched.bm25_topk(corp["index"], corp["qp"], corp["qt"], 192, q_group=want, id_base=base)
    _assert_topk(r, ref, 192, "filtered k=192", corp, id_base=base)
    assert (r.counts[want == 9] == 0).all()


def test_deep_shards_merge_to_the_global_index(corp):
    st = corp["stats"]
    parts = []
    for lo, hi in [(0, 333_333), (333_333, 777_777), (777_777, N_DOCS)]:
        ix = Bm25Index(st, device=DEV, doc_lo=lo, doc_hi=hi)
        assert ix.post_pk is not None
        parts.append(batched.bm25_topk(ix, corp["qp"], corp["qt"], 192, id_base=lo))
        del ix
    merged = batched.merge_topk(torch.cat([r.scores for r in parts], 1).contiguous(),
                                torch.cat([r.ids for r in parts], 1).contiguous(), 192)
    _assert_topk(merged, _ref1024(corp), 192, "3 shards merged k=192", corp)


# -------------------------------------------------------- 3. blocked score rows: bm25s float32, negative idf
def test_blocked_rows_bm25s_float32(corp):
    t0 = time.perf_counter()
    st = corp["stats"]
    st1 = Bm25Stats.from_counts(N_DOCS, VOCAB, int(corp["doc_ptr"][-1]), st.doc_len, st.df, st.indptr, st.post_doc,
                                st.post_tf, np.zeros(VOCAB, np.uint64), bm25_type=1)
    ix = Bm25Index(st1, device=DEV)
    assert ix.post_w.dtype == torch.float32 and ix.post_pk is None
    idf32 = torch.from_numpy(st1.idf.astype(np.float32)).to(DEV)
    w32 = torch.empty(ix.n_postings, dtype=torch.float32, device=DEV)
    for s, e in _chunks(ix.n_postings):
        w32[s:e] = bm25s_weights(st.post_tf[s:e], st.doc_len[st.post_doc[s:e].long()],
                                 idf32[_term_of(st.indptr, s, e)], st1.avgdl)
    assert torch.equal(ix.post_w.view(torch.int32), w32.view(torch.int32))
    bp, bt = corp["batch"]
    qp, qt = bp[:2001] - bp[0], bt[:int(bp[2000])]
    got = batched.bm25_topk(ix, qp, qt, 192)
    want = _blocked_rows_topk(ix, qp, qt, 192)
    assert torch.equal(got.counts, want.counts) and torch.equal(got.ids, want.ids)
    assert torch.equal(got.scores.view(torch.int32), want.scores.view(torch.int32))
    # the reference rows for a sample
    df = st.df.cpu().numpy()
    sample = list(range(0, 2000, 50))
    rows = torch.stack([bm25s_row(corp["batch_lists"][i], corp["indptr_h"], st.post_doc, w32, df, N_DOCS)
                        for i in sample])
    ids, sc, cnt = canonical_topk(rows, 192)
    assert torch.equal(got.counts[sample].long(), cnt.clamp(max=192))
    valid = torch.arange(192, device=DEV)[None, :] < cnt.clamp(max=192)[:, None]
    assert torch.equal(got.ids[sample].long(), torch.where(valid, ids[:, :192], torch.full_like(ids[:, :192], -1)))
    assert bool(((got.scores[sample] == sc[:, :192].float()) | ~valid).all())
    _report("bm25s blocked rows", dict(queries=2000, k=192, seconds=time.perf_counter() - t0))


def test_blocked_rows_negative_idf():
    from oracle import bm25 as obm
    # five terms in ~90% of the documents and one in ~30%: the mean idf is negative (as in test_gpu_retrieval.py)
    rng = np.random.default_rng(17)
    docs = []
    for i in range(20_000):
        d = [t for t in range(5) if rng.random() < 0.9] * int(rng.integers(1, 3))
        if rng.random() < 0.3:
            d += [5] * int(rng.integers(1, 4))
        docs.append(np.array(d if d else [0], dtype=np.int32))
    tokens = torch.from_numpy(np.concatenate(docs)).to(torch.int32)
    ptr = torch.tensor(np.cumsum([0] + [len(d) for d in docs]), dtype=torch.int64)
    o = obm.OkapiCSR(docs, 6)
    ix = Bm25Index(Bm25Stats.from_tokens(tokens, ptr, 6), device=DEV)
    assert not ix.monotone and ix.post_pk is None
    lists = [[int(t) for t in rng.integers(0, 6, int(rng.integers(1, 7)))] for _ in range(2000)]
    qp, qt = _pack(lists)
    got = batched.bm25_topk(ix, qp, qt, 192)
    want = _blocked_rows_topk(ix, qp, qt, 192)
    assert torch.equal(got.counts, want.counts) and torch.equal(got.ids, want.ids)
    assert torch.equal(got.scores.view(torch.int64), want.scores.view(torch.int64))
    rows = torch.from_numpy(np.stack([o.get_scores(lists[i]) for i in range(0, 2000, 100)])).to(DEV)
    ids, sc, cnt = canonical_topk(rows, 192)
    sample = list(range(0, 2000, 100))
    assert torch.equal(got.counts[sample].long(), cnt.clamp(max=192))
    valid = torch.arange(192, device=DEV)[None, :] < cnt.clamp(max=192)[:, None]
    assert torch.equal(got.ids[sample].long(), torch.where(valid, ids[:, :192], torch.full_like(ids[:, :192], -1)))
    assert bool(((got.scores[sample].view(torch.int64) == sc[:, :192].view(torch.int64)) | ~valid).all())


# ------------------------------------------------------------------------------------- 4. batch scale
def test_batch_scale_k192(corp):
    t0 = time.perf_counter()
    L = _lib.lib()
    ix = corp["index"]
    bp, bt = corp["batch"]
    k = 192
    need = L.ezr_bm25_topk_workspace(ix.struct, N_BATCH, k)
    # per query: candidate ids, lower and upper bounds (4 B each) and exact scores (8 B) for list_cap(k) entries, the
    # plan table (32 ranges x 16 tokens x 8 B) and 8 ints of state; plus one block of score rows (at most 1 GiB) and
    # its select workspace (< 16 MiB)
    bound = N_BATCH * (20 * list_cap(k) + 4096 + 32 + 2048) + (1 << 30) + (1 << 24)
    assert need <= bound, (need, bound)
    assert need < N_BATCH * N_DOCS * 8 // 20
    torch.cuda.synchronize()
    t1 = time.perf_counter()
    got = batched.bm25_topk(ix, bp, bt, k)
    torch.cuda.synchronize()
    call_s = time.perf_counter() - t1
    want = _blocked_rows_topk(ix, bp, bt, k)
    assert torch.equal(got.counts, want.counts) and torch.equal(got.ids, want.ids)
    assert torch.equal(got.scores.view(torch.int64), want.scores.view(torch.int64))
    again = batched.bm25_topk(ix, bp, bt, k)
    assert _same_bytes(got, again)
    # a 512-query sample against the device reference
    sample = list(range(0, N_BATCH, N_BATCH // 512))[:512]
    sub = dict(corp, lists=[corp["batch_lists"][i] for i in sample], names={})
    ref = _ref_topk(sub, list(range(len(sample))), k)
    r = batched.TopK(got.scores[sample], got.ids[sample], got.counts[sample])
    _assert_topk(r, ref, k, "batch sample k=192", sub)
    _report("batch k=192", dict(queries=N_BATCH, workspace_gb=need / 2 ** 30, bound_gb=bound / 2 ** 30,
                                call_s=call_s, seconds=time.perf_counter() - t0))


def test_dual_sparse_fusion_at_batch_scale(corp):
    ix = corp["index"]
    bp, bt = corp["batch"]
    got = batched.dual_sparse_fusion(ix, ix, bp, bt, bp, bt, 192, 6, 256)
    a = _blocked_rows_topk(ix, bp, bt, 192)
    b = batched.bm25_topk(ix, bp, bt, 6)
    ib = torch.full((N_BATCH, 192), -1, dtype=torch.int32, device=DEV)
    sb = torch.zeros(N_BATCH, 192, dtype=torch.float64, device=DEV)
    ib[:, :6], sb[:, :6] = b.ids, b.scores
    want = batched.fusion_simple(a.ids, a.scores, a.counts, ib, sb, b.counts, 256)
    assert _same_bytes(got, want)
