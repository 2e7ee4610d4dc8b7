"""GPU: BM25 top-k on the benchmark corpus (bench.py configs[2]: 1M chunks, a 200k vocabulary, 123 document ranges of
8192) against the torch restatement in tests/_bm25_ref.py, bit for bit.

Smaller corpora never reach the code of the two-phase path (csrc/bm25_pk.cuh) that only runs at scale: the bound
updates between range chunks, the steady state at kPkMaxChunk (32) ranges per launch, the skip mask (a query's first
32 tokens), the plan table (16 tokens, later ones resolved inside the candidate CTAs), and the hand-off of overflowed
queries to the ordered kernel across all 123 ranges.  Two groups of documents are rewritten so that both overflow
routes are certain (see ``corp``), and constructed queries cross every token-count limit of the kernels.

The reference (tests/_bm25_ref.py, checked against the oracle classes in tests/test_bm25_ref_cpu.py) adds the terms
of a query in token order, exactly as rank_bm25 does; the kernels must return the same ids, counts and score bytes in
the canonical order (score descending, id descending).  What each case actually ran is printed (``pytest -s``).

The corpus has 2.97e8 tokens and 2.85e8 postings (the longest list 374,971).  Peak device memory of the whole file
was 14.3 GB on an H100 80GB HBM3 (700 W power limit), and the file ran in about 20 s there.  Per-posting reference
arithmetic goes in chunks of 2^25 postings and reference rows in blocks of 32 queries to keep that peak low.
"""
import time

import numpy as np
import pytest
import torch

from _bm25_ref import FIRST_ABSENT, bm25s_row, bm25s_weights, canonical_topk, counts, okapi_row, okapi_weights
from easyrag_b200 import _lib, batched, dist, synth
from easyrag_b200.index import Bm25Index, Bm25Stats
from oracle import bm25 as obm

pytestmark = pytest.mark.gpu
DEV = "cuda"
SEED = 20240922 + 3            # bench.py's SEED: make_sparse_corpus(SEED), make_queries(SEED + 1)
N_DOCS, V0 = 1_000_000, 200_000
T_D, T_E = V0, V0 + 1          # terms only the rewritten documents hold
VOCAB = V0 + 2
N_D, E_RUN = 3000, 600         # copies of D (spread over every range), consecutive copies of E (inside one range)
KPK_LIST_CAP, KPK_LOCAL_CAP, KPK_MAX_CHUNK, KPK_MAX_TERMS = 1024, 512, 32, 4096    # csrc/bm25_pk.cuh
DEFAULT_PLAN, DEFAULT_SKIP, DEFAULT_SPAN = 1, 0, 4                                 # csrc/bm25.cu
CH = 1 << 25                   # postings per chunk of the per-posting reference arithmetic
QB = 32                        # queries per block of 1M-column reference rows


def _report(what, info):
    info = dict(info, peak_gb=torch.cuda.max_memory_allocated() / 2 ** 30)
    print(f"\n[bm25-scale] {what}: " + ", ".join(f"{k}={v:.4g}" if isinstance(v, float) else f"{k}={v}"
                                                for k, v in info.items()))


@pytest.fixture(scope="module", autouse=True)
def _ready(lib_built):
    _lib.require_cuda()


def _chunks(n):
    for s in range(0, n, CH):
        yield s, min(n, s + CH)


def _term_of(indptr, s, e):
    """term of postings s..e-1 (indptr int64 on the device)."""
    return torch.searchsorted(indptr[1:], torch.arange(s, e, device=DEV), right=True)


def _pack(lists):
    ptr = torch.tensor(np.cumsum([0] + [len(q) for q in lists]), dtype=torch.int32, device=DEV)
    terms = torch.tensor([t for q in lists for t in q] or [0], dtype=torch.int32, device=DEV)
    return ptr, terms


# ------------------------------------------------------------------------------------------------- the corpus
@pytest.fixture(scope="module")
def corp():
    """bench.py's corpus and queries, with two groups of documents rewritten on the device:

    (a) ~3000 documents spread over all 123 ranges become copies of one document D with term T_D appended three
        times.  The query [T_D] then ties all copies exactly (same tf, same length) and scores 0 elsewhere: more ties
        than a query's candidate list holds (kPkListCap = 1024), so the query must overflow to the ordered kernel,
        which then runs over all 123 ranges.
    (b) 600 consecutive documents of range 50 become copies of another document E with T_E appended.  The query
        [T_E] puts 600 crossing documents into one (query, range) CTA, more than its local list holds
        (kPkLocalCap = 512): that CTA overflows.
    """
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    c = synth.make_sparse_corpus(N_DOCS, V0, SEED, device=DEV)
    qs = synth.make_queries(c, 512, SEED + 1)
    ptr_h = c.doc_ptr.cpu()
    tok = c.tokens
    D, E = 4242, 777_777
    e0 = 50 * 8192 + 1000
    a_ids = [int(x) for x in (torch.arange(N_D) * (N_DOCS - 200) // (N_D - 1) + 100)]
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
    indptr = stats.indptr
    # reference weights from the counted postings (checked against the restated counts in test_build_at_scale) and
    # the (term, document) key of every posting
    idf_dev = torch.from_numpy(stats.idf).to(DEV)
    ref_w = torch.empty(P, dtype=torch.float64, device=DEV)
    key = torch.empty(P, dtype=torch.int64, device=DEV)
    for s, e in _chunks(P):
        t = _term_of(indptr, s, e)
        d = stats.post_doc[s:e].long()
        ref_w[s:e] = okapi_weights(stats.post_tf[s:e], stats.doc_len[d], idf_dev[t], stats.avgdl)
        key[s:e] = t * N_DOCS + d

    # constructed queries
    df = stats.df.cpu().numpy()
    present = np.nonzero(df)[0]
    top = np.argsort(df, kind="stable")[-300:]                 # the longest posting lists
    rng = np.random.default_rng(8)
    mix = lambda m: [int(t) for t in rng.permutation(np.concatenate([rng.choice(top, m // 2),
                                                                       rng.choice(present, m - m // 2)]))]
    d_tokens = [int(t) for t in d_new[:-3].cpu()]
    lists = [[int(t) for t in q] for q in qs.term_lists()]
    named = dict(plan17=mix(17), plan20=mix(20), batch40=mix(40), batch40b=mix(40), rescore100=mix(100),
                 huge4200=[int(t) for t in rng.choice(present, 4200)],
                 dup=[int(top[-1])] * 7 + [int(present[5])] + [int(top[-2])] * 3,
                 oov=[-1, -1, VOCAB + 5], empty=[], tieD=[T_D], tieE=[T_E], mixD=d_tokens + [T_D])
    names = {}
    for nm, q in named.items():
        names[nm] = len(lists)
        lists.append(q)
    qp, qt = _pack(lists)
    prefix = 20_000
    out = dict(tokens=tokens, doc_ptr=doc_ptr, stats=stats, index=index, ordered=index.ordered_view(), groups=groups,
               ref_w=ref_w, key=key, indptr_h=indptr.cpu().numpy(), lists=lists, names=names, qp=qp, qt=qt,
               a_ids=a_ids, cache={},
               prefix_tokens=tokens[:int(doc_ptr[prefix])].clone(), prefix_ptr=doc_ptr[:prefix + 1].clone())
    _report("corpus", dict(docs=N_DOCS, vocab=VOCAB, tokens=int(doc_ptr[-1]), postings=P, ranges=index.n_ranges,
                           longest_list=int(df.max()), copies_of_D=len(a_ids), copies_of_E=E_RUN, queries=len(lists),
                           D_len=len(d_tokens), seconds=time.perf_counter() - t0))
    return out


def _okapi_rows(corp, qidx):
    st = corp["stats"]
    return torch.stack([okapi_row(corp["lists"][i], corp["indptr_h"], st.post_doc, corp["ref_w"], st.idf, N_DOCS)
                        for i in qidx])


def _ref_topk(corp, qidx, k, want=None, rows_fn=_okapi_rows):
    """canonical top-k of the reference rows of queries ``qidx``; ``want`` [len(qidx)] = q_group filter."""
    ids, sc, cnt = [], [], []
    for b in range(0, len(qidx), QB):
        blk = qidx[b:b + QB]
        rows = rows_fn(corp, blk)
        al = None
        if want is not None:
            w = want[b:b + QB]
            al = (w[:, None] == -1) | (corp["groups"][None, :] == w[:, None])
        i, s, c = canonical_topk(rows, k, al)
        ids.append(i), sc.append(s), cnt.append(c)
        del rows, al
    return torch.cat(ids), torch.cat(sc), torch.cat(cnt)


def _ref33(corp):
    """The unfiltered reference top-33 of every query (the top-k for every k <= 32, and the (k+1)-th for ties)."""
    if "ref33" not in corp["cache"]:
        corp["cache"]["ref33"] = _ref_topk(corp, list(range(len(corp["lists"]))), 33)
    return corp["cache"]["ref33"]


def _assert_topk(res, ref, k, what, corp, id_base=0):
    """ids, counts and score bytes of ``res`` equal to the reference top-k; the first differing query is named."""
    ids, sc, cnt = ref
    want_cnt = cnt.clamp(max=k)
    valid = torch.arange(k, device=DEV)[None, :] < want_cnt[:, None]
    want_ids = torch.where(valid, ids[:, :k] + id_base, torch.full_like(ids[:, :k], -1))
    bits = torch.int64 if res.scores.dtype == torch.float64 else torch.int32
    bad = (res.counts.long() != want_cnt) | (res.ids.long() != want_ids).any(1) | \
          ((res.scores.view(bits) != sc[:, :k].to(res.scores.dtype).view(bits)) & valid).any(1)
    if bad.any():
        qi = int(torch.nonzero(bad)[0])
        nm = [n for n, j in corp["names"].items() if j == qi]
        raise AssertionError(
            f"{what}: {int(bad.sum())} queries differ; first: query {qi} {nm} ({len(corp['lists'][qi])} tokens), count "
            f"{int(res.counts[qi])} vs {int(want_cnt[qi])}\n  got ids {res.ids[qi].tolist()}\n  want ids "
            f"{want_ids[qi].tolist()}\n  got scores {res.scores[qi].tolist()}\n  want scores {sc[qi, :k].tolist()}")


def _same_bytes(a, b):
    return (torch.equal(a.counts, b.counts) and torch.equal(a.ids, b.ids)
            and torch.equal(a.scores.view(torch.int64), b.scores.view(torch.int64)))


# ----------------------------------------------------------------------------------------- 1. build at scale
def test_build_at_scale(corp):
    t0 = time.perf_counter()
    st, ix = corp["stats"], corp["index"]
    tokens, doc_ptr = corp["tokens"], corp["doc_ptr"]
    key = corp["key"]
    # counts and postings, one placement block of 8192 documents at a time
    df = torch.zeros(VOCAB, dtype=torch.int64, device=DEV)
    first = torch.full((VOCAB,), FIRST_ABSENT, dtype=torch.int64, device=DEV)
    n_blocks = 0
    for lo in range(0, N_DOCS, 8192):
        hi = min(N_DOCS, lo + 8192)
        r = counts(tokens, doc_ptr, VOCAB, lo, hi)
        m = (st.post_doc >= lo) & (st.post_doc < hi)
        assert torch.equal(key[m], r["key"]), f"postings of block {lo // 8192}"
        assert torch.equal(st.post_tf[m].long(), r["tf"]), f"tf of block {lo // 8192}"
        assert torch.equal(st.doc_len[lo:hi].long(), r["doc_len"])
        df += r["df"]
        torch.minimum(first, r["first_pos"], out=first)
        n_blocks += 1
        del r, m
    assert n_blocks == 123
    assert torch.equal(st.df, df)
    indptr = torch.zeros(VOCAB + 1, dtype=torch.int64, device=DEV)
    torch.cumsum(df, 0, out=indptr[1:])
    assert torch.equal(st.indptr, indptr)
    assert bool((key[1:] > key[:-1]).all()), "postings not term-major with documents ascending"
    corp.pop("tokens")                                         # the raw corpus is not needed past this point
    # host-side statistics from the restated counts
    ref = Bm25Stats.from_counts(N_DOCS, VOCAB, int(doc_ptr[-1]), st.doc_len, df, indptr, st.post_doc[:0],
                                st.post_tf[:0], first.cpu().numpy().astype(np.uint64))
    assert st.avgdl == ref.avgdl and st.average_idf == ref.average_idf and st.idf.tobytes() == ref.idf.tobytes()
    # weights
    assert torch.equal(ix.post_w.view(torch.int64), corp["ref_w"].view(torch.int64))
    # range offsets: lower bound of each range's first document in the term's postings, for a sample of terms
    dfh = df.cpu().numpy()
    rng = np.random.default_rng(9)
    sample = np.unique(np.concatenate([np.argsort(dfh, kind="stable")[-40:], rng.choice(np.nonzero(dfh)[0], 300),
                                       [T_D, T_E], rng.choice(VOCAB, 20)]))
    ro = ix.range_off.view(VOCAB, ix.n_ranges + 1)
    starts = torch.arange(ix.n_ranges + 1, device=DEV, dtype=torch.int32) * 8192
    for t in sample.tolist():
        s, e = int(indptr[t]), int(indptr[t + 1])
        want = torch.searchsorted(st.post_doc[s:e], starts).to(torch.int32)
        assert torch.equal(ro[int(t)], want), f"range_off of term {t}"
    # packed postings and per-term maxima (definition as in test_bm25_pack_matches_definition)
    wbits = 32 - 13
    mask = (1 << wbits) - 1
    tmax = torch.zeros(VOCAB, dtype=torch.int64, device=DEV)
    for s, e in _chunks(ix.n_postings):
        w = ix.post_w[s:e]
        wq = torch.ceil(w * 2.0 ** ix.pk_scale_log2).long()
        assert int(wq.max()) < (1 << (wbits - 1)) and bool((wq[w > 0] >= 1).all())
        pk = ix.post_pk[s:e].long() & 0xffffffff
        assert torch.equal(pk >> wbits, (st.post_doc[s:e] % 8192).long())
        assert torch.equal(pk & mask, wq)
        tmax.scatter_reduce_(0, _term_of(st.indptr, s, e), wq, reduce="amax")
    assert torch.equal(ix.term_max.long(), tmax)
    _report("build", dict(blocks=n_blocks, longest_list=int(dfh.max()), terms_range_checked=sample.size,
                          seconds=time.perf_counter() - t0))


# --------------------------------------------------------------------------- 2. two-phase top-k, bit exact
def test_two_phase_topk_bit_exact(corp):
    t0 = time.perf_counter()
    ref = _ref33(corp)
    ids, sc, cnt = ref
    nm = corp["names"]
    # the constructed regimes are there: mass ties beyond the list capacities, 0 elsewhere
    rows = _okapi_rows(corp, [nm["tieD"], nm["tieE"]])
    n_tie = (rows == rows.max(1, keepdim=True).values).sum(1).tolist()
    assert n_tie[0] == len(corp["a_ids"]) > KPK_LIST_CAP and n_tie[1] == E_RUN > KPK_LOCAL_CAP
    assert int((rows > 0).sum()) == n_tie[0] + n_tie[1]
    del rows
    assert len(corp["lists"][nm["huge4200"]]) > KPK_MAX_TERMS
    L = _lib.lib()
    L.ezr_profile_enable(1)
    try:
        for k in (1, 10, 32):
            L.ezr_profile_reset()
            a = batched.bm25_topk(corp["index"], corp["qp"], corp["qt"], k)
            torch.cuda.synchronize()
            assert _lib.profile_read("bm25_cand")[1] == 1 and _lib.profile_read("bm25_rescore")[1] == 1
            _assert_topk(a, ref, k, f"two-phase k={k}", corp)
            b = batched.bm25_topk(corp["ordered"], corp["qp"], corp["qt"], k)
            assert _same_bytes(a, b), f"ordered view k={k}"
    finally:
        L.ezr_profile_enable(0)
    ties = {}
    for k in (1, 10, 32):
        straddle = (cnt > k) & (sc[:, k - 1] == sc[:, k])
        inside = ((sc[:, :k - 1] == sc[:, 1:k]) & (torch.arange(1, k, device=DEV)[None, :] < cnt[:, None])).any(1)
        ties[f"tie_at_kth_k{k}"] = int(straddle.sum())
        ties[f"tie_inside_k{k}"] = int(inside.sum())
    # score rows of 16 queries, byte for byte
    sel = list(range(8)) + [nm[x] for x in ("plan20", "batch40", "rescore100", "dup", "oov", "empty", "tieD", "mixD")]
    qp, qt = _pack([corp["lists"][i] for i in sel])
    got = batched.bm25_scores(corp["index"], qp, qt)
    want = _okapi_rows(corp, sel)
    assert torch.equal(got.view(torch.int64), want.view(torch.int64))
    del got, want
    _report("two-phase top-k", dict(queries=len(corp["lists"]), **ties, seconds=time.perf_counter() - t0))


# ------------------------------------------------------------------------------------- 3. switch matrix
def test_switch_matrix(corp):
    t0 = time.perf_counter()
    L = _lib.lib()
    ref = _ref33(corp)
    ix, qp, qt = corp["index"], corp["qp"], corp["qt"]
    base = {k: batched.bm25_topk(ix, qp, qt, k) for k in (1, 10, 32)}
    n = 0
    try:
        for plan in (0, 1):
            for skip in (0, 1):
                for span in (1, 4, 8, 32):
                    _lib.check(L.ezr_bm25_set_plan(plan))
                    _lib.check(L.ezr_bm25_set_skipping(skip))
                    _lib.check(L.ezr_bm25_set_span(span))
                    for k in (1, 10, 32):
                        r = batched.bm25_topk(ix, qp, qt, k)
                        what = f"plan={plan} skip={skip} span={span} k={k}"
                        _assert_topk(r, ref, k, what, corp)
                        assert _same_bytes(r, base[k]), what
                        n += 1
    finally:
        L.ezr_bm25_set_plan(DEFAULT_PLAN)
        L.ezr_bm25_set_skipping(DEFAULT_SKIP)
        L.ezr_bm25_set_span(DEFAULT_SPAN)
    _report("switch matrix", dict(runs=n, seconds=time.perf_counter() - t0))


# ------------------------------------------------------------------------------------- 4. chunk schedule
def _chunks_of(n_ranges, span):
    """pk_launch's range chunks (csrc/bm25.cu), restated: doubling from ``span`` after the first two chunks, no last
    chunk under half a span, at most kPkMaxChunk ranges (the plan table's size)."""
    out, r0, first = [], 0, span
    while r0 < n_ranges:
        ln = min(n_ranges - r0, span)
        if span < KPK_MAX_CHUNK and n_ranges - (r0 + ln) < span // 2:
            ln = n_ranges - r0
        ln = min(ln, KPK_MAX_CHUNK)
        out.append(ln)
        r0 += ln
        if r0 > first and span < KPK_MAX_CHUNK:
            span *= 2
    return out


def test_chunk_schedule_pinned(corp):
    assert _chunks_of(123, 4) == [4, 4, 8, 16, 32, 32, 27]
    assert _chunks_of(123, 32) == [32, 32, 32, 27]
    assert _chunks_of(18, 4) == [4, 4, 10]                  # the largest schedule the 140k-document test runs
    L = _lib.lib()
    qp, qt = _pack(corp["lists"][:16])

    def launches():
        torch.cuda.synchronize()
        a = L.ezr_launch_count()
        batched.bm25_topk(corp["index"], qp, qt, 10)
        torch.cuda.synchronize()
        return L.ezr_launch_count() - a

    seen = {}
    try:
        for span in (1, 4, 8, 32):
            _lib.check(L.ezr_bm25_set_span(span))
            _lib.check(L.ezr_bm25_set_plan(1))
            on = launches()
            _lib.check(L.ezr_bm25_set_plan(0))
            off = launches()
            seen[span] = _chunks_of(123, span)
            assert on - off == len(seen[span]), f"span {span}: {on - off} plan launches, {len(seen[span])} chunks"
    finally:
        L.ezr_bm25_set_plan(DEFAULT_PLAN)
        L.ezr_bm25_set_span(DEFAULT_SPAN)
    _report("chunk schedule", dict(ranges=corp["index"].n_ranges, **{f"span{s}": c for s, c in seen.items()}))


# ------------------------------------------------------------------------------------- 5. filters, id_base
def test_filters_and_id_base(corp):
    t0 = time.perf_counter()
    nq = len(corp["lists"])
    pattern = torch.tensor([-1, 0, 1, 2, 3, 9], dtype=torch.int32, device=DEV)      # 9: no document has it
    want = pattern[torch.arange(nq, device=DEV) % pattern.numel()]
    base = 2 ** 31 - 1 - N_DOCS
    ref = _ref_topk(corp, list(range(nq)), 32, want=want)
    for k in (10, 32):
        r = batched.bm25_topk(corp["index"], corp["qp"], corp["qt"], k, q_group=want, id_base=base)
        _assert_topk(r, ref, k, f"filtered k={k}", corp, id_base=base)
        assert (r.counts[want == 9] == 0).all()
        o = batched.bm25_topk(corp["ordered"], corp["qp"], corp["qt"], k, q_group=want, id_base=base)
        assert _same_bytes(r, o), f"ordered view, filtered k={k}"
    _report("filters", dict(queries=nq, id_base=base, results=int(ref[2].clamp(max=32).sum()),
                            seconds=time.perf_counter() - t0))


# ---------------------------------------------------------------------------------------------- 6. shards
def test_shards_equal_the_global_index(corp):
    t0 = time.perf_counter()
    st, gix, key = corp["stats"], corp["index"], corp["key"]
    ref = _ref33(corp)
    terms = torch.arange(VOCAB, device=DEV) * N_DOCS
    splits = {"8 shards": [dist.shard_bounds(N_DOCS, 8, r, align=64) for r in range(8)],
              "odd cuts": [(0, 333_333), (333_333, 777_777), (777_777, N_DOCS)]}
    for what, bounds in splits.items():
        parts = {10: [], 32: []}
        for lo, hi in bounds:
            ix = Bm25Index(st, device=DEV, doc_lo=lo, doc_hi=hi)
            a = torch.searchsorted(key, terms + lo)
            b = torch.searchsorted(key, terms + hi)
            want_ptr = torch.zeros(VOCAB + 1, dtype=torch.int64, device=DEV)
            torch.cumsum(b - a, 0, out=want_ptr[1:])
            assert torch.equal(ix.indptr, want_ptr), f"{what} [{lo}, {hi}): indptr"
            m = (st.post_doc >= lo) & (st.post_doc < hi)
            assert torch.equal(ix.post_doc, st.post_doc[m] - lo), f"{what} [{lo}, {hi}): postings"
            assert torch.equal(ix.post_w.view(torch.int64), gix.post_w[m].view(torch.int64)), f"{what}: weights"
            del m
            for k in parts:
                r = batched.bm25_topk(ix, corp["qp"], corp["qt"], k, id_base=lo)
                parts[k].append(r)
            del ix
        for k, rs in parts.items():
            merged = batched.merge_topk(torch.cat([r.scores for r in rs], 1).contiguous(),
                                        torch.cat([r.ids for r in rs], 1).contiguous(), k)
            _assert_topk(merged, ref, k, f"{what} merged k={k}", corp)
    _report("shards", dict(shards=[hi - lo for lo, hi in splits["8 shards"]][:2], seconds=time.perf_counter() - t0))


# --------------------------------------------------------------------------------------- 7. k > 32 at 1M columns
def test_large_k_score_rows(corp):
    t0 = time.perf_counter()
    nm = corp["names"]
    sel = [nm["tieD"], nm["tieE"], nm["mixD"], nm["dup"], nm["batch40"]] + list(range(7))
    ref = _ref_topk(corp, sel, 1024)
    qp, qt = _pack([corp["lists"][i] for i in sel])
    for k in (33, 256, 1024):
        r = batched.bm25_topk(corp["index"], qp, qt, k)
        _assert_topk(r, ref, k, f"k={k}", dict(corp, names={n: sel.index(j) for n, j in nm.items() if j in sel},
                                                lists=[corp["lists"][i] for i in sel]))
    _report("k > 32", dict(queries=len(sel), counts=ref[2].tolist()[:3], seconds=time.perf_counter() - t0))


# ----------------------------------------------------------------------------------------- 8. bm25s float32
def test_bm25s_float32_at_scale(corp):
    t0 = time.perf_counter()
    st = corp["stats"]
    # the same counted postings, bm25s statistics (its idf does not depend on the first-seen term order)
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
    nm = corp["names"]
    sel = list(range(116)) + [nm[x] for x in ("plan17", "plan20", "batch40", "rescore100", "huge4200", "dup", "oov",
                                              "empty", "tieD", "tieE", "mixD")]
    df = st.df.cpu().numpy()
    rows_fn = lambda c, qidx: torch.stack([bm25s_row(c["lists"][i], c["indptr_h"], st.post_doc, w32, df, N_DOCS)
                                           for i in qidx])
    ref = _ref_topk(corp, sel, 32, rows_fn=rows_fn)
    qp, qt = _pack([corp["lists"][i] for i in sel])
    sub = dict(corp, names={n: sel.index(j) for n, j in nm.items() if j in sel}, lists=[corp["lists"][i] for i in sel])
    for k in (1, 10, 32):
        _assert_topk(batched.bm25_topk(ix, qp, qt, k), ref, k, f"bm25s k={k}", sub)
    del ix, w32
    _report("bm25s", dict(queries=len(sel), ranges=123, seconds=time.perf_counter() - t0))


# --------------------------------------------------------------------------------- 9. the device reference
def test_device_reference_equals_okapi_csr(corp):
    tok, ptr = corp["prefix_tokens"], corp["prefix_ptr"]
    n = ptr.numel() - 1
    docs = [d for d in synth.SparseCorpus(tokens=tok.cpu(), doc_ptr=ptr.cpu(), vocab=VOCAB).doc_lists()]
    o = obm.OkapiCSR(docs, VOCAB)
    lists = corp["lists"][:20] + [corp["lists"][corp["names"][x]] for x in ("batch40", "dup", "oov", "tieD", "mixD")]
    for dev in (DEV, "cpu"):
        r = counts(tok.to(dev), ptr.to(dev), VOCAB)
        indptr = torch.zeros(VOCAB + 1, dtype=torch.int64, device=dev)
        torch.cumsum(r["df"], 0, out=indptr[1:])
        st = Bm25Stats.from_counts(n, VOCAB, int(ptr[-1]), r["doc_len"], r["df"], indptr, r["doc"], r["tf"],
                                   r["first_pos"].cpu().numpy().astype(np.uint64))
        assert st.idf.tobytes() == o.idf.tobytes()
        w = okapi_weights(r["tf"], r["doc_len"][r["doc"]], torch.from_numpy(st.idf).to(dev)[r["term"]], st.avgdl)
        assert w.cpu().numpy().tobytes() == np.concatenate([o.contributions(t) for t in np.nonzero(o.df)[0]]).tobytes()
        ih = indptr.cpu().numpy()
        for q in lists:
            got = okapi_row(q, ih, r["doc"], w, st.idf, n)
            assert got.device.type == torch.device(dev).type
            assert got.cpu().numpy().tobytes() == o.get_scores(q).tobytes(), (dev, q[:8])
    _report("device reference", dict(docs=n, queries=len(lists)))
