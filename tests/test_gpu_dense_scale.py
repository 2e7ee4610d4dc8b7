"""GPU: the wgmma dense top-k (csrc/dense_tc.cu) at benchmark scale, where every persistent CTA walks several
(corpus split, query block) work units, against fp64 references.

At this scale the code that only runs from a CTA's second unit onward is exercised: the per-query seed (a unit starts
from the k-th score that earlier units of the same query published with ``atomicMax``), the reload of the query block
on a unit change (``a_empty`` / ``a_full`` phases; the register-held query chunks of the 128-query form), and ties
between ids of different splits once a seed is set.  Every case asserts, with a restatement of the kernel's cost model
(``ts_choose_splits`` / ``tc_rows_per_slice``) and the device's SM count, that it runs at least two units per CTA, so
a change of the cost model cannot quietly turn these into single-wave tests.

Integer inputs in [-2, 2] make every score exact in fp32, so ids, counts and score bits must equal the canonical
(score desc, id desc) fp64 top-k.  Unit vectors (the benchmark's data) are checked against fp64 with the kernel's own
error bound (tests/_bounds.py ``dense_score_bound``).  ``ezr_normalize_rows``, which every stored row and query goes
through, is checked against fp64 as well.  The measured figures are printed (``pytest -s``).
"""
import pytest
import torch

from _bounds import (NORM_FLOOR, check_bf16, check_dense_topk, dense_delta_max, dense_score_bound,
                     l2_normalize_exact_and_delta, rejects)
from _topk_ref import fp64_top
from easyrag_b200 import _lib, batched, synth
from easyrag_b200.index import DenseIndex, normalize_rows

pytestmark = pytest.mark.gpu
DEV = "cuda"
N_ROWS = 1_000_000
N_ODD = 1_000_077            # not a multiple of any corpus tile: a partial tail tile
KMAX = 16                    # the top-16 reference of a data set holds the top-k for every k <= 16
BENCH_SEED = 20240922 + 3    # bench.py's SEED: its corpus and queries are make_dense_corpus(SEED + 2) / _queries(SEED + 3)

# public kernel form (ezr_dense_set_kernel) -> (64-query blocks per CTA, corpus tile rows, CTAs per cluster, name),
# as dense_tc.cu kForms
FORMS = {2: (2, 128, 1, b"wgmma"), 3: (1, 64, 1, b"wgmma-q64"), 4: (1, 128, 1, b"wgmma-q64-n128"),
         5: (1, 128, 2, b"wgmma-q64-n128-mc2")}


@pytest.fixture(scope="module", autouse=True)
def _ready(lib_built):
    _lib.require_cuda()


def _report(what, info):
    print(f"\n[dense-scale] {what}: " + ", ".join(f"{k}={v:.5g}" if isinstance(v, float) else f"{k}={v}"
                                               for k, v in info.items()))


# ------------------------------------------------------------------------------ the work decomposition
def _auto_form(dim, nq):
    return 2 if dim <= 768 and nq > 64 else 4          # ezr_dense_topk's automatic choice


def _choose_splits(qblocks, n_rows, dim, sms, tn):
    """ts_choose_splits (csrc/dense_tc.cu), restated."""
    tiles = (n_rows + tn - 1) // tn
    max_s = max(1, min(tiles // 4, sms))
    t_corpus = n_rows * dim * 2 / 45e9
    eps = 20e-6 / max(t_corpus, 1e-9)
    best, best_cost = 1, 1e30
    for s in range(1, max_s + 1):
        waves = (qblocks * s + sms - 1) // sms
        cost = waves * (1.0 / s + eps)
        if cost < best_cost * (1 - 1e-9):
            best, best_cost = s, cost
    return best


def _schedule(form, n_rows, dim, nq):
    """-> dict(splits, rows_per_slice, units, units_per_cta) of dense_tc_topk for this launch."""
    qw, tn, cl, _ = FORMS[form]
    sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    groups = -(-(-(-nq // (64 * qw))) // cl)                        # work units per corpus split
    s = _choose_splits(groups, n_rows, dim, sms // cl, tn)
    rows_per_slice = -(-(-(-n_rows // tn)) // s) * tn               # tc_rows_per_slice
    s = -(-n_rows // rows_per_slice)                                # only the non-empty splits
    units = s * groups
    return dict(splits=s, rows_per_slice=rows_per_slice, units=units, units_per_cta=units / min(units, sms // cl),
                sms=sms)


def _multi_wave(form, n_rows, dim, nq, what):
    sch = _schedule(form, n_rows, dim, nq)
    _report(f"{what} schedule (form {form})", sch)
    assert sch["units_per_cta"] >= 2, f"{what}: form {form} runs {sch['units_per_cta']:.2f} units per CTA (need >= 2)"
    return sch


# ----------------------------------------------------------------------------------------------- helpers
def _ints(rows, dim, lo, hi, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randint(lo, hi + 1, (rows, dim), generator=g, device=DEV, dtype=torch.int8).to(torch.bfloat16)


def _dense(index, q, k, form=0, q_group=None):
    """One ezr_dense_topk call with the kernel form forced (0 = automatic); asserts which kernel ran."""
    L = _lib.lib()
    _lib.check(L.ezr_dense_set_kernel(form))
    try:
        res = batched.dense_topk(index, q, k, q_group=q_group)
        torch.cuda.synchronize()
        ran = L.ezr_dense_last_kernel()
    finally:
        L.ezr_dense_set_kernel(0)
    assert ran == FORMS[form or _auto_form(index.dim, q.shape[0])][3]
    return res


def _same_bytes(a, b):
    return (torch.equal(a.counts, b.counts) and torch.equal(a.ids, b.ids)
            and torch.equal(a.scores.view(torch.int32), b.scores.view(torch.int32)))


def _assert_exact(res, ref, k, what, sch, id_base=0, qw=128):
    """ids, counts and score bits (so +0.0, never -0.0) equal to the canonical fp64 top-k (``ref`` = fp64_top of the
    same data).  A mismatch reports the first query that differs, its query block and the corpus split of each id.
    Returns the number of results compared."""
    ids, sc, valid = ref[0][:, :k], ref[1][:, :k], ref[2][:, :k]
    cnt = valid.sum(1)
    want_ids = torch.where(valid, ids + id_base, torch.full_like(ids, -1))
    got_ids = res.ids.long()
    bad = (res.counts.long() != cnt) | (got_ids != want_ids).any(1) | \
          ((res.scores.view(torch.int32) != sc.float().view(torch.int32)) & valid).any(1)
    if bad.any():
        qi = int(torch.nonzero(bad)[0])
        rps = sch["rows_per_slice"]
        split = lambda t: [int(i) // rps if i >= 0 else -1 for i in (t - id_base).tolist()]
        raise AssertionError(
            f"{what}: {int(bad.sum())} queries differ; first: query {qi} (query block {qi // qw}), count "
            f"{int(res.counts[qi])} vs {int(cnt[qi])}\n  got ids {got_ids[qi].tolist()} (splits {split(got_ids[qi])})"
            f"\n  got scores {res.scores[qi].tolist()}\n  want ids {want_ids[qi].tolist()} (splits "
            f"{split(want_ids[qi])})\n  want scores {sc[qi].float().tolist()}")
    return int(cnt.sum())


def _index_topk_abi(corpus, ld, q, k):
    """ezr_dense_topk straight through the C ABI with a row stride ``ld`` >= dim."""
    L = _lib.lib()
    n, dim = corpus.shape[0], q.shape[1]
    nq = q.shape[0]
    out_s = torch.empty(nq, k, dtype=torch.float32, device=DEV)
    out_i = torch.empty(nq, k, dtype=torch.int32, device=DEV)
    out_c = torch.empty(nq, dtype=torch.int32, device=DEV)
    ws = torch.empty(L.ezr_dense_topk_workspace(n, dim, nq, k), dtype=torch.uint8, device=DEV)
    _lib.check(L.ezr_dense_topk(_lib.ptr(corpus), n, dim, ld, _lib.ptr(q), nq, q.stride(0), k, None, None, 0,
                                _lib.ptr(out_s), _lib.ptr(out_i), _lib.ptr(out_c), _lib.ptr(ws), ws.numel(),
                                _lib.stream_ptr()), "ezr_dense_topk")
    torch.cuda.synchronize()
    return batched.TopK(out_s, out_i, out_c)


# ------------------------------------------------------------------ A: the bench shape, exact integers
N_Q_A = 10_001               # 78 full 128-query blocks and one of 17 rows


@pytest.fixture(scope="module")
def case_a():
    c = _ints(N_ROWS, 768, -2, 2, 1)
    q = _ints(N_Q_A, 768, -2, 2, 2)
    return dict(c=c, q=q, index=DenseIndex(c, device=DEV), ref=fp64_top(q, c, KMAX, integer=True))


def test_a_bench_shape_bit_exact_with_ties_across_splits(case_a):
    k = 10
    sch = _multi_wave(2, N_ROWS, 768, N_Q_A, "A")
    res = _dense(case_a["index"], case_a["q"], k)
    _assert_exact(res, case_a["ref"], k, "A", sch)
    ids, sc, _ = case_a["ref"]
    tie = sc[:, k - 1] == sc[:, k]                               # the k-th and (k+1)-th score tie: the id decides
    split_tie = tie & (ids[:, k - 1] // sch["rows_per_slice"] != ids[:, k] // sch["rows_per_slice"])
    _report("A", dict(queries=N_Q_A, tie_at_kth=tie.double().mean().item(),
                      tie_at_kth_across_splits=split_tie.double().mean().item()))
    assert tie.double().mean().item() >= 0.05
    # control: the same reference with ties ordered by id ascending must disagree
    asc = fp64_top(case_a["q"], case_a["c"], k, integer=True, ids_asc=True)
    assert not torch.equal(res.ids.long(), asc[0])


# ------------------------------------------------------------ E: independence of schedule and layout
def test_e_stage_cap_does_not_change_the_result(case_a):
    L = _lib.lib()
    runs = {}
    try:
        for cap in (2, 3, 0):
            _lib.check(L.ezr_dense_set_stage_cap(cap))
            runs[cap] = _dense(case_a["index"], case_a["q"], 10)
    finally:
        L.ezr_dense_set_stage_cap(0)
    sch = _schedule(2, N_ROWS, 768, N_Q_A)
    for cap, r in runs.items():
        _assert_exact(r, case_a["ref"], 10, f"A with stage cap {cap}", sch)
        assert _same_bytes(r, runs[0]), f"stage cap {cap}"


def test_e_spare_capacity_rows_are_never_read(case_a):
    c, q = case_a["c"], case_a["q"]
    spare = 4096
    index = DenseIndex(c, device=DEV, capacity=N_ROWS + spare)
    tail = index.rows_for_append(spare)                          # behind the live rows, not committed
    sign = torch.where(torch.arange(spare, device=DEV) % 2 == 0, 1.0, -1.0)
    tail.copy_((64.0 * sign)[:, None].expand(spare, c.shape[1]))   # any query would rank one of them first
    assert index.n_rows == N_ROWS
    assert _same_bytes(_dense(index, q, 10), _dense(case_a["index"], q, 10))


def test_e_row_stride_wider_than_dim(case_a):
    c, q = case_a["c"], case_a["q"]
    wide = torch.full((N_ROWS, 768 + 64), 64.0, dtype=torch.bfloat16, device=DEV)
    wide[:, :768] = c
    L = _lib.lib()
    res = _index_topk_abi(wide, wide.stride(0), q, 10)
    assert L.ezr_dense_last_kernel() == b"wgmma"
    assert _same_bytes(res, _dense(case_a["index"], q, 10))


# ------------------------------------------------------- B: k x register query chunks, form 2, at scale
B_KS = [1, 4, 5, 8, 12, 16]            # 4 register chunks for k <= 8, 2 for k = 12, none for k = 16


@pytest.mark.parametrize("dim", [64, 128, 192, 576, 704, 768])
def test_b_register_chunks_times_k_bit_exact(dim):
    # dims 64 / 128 / 192 hold fewer k-chunks than the 4 (k <= 8) or 2 (k = 12, dim 64) register chunks; 576 / 704 /
    # 768 stream 9 / 11 / 12 k-chunks
    nq = 10_000
    sch = _multi_wave(2, N_ROWS, dim, nq, f"B dim {dim}")
    c = _ints(N_ROWS, dim, -2, 2, 100 + dim)
    q = _ints(nq, dim, -2, 2, 200 + dim)
    ref = fp64_top(q, c, KMAX, integer=True)
    index = DenseIndex(c, device=DEV)
    for k in B_KS:
        _assert_exact(_dense(index, q, k, form=2), ref, k, f"B dim {dim} k {k}", sch)


# ---------------------------------------------------------------------------- C: the other forms at scale
@pytest.mark.parametrize("dim", [768, 832, 1024])
def test_c_q64_forms_bit_exact(dim):
    c = _ints(N_ROWS, dim, -2, 2, 300 + dim)
    q = _ints(10_000, dim, -2, 2, 400 + dim)
    ref = fp64_top(q, c, 10, integer=True)
    index = DenseIndex(c, device=DEV)
    for form in (3, 4, 5):
        nq = 4000 if form == 5 else 10_000                    # the cluster-pair form: fewer queries, still multi-wave
        sch = _multi_wave(form, N_ROWS, dim, nq, f"C dim {dim}")
        _assert_exact(_dense(index, q[:nq], 10, form=form), tuple(t[:nq] for t in ref), 10, f"C dim {dim} form {form}",
                      sch, qw=64)


# ---------------------------------------------------------------------------- D: seeds, ties and signs
N_Q_D = 4000
ZERO_EVERY = 50


@pytest.fixture(scope="module")
def case_d():
    """Row j = row (j mod 997) of a random integer block: every top score is shared by ~1000 ids spread over all
    splits.  Every 50th query is all zero (every score 0, with -0.0 products from negative corpus entries)."""
    base = _ints(997, 768, -2, 2, 500)
    c = base[torch.arange(N_ODD, device=DEV) % 997].contiguous()
    q = _ints(N_Q_D, 768, -2, 2, 501)
    q[::ZERO_EVERY] = 0
    return dict(c=c, q=q, index=DenseIndex(c, device=DEV), ref=fp64_top(q, c, KMAX, integer=True))


@pytest.mark.parametrize("form", [2, 3, 4, 5])
def test_d_duplicated_rows_and_zero_queries(case_d, form):
    k = 10
    sch = _multi_wave(form, N_ODD, 768, N_Q_D, "D duplicated rows")
    ids, sc, _ = case_d["ref"]
    live = torch.ones(N_Q_D, dtype=torch.bool, device=DEV)
    live[::ZERO_EVERY] = False
    assert (sc[live, 0] == sc[live, KMAX - 1]).all()           # the whole top-16 ties on every non-zero query
    res = _dense(case_d["index"], case_d["q"], k, form=form)
    _assert_exact(res, case_d["ref"], k, f"D duplicated rows, form {form}", sch, qw=FORMS[form][0] * 64)
    zero = res.ids[~live].long()
    assert (zero == torch.arange(N_ODD - 1, N_ODD - 1 - k, -1, device=DEV)).all()
    assert (res.scores[~live].view(torch.int32) == 0).all()    # +0.0 bit for bit


@pytest.mark.parametrize("form", [2, 4])
def test_d_all_scores_negative_no_phantom_rows(form):
    # no score is positive, so no unit publishes a seed; a zero-filled row past the end of the corpus would score 0
    # and beat every real row
    c = _ints(N_ODD, 768, 0, 2, 510)
    q = _ints(N_Q_D, 768, -2, -1, 511)
    sch = _multi_wave(form, N_ODD, 768, N_Q_D, "D negative scores")
    ref = fp64_top(q, c, 10, integer=True)
    assert (ref[1] < 0).all()
    res = _dense(DenseIndex(c, device=DEV), q, 10, form=form)
    assert ((res.ids >= 0) & (res.ids < N_ODD)).all()
    _assert_exact(res, ref, 10, f"D negative scores, form {form}", sch, qw=FORMS[form][0] * 64)


@pytest.mark.parametrize("form", [2, 4])
def test_d_filters_at_scale(case_d, form):
    k, row_lo = 10, 2 ** 31 - 2_000_000
    rare = 7
    groups = synth.make_groups(N_ODD, 4, 520, device=DEV)
    groups[-3:] = rare                                         # a class of 3 (< k) rows, at the end of the corpus
    pattern = torch.tensor([-1, -2, rare, 0, 3], dtype=torch.int32, device=DEV)    # -2: no such class
    want = pattern[torch.arange(N_Q_D, device=DEV) % 5]
    sch = _multi_wave(form, N_ODD, 768, N_Q_D, "D filters")
    ref = fp64_top(case_d["q"], case_d["c"], k, integer=True,
                   allowed=lambda q0, q1, c0, c1: (want[q0:q1, None] == -1) | (groups[None, c0:c1] == want[q0:q1, None]))
    index = DenseIndex(case_d["c"], device=DEV, doc_group=groups, row_lo=row_lo)
    res = _dense(index, case_d["q"], k, form=form, q_group=want)
    n = _assert_exact(res, ref, k, f"D filters, form {form}", sch, id_base=row_lo, qw=FORMS[form][0] * 64)
    cnt = res.counts.long()
    assert (cnt[want == -2] == 0).all() and (cnt[want == rare] == 3).all() and (cnt[want == 0] == k).all()
    assert (res.ids[want == rare][:, :3].long() >= row_lo + N_ODD - 3).all()
    _report(f"D filters form {form}", dict(results=n))


# ----------------------------------------------------------- F: unit vectors against fp64, derived bound
@pytest.mark.parametrize("dim", [768, 1024])
def test_f_unit_vectors_within_derived_bound(dim):
    k, nq = 10, 10_000
    c = synth.make_dense_corpus(N_ROWS, dim, BENCH_SEED + 2, device=DEV)
    q = synth.make_dense_queries(c, nq, BENCH_SEED + 3)
    form = _auto_form(dim, nq)
    sch = _multi_wave(form, N_ROWS, dim, nq, f"F dim {dim}")
    res = _dense(DenseIndex(c, device=DEV), q, k)
    assert (res.counts == k).all()
    top_i, top_s, _ = fp64_top(q, c, KMAX, integer=False)
    exact, delta = dense_score_bound(q, c, res.ids.long())
    c_max = max(c[i:i + 131072].double().norm(dim=1).max().item() for i in range(0, N_ROWS, 131072))
    dmax = dense_delta_max(q, c_max)
    info = check_dense_topk(res.scores, res.ids, exact, delta, top_s, top_i, dmax, N_ROWS, f"F dim {dim}")
    _report(f"F dim {dim} form {form}", dict(info, units_per_cta=sch["units_per_cta"]))
    # negative controls on the first 512 queries
    m = 512
    sub = lambda **kw: dict(dict(scores=res.scores[:m], ids=res.ids[:m], exact=exact[:m], delta=delta[:m],
                                 top_vals=top_s[:m], top_ids=top_i[:m], dmax=dmax[:m]), **kw)
    chk = lambda a: check_dense_topk(a["scores"], a["ids"], a["exact"], a["delta"], a["top_vals"], a["top_ids"],
                                     a["dmax"], N_ROWS, f"F dim {dim} control")
    chk(sub())
    # (a) a reference without the last 16 dims
    wi, ws, _ = fp64_top(q[:m], c, KMAX, integer=False, drop_dims=16)
    we = (q[:m, :-16].double()[:, None, :] * c[res.ids[:m].long(), :-16].double()).sum(-1)
    assert rejects(chk, sub(top_vals=ws, top_ids=wi, exact=we))
    # (b) the best id of one query replaced by the fp64 (k+1)-th (its score the fp32 rounding of its fp64 score)
    sep = (top_s[:m, 0] - top_s[:m, k - 1] > 2 * dmax[:m]) & ~(top_i[:m, k:k + 1] == res.ids[:m].long()).any(1)
    qi = int(torch.nonzero(sep)[0])
    gi, gs, ge = res.ids[:m].long().clone(), res.scores[:m].clone(), exact[:m].clone()
    j = int((gi[qi] == top_i[qi, 0]).nonzero()[0])
    gi[qi, j], gs[qi, j], ge[qi, j] = top_i[qi, k], top_s[qi, k].float(), top_s[qi, k]
    order = torch.argsort(gi[qi], descending=True)
    order = order[torch.argsort(gs[qi][order], descending=True, stable=True)]
    gi[qi], gs[qi], ge[qi] = gi[qi][order], gs[qi][order], ge[qi][order]
    gd = delta[:m].clone()
    gd[qi] = gd[qi][order]
    assert rejects(chk, sub(ids=gi, scores=gs, exact=ge, delta=gd))


# --------------------------------------------------------------------- ezr_normalize_rows against fp64
NORM_ROWS = 300


def _norm_input(dim, ld, f32, seed):
    """Rows of N(0, 1) at scales from 1e-3 to 1e3; rows 0-15 with norms near 1e-13 and 1e-14 (below the 1e-12 floor:
    the kernel scales them by 1 / 1e-12f); rows 16-19 zero."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(NORM_ROWS, ld, generator=g, device=DEV)
    x = x * torch.exp(3 * torch.randn(NORM_ROWS, 1, generator=g, device=DEV)).clamp(1e-3, 1e3)
    x[:16] = x[:16] / x[:16, :dim].norm(dim=1, keepdim=True) * torch.where(torch.arange(16, device=DEV) % 2 == 0,
                                                                           1e-13, 1e-14)[:, None]
    x[16:20] = 0.0
    x = x if f32 else x.to(torch.bfloat16)
    return x[:, :dim]


@pytest.mark.parametrize("f32", [True, False], ids=["fp32", "bf16"])
@pytest.mark.parametrize("dim,ldx,ldo", [(768, 768, 768), (1024, 1031, 1088), (3584, 3584, 3600)])
def test_normalize_rows_vs_fp64(dim, ldx, ldo, f32):
    x = _norm_input(dim, ldx, f32, 600 + dim)
    nrm = x.double().norm(dim=1)
    assert (nrm[:16] < 0.5 * NORM_FLOOR).all() and (nrm[20:] > 1e3 * NORM_FLOOR).all()
    buf = torch.full((NORM_ROWS, ldo), 7.0, dtype=torch.bfloat16, device=DEV)
    out = normalize_rows(x, buf[:, :dim])
    torch.cuda.synchronize()
    assert (buf[:, dim:] == 7.0).all(), "wrote past dim"
    exact, delta = l2_normalize_exact_and_delta(x)
    info = check_bf16(out, exact, delta, f"normalize {dim}", median_ulps=0.01)
    _report(f"normalize dim={dim} ldx={ldx} ldo={ldo} {'fp32' if f32 else 'bf16'} in", info)
    zero = out[16:20]
    assert (zero == 0).all() and not torch.signbit(zero.float()).any(), "zero rows must give +0.0"
    assert (out[:16].double().norm(dim=1) < 0.5).all()           # scaled by 1e12, not normalised
    # controls: normalising the tiny rows to unit length; a norm that leaves out the last 32 columns
    X = x.double()
    unit = torch.nan_to_num(X / X.norm(dim=1, keepdim=True))
    assert rejects(check_bf16, out, unit, delta, "control: no floor", median_ulps=0.01)
    short = X / X[:, :-32].norm(dim=1, keepdim=True).clamp_min(NORM_FLOOR)
    assert rejects(check_bf16, out, short, delta, "control: 32 columns short", median_ulps=0.01)
