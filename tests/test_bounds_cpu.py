"""CPU: the bf16 error-bound checker of tests/_bounds.py accepts correct roundings and rejects biased or wrong ones;
the cross-encoder head's bound holds for an fp32 emulation of the kernel and rejects wrong references; the dense
top-k score bound holds for an emulated truncating k16 accumulator, stays tight, and the membership check built on
it rejects a wrong reference and a result that leaves out a clearly better row."""
import pytest
import torch

from _bounds import (Z_ONE, Z_SUB, Z_ZERO, check_bf16, check_dense_topk, check_sigmoid, cross_head_bound,
                     cross_head_case, cross_head_logit, dense_delta_max, dense_score_bound, rejects, round_bf16,
                     ulp_bf16, ulp_f32)

N = 200_000


@pytest.fixture(scope="module")
def exact():
    g = torch.Generator().manual_seed(3)
    x = torch.randn(N, generator=g, dtype=torch.float64) * torch.exp(torch.randn(N, generator=g, dtype=torch.float64))
    x[:4] = torch.tensor([0.0, 1.0, -2.0 ** -130, 3.0 * 2 ** 100], dtype=torch.float64)   # zero, binade edge, subnormal
    return x


def test_ulp_and_rounding_of_known_values():
    x = torch.tensor([1.0, 1.5, -2.0, 0.75, 3.0 * 2 ** -20, 0.0], dtype=torch.float64)
    assert ulp_bf16(x).tolist() == [2 ** -7, 2 ** -7, 2 ** -6, 2 ** -8, 2 ** -26, 2 ** -133]
    # halfway cases go to the even neighbour; the result agrees with torch's fp32 -> bf16 conversion (one rounding)
    t = torch.tensor([1 + 2 ** -8, 1 + 3 * 2 ** -8, 1 + 2 ** -9, -(1 + 2 ** -8)], dtype=torch.float64)
    assert round_bf16(t).tolist() == [1.0, 1 + 2 ** -6, 1.0, -1.0]
    f = torch.randn(10_000, generator=torch.Generator().manual_seed(1))
    assert torch.equal(round_bf16(f.double()), f.to(torch.bfloat16).double())


def test_accepts_round_to_nearest(exact):
    info = check_bf16(round_bf16(exact).to(torch.bfloat16), exact, 0.0, "rn", median_ulps=0.0)
    assert info["rate"] == 1.0 and abs(info["bias"]) < 0.01


def test_accepts_values_perturbed_within_delta(exact):
    # a kernel whose fp32 result is off by up to delta before the final rounding: the error bound holds, and with
    # delta a small fraction of an ulp nearly every element still rounds to the exact value's nearest bf16
    delta = 0.004 * ulp_bf16(exact)
    g = torch.Generator().manual_seed(4)
    pert = exact + (2 * torch.rand(N, generator=g, dtype=torch.float64) - 1) * delta
    info = check_bf16(round_bf16(pert).to(torch.bfloat16), exact, delta, "perturbed", median_ulps=0.01)
    assert info["rate"] >= 0.99


def test_rejects_rounding_toward_zero(exact):
    u = ulp_bf16(exact)
    trunc = torch.trunc(exact / u) * u                       # within one ulp everywhere: only the bias shows it
    assert rejects(check_bf16, trunc.to(torch.bfloat16), exact, 0.0, "trunc", median_ulps=0.0)
    with pytest.raises(AssertionError, match="bias"):
        check_bf16(trunc.to(torch.bfloat16), exact, 0.0, "trunc", median_ulps=0.0, min_rate=0.0)


def test_rejects_one_element_two_ulps_past_delta(exact):
    delta = 0.25 * ulp_bf16(exact)
    got = round_bf16(exact)
    i = 1234
    got[i] = round_bf16(exact[i] + torch.sign(exact[i]) * (delta[i] + 2 * ulp_bf16(exact[i])))
    with pytest.raises(AssertionError, match="worst element 1234"):
        check_bf16(got.to(torch.bfloat16), exact, delta, "one off", median_ulps=0.5)


def test_rejects_two_percent_flipped_by_one_ulp(exact):
    # 2 % of the elements take the other bf16 neighbour of the exact value: still within one ulp and unbiased, so only
    # the correct-rounding rate can catch it
    u = ulp_bf16(exact)
    lo = torch.floor(exact / u) * u
    near = round_bf16(exact)
    other = torch.where(near == lo, lo + u, lo)
    flip = torch.zeros(N, dtype=torch.bool)
    flip[torch.randperm(N, generator=torch.Generator().manual_seed(5))[: N // 50]] = True
    got = torch.where(flip, other, near)
    with pytest.raises(AssertionError, match=r"correctly rounded 98\.0"):
        check_bf16(got.to(torch.bfloat16), exact, 0.0, "flipped", median_ulps=0.0)
    check_bf16(got.to(torch.bfloat16), exact, 0.0, "flipped", median_ulps=0.0, min_rate=0.97)   # nothing else fails


def test_preconditions():
    x = torch.randn(1000, dtype=torch.float64)
    with pytest.raises(AssertionError, match="too few"):
        check_bf16(round_bf16(x).to(torch.bfloat16), x, 0.0, "small", median_ulps=0.0)
    y = torch.randn(N, dtype=torch.float64)
    with pytest.raises(AssertionError, match="vacuous"):
        check_bf16(round_bf16(y).to(torch.bfloat16), y, 10 * ulp_bf16(y), "loose", median_ulps=2.0)
    with pytest.raises(AssertionError):
        rejects(check_bf16, round_bf16(y).to(torch.bfloat16), y, 10 * ulp_bf16(y), "loose", median_ulps=2.0)


# ------------------------------------------------------------------------------------- cross-encoder head
HEAD_PAIRS = 6000
HEAD_MEDIAN_ULPS = 128     # the same figure the GPU test holds the bound to (tests/test_gpu_bert_shapes.py)


def _ulps_off(exact, k):
    """An fp32 result within 2 ulp of ``exact`` (fp64), as tanhf / expf guarantee: the nearest fp32 value moved by
    ``k`` ulps, or left nearest where that would leave the 2-ulp band."""
    near = exact.float()
    u = ulp_f32(exact)
    cand = (near.double() + k * u).float()
    ok = (cand.double() - exact).abs() <= 2 * u
    return torch.where(ok, cand, near)


def _emulate_head(rows, w, b, k_tanh, k_exp):
    """csrc/rerank.cu cross_pair_sigmoid in fp32 on the CPU, in the kernel's order: lane i % 32 accumulates element i
    with fmaf, then the xor-shuffle tree adds the lanes.  fmaf is emulated as the fp64 value of t * w + acc (the
    product is exact there) rounded to fp32: a double rounding, at most 2^-29 relative away from fmaf's one."""
    t = _ulps_off(torch.tanh(rows.double()), k_tanh).clamp(-1, 1).double()
    n, d = rows.shape
    wd = w.double()
    acc = torch.zeros(n, 32, dtype=torch.float32)
    for i0 in range(0, d, 32):
        m = min(32, d - i0)
        acc[:, :m] = (t[:, i0:i0 + m] * wd[i0:i0 + m] + acc[:, :m].double()).float()
    lane = torch.arange(32)
    for o in (16, 8, 4, 2, 1):
        acc = acc + acc[:, lane ^ o]
    z = acc[:, 0] + torch.tensor(b, dtype=torch.float32)
    e = _ulps_off(torch.exp(-z.double()), k_exp)              # +inf past FLT_MAX
    one = torch.ones((), dtype=torch.float32)
    return one / (one + e)


@pytest.fixture(scope="module", params=[768, 1000], ids=["d768", "d1000-ragged-lanes"])
def head(request):
    d = request.param
    rows, w, b = cross_head_case(HEAD_PAIRS, d, 90 + d)
    z, s, ds = cross_head_bound(rows, w, b)
    return rows, w, b, z, s, ds


def test_head_case_fills_every_band(head):
    *_, z, _, _ = head
    for lo, hi in ((-1, 1), (Z_ONE, 40), (Z_SUB[0], Z_SUB[1]), (-120, Z_ZERO)):
        share = ((z > lo) & (z < hi)).double().mean().item()
        assert share > 0.15, (lo, hi, share)


def test_head_bound_holds_for_the_emulated_kernel(head):
    rows, w, b, z, s, ds = head
    g = torch.Generator().manual_seed(5)
    k_t = torch.randint(-2, 3, rows.shape, generator=g)
    k_e = torch.randint(-2, 3, (rows.shape[0],), generator=g)
    got = _emulate_head(rows, w, b, k_t, k_e)
    info = check_sigmoid(got, z, s, ds, "emulated head", median_ulps=HEAD_MEDIAN_ULPS, min_elems=HEAD_PAIRS)
    # worst case within the functions' accuracy: every tanhf 2 ulp towards sign(w) (all push z up), expf 2 ulp down
    sw = torch.sign(w).long()[None, :].expand(rows.shape)
    up = _emulate_head(rows, w, b, 2 * sw, torch.full((rows.shape[0],), -2))
    info_up = check_sigmoid(up, z, s, ds, "emulated head, errors aligned", median_ulps=HEAD_MEDIAN_ULPS,
                            min_elems=HEAD_PAIRS, max_bias=1.0)
    print(f"\n[bounds] head emulation: random {info}; aligned {info_up}")
    assert info_up["bias"] > info["bias"]                    # the aligned errors show in the mean


@pytest.mark.parametrize("control", ["bias dropped", "tanh rounded to bf16", "tanh omitted", "w_out shifted by one"])
def test_head_bound_rejects_wrong_references(head, control):
    rows, w, b, z, s, ds = head
    got = _emulate_head(rows, w, b, torch.zeros(rows.shape, dtype=torch.long),
                        torch.zeros(rows.shape[0], dtype=torch.long))
    if control == "bias dropped":
        zw = cross_head_logit(rows, w, 0.0)
    elif control == "tanh rounded to bf16":
        zw = cross_head_logit(rows, w, b, tanh=lambda x: round_bf16(torch.tanh(x)))
    elif control == "tanh omitted":
        zw = cross_head_logit(rows, w, b, tanh=lambda x: x)
    else:
        zw = cross_head_logit(rows, torch.roll(w, 1), b)
    assert rejects(check_sigmoid, got, zw, torch.sigmoid(zw), ds, control, median_ulps=HEAD_MEDIAN_ULPS,
                   min_elems=HEAD_PAIRS)


def test_head_bound_preconditions(head):
    rows, w, b, z, s, ds = head
    got = _emulate_head(rows, w, b, torch.zeros(rows.shape, dtype=torch.long),
                        torch.zeros(rows.shape[0], dtype=torch.long))
    with pytest.raises(AssertionError, match="vacuous"):
        check_sigmoid(got, z, s, 1e3 * ds, "loose", median_ulps=HEAD_MEDIAN_ULPS, min_elems=HEAD_PAIRS)
    with pytest.raises(AssertionError, match="too few"):
        check_sigmoid(got[:10], z[:10], s[:10], ds[:10], "small", median_ulps=HEAD_MEDIAN_ULPS)
    sub = (z > Z_SUB[0]) & (z < Z_SUB[1])
    flushed = torch.where(sub, torch.zeros_like(got), got)
    with pytest.raises(AssertionError, match="flushed"):                 # a bound wide enough to pass zeros there
        check_sigmoid(flushed, z, s, torch.where(sub, 2 * s, ds), "ftz", median_ulps=HEAD_MEDIAN_ULPS,
                      min_elems=HEAD_PAIRS, max_bias=1.0)
    neg0 = torch.where(z < Z_ZERO, torch.full_like(got, -0.0), got)
    with pytest.raises(AssertionError, match=r"\+0\.0"):
        check_sigmoid(neg0, z, s, ds, "-0", median_ulps=HEAD_MEDIAN_ULPS, min_elems=HEAD_PAIRS)


# --------------------------------------------------------------------------------------------- dense top-k
DENSE_ROWS, DENSE_DIM, DENSE_Q, DENSE_KEEP, DENSE_TOPK = 20_000, 768, 64, 64, 10
DENSE_MEDIAN_ULPS = 1024     # median bound of a returned score, in fp32 ulps of the score (the GPU test's 1e-3
                             # tolerance it replaces is ~17000 ulps at 0.5)


def _to_f32(x, mode):
    """fp64 -> fp32 rounded to nearest ("rn") or toward zero ("rz"), as fp64."""
    r = x.float().double()
    if mode == "rz":
        over = r.abs() > x.abs()
        r = torch.where(over, torch.nextafter(r.float(), torch.zeros_like(r.float())).double(), r)
    return r


def _emulate_dense(q, rows, mode):
    """fp32 accumulation over k16 steps of the exact products of q [Q, d] with rows [Q, m, d]: each step adds its 16
    products (summed exactly) to the accumulator and rounds the result to fp32 (``mode``)."""
    p = q.double()[:, None, :] * rows.double()
    steps = p.view(*p.shape[:2], -1, 16).sum(-1)
    acc = torch.zeros(p.shape[:2], dtype=torch.float64)
    for j in range(steps.shape[-1]):
        acc = _to_f32(acc + steps[..., j], mode)
    return acc


@pytest.fixture(scope="module")
def dense():
    from easyrag_b200 import synth
    c = synth.make_dense_corpus(DENSE_ROWS, DENSE_DIM, 61)
    q = synth.make_dense_queries(c, DENSE_Q, 62)
    sims = q.double() @ c.double().T
    top_vals, top_ids = sims.topk(DENSE_KEEP, dim=1)
    # the emulated kernel's top-k, among the fp64 top 64 (its errors are far below the gaps that far down)
    emu = _emulate_dense(q, c[top_ids], "rz")
    order = torch.argsort(top_ids, dim=1, descending=True)                 # id desc, then a stable sort by score
    emu_s, emu_i = emu.gather(1, order), top_ids.gather(1, order)
    order = torch.argsort(emu_s, dim=1, descending=True, stable=True)[:, :DENSE_TOPK]
    got_s, got_i = emu_s.gather(1, order).float(), emu_i.gather(1, order)
    exact, delta = dense_score_bound(q, c, got_i)
    dmax = dense_delta_max(q, c.double().norm(dim=1).max().item())
    return dict(c=c, q=q, top_vals=top_vals, top_ids=top_ids, got_s=got_s, got_i=got_i, exact=exact, delta=delta,
                dmax=dmax)


@pytest.mark.parametrize("mode", ["rz", "rn"])
def test_dense_bound_holds_for_emulated_accumulator(dense, mode):
    c, q, ids = dense["c"], dense["q"], dense["top_ids"]
    emu = _emulate_dense(q, c[ids], mode)
    exact, delta = dense_score_bound(q, c, ids)
    ratio = ((emu - exact).abs() / delta).max().item()
    print(f"\n[bounds] dense emulation ({mode}): worst |err| / delta = {ratio:.4g}")
    assert ratio <= 1
    assert (delta <= dense_delta_max(q, c.double().norm(dim=1).max().item())[:, None]).all()


def test_dense_bound_is_not_vacuous(dense):
    med = (dense["delta"] / ulp_f32(dense["exact"])).median().item()
    print(f"\n[bounds] dense: median delta = {med:.4g} fp32 ulps, median delta max = "
          f"{dense['dmax'].median().item():.3g}")
    assert med <= DENSE_MEDIAN_ULPS
    assert dense["dmax"].max().item() < 2e-4                 # unit vectors, d 768: 17 * 2^-23 * 49


def _check(d, **over):
    a = dict(d, **over)
    return check_dense_topk(a["got_s"], a["got_i"], a["exact"], a["delta"], a["top_vals"], a["top_ids"], a["dmax"],
                            DENSE_ROWS, "emulated dense")


def test_dense_membership_accepts_emulated_and_rejects_controls(dense):
    info = _check(dense)
    print(f"\n[bounds] dense membership: {info}")
    assert info["worst"] <= 1
    c, q, k = dense["c"], dense["q"], DENSE_TOPK
    # (a) a reference without the last 16 dims
    cs, qs = c[:, :-16], q[:, :-16]
    tv, ti = (qs.double() @ cs.double().T).topk(DENSE_KEEP, dim=1)
    ex = (qs.double()[:, None, :] * cs[dense["got_i"]].double()).sum(-1)
    assert rejects(_check, dense, top_vals=tv, top_ids=ti, exact=ex)
    # (b) the best id of one query replaced by the fp64 (k+1)-th, its score the fp32 rounding of its fp64 score
    tv, ti = dense["top_vals"], dense["top_ids"]
    sep = (tv[:, 0] - tv[:, k - 1] > 2 * dense["dmax"]) & ~(ti[:, k:k + 1] == dense["got_i"]).any(1)
    qi = int(torch.nonzero(sep)[0])
    gi, gs, ge, gd = (dense[n].clone() for n in ("got_i", "got_s", "exact", "delta"))
    j = int((gi[qi] == ti[qi, 0]).nonzero()[0])
    gi[qi, j], gs[qi, j], ge[qi, j] = ti[qi, k], tv[qi, k].float(), tv[qi, k]
    order = torch.argsort(gi[qi], descending=True)
    order = order[torch.argsort(gs[qi][order], descending=True, stable=True)]
    gi[qi], gs[qi], ge[qi], gd[qi] = gi[qi][order], gs[qi][order], ge[qi][order], gd[qi][order]
    with pytest.raises(AssertionError, match="not returned"):
        _check(dense, got_i=gi, got_s=gs, exact=ge, delta=gd)
    assert rejects(_check, dense, got_i=gi, got_s=gs, exact=ge, delta=gd)
