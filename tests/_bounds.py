"""Test infrastructure: error-bound checks for kernels whose result is a bf16 rounding of an fp32 computation.

A kernel that computes ``f`` in fp32 and rounds once to bf16 returns ``bf16_rn(f + e)`` with ``|e| <= delta`` (the
fp32 error of its accumulation and epilogue, bounded per test).  ``check_bf16`` compares such an output with the fp64
value of ``f`` on the same bf16 inputs and asserts three things: every element lies within ``delta`` plus one bf16
ulp; at least 99 % of the elements are exactly the round-to-nearest bf16 value of the fp64 result; and the rounding is
unbiased (a kernel that truncates instead of rounding to nearest shows a mean signed error of about -0.5 ulp).

``ln_exact_and_delta`` is the fp64 LayerNorm and the bound of the norm kernels' fp32 error.  ``cross_head_bound`` /
``check_sigmoid`` do the same for the cross-encoder head (csrc/rerank.cu), whose result is an fp32 sigmoid rather
than a bf16 rounding.  ``dense_score_bound`` / ``check_dense_topk`` bound the fp32 scores of the wgmma dense top-k
(csrc/dense_tc.cu) and check its result lists against an fp64 top list.  Used by tests/test_gpu_model_shapes.py,
tests/test_gpu_bert_shapes.py and tests/test_gpu_dense_scale.py; checked itself by tests/test_bounds_cpu.py.
"""
import math

import torch
import torch.nn.functional as F

U32 = 2.0 ** -24                 # unit roundoff of fp32 (round to nearest)
BF16_MIN_ULP = 2.0 ** -133       # ulp of the smallest bf16 subnormal (bf16 shares fp32's exponent range)
F32_MIN_ULP = 2.0 ** -149        # spacing of fp32 subnormals
F32_MIN_NORMAL = 2.0 ** -126


def ulp_bf16(x: torch.Tensor) -> torch.Tensor:
    """fp64 ulp of bf16 at |x|: 2^(e - 7) for |x| in [2^e, 2^(e+1)), from the exponent alone."""
    x = x.double().abs()
    _, e = torch.frexp(x)                                  # x = m 2^e, m in [0.5, 1)
    u = torch.ldexp(torch.ones_like(x), (e - 8).to(torch.int32))
    return torch.where(x > 0, u.clamp_min(BF16_MIN_ULP), torch.full_like(x, BF16_MIN_ULP))


def round_bf16(x: torch.Tensor) -> torch.Tensor:
    """fp64 -> nearest bf16 value (ties to even), as fp64.  Done in fp64 directly: ``.to(torch.bfloat16)`` on a double
    tensor may round twice (through fp32)."""
    x = x.double()
    u = ulp_bf16(x)
    return torch.round(x / u) * u                          # x / u is exact (u is a power of two); round = half-to-even


def check_bf16(got: torch.Tensor, exact: torch.Tensor, delta, what: str, median_ulps: float, ulps: float = 1.0,
               min_rate: float = 0.99, max_bias: float = 0.05, min_elems: int = 100_000) -> dict:
    """Assert that ``got`` (bf16) is the bf16 rounding of ``exact`` (fp64) up to a pre-rounding error ``delta`` (fp64,
    per element or scalar).  ``median_ulps``: the bound itself must stay tight -- median(delta / ulp(exact)) below it.
    ``ulps``: bf16 ulps allowed per element beyond ``delta`` (1 = the final rounding; 2 where the kernel rounds to
    bf16 twice).  Returns the measured rate / bias / worst excess for the report."""
    got = got.double().reshape(-1)
    exact = exact.double().reshape(-1).to(got.device)
    delta = torch.as_tensor(delta, dtype=torch.float64, device=got.device)
    delta = delta.reshape(-1).expand(exact.shape) if delta.numel() == 1 else delta.reshape(-1)
    n = got.numel()
    assert n >= min_elems, f"{what}: {n} elements are too few to measure a rounding bias (need {min_elems})"
    assert torch.isfinite(got).all(), f"{what}: non-finite output"
    u_ex = ulp_bf16(exact)
    med = (delta / u_ex).median().item()
    assert med <= median_ulps, f"{what}: bound is vacuous: median delta = {med:.3g} ulp > {median_ulps}"
    err = (got - exact).abs()
    lim = delta + ulps * ulp_bf16(exact.abs() + delta)
    excess = err / lim
    worst = int(torch.argmax(excess))
    rate = (got == round_bf16(exact)).double().mean().item()
    bias = (torch.sign(exact) * (got - exact) / u_ex).mean().item()
    info = dict(rate=rate, bias=bias, worst=excess[worst].item(), median_delta_ulps=med, n=n)
    msg = (f"{what}: worst element {worst}: got {got[worst].item():.9g}, exact {exact[worst].item():.9g}, "
           f"|err| {err[worst].item():.3g} vs bound {lim[worst].item():.3g} (delta {delta[worst].item():.3g}); "
           f"correctly rounded {rate:.4%}, bias {bias:+.4f} ulp, median delta {med:.3g} ulp")
    assert (err <= lim).all(), msg
    assert rate >= min_rate, msg
    assert abs(bias) <= max_bias, msg
    return info


def rejects(fn, *args, **kw) -> bool:
    """True when the check ``fn`` fails on the error itself (a negative control: a wrong reference must not pass).
    Failed preconditions (too few elements, a vacuous bound) are re-raised: they would reject for the wrong reason."""
    try:
        fn(*args, **kw)
    except AssertionError as e:
        if "worst element" not in str(e) and "rms error" not in str(e):
            raise
        return True
    return False


def ulp_f32(x: torch.Tensor) -> torch.Tensor:
    """fp64 ulp of fp32 at |x|: 2^(e - 23) for |x| in [2^e, 2^(e+1)), 2^-149 among the subnormals."""
    x = x.double().abs()
    _, e = torch.frexp(x)
    u = torch.ldexp(torch.ones_like(x), (e - 24).to(torch.int32))
    return torch.where(x > 0, u.clamp_min(F32_MIN_ULP), torch.full_like(x, F32_MIN_ULP))


# ------------------------------------------------------------------------------------------------ LayerNorm
def ln_exact_and_delta(x, gamma, beta, eps):
    """LayerNorm in fp64 and the bound on the kernel's fp32 error before its one bf16 rounding (ops.cu norm kernels:
    two-pass mean / variance)."""
    dim = x.shape[1]
    X, G, B = x.double(), gamma.double(), beta.double()
    mu = X.mean(-1, keepdim=True)
    d = X - mu
    var = d.pow(2).mean(-1, keepdim=True)
    r = torch.rsqrt(var + eps)
    exact = d * r * G + B
    chain = dim / 32 + 10                 # longest fp32 addition chain of a row sum: dim / 32 serial adds per lane
                                          # (dim / 128 in the block kernel) + 5 shuffle levels (+ 5 block levels)
    e_mu = (chain + 1) * U32 * X.abs().mean(-1, keepdim=True)    # the row sum, then the division by dim
    e_var = ((chain + 3) * U32                                   # sum of squares (+ square, division, eps add)
             + 2 * e_mu * d.abs().mean(-1, keepdim=True) / var   # each d carries the mean's error
             + e_mu ** 2 / var)
    e_r = 0.5 * e_var + 2.0 ** -22 + U32                         # sqrt halves it; rsqrtf <= 2 ulp; the eps add
    delta = (G.abs() * r * (e_mu + U32 * d.abs())                # x - mean: the mean's error, then its rounding
             + (G * d * r).abs() * (e_r + 2 * U32)               # rstd's error; (d * rstd) * gamma rounded twice
             + U32 * ((G * d * r).abs() + B.abs()))              # + beta rounded
    return exact, delta


# ------------------------------------------------------------------------------------- cross-encoder head
# cross_pair_sigmoid (csrc/rerank.cu) computes, for one pair on one warp,
#     acc_lane = fmaf(tanhf(row[i]), w[i], acc_lane)   for i = lane, lane + 32, ...   (ceil(d / 32) steps)
#     acc      = xor-shuffle sum of the 32 lane sums                                   (5 levels)
#     s        = 1.f / (1.f + expf(-(acc + b)))
# in fp32 without fast-math: tanhf and expf err by at most 2 ulp (CUDA C Programming Guide, single-precision
# mathematical functions), the division is IEEE and keeps subnormal results.
TANHF_ULPS = 2
EXPF_ULPS = 2
Z_ONE = 17.4               # e^-z < 2^-25 from here: 1 + expf(-z) rounds to 1 and the score is exactly 1.0f
Z_SUB = (-88.72, -87.34)   # e^z below 2^-126 = e^-87.3365: a subnormal score (expf(-z) is still finite: it
                           # overflows at z < -ln(FLT_MAX) = -88.7228)
Z_ZERO = -88.8             # expf(-z) is +inf, 1 / inf = +0.0 (torch.sigmoid on the CPU returns +0.0 there as well)


def cross_head_logit(rows, w, b, tanh=torch.tanh):
    """fp64 logit tanh(rows) . w + b of each pair; ``rows`` [P, d] (bf16), ``w`` [d] (fp32), ``b`` an fp32 value.
    ``tanh`` replaces the activation to build negative controls."""
    return tanh(rows.double()) @ w.double() + b


def cross_head_bound(rows, w, b):
    """-> (z, s, ds): fp64 logit and sigmoid of each pair, and the bound on |kernel score - s|."""
    R, W = rows.double(), w.double()
    n, d = R.shape
    t = torch.tanh(R)
    prod = t * W                                            # fmaf: the product is not rounded on its own
    z = prod.sum(1) + b
    steps = -(-d // 32)
    lanes = F.pad(prod, (0, steps * 32 - d)).view(n, steps, 32)   # element i: lane i % 32, step i // 32
    part = lanes.cumsum(1)                                  # each lane's running sum after each fmaf
    e_chain = part.abs().sum((1, 2))                        # every fmaf rounds once, relative to its result
    node = part[:, -1]
    e_tree = torch.zeros_like(z)
    while node.shape[1] > 1:                                # the 5 shuffle levels: lane i adds lane i ^ o
        h = node.shape[1] // 2
        node = node[:, :h] + node[:, h:]
        e_tree = e_tree + node.abs().sum(1)                 # each add rounds once (31 adds reach lane 0)
    dz = (TANHF_ULPS * (W.abs() * ulp_f32(t)).sum(1)        # tanhf <= 2 ulp per term, weighted by |w_i|
          + U32 * (e_chain + e_tree)                        # the fmaf chains and the shuffle tree
          + U32 * z.abs()) * (1 + 2.0 ** -10)               # acc + b rounded; the factor covers second-order terms
                                                            # (rounding the already-perturbed sums: < 1e-4 relative)
    s = torch.sigmoid(z)
    ds = (s * (1 - s) * dz * torch.exp(dz)                  # dz through the sigmoid: s(1-s) changes by at most a
                                                            # factor e^dz across [z - dz, z + dz]
          + s * (1 - s) * EXPF_ULPS * 2.0 ** -23 * (1 + 2.0 ** -20)   # expf <= 2 ulp, relative 2^-22 of e = e^-z;
                                                                      # enters s scaled by e / (1 + e) = 1 - s
          + U32 * s                                         # 1 + e rounded: relative u on 1 + e and on s
          + U32 * s + 2.0 ** -150)                          # the division: relative u, or half a subnormal ulp
    return z, s, ds


def check_sigmoid(got, z, s, ds, what, median_ulps: float, max_bias: float = 0.05,
                  min_elems: int = 100_000) -> dict:
    """Assert that fp32 scores ``got`` are the sigmoids ``s`` (fp64) of logits ``z`` within ``ds``, except past the
    overflow of expf(-z) (z <= Z_SUB[0]), where the kernel returns 0; that the mean signed error is small against the
    bound; and the saturation bands: exactly 1.0 for z >= Z_ONE, a positive subnormal (never flushed) for z in Z_SUB,
    +0.0 (never -0.0) for z < Z_ZERO.  ``median_ulps``: median(ds / fp32 ulp of s) among |z| < 1 must stay below it."""
    got = got.double().reshape(-1).to(s.device)
    n = got.numel()
    assert n >= min_elems, f"{what}: {n} pairs are too few (need {min_elems})"
    assert not torch.isnan(got).any(), f"{what}: NaN score"
    mid = z.abs() < 1
    med = (ds[mid] / ulp_f32(s[mid])).median().item()
    assert med <= median_ulps, f"{what}: bound is vacuous: median bound = {med:.3g} fp32 ulp > {median_ulps}"
    live = z > Z_SUB[0]
    err = got - s
    excess = torch.where(live, err.abs() / ds, torch.zeros_like(s))
    worst = int(torch.argmax(excess))
    bias = (err[live] / ds[live]).mean().item()
    info = dict(worst=excess[worst].item(), bias=bias, median_bound_ulps=med, n=n)
    msg = (f"{what}: worst element {worst}: z {z[worst].item():.9g}, got {got[worst].item():.9g}, "
           f"exact {s[worst].item():.9g}, |err| {err[worst].abs().item():.3g} vs bound {ds[worst].item():.3g}; "
           f"mean signed error {bias:+.4f} of the bound")
    assert excess[worst] <= 1, msg
    assert abs(bias) <= max_bias, msg
    one, zero = z >= Z_ONE, z < Z_ZERO
    sub = (z > Z_SUB[0]) & (z < Z_SUB[1])
    assert (got[one] == 1.0).all(), f"{what}: {int((got[one] != 1).sum())} scores below 1.0 for z >= {Z_ONE}"
    gz = got[zero]
    assert (gz == 0).all() and not torch.signbit(gz).any(), f"{what}: scores other than +0.0 for z < {Z_ZERO}"
    gs = got[sub]
    assert ((gs > 0) & (gs < F32_MIN_NORMAL)).all(), f"{what}: {int((gs == 0).sum())} subnormal scores flushed"
    return info


def cross_head_case(n_pairs: int, dim: int, seed: int, device="cpu"):
    """Head inputs -> (rows bf16 [n, dim], w_out fp32 [dim], b_out): rows at the scale of a Linear output (N(0, 1)),
    2 % of the entries at |x| >= 9.5, where tanhf is exactly +-1; an output row with fp32 values that are not bf16
    values; logits spread over five bands in equal shares: |z| < 1, [-16, 16], z >= 17.5 (score 1.0f),
    (-88.6, -87.45) (subnormal score) and [-100, -89] (score 0).  Every 8th channel steers its pair's logit into its
    band: those carry |w| in [1.2, 1.8], and their row values are set so the pair's tanh sum lands on the target."""
    g = torch.Generator(device=device).manual_seed(seed)
    u = lambda *s: torch.rand(*s, generator=g, device=device, dtype=torch.float64)
    sign = lambda *s: torch.where(u(*s) < 0.5, -1.0, 1.0).to(torch.float64)
    steer = torch.arange(dim, device=device) % 8 == 7
    w = (torch.randn(dim, generator=g, device=device) * 0.05).double()
    w[steer] = sign(int(steer.sum())) * (1.2 + 0.6 * u(int(steer.sum())))
    w = w.float()
    b = -0.37109375 - 2.0 ** -20                              # an fp32 value, not a bf16 one
    x = torch.randn(n_pairs, dim, generator=g, device=device, dtype=torch.float64)
    big = u(n_pairs, dim) < 0.02
    x = torch.where(big, sign(n_pairs, dim) * (9.5 + 20 * u(n_pairs, dim)), x)
    bands = torch.tensor([[-1, 1], [-16, 16], [17.5, 30], [-88.6, -87.45], [-100, -89]], dtype=torch.float64,
                         device=device)
    pick = bands[torch.randint(0, 5, (n_pairs,), generator=g, device=device)]
    target = pick[:, 0] + (pick[:, 1] - pick[:, 0]) * u(n_pairs)
    xs = x[:, ~steer].to(torch.bfloat16)
    rest = torch.tanh(xs.double()) @ w[~steer].double() + b
    ws = w[steer].double()
    c = ((target - rest) / ws.abs().sum()).clamp(-1, 1)[:, None] * torch.sign(ws)[None, :]
    xv = torch.where(c.abs() >= math.tanh(9.5), torch.sign(c) * 12.0, torch.atanh(c.clamp(-0.999999, 0.999999)))
    x[:, ~steer] = xs.double()
    x[:, steer] = xv
    return x.to(torch.bfloat16), w, b


# ------------------------------------------------------------------------------------------ dense top-k
# The wgmma dense kernels (csrc/dense_tc.cu) compute each score as an fp32 accumulation over d / 16 k16 steps of
# bf16 x bf16 products, which are exact in fp32.  How the tensor core adds the 16 products of a step to the
# accumulator is not documented for Hopper: the products are aligned to the largest exponent and the sum may be
# truncated rather than rounded.  Each step is therefore allowed 17 units of 2^-23 relative to |S_j| + sum |p_i|
# (16 aligned products and the accumulator, each losing up to one ulp, plus the truncated result), where S_j is
# the exact partial sum after step j.  Not fitted to a measurement: the ratio an H100 shows is reported, not used.
DENSE_STEP_ULPS = 17
DENSE_K = 16                     # products per wgmma k step (bf16)


def dense_score_bound(q: torch.Tensor, c: torch.Tensor, ids: torch.Tensor, chunk: int = 1024):
    """-> (exact, delta) [Q, k] fp64: the score of each (query, returned id) pair and the bound on the kernel's fp32
    error in it.  ``q`` [Q, d], ``c`` [n, d] bf16 on one device; ``ids`` [Q, k] row indices (>= 0)."""
    nq, d = q.shape
    assert d % DENSE_K == 0
    k = ids.shape[1]
    exact = torch.empty(nq, k, dtype=torch.float64, device=q.device)
    delta = torch.empty_like(exact)
    for q0 in range(0, nq, chunk):
        qq = q[q0:q0 + chunk].double()
        rows = c[ids[q0:q0 + chunk].long()].double()                   # [Qc, k, d]
        p = qq[:, None, :] * rows                                       # exact: 8 + 8 significant bits
        steps = p.view(p.shape[0], k, d // DENSE_K, DENSE_K)
        part = steps.sum(-1).cumsum(-1)                                 # S_j after each k16 step
        exact[q0:q0 + chunk] = part[..., -1]
        delta[q0:q0 + chunk] = DENSE_STEP_ULPS * 2.0 ** -23 * (part.abs().sum(-1) + p.abs().sum(-1))
    return exact, delta


def dense_delta_max(q: torch.Tensor, c_norm_max: float):
    """[Q] fp64: an upper bound of ``dense_score_bound`` over every row of a corpus whose largest row norm is
    ``c_norm_max``: |S_j| <= ||q|| ||c|| for each of the d / 16 steps, and sum |p_i| <= ||q|| ||c|| (Cauchy-Schwarz)."""
    d = q.shape[1]
    return DENSE_STEP_ULPS * 2.0 ** -23 * (d / DENSE_K + 1) * q.double().norm(dim=1) * c_norm_max


def check_dense_topk(scores, ids, exact, delta, top_vals, top_ids, dmax, n_rows, what) -> dict:
    """Assert that a top-k result (``scores`` fp32 / ``ids`` [Q, k], every query with k results) is the fp64 top-k up
    to the kernel's error.  ``exact`` / ``delta``: fp64 score of each returned id and its bound (dense_score_bound);
    ``top_vals`` / ``top_ids`` [Q, K > k]: the fp64 top list, descending; ``dmax`` [Q]: dense_delta_max.
      * every returned score lies within delta of its id's fp64 score;
      * every id whose fp64 score beats the fp64 k-th by more than 2 dmax is returned (nothing clearly better left out);
      * no returned id scores below the fp64 k-th - 2 dmax;
      * ids are distinct rows, scores non-increasing, equal scores ordered by id descending.
    Returns the measured figures: worst |err| / delta, the share of scores equal to the fp32 rounding of the fp64
    score, and the queries whose fp64 (k+1)-th lies within 2 dmax of the k-th (where either id may be returned)."""
    nq, k = ids.shape
    dev = exact.device
    scores, ids = scores.to(dev), ids.to(dev).long()
    top_vals, top_ids, dmax = top_vals.to(dev), top_ids.to(dev).long(), dmax.to(dev)
    assert top_ids.shape[1] > k
    assert ((ids >= 0) & (ids < n_rows)).all(), f"{what}: ids outside [0, {n_rows})"
    srt = ids.sort(1).values
    assert (srt[:, 1:] != srt[:, :-1]).all(), f"{what}: a row returned twice"
    g = scores.double()
    ratio = (g - exact).abs() / delta
    w = int(torch.argmax(ratio))
    wq, wj = divmod(w, k)
    assert ratio.max() <= 1, (f"{what}: worst element query {wq} rank {wj} (id {int(ids[wq, wj])}): got "
                              f"{g[wq, wj].item():.9g}, fp64 {exact[wq, wj].item():.9g}, bound "
                              f"{delta[wq, wj].item():.3g}")
    kth = top_vals[:, k - 1]
    margin = 2 * dmax
    must = top_vals[:, :k] > (kth + margin)[:, None]
    found = (top_ids[:, :k, None] == ids[:, None, :]).any(-1)
    miss = must & ~found
    if miss.any():
        mq, mj = (int(x) for x in torch.nonzero(miss)[0])
        raise AssertionError(f"{what}: worst element query {mq}: id {int(top_ids[mq, mj])} (fp64 {top_vals[mq, mj].item():.9g}"
                             f", rank {mj}) beats the k-th ({kth[mq].item():.9g}) by more than {margin[mq].item():.3g} "
                             f"and is not returned")
    low = exact < (kth - margin)[:, None]
    if low.any():
        lq, lj = (int(x) for x in torch.nonzero(low)[0])
        raise AssertionError(f"{what}: worst element query {lq}: returned id {int(ids[lq, lj])} scores "
                             f"{exact[lq, lj].item():.9g} in fp64, below the k-th {kth[lq].item():.9g} - {margin[lq].item():.3g}")
    ds, di = scores[:, 1:] - scores[:, :-1], ids[:, 1:] - ids[:, :-1]
    bad = (ds > 0) | ((ds == 0) & (di > 0))
    assert not bad.any(), f"{what}: query {int(torch.nonzero(bad)[0, 0])}: not in (score desc, id desc) order"
    return dict(worst=ratio.max().item(), rn_share=(g == exact.float().double()).double().mean().item(),
                ambiguous=int((top_vals[:, k] >= kth - margin).sum()), queries=nq,
                median_delta=delta.median().item(), median_dmax=dmax.median().item())


# ------------------------------------------------------------------------------------------ L2 normalisation
# normalize_rows_kernel (csrc/dense.cu), one warp per row, fp32 without fast-math:
#     q   = sum of x_i^2: lane i % 32 runs ceil(d / 32) fmaf steps, then 5 xor-shuffle adds
#     inv = 1.0f / fmaxf(sqrtf(q), 1e-12f)      (sqrtf and the division are IEEE, correctly rounded)
#     out = bf16(x_i * inv)
NORM_FLOOR = float(torch.tensor(1e-12, dtype=torch.float32))    # the fp32 value of 1e-12f


def l2_normalize_exact_and_delta(x):
    """-> (exact, delta): the fp64 value of the kernel's function (rows below the 1e-12f floor are scaled by
    1 / 1e-12f, not normalised) and the bound on its fp32 error before the bf16 rounding.  Rows within a few ulps
    of the floor are not covered (either branch may be taken there)."""
    X = x.double()
    nrm = X.norm(dim=1, keepdim=True)
    exact = X / nrm.clamp_min(NORM_FLOOR)
    steps = -(-x.shape[1] // 32)
    rel = torch.where(nrm >= NORM_FLOOR,
                      (steps + 5) * U32 / 2          # q: every fmaf / shuffle add rounds relative to a partial sum
                                                     # <= q, so |q err| <= (steps + 5) u q; sqrt halves it
                      + U32                          # sqrtf
                      + 2 * U32,                     # 1 / norm; x * inv
                      torch.full_like(nrm, 2 * U32))   # below the floor: 1 / 1e-12f and x * inv
    return exact, exact.abs() * rel * (1 + 2.0 ** -10)   # the factor covers second-order terms
