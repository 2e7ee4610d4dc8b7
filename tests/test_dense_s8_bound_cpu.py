"""The certified int8 candidate bound of csrc/dense_s8.cu, checked in numpy (no GPU).

A numpy emulation of the quantizer, of s^ = fl(fl(a_q a_r) * (float)S) and of rescore (fp32, increasing coordinate
order, separate multiply and add) checks |rescore - s^| <= D_q on every (query, row) pair, and that the rows with
s^ >= T - 2 D_q under the worst admissible T (the k-th best s^ itself) contain the exact rescore top-k.  A negative
control builds a case whose answer row the certified margin keeps and half of it loses.
"""
import numpy as np
import pytest

U = 2.0 ** -24


def bf16(x):
    """Round float32 values to bf16 (nearest even) and return them as float32."""
    b = np.asarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    b = (b + 0x7FFF + ((b >> 16) & 1)) & 0xFFFF0000
    return b.astype(np.uint32).view(np.float32)


def quantize(x):
    x = x.astype(np.float32)
    scale = (np.abs(x).max(1) / np.float32(127)).astype(np.float32)
    safe = np.where(scale > 0, scale, np.float32(1))
    r = np.clip(np.rint((x / safe[:, None]).astype(np.float32)), -127, 127)
    r = np.where(scale[:, None] > 0, r, 0).astype(np.int32)
    a = scale[:, None].astype(np.float64) * r
    e = np.sqrt(((x.astype(np.float64) - a) ** 2).sum(1)).astype(np.float32)
    n = np.sqrt((a ** 2).sum(1)).astype(np.float32)
    # rounded up to fp32, as the kernel's __double2float_ru
    e64 = np.sqrt(((x.astype(np.float64) - a) ** 2).sum(1))
    n64 = np.sqrt((a ** 2).sum(1))
    e = np.where(e.astype(np.float64) < e64, np.nextafter(e, np.float32(np.inf)), e)
    n = np.where(n.astype(np.float64) < n64, np.nextafter(n, np.float32(np.inf)), n)
    return r, scale, e, n


def margin(eq, nq, emax, nmax, dim):
    """2 D_q of the kernel header, fp64."""
    gam = dim * U / (1 - dim * U)
    d = (nq * emax + eq * nmax + eq * emax + gam * (nq + eq) * (nmax + emax) + dim * 2.0 ** -149
         + (2 * U + U * U) * nq * nmax + 2.0 ** -125)
    return 2 * d * (1 + 2.0 ** -20)


def s_hat(q_r, q_s, c_r, c_s):
    S = (q_r.astype(np.int64) @ c_r.T.astype(np.int64)).astype(np.float32)     # exact: |S| < 2^24
    a = (q_s[:, None] * c_s[None, :]).astype(np.float32)
    return (a * S).astype(np.float32)


def rescore(q, c):
    acc = np.zeros((q.shape[0], c.shape[0]), dtype=np.float32)
    for i in range(q.shape[1]):
        acc = (acc + (q[:, i:i + 1] * c[None, :, i]).astype(np.float32)).astype(np.float32)
    return acc + np.float32(0)


def unit(rng, n, dim):
    x = rng.standard_normal((n, dim)).astype(np.float32)
    return bf16(x / np.linalg.norm(x, axis=1, keepdims=True))


def data(kind, dim, rng):
    c = unit(rng, 400, dim)
    q = unit(rng, 12, dim)
    if kind == "dominant":
        c[::7] = bf16(np.full(dim, 1e-3, np.float32))
        c[::7, 3] = 1.0
        q[0] = c[7]
    elif kind == "zero":
        c[5] = 0
        q[1] = 0
    elif kind == "clustered":
        q = bf16(c[:12] + 0.3 * unit(rng, 12, dim))
    return q, c


def canonical(s, k):
    order = np.lexsort((-np.arange(s.size), -s.astype(np.float64)))
    return order[:k]


@pytest.mark.parametrize("dim", [128, 256, 768, 1024])
@pytest.mark.parametrize("kind", ["unit", "dominant", "zero", "clustered"])
def test_bound_holds_and_candidates_cover_topk(dim, kind):
    rng = np.random.default_rng(dim * 7 + len(kind))
    q, c = data(kind, dim, rng)
    cr, cs, ce, cn = quantize(c)
    qr, qs, qe, qn = quantize(q)
    emax, nmax = float(ce.max()), float(cn.max())
    sh = s_hat(qr, qs, cr, cs).astype(np.float64)
    sp = rescore(q, c).astype(np.float64)
    for i in range(q.shape[0]):
        m = margin(float(qe[i]), float(qn[i]), emax, nmax, dim)
        assert (np.abs(sp[i] - sh[i]) <= m / 2).all()
        for k in (1, 10, 16):
            T = np.sort(sh[i])[::-1][k - 1]               # the largest admissible T
            thr = np.float32(T - m)                       # the kernel rounds this down; float64 here is exact enough
            emitted = set(np.nonzero(sh[i] >= min(float(thr), T - m))[0].tolist())
            assert set(canonical(sp[i].astype(np.float32), k).tolist()) <= emitted


def constructed_case():
    """Two rows whose quantization errors are as large as Cauchy-Schwarz allows and point in opposite directions.

    d = 128, q = (1/16, ..., 1/16).  Both rows hold 127/128 in coordinate 0, so their scale is exactly 2^-7, and
    half-step values (j + 0.5) 2^-7 elsewhere, which round half to even by a full half step.  Row A uses j = 2
    (rounds down: s^ under-estimates the score by ~0.031), row B mixes j = 1 and j = 3 (rounds up: s^
    over-estimates by ~0.031).  A's score is higher by 2^-4 2^-7 = 4.9e-4, so A is the top-1 answer, yet its s^
    lies below s^_B = T by almost 2 D_q: only the full certified margin keeps it."""
    dim = 128
    q = np.full((1, dim), 1 / 16, np.float32)
    a = np.full(dim, 2.5 / 128, np.float32)
    b = np.full(dim, 3.5 / 128, np.float32)
    b[1:65] = 1.5 / 128
    a[0] = b[0] = 127 / 128
    c = np.stack([a, b])
    assert np.array_equal(bf16(c), c) and np.array_equal(bf16(q), q)
    return q, c


def test_half_margin_loses_an_answer_row():
    """Negative control: in the constructed case, the rows with s^ >= T - 2 D_q (the kernel's rule, the same
    ``margin()`` as the coverage test, T = the top s^) contain the answer; with the margin halved they do not."""
    q, c = constructed_case()
    cr, cs, ce, cn = quantize(c)
    qr, qs, qe, qn = quantize(q)
    assert cs[0] == cs[1] == 2.0 ** -7
    sh = s_hat(qr, qs, cr, cs).astype(np.float64)[0]
    sp = rescore(q, c)[0]
    m = margin(float(qe[0]), float(qn[0]), float(ce.max()), float(cn.max()), q.shape[1])
    assert (np.abs(sp.astype(np.float64) - sh) <= m / 2).all()          # the bound holds here too
    answer = canonical(sp, 1)[0]
    assert answer == 0 and sh[1] > sh[0]                                 # s^ ranks the rows the other way
    T = sh.max()
    assert sh[answer] >= T - m                                           # kept under the certified margin
    assert sh[answer] < T - m / 2                                        # lost under half of it
