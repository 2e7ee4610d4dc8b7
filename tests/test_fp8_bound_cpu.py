"""The error bound of the FP8 GEMM path (tests/_bounds_fp8.py: fp8_gemm_bound), checked on a numpy emulation of the
kernels (no GPU), and the argument checks of the FP8 entry points.

The emulation follows csrc/encoder/quant_fp8.cu and gemm_fp8.cu step by step: power-of-two scales, e4m3 rounding to
nearest-even, per 128-K chunk an MMA chain of four k32 steps under the bound's accumulator model (addends aligned to
the largest exponent and truncated to 13 fraction bits, the sum truncated to 14 bits), the fp32 promotion after
every chunk, the exact rescale, the epilogue in fp32 and the bf16 store.  The bound must hold on it, and must reject
four faults: truncating instead of rounding, one scale for the whole tensor instead of one per row, no promotion
(the reduced-precision chain run over all of K = 18944), and the scales applied twice.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from _bounds import rejects, round_bf16
from _bounds_fp8 import (FP8_CHUNK, FP8_K_STEP, FP8_MAX, FP8_MMA_FRAC, check_fp8, e4m3_rn, fp8_gemm_bound,
                         pow2_scale, quant_rows_ref)


# ------------------------------------------------------------------------------------------- numpy emulation
def np_pow2_scale(amax):
    m, e = np.frexp(np.asarray(amax, np.float64))
    s = np.ldexp(1.0, np.where(m <= 0.875, e - 9, e - 8))
    return np.where(amax > 0, s, 1.0)


def np_e4m3(x, trunc=False):
    """float64 -> e4m3 value, round to nearest-even (or toward zero), |x| <= 448."""
    x = np.asarray(x, np.float64)
    _, e = np.frexp(x)
    ulp = np.ldexp(1.0, np.maximum(e - 1, -6) - 3)
    r = np.trunc(x / ulp) if trunc else np.round(x / ulp)     # np.round: half to even
    return np.where(x == 0, 0.0, r * ulp)


def np_quant(x, per_tensor=False, trunc=False):
    amax = np.abs(x).max(1)
    s = np_pow2_scale(np.full_like(amax, amax.max()) if per_tensor else amax)
    return np_e4m3(x / s[:, None], trunc), s


def _trunc_sig(v, mx, bits):
    """v truncated toward zero to the grid 2^(floor(log2 mx) - bits) (mx > 0 elementwise or v == 0)."""
    _, e = np.frexp(np.where(mx > 0, mx, 1.0))
    grid = np.ldexp(1.0, e - 1 - bits)
    return np.where(mx > 0, np.trunc(v / grid) * grid, 0.0)


def mma_step(s, p):
    """One k32 step of the modelled fp8 MMA: s [n] partial sums, p [n, 32] exact products."""
    add = np.concatenate([s[:, None], p], 1)
    mx = np.abs(add).max(1)
    t = _trunc_sig(add, mx[:, None], FP8_MMA_FRAC).sum(1)
    return _trunc_sig(t, np.abs(t), FP8_MMA_FRAC)


def f32(x):
    return np.asarray(x, np.float64).astype(np.float32).astype(np.float64)


def gelu_f32(x):
    from math import erf, sqrt
    return f32(np.vectorize(lambda v: 0.5 * v * (1 + erf(v / sqrt(2))))(x))


def emulate(qa, sa, qw, sw, bias=None, res=None, epi=0, promote=True, scale_twice=False):
    """The kernel's arithmetic for every (row, column) of qa [M, K] x qw [N, K] -> bf16 values as float64."""
    m, k = qa.shape
    n = qw.shape[0]
    p = (qa[:, None, :] * qw[None, :, :]).reshape(m * n, k)          # e4m3 x e4m3: exact
    acc = np.zeros(m * n)
    s = np.zeros(m * n)
    for j in range(k // FP8_K_STEP):
        if promote and j % (FP8_CHUNK // FP8_K_STEP) == 0:
            s = np.zeros(m * n)
        s = mma_step(s, p[:, j * FP8_K_STEP:(j + 1) * FP8_K_STEP])
        if promote and (j + 1) % (FP8_CHUNK // FP8_K_STEP) == 0:
            acc = f32(acc + s)
    if not promote:
        acc = f32(s)
    scale = (sa[:, None] * sw[None, :]).reshape(-1)
    x = acc * scale                                                  # exact (powers of two)
    if scale_twice:
        x = x * scale
    x = x.reshape(m, n)
    if epi == 2:
        g = x.reshape(m, -1, 2, 64)
        gate, up = g[:, :, 0].reshape(m, -1), g[:, :, 1].reshape(m, -1)
        x = f32(f32(gate / f32(1 + np.exp(-gate))) * up)
    else:
        if bias is not None:
            x = f32(x + bias[None, :])
        if epi == 1:
            x = gelu_f32(x)
    if res is not None:
        x = f32(x + res)
    return round_bf16(torch.from_numpy(x)).numpy()


def _bound(a, w, qa, sa, qw, sw, bias=None, res=None, epi=0):
    T = lambda v: None if v is None else torch.from_numpy(np.asarray(v, np.float64))
    return fp8_gemm_bound(T(qa), T(sa), T(qw), T(sw), T(bias), T(res), epi, a=T(a), w=T(w))


def _bf16(x):
    return torch.from_numpy(np.asarray(x, np.float32)).to(torch.bfloat16).double().numpy()


def _check(got, exact, delta, what):
    return check_fp8(torch.from_numpy(got), exact, delta, what)


# ------------------------------------------------------------------------------------------- the emulation itself
def test_scale_and_rounding_match_definitions():
    amax = np.concatenate([FP8_MAX * np.ldexp(1.0, np.arange(-140, 120)),            # exactly 448 * 2^k
                           FP8_MAX * np.ldexp(1.0, np.arange(-140, 120)) * (1 + 2.0 ** -7),
                           np.random.default_rng(1).lognormal(0, 20, 2000)])
    amax = amax[np.isfinite(amax) & (amax < 3e38)]
    s = np_pow2_scale(amax)
    assert (amax / s <= FP8_MAX).all() and (amax / s > FP8_MAX / 2).all()            # the smallest such power of two
    assert np.array_equal(s, pow2_scale(torch.from_numpy(amax)).numpy())
    assert np_pow2_scale(np.array([0.0]))[0] == 1.0
    # every e4m3 value, midpoints (ties to even) and points between, against torch's own float8 conversion
    grid = torch.arange(256, dtype=torch.uint8).view(torch.float8_e4m3fn).double()
    grid = grid[torch.isfinite(grid)].unique()
    mid = (grid[1:] + grid[:-1]) / 2
    x = torch.cat([grid, mid, grid[1:] * 0.3 + grid[:-1] * 0.7]).clamp(-FP8_MAX, FP8_MAX)
    ref = x.float().to(torch.float8_e4m3fn).double()
    assert torch.equal(torch.from_numpy(np_e4m3(x.numpy())), ref)
    assert torch.equal(e4m3_rn(x), ref)
    # the stated quantisation error: max(2^-4 |x|, 2^-10 s) with s = 1 here
    assert ((e4m3_rn(x) - x).abs() <= torch.maximum(x.abs() * 2.0 ** -4, torch.full_like(x, 2.0 ** -10))).all()


def test_mma_model_truncates_to_14_bits():
    s = mma_step(np.array([1.0]), np.full((1, 32), 2.0 ** -15))     # each addend below the 2^-13 grid of the sum
    assert s[0] == 1.0
    s = mma_step(np.array([0.0]), np.array([[1.0 + 2.0 ** -13] + [0.0] * 31]))
    assert s[0] == 1.0 + 2.0 ** -13
    s = mma_step(np.array([0.0]), np.array([[1.0 + 2.0 ** -14] + [0.0] * 31]))
    assert s[0] == 1.0


# ---------------------------------------------------------------------------------------- the bound holds
EPI_CASES = [(0, False, False), (0, True, True), (1, True, False), (2, False, False)]


@pytest.mark.parametrize("epi,has_bias,has_res", EPI_CASES)
def test_bound_holds_on_emulation(epi, has_bias, has_res):
    rng = np.random.default_rng(10 + epi)
    m, k, n = 5, 3584, 256 if epi == 2 else 24
    a = _bf16(rng.standard_normal((m, k)))
    a[1] *= 2.0 ** -20                                                # rows at very different scales
    a[2, :7] = 0.0
    a[3, 5] = 300.0                                                   # one huge element: the rest turn subnormal
    w = _bf16(rng.standard_normal((n, k)) * 0.02)
    bias = _bf16(rng.standard_normal(n) * 0.02) if has_bias else None
    n_out = n // 2 if epi == 2 else n
    res = _bf16(rng.standard_normal((m, n_out))) if has_res else None
    qa, sa = np_quant(a)
    qw, sw = np_quant(w)
    got = emulate(qa, sa, qw, sw, bias, res, epi)
    exact, delta = _bound(a, w, qa, sa, qw, sw, bias, res, epi)
    info = _check(got, exact, delta, f"emulation epi={epi}")
    print(f"\n[fp8 bound] emulation epi={epi}: " + ", ".join(f"{kk}={v:.4g}" for kk, v in info.items()))


# --------------------------------------------------------------------------------------- negative controls
def _offset_case(rng, m, k, n):
    """Positive values 0.9 of an e4m3 ulp above a grid point: rounding to nearest moves each by 0.1 ulp, truncation
    by 0.9 ulp (beyond the half-ulp term), and every error has the same sign."""
    e = lambda *s: np.ldexp(1.0 + 0.9 / 8, rng.integers(-3, 4, s))
    return _bf16(e(m, k)), _bf16(e(n, k) * 2.0 ** -6)


def test_rejects_truncation():
    rng = np.random.default_rng(3)
    a, w = _offset_case(rng, 4, 1024, 8)
    qa, sa = np_quant(a)
    qw, sw = np_quant(w)
    exact, delta = _bound(a, w, qa, sa, qw, sw)
    _check(emulate(qa, sa, qw, sw), exact, delta, "rounded")
    ta, _ = np_quant(a, trunc=True)
    tw, _ = np_quant(w, trunc=True)
    assert rejects(_check, emulate(ta, sa, tw, sw), exact, delta, "truncated")


def test_rejects_per_tensor_scale():
    rng = np.random.default_rng(4)
    # positive operands, so the error of a row quantised with another row's scale cannot cancel
    a = _bf16(rng.uniform(0.5, 1.0, (4, 1024)) * np.ldexp(1.0, np.array([8, 0, -8, -14]))[:, None])
    w = _bf16(rng.uniform(0.5, 1.0, (8, 1024)) * 0.02)
    qa, sa = np_quant(a)
    qw, sw = np_quant(w)
    exact, delta = _bound(a, w, qa, sa, qw, sw)
    _check(emulate(qa, sa, qw, sw), exact, delta, "per row")
    pa, ps = np_quant(a, per_tensor=True)
    assert rejects(_check, emulate(pa, ps, qw, sw), exact, delta, "per tensor")


def test_rejects_no_promotion_at_k_18944():
    rng = np.random.default_rng(5)
    a = _bf16(rng.uniform(0.5, 1.0, (3, 18944)))
    w = _bf16(rng.uniform(0.5, 1.0, (4, 18944)) * 0.02)
    qa, sa = np_quant(a)
    qw, sw = np_quant(w)
    exact, delta = _bound(a, w, qa, sa, qw, sw)
    _check(emulate(qa, sa, qw, sw), exact, delta, "promoted")
    assert rejects(_check, emulate(qa, sa, qw, sw, promote=False), exact, delta, "not promoted")


def test_rejects_scale_applied_twice():
    rng = np.random.default_rng(6)
    a = _bf16(rng.standard_normal((4, 512)))
    w = _bf16(rng.standard_normal((8, 512)) * 0.02)
    qa, sa = np_quant(a)
    qw, sw = np_quant(w)
    exact, delta = _bound(a, w, qa, sa, qw, sw)
    _check(emulate(qa, sa, qw, sw), exact, delta, "once")
    assert rejects(_check, emulate(qa, sa, qw, sw, scale_twice=True), exact, delta, "twice")


def test_quant_rows_ref_matches_emulation():
    rng = np.random.default_rng(7)
    x = _bf16(rng.standard_normal((6, 256)) * np.ldexp(1.0, rng.integers(-30, 30, (6, 1))))
    q, s = quant_rows_ref(torch.from_numpy(x))
    nq, ns = np_quant(x)
    assert np.array_equal(q.numpy(), nq) and np.array_equal(s.numpy(), ns)


# --------------------------------------------------------------------------------------- argument checks
def test_fp8_entry_points_check_arguments(lib_built):
    from easyrag_b200 import _lib
    L = _lib.lib()
    buf = (C.c_uint8 * 4096)()
    base = (C.addressof(buf) + 15) // 16 * 16
    p = C.c_void_p(base)
    f = C.cast(C.c_void_p(base), C.POINTER(C.c_float))
    null = C.c_void_p(0)
    # K % 128
    assert L.ezr_gemm_fp8(p, f, 8, 192, 192, p, f, 8, 192, null, null, 0, p, 8, 0, null) == -1
    assert b"K % 128" in L.ezr_last_error()
    # strides and alignment
    assert L.ezr_gemm_fp8(p, f, 8, 128, 136, p, f, 8, 128, null, null, 0, p, 8, 0, null) == -1
    assert L.ezr_gemm_fp8(C.c_void_p(base + 8), f, 8, 128, 128, p, f, 8, 128, null, null, 0, p, 8, 0, null) == -1
    assert b"aligned" in L.ezr_last_error()
    # SwiGLU needs N % 128, scales are required, the epilogue must exist
    assert L.ezr_gemm_fp8(p, f, 8, 128, 128, p, f, 192, 128, null, null, 0, p, 96, 2, null) == -1
    assert L.ezr_gemm_fp8(p, null, 8, 128, 128, p, f, 8, 128, null, null, 0, p, 8, 0, null) == -1
    assert L.ezr_gemm_fp8(p, f, 8, 128, 128, p, f, 8, 128, null, null, 0, p, 8, 3, null) == -1
    # quantisers: cols % 8, 16-byte input, strides
    assert L.ezr_quant_rows_fp8(p, 12, 2, 12, p, 16, f, null) == -1
    assert L.ezr_quant_rows_fp8(C.c_void_p(base + 2), 16, 2, 16, p, 16, f, null) == -1
    assert L.ezr_quant_weight_fp8(p, 8, 2, 16, p, 16, f, null) == -1
    assert L.ezr_rmsnorm_fp8(p, 16, p, C.c_float(1e-6), 2, 8192, null, 0, p, 8192, f, null) == -1
    assert L.ezr_layernorm_fp8(p, 16, p, null, C.c_float(1e-6), 2, 16, null, 0, p, 16, f, null) == -1


def test_unknown_precision_is_rejected():
    from easyrag_b200.encoder import BertConfig, BertEncoder, Qwen2Config, Qwen2Encoder
    qc = Qwen2Config(vocab_size=8, hidden_size=128, intermediate_size=128, num_hidden_layers=1,
                     num_attention_heads=2, num_key_value_heads=2)
    bc = BertConfig(vocab_size=8, hidden_size=128, intermediate_size=128, num_hidden_layers=1, num_attention_heads=2)
    for bad in ("fp16", "FP8", "int8", None):
        with pytest.raises(ValueError, match="precision"):
            Qwen2Encoder(qc, {}, device="cpu", precision=bad)
        with pytest.raises(ValueError, match="precision"):
            BertEncoder(bc, {}, device="cpu", precision=bad)
