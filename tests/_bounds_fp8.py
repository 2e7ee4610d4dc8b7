"""Test infrastructure: the error bound of the FP8 encoder GEMMs (csrc/encoder/quant_fp8.cu, gemm_fp8.cu).

``fp8_gemm_bound`` bounds the kernel's output against fp64, either on the dequantised operands (accumulation and
epilogue only) or on the original bf16 operands (adding the quantisation term); ``check_fp8`` asserts it elementwise
and reports the worst error / bound.  ``pow2_scale`` / ``e4m3_rn`` / ``quant_rows_ref`` restate the quantisers.
Builds on the bf16 helpers of ``_bounds.py``.  Used by tests/test_gpu_encoder_fp8.py; checked itself on a numpy
emulation of the kernels by tests/test_fp8_bound_cpu.py.
"""
import math

import torch

from _bounds import U32, round_bf16, ulp_bf16


# The e4m3 path (csrc/encoder/quant_fp8.cu, gemm_fp8.cu) computes, for one output,
#     q_a = e4m3_rn(a / s_a), q_w = e4m3_rn(w / s_w)       power-of-two scales, one per activation row / weight row
#     per 128-K chunk: an MMA chain of 4 k32 steps from zero (reduced-precision accumulation inside the tensor core)
#     acc = fp32(acc + chunk)                              the promotion, once per chunk
#     x = (acc * s_a) * s_w                                exact: both scales are powers of two
#     then the bf16 kernel's epilogue (bias, GELU / SwiGLU, residual) and one bf16 rounding.
# The bound has three parts:
#   quantisation  |q(x) s - x| <= max(2^-4 |x|, 2^-10 s): half an e4m3 ulp, 2^-4 relative to a normal value (3
#                 mantissa bits), 2^-10 s absolute among the subnormals (spacing 2^-9 s).  |x / s| <= 448 by the
#                 choice of s, so nothing saturates.
#   accumulation  inside the MMA, per k32 step: Hopper's fp8 accumulation is undocumented; published reports
#                 (DeepSeek-V3, 3.3.2) find about 14 bits kept.  Modelled as: the 32 products and the chain's partial
#                 sum are aligned to the largest exponent and truncated to FP8_MMA_FRAC fraction bits (each loses
#                 less than 2^-13 of the largest addend, |S_{j-1}| + max |p_i| bounds that), then the sum is truncated
#                 to 14 bits: 2^-13 (34 |S_{j-1}| + 33 max_a max_w + |P_j|) per step, S the chunk's exact partial.
#                 Each promotion adds one fp32 rounding of the running total.
#   epilogue      the bf16 kernel's terms (bias add, GELU / SwiGLU propagation, residual add), then the bf16 store.
FP8_MAX = 448.0
FP8_MMA_FRAC = 13                # fraction bits kept by the modelled in-MMA accumulator (14-bit significand)
FP8_K_STEP = 32                  # products per wgmma k step (e4m3)
FP8_CHUNK = 128                  # promotion interval (gemm_fp8.cu)


def pow2_scale(amax: torch.Tensor) -> torch.Tensor:
    """s = 2^ceil(log2(amax / 448)) per element of ``amax`` (1 where amax == 0), fp64, from the exponent alone."""
    amax = amax.double()
    m, e = torch.frexp(amax)                                        # amax = m 2^e, m in [0.5, 1)
    ex = torch.where(m <= 0.875, e - 9, e - 8)
    return torch.where(amax > 0, torch.ldexp(torch.ones_like(amax), ex.to(torch.int32)), torch.ones_like(amax))


def e4m3_rn(x: torch.Tensor, trunc: bool = False) -> torch.Tensor:
    """fp64 -> nearest e4m3 value (ties to even), as fp64; |x| <= 448 assumed.  ``trunc`` rounds toward zero instead
    (a negative control)."""
    x = x.double()
    _, e = torch.frexp(x)                                           # |x| in [2^(e-1), 2^e)
    ulp = torch.ldexp(torch.ones_like(x), (torch.clamp(e - 1, min=-6) - 3).to(torch.int32))
    r = torch.trunc(x / ulp) if trunc else torch.round(x / ulp)
    return torch.where(x == 0, x, r * ulp)


def quant_rows_ref(x: torch.Tensor, per_tensor: bool = False, trunc: bool = False):
    """-> (q, s): e4m3 values (fp64) and the fp64 scales [rows] of ``x`` as the kernels quantise it.  ``per_tensor``
    uses one scale for the whole matrix (a negative control)."""
    X = x.double()
    amax = X.abs().amax(1)
    s = pow2_scale(amax.max().expand_as(amax) if per_tensor else amax)
    return e4m3_rn(X / s[:, None], trunc=trunc), s


def fp8_quant_err(x: torch.Tensor, s: torch.Tensor) -> torch.Tensor:
    """Bound on |q(x) s - x| per element, rows scaled by ``s``."""
    X = x.double()
    return torch.maximum(X.abs() * 2.0 ** -4, s.double()[:, None] * 2.0 ** -10)


def fp8_accum_delta(A: torch.Tensor, W: torch.Tensor) -> torch.Tensor:
    """Accumulation part of the bound for dequantised operands A [M, K], W [N, K] (fp64, the exact values the kernel
    multiplies): the in-MMA allowance of every k32 step and the fp32 rounding of every promotion."""
    m, k = A.shape
    n = W.shape[0]
    assert k % FP8_CHUNK == 0
    e = torch.zeros(m, n, dtype=torch.float64, device=A.device)
    total = torch.zeros_like(e)
    s = torch.zeros_like(e)
    for j in range(k // FP8_K_STEP):
        sl = slice(j * FP8_K_STEP, (j + 1) * FP8_K_STEP)
        if j % (FP8_CHUNK // FP8_K_STEP) == 0:
            s.zero_()
        p = A[:, sl] @ W[:, sl].T
        amw = A[:, sl].abs().amax(1)[:, None] * W[:, sl].abs().amax(1)[None, :]
        e += 2.0 ** -FP8_MMA_FRAC * (34 * s.abs() + 33 * amw + p.abs())
        s += p
        if (j + 1) % (FP8_CHUNK // FP8_K_STEP) == 0:
            total += s
            e += U32 * total.abs()                                  # acc = fp32(acc + chunk)
    return e * (1 + 2.0 ** -5)          # second order: the chain's computed partials exceed the exact ones by < 2 %


def _gelu64(x):
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def _silu64(x):
    return x / (1.0 + torch.exp(-x))


def split_gate_up(t: torch.Tensor, block: int):
    """[M, 2 ffn] with gate / up columns interleaved per ``block`` -> (gate, up)."""
    b = t.view(t.shape[0], -1, 2, block)
    return b[:, :, 0].reshape(t.shape[0], -1), b[:, :, 1].reshape(t.shape[0], -1)


def fp8_epilogue(acc, e_acc, bias, res, epi, block: int = 64):
    """-> (exact, delta): the epilogue of gemm_fp8.cu (= gemm_tc.cu's) applied to the fp64 accumulator ``acc`` whose
    kernel value is within ``e_acc``; delta bounds the fp32 error before the bf16 store.  epi: 0 none, 1 GELU,
    2 SwiGLU (gate / up interleaved per ``block`` columns)."""
    if epi == 2:
        g, u = split_gate_up(acc, block)
        eg, eu = split_gate_up(e_acc, block)
        if bias is not None:
            bg, bu = split_gate_up(bias.double()[None, :], block)
            g, u = g + bg, u + bu
            eg, eu = eg + U32 * (g.abs() + eg), eu + U32 * (u.abs() + eu)
        sg = _silu64(g)
        out = sg * u
        delta = (1.1 * u.abs() * eg + sg.abs() * eu + 1.1 * eg * eu
                 + out.abs() * ((2.0 + 1.173 * g.abs()) * 2.0 ** -23 + 3 * U32))   # as gemm_tc.cu's SwiGLU bound
    else:
        out, delta = acc, e_acc
        if bias is not None:
            out = acc + bias.double()
            delta = delta + U32 * (out.abs() + delta)
        if epi == 1:
            pre = out
            out = _gelu64(pre)
            delta = 1.13 * delta + torch.maximum(torch.full_like(out, 4.7e-7), 2.3e-4 * out.abs())
    if res is not None:
        out = out + res.double()
        delta = delta + U32 * (out.abs() + delta)
    return out, delta


def fp8_gemm_bound(qa, sa, qw, sw, bias=None, res=None, epi=0, a=None, w=None):
    """-> (exact, delta) for gemm_fp8 on e4m3 operands ``qa`` [M, K] / ``qw`` [N, K] with scales ``sa`` [M] / ``sw``
    [N].  Without ``a`` / ``w``: exact is the fp64 value on the dequantised operands and delta covers accumulation,
    epilogue (isolating the kernel's arithmetic).  With the original operands ``a`` / ``w``: exact is their fp64
    value and delta adds the quantisation term."""
    A = qa.double() * sa.double()[:, None]
    W = qw.double() * sw.double()[:, None]
    e = fp8_accum_delta(A, W)
    if a is None:
        acc = A @ W.T
    else:
        ea, ew = fp8_quant_err(a, sa), fp8_quant_err(w, sw)
        Aa, Wa = a.double().abs(), w.double().abs()
        e = e + Aa @ ew.T + ea @ Wa.T + ea @ ew.T
        acc = a.double() @ w.double().T
    return fp8_epilogue(acc, e, bias, res, epi)


def check_fp8(got: torch.Tensor, exact: torch.Tensor, delta: torch.Tensor, what: str) -> dict:
    """Assert |got - exact| <= delta + one bf16 ulp everywhere; report the worst ratio and the rounding share."""
    got = got.double().reshape(-1)
    exact = exact.double().reshape(-1).to(got.device)
    delta = delta.double().reshape(-1).to(got.device)
    assert torch.isfinite(got).all(), f"{what}: non-finite output"
    err = (got - exact).abs()
    lim = delta + ulp_bf16(exact.abs() + delta)
    ratio = err / lim
    worst = int(torch.argmax(ratio))
    info = dict(worst=ratio[worst].item(), median_err_over_bound=(err / lim).median().item(),
                median_bound_ulps=(delta / ulp_bf16(exact)).median().item(),
                rn_share=(got == round_bf16(exact)).double().mean().item(), n=got.numel())
    assert ratio[worst] <= 1, (f"{what}: worst element {worst}: got {got[worst].item():.9g}, exact "
                               f"{exact[worst].item():.9g}, |err| {err[worst].item():.3g} vs bound {lim[worst].item():.3g}")
    return info
