"""Test infrastructure: error-bound checks for kernels whose result is a bf16 rounding of an fp32 computation.

A kernel that computes ``f`` in fp32 and rounds once to bf16 returns ``bf16_rn(f + e)`` with ``|e| <= delta`` (the
fp32 error of its accumulation and epilogue, bounded per test).  ``check_bf16`` compares such an output with the fp64
value of ``f`` on the same bf16 inputs and asserts three things: every element lies within ``delta`` plus one bf16
ulp; at least 99 % of the elements are exactly the round-to-nearest bf16 value of the fp64 result; and the rounding is
unbiased (a kernel that truncates instead of rounding to nearest shows a mean signed error of about -0.5 ulp).
Used by tests/test_gpu_model_shapes.py; checked itself by tests/test_bounds_cpu.py.
"""
import torch

U32 = 2.0 ** -24                 # unit roundoff of fp32 (round to nearest)
BF16_MIN_ULP = 2.0 ** -133       # ulp of the smallest bf16 subnormal (bf16 shares fp32's exponent range)


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
