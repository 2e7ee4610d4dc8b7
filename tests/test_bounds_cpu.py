"""CPU: the bf16 error-bound checker of tests/_bounds.py accepts correct roundings and rejects biased or wrong ones."""
import pytest
import torch

from _bounds import check_bf16, rejects, round_bf16, ulp_bf16

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
