"""CPU: the rounding model behind the exact length-2 attention case of tests/test_gpu_encode_batches.py.

For a sequence of two tokens whose logits are equal, the wgmma attention kernel (csrc/encoder/attention_tc.cuh)
computes, in fp32: p = ex2(fma(s, scale log2 e, -m scale log2 e)) for both keys, P = bf16(p) as the A operand of
O = P V, l = p + p, and out = bf16_rn(O * (1 / l)).  This emulates those steps with numpy fp32 and torch's bf16
rounding, for V values of magnitude [0.25, 4) as the GPU test draws them, and checks the two claims the GPU test rests
on: with p = 1 (logits exactly 0) the output is the round-to-nearest-even bf16 of the exact mean of the two V rows,
ties included; with p a few fp32 ulps off 1 (equal logits s that are not 0: the fma leaves the rounding error of
s scale log2 e, up to 2^-24 |s scale log2 e|, and ex2.approx adds up to 2 ulps) it is the same except on a tie, where
it may be the other neighbour.
"""
import numpy as np
import torch

from _bounds import round_bf16, ulp_bf16


def _v_pairs(n, seed):
    g = torch.Generator().manual_seed(seed)
    mag = torch.exp2(torch.rand(2, n, generator=g) * 4 - 2)
    sign = torch.where(torch.rand(2, n, generator=g) < 0.5, -1.0, 1.0)
    v = (mag * sign).to(torch.bfloat16)
    return v[0], v[1]


def _kernel_out(v0, v1, p):
    """The kernel's steps in fp32 for probability p (both keys) -> bf16 output as fp64."""
    p = np.float32(p)
    pb = np.float32(torch.tensor(float(p)).to(torch.bfloat16).item())            # P as the bf16 A operand
    o = pb * v0.float().numpy() + pb * v1.float().numpy()                        # fp32 accumulation of P V
    inv = np.float32(1) / (p + p)
    return torch.from_numpy((o * inv).astype(np.float32)).to(torch.bfloat16).double()


def test_length_two_rounding_model():
    v0, v1 = _v_pairs(200_000, 3)
    a, b = v0.double(), v1.double()
    assert torch.equal(torch.from_numpy(v0.float().numpy() + v1.float().numpy()).double(), a + b)   # exact in fp32
    mean = (a + b) / 2
    want = round_bf16(mean)
    tie = (mean - want).abs() == ulp_bf16(mean) / 2
    other = 2 * mean - want
    assert tie.double().mean().item() > 0.2
    # logits exactly 0: p = 1, the output is the rounded mean everywhere
    assert torch.equal(_kernel_out(v0, v1, 1.0), want)
    # a kernel that truncated instead of rounding to nearest even would differ on the ties the GPU test meets
    trunc = torch.sign(mean) * torch.floor(mean.abs() / ulp_bf16(mean)) * ulp_bf16(mean)
    assert (trunc != want).double().mean().item() > 0.1
    # equal logits that are not 0: p within 8 fp32 ulps of 1
    for p in [1 - k * 2 ** -24 for k in (1, 2, 4, 8)] + [1 + k * 2 ** -23 for k in (1, 2, 4, 8)]:
        got = _kernel_out(v0, v1, p)
        assert torch.equal(got[~tie], want[~tie]), p
        assert ((got == want) | (got == other))[tie].all(), p
