"""GPU: the encoder kernels and dense search at the shapes of the models the pipeline runs, against fp64 references.

Shapes: gte-Qwen2-7B-instruct (d 3584, 28 query / 4 KV heads of 128, FFN 18944, texts up to 8192 tokens) and the
XLM-R-large-shaped cross-encoders (bge-reranker-large / -v2-m3: d 1024, 16 heads of 64, FFN 4096).  Every reference
is computed in float64 with plain torch ops on the same bf16 inputs (products of bf16 values are exact in fp64).
GEMM and norm outputs go through ``_bounds.check_bf16``: an error bound derived from each kernel's rounding points
(every term commented with the kernel step it covers), a correct-rounding rate and a rounding-bias test.  Each test
also runs negative controls -- references that are wrong in a small, specific way -- and asserts the checks reject
them.  The figures each check measures are printed (``pytest -s``).
"""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from _attn_ref import _attn_check, _attn_ref
from _bounds import U32, check_bf16, ln_exact_and_delta, rejects, round_bf16, ulp_bf16
from _topk_ref import canonical_topk
from oracle import encoder as oenc
from oracle import retrieve as ort
from easyrag_b200 import _lib, batched, encoder as enc, synth
from easyrag_b200.encoder import PackedBatch, Qwen2Config, Qwen2Encoder, random_state
from easyrag_b200.index import DenseIndex

pytestmark = pytest.mark.gpu
DEV = "cuda"
W_STD = 0.02           # encoder.random_state's default weight std
LAM = 4.0              # probabilistic accumulation bound (Higham & Mary 2019): |err| <= LAM sqrt(K) u sum|a_i b_i| fails
                       # with probability <= 2 exp(-LAM^2 / 2) per element under independent rounding errors; the real
                       # error is far smaller: bf16 products are exact in fp32 and only K / 16 partial sums round
COS_TOL = 1e-3         # cosine scores of the bf16 dense route (the north star's tolerance)


@pytest.fixture(scope="module", autouse=True)
def _ready(lib_built):
    _lib.require_cuda()


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _randn(*shape, seed, std=1.0):
    return (torch.randn(*shape, generator=_gen(seed), device=DEV) * std).to(torch.bfloat16)


def _report(what, info):
    print(f"\n[bounds] {what}: " + ", ".join(f"{k}={v:.5g}" if isinstance(v, float) else f"{k}={v}"
                                          for k, v in info.items()))


# ------------------------------------------------------------------------------------------------ GEMM
# (name, M, K, N, bias, epilogue, residual, least correctly rounded share)
# The share of outputs equal to the fp64 result rounded to nearest falls with K: the fp32 accumulation of wgmma errs
# by an amount that grows about linearly in K relative to a bf16 ulp of the result (measured on an H100 80GB HBM3:
# 99.95 % at K = 1024, 99.8 % at 3584, 99.74 % at 4096, 98.96 % at 18944, every error inside the fp32 bound and the
# rounding bias within 0.004 ulp).  The kernel is deterministic, so the K = 18944 case keeps a stated 98.5 %.
GEMM_CASES = [
    ("qwen2-qkv", 333, 3584, 4608, True, enc.EPI_NONE, False, 0.99),
    ("qwen2-o-proj-inplace", 300, 3584, 3584, False, enc.EPI_NONE, True, 0.99),
    ("qwen2-swiglu", 333, 3584, 2 * 18944, False, enc.EPI_SWIGLU, False, 0.99),
    ("qwen2-down-inplace", 77, 18944, 3584, False, enc.EPI_NONE, True, 0.985),
    ("xlmr-qkv", 512, 1024, 3072, True, enc.EPI_NONE, False, 0.99),
    ("xlmr-ffn1-gelu", 333, 1024, 4096, True, enc.EPI_GELU, False, 0.99),
    ("xlmr-ffn2", 200, 4096, 1024, True, enc.EPI_NONE, True, 0.99),
]


def _gelu64(x):
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def _silu64(x):
    return x / (1.0 + torch.exp(-x))


def _split_gate_up(t):
    """[M, 2 ffn] in the interleaved layout (blocks of 128 gate columns, then their 128 up columns) -> gate, up."""
    m = t.shape[0]
    b = t.view(m, -1, 2, 128)
    return b[:, :, 0].reshape(m, -1), b[:, :, 1].reshape(m, -1)


def _gemm_exact(a, w, bias, res, epi, kdrop=0, bias_shift=False, swap_block=False):
    """fp64 value of the GEMM's function on the same bf16 inputs; the keyword arguments build the negative controls."""
    A, W = a.double(), w.double()
    if kdrop:
        A, W = A[:, :-kdrop], W[:, :-kdrop]
    acc = A @ W.T
    if epi == enc.EPI_SWIGLU:
        g, u = _split_gate_up(acc)
        if swap_block:
            g, u = g.clone(), u.clone()
            g[:, :128], u[:, :128] = u[:, :128].clone(), g[:, :128].clone()
        out = _silu64(g) * u
    else:
        out = acc
        if bias is not None:
            out = out + (torch.roll(bias.double(), 1) if bias_shift else bias.double())
        if epi == enc.EPI_GELU:
            out = _gelu64(out)
    if res is not None:
        out = out + res.double()
    return out


def _gemm_delta(a, w, bias, res, epi):
    """Per-element bound on the kernel's fp32 error before its final bf16 rounding (gemm_tc.cu)."""
    k = a.shape[1]
    A, W = a.double(), w.double()
    acc = A @ W.T
    absacc = A.abs() @ W.abs().T
    e_acc = LAM * math.sqrt(k) * U32 * absacc              # wgmma fp32 accumulation of the K products
    if epi == enc.EPI_SWIGLU:
        g, u = _split_gate_up(acc)
        eg, eu = _split_gate_up(e_acc)
        s = _silu64(g)
        out = s * u
        delta = (1.1 * u.abs() * eg                        # gate accumulation error through silu' (|silu'| <= 1.0998)
                 + s.abs() * eu                            # up accumulation error times silu(gate)
                 + 1.1 * eg * eu                           # second-order product of the two
                 + out.abs() * ((2.0 + 1.173 * g.abs()) * 2.0 ** -23   # __expf(-g): <= 2 + floor(|1.173 g|) fp32 ulps
                                                                          # (CUDA C Programming Guide); enters silu
                                                                          # scaled by e / (1 + e) <= 1
                                + U32                      # 1 + e rounded to fp32 (relative effect on silu <= u)
                                + U32                      # IEEE fp32 division g / (1 + e)
                                + U32))                    # silu(g) * up rounded to fp32
    else:
        pre = acc if bias is None else acc + bias.double()
        delta = e_acc
        if bias is not None:
            delta = delta + U32 * (absacc + bias.double().abs())   # fp32 rounding of acc + bias
        out = pre
        if epi == enc.EPI_GELU:
            out = _gelu64(pre)
            delta = (1.13 * delta                          # accumulation / bias error through gelu' (max 1.129)
                     + torch.maximum(torch.full_like(out, 4.7e-7), 2.3e-4 * out.abs()))
                     # gelu_erf's own stated accuracy (4.7e-7 absolute or 2.3e-4 relative): the weaker of the two
    if res is not None:
        delta = delta + U32 * (out.abs() + delta + res.double().abs())   # fp32 rounding of the residual add
    return delta


@pytest.mark.parametrize("case", GEMM_CASES, ids=[c[0] for c in GEMM_CASES])
def test_gemm_model_shapes_within_fp32_bound(case):
    name, m, k, n, has_bias, epi, has_res, min_rate = case
    seed = 1000 + k + n + m
    a = _randn(m, k, seed=seed)                                                 # activations ~ N(0, 1)
    w = _randn(n, k, seed=seed + 1, std=W_STD)
    bias = _randn(n, seed=seed + 2, std=W_STD) if has_bias else None
    n_out = n // 2 if epi == enc.EPI_SWIGLU else n
    res = _randn(m, n_out, seed=seed + 3) if has_res else None
    if has_res:                                    # in place, as the layers call it: out = residual = x
        x = res.clone()
        got = enc.gemm(a, w, bias=bias, residual=x, out=x, epilogue=epi)
        assert got.data_ptr() == x.data_ptr()
    else:
        got = enc.gemm(a, w, bias=bias, epilogue=epi)
    assert got.shape == (m, n_out)
    exact = _gemm_exact(a, w, bias, res, epi)
    delta = _gemm_delta(a, w, bias, res, epi)
    info = check_bf16(got, exact, delta, name, median_ulps=1.5, min_rate=min_rate)
    _report(f"gemm {name} M={m} K={k} N={n}", info)
    # negative controls: the same checks must reject references that are wrong in a small way
    ctl = {"last 16 K columns dropped": _gemm_exact(a, w, bias, res, epi, kdrop=16)}
    if has_bias:
        ctl["bias shifted by one column"] = _gemm_exact(a, w, bias, res, epi, bias_shift=True)
    if epi == enc.EPI_SWIGLU:
        ctl["gate and up swapped in one 128-column block"] = _gemm_exact(a, w, bias, res, epi, swap_block=True)
    for what, wrong in ctl.items():
        assert rejects(check_bf16, got, wrong, delta, f"{name} control", median_ulps=1.5, min_rate=min_rate), \
            f"{name}: accepted {what}"


# ---------------------------------------------------------------------------------------------- norms
NORM_ROWS = 203                        # not a multiple of the warp kernel's 8 rows per CTA


def _norm_input(dim, seed, ld=None, offset_rows=False):
    """Rows of N(0, 1) with four outlier channels about 1000x the rest (as in real Qwen2 residual streams).
    ``offset_rows``: the second half of the rows sits on a large common offset instead (centred near 32, spread 0.3:
    mean ~ 100x the std), which defeats a one-pass fp32 variance.  ``ld``: row stride of the buffer the rows are a
    view of."""
    ld = ld or dim
    g = _gen(seed)
    x = torch.randn(NORM_ROWS, ld, generator=g, device=DEV)
    ch = torch.randperm(dim, generator=g, device=DEV)[:4]
    x[:, ch] *= 1000.0
    half = NORM_ROWS // 2
    if offset_rows:
        x[half:] = 32.0 + 0.3 * torch.randn(NORM_ROWS - half, ld, generator=g, device=DEV)
    buf = x.to(torch.bfloat16)
    return buf[:, :dim]


def _rms_exact(x, gamma, eps):
    """Qwen2RMSNorm's rounding points with fp64 statistics: y = bf16(x * rstd), out = gamma * y (then bf16)."""
    X = x.double()
    rstd = torch.rsqrt(X.pow(2).mean(-1, keepdim=True) + eps)
    return gamma.double() * round_bf16(X * rstd)


RMS_CASES = [  # (dim, row stride): warp kernel MAXC = 16 (1032..4096), MAXC = 4 (<= 1024); block kernel otherwise
    (3584, None), (1536, None), (4096, None), (1032, None), (1024, None), (5120, None), (3588, None), (3584, 3587)]


@pytest.mark.parametrize("dim,ld", RMS_CASES, ids=[f"{d}" + (f"-ld{l}" if l else "") for d, l in RMS_CASES])
def test_rmsnorm_model_dims(dim, ld):
    x = _norm_input(dim, 7 + dim, ld)
    gamma = (1 + 0.1 * torch.randn(dim, generator=_gen(8 + dim), device=DEV)).to(torch.bfloat16)
    got = enc.rmsnorm(x, gamma, 1e-6)
    exact = _rms_exact(x, gamma, 1e-6)
    # delta = 0: the kernel's last step, bf16 gamma x bf16 y, is exact in fp32 before its rounding.  The bf16 rounding
    # of y in the middle may flip by one ulp where the fp32 rstd differs from fp64 in its last bits.  One ulp of y is at
    # most 2^-7 |y|, which is up to 2 ulps of gamma * y (a bf16 ulp spans 2^-8 to 2^-7 of the value), and the final
    # rounding of a flipped product adds up to one more (measured on an H100: 2.26 ulps at dim 4096): 3 ulps per element
    info = check_bf16(got, exact, 0.0, f"rmsnorm {dim}", median_ulps=0.0, ulps=3.0)
    _report(f"rmsnorm dim={dim} ld={ld or dim}", info)
    wrong = _rms_exact(x, torch.roll(gamma, 1), 1e-6)
    assert rejects(check_bf16, got, wrong, 0.0, "rms control", median_ulps=0.0, ulps=3.0)
    wrong = exact * (1 + 2.0 ** -7)                                 # a 1/128 relative scale error of rstd
    assert rejects(check_bf16, got, wrong, 0.0, "rms control", median_ulps=0.0, ulps=3.0)


LN_CASES = [(1024, 1e-5, None), (1024, 1e-5, 1029), (768, 1e-12, None), (768, 1e-12, 771)]   # warp / block kernel


@pytest.mark.parametrize("dim,eps,ld", LN_CASES, ids=[f"{d}-{'block' if l else 'warp'}" for d, _, l in LN_CASES])
def test_layernorm_model_dims(dim, eps, ld):
    x = _norm_input(dim, 17 + dim, ld, offset_rows=True)
    gamma = (1 + 0.1 * torch.randn(dim, generator=_gen(18 + dim), device=DEV)).to(torch.bfloat16)
    beta = _randn(dim, seed=19 + dim, std=0.1)
    got = enc.layernorm(x, gamma, beta, eps)
    exact, delta = ln_exact_and_delta(x, gamma, beta, eps)
    info = check_bf16(got, exact, delta, f"layernorm {dim}", median_ulps=0.1)
    _report(f"layernorm dim={dim} eps={eps} ld={ld or dim}", info)
    # control: a one-pass variance E[x^2] - E[x]^2 accumulated serially in fp32 (what the offset rows defeat)
    X = x.float()
    s = torch.zeros(NORM_ROWS, device=DEV)
    q = torch.zeros(NORM_ROWS, device=DEV)
    for j in range(dim):
        s += X[:, j]
        q += X[:, j] * X[:, j]
    var1 = (q / dim - (s / dim) ** 2).clamp_min(0).double()[:, None]
    wrong = (x.double() - x.double().mean(-1, keepdim=True)) * torch.rsqrt(var1 + eps) * gamma.double() + beta.double()
    assert rejects(check_bf16, got, wrong, delta, "ln control", median_ulps=0.1)


# ---------------------------------------------------------------------------------------------- pooling
def _pool(h, cu, pool, final_norm, gamma, eps, l2):
    L = _lib.lib()
    n_seq, dim = cu.numel() - 1, h.shape[1]
    ob = torch.empty(n_seq, dim, dtype=torch.bfloat16, device=DEV)
    of = torch.empty(n_seq, dim, dtype=torch.float32, device=DEV)
    _lib.check(L.ezr_pool_normalize(_lib.ptr(h), h.stride(0), _lib.ptr(cu), n_seq, pool, final_norm, _lib.ptr(gamma),
                                    eps, l2, dim, _lib.ptr(ob), _lib.ptr(of), _lib.stream_ptr()), "ezr_pool_normalize")
    torch.cuda.synchronize()
    return ob, of


@pytest.mark.parametrize("dim", [3584, 1536])
def test_pool_last_token_rmsnorm_bf16_l2_matches_torch_bf16_ops(dim):
    """Qwen2Encoder's pooling: last token, final RMSNorm, F.normalize on a bf16 tensor (gte_embeddings.py:42-50,70)."""
    g = torch.Generator().manual_seed(dim)
    lens = torch.randint(1, 40, (64,), generator=g).tolist()
    h = _randn(sum(lens), dim, seed=30 + dim, std=3.0)
    gamma = (1 + 0.1 * torch.randn(dim, generator=_gen(31 + dim), device=DEV)).to(torch.bfloat16)
    cu = torch.tensor(np.cumsum([0] + lens), dtype=torch.int32, device=DEV)
    ob, of = _pool(h, cu, enc.POOL_LAST, 1, gamma, 1e-6, 1)
    last = h[cu[1:].long() - 1]                                         # pooled bf16 rows
    y = oenc._rms(last, gamma, 1e-6)                                     # bf16 in, bf16 out (torch bf16 ops)
    ref = F.normalize(y, p=2, dim=1)                                     # norm rounded to bf16, then the division
    assert ref.dtype == torch.bfloat16
    same = (ob == ref)
    diff = (ob.double() - ref.double()).abs()
    _report(f"pool last+rms+bf16-l2 dim={dim}", dict(identical=same.double().mean().item(),
                                                      rows_identical=int(same.all(1).sum()), rows=len(lens)))
    # bit-identical except where the bf16-rounded norm (or an intermediate bf16 of the RMSNorm) lands on the other side
    # of a rounding boundary: then by one ulp
    assert (diff <= ulp_bf16(ref.double())).all()
    assert same.double().mean().item() >= 0.999
    assert torch.equal(of, ob.float())                                   # l2 = 1: the float copy is the bf16 row
    # control: fp32 normalisation semantics (unrounded norm) differs on many elements
    ref2 = (y.float() / y.float().norm(dim=1, keepdim=True)).to(torch.bfloat16)
    assert (ref2 != ob).double().mean().item() > 0.01


@pytest.mark.parametrize("l2", [0, 2])
def test_pool_mean_8192_and_1_token(l2):
    dim, lens = 3584, [8192, 1]
    h = (torch.randn(sum(lens), dim, generator=_gen(40 + l2), device=DEV)
         + torch.randn(dim, generator=_gen(41), device=DEV)).to(torch.bfloat16)       # per-channel offsets
    cu = torch.tensor(np.cumsum([0] + lens), dtype=torch.int32, device=DEV)
    ob, of = _pool(h, cu, enc.POOL_MEAN, 0, None, 0.0, l2)
    assert torch.equal(ob, of.to(torch.bfloat16))                         # the bf16 row is the rounded float row
    o = 0
    for i, n in enumerate(lens):
        H = h[o:o + n].double()
        mean = H.mean(0)
        e_mean = LAM * math.sqrt(n) * U32 * H.abs().sum(0) / n + U32 * mean.abs()   # serial fp32 sum; the division
        if l2 == 0:
            exact, bound = mean, e_mean
        else:
            nrm = mean.norm()
            exact = mean / nrm
            chain = dim / 256 + 10                                        # block sum of the squares (256 threads)
            bound = e_mean / nrm + exact.abs() * (e_mean.norm() / nrm + (chain + 3) * U32)   # mean, norm, division
        err = (of[i].double() - exact).abs()
        assert (err <= bound).all(), f"seq {i} (len {n}): worst {(err / bound).max().item():.3g} of the bound"
        assert (bound / exact.abs().clamp_min(1e-30)).median().item() < 1e-3     # well under a bf16 ulp (2^-8)
        o += n


# -------------------------------------------------------------------------------------------- attention
ATTN_CASES = [  # (H, KV, hd, lengths)
    (28, 4, 128, [1, 8, 48, 129, 4097, 300, 1024, 8192]),      # gte-Qwen2-7B: GQA group 7; 8192 ends the buffer
    (16, 16, 64, [512, 1, 77, 256, 129, 500, 64, 3, 511]),     # XLM-R-large cross-encoder
]


@pytest.mark.parametrize("H,KV,hd,lens", ATTN_CASES, ids=["qwen2-7b", "xlmr-large"])
def test_attention_model_shapes_vs_fp64(H, KV, hd, lens):
    t = sum(lens)
    qkv = _randn(t, (H + 2 * KV) * hd, seed=50 + H, std=0.8)
    cu = torch.tensor(np.cumsum([0] + lens), dtype=torch.int32, device=DEV)
    got = enc.attention(qkv, cu, max(lens), H, KV, hd).view(t, H, hd)
    torch.cuda.synchronize()
    assert _lib.lib().ezr_attn_last_kernel() == b"wgmma"
    scale = 1.0 / math.sqrt(hd)
    ref = _attn_ref(qkv, lens, H, KV, hd, scale)
    offs = np.cumsum([0] + lens)
    worst = 0.0
    for b, n in enumerate(lens):
        worst = max(worst, _attn_check(got[offs[b]:offs[b] + n], ref[b], n, f"seq {b} (len {n})"))
    _report(f"attention H={H} KV={KV} hd={hd}", dict(worst_rms_ratio=worst, tokens=t))
    # negative controls, each on the sequence where it shows
    b = int(np.argmax(lens))
    n = lens[b]
    g_b = got[offs[b]:offs[b] + n]
    tile = (n // 2) // 64 * 64                                        # one 64-key tile in the middle of the longest
    wrong = _attn_ref(qkv, lens, H, KV, hd, scale, seqs=[b], drop=(b, tile, tile + 64))[b]
    assert rejects(_attn_check, g_b, wrong, n, "control: one key tile dropped")
    if H != KV:
        group = H // KV
        kv_map = [h // group + (1 if h % group == group - 1 else 0) for h in range(H)]
        kv_map = [x % KV for x in kv_map]                             # last head of each group -> the next KV head
        wrong = _attn_ref(qkv, lens, H, KV, hd, scale, seqs=[b], kv_of_head=kv_map)[b]
        assert rejects(_attn_check, g_b, wrong, n, "control: head paired with the next KV head")
    if hd == 128:
        b2 = lens.index(300)
        wrong = _attn_ref(qkv, lens, H, KV, hd, 1.0 / 8.0, seqs=[b2])[b2]      # the softmax scale of head dim 64
        assert rejects(_attn_check, got[offs[b2]:offs[b2] + 300], wrong, 300, "control: scale 1/sqrt(64)")


# ------------------------------------------------------------------------------- Qwen2 encoder end to end
def test_qwen2_encoder_gte_qwen2_7b_width_vs_oracle():
    """Two layers of the real width: d 3584, 28 / 4 heads, FFN 18944, rope_theta 1e6."""
    cfg = Qwen2Config(vocab_size=1000, hidden_size=3584, intermediate_size=18944, num_hidden_layers=2,
                      num_attention_heads=28, num_key_value_heads=4, max_position_embeddings=8192, rope_theta=1e6)
    state = random_state("qwen2", cfg, 71)
    g = torch.Generator().manual_seed(72)
    lens = [1, 17, 48, 300, 1024]
    seqs = [torch.randint(1, cfg.vocab_size, (n,), generator=g).tolist() for n in lens]
    ids, mask = oenc.pad_left(seqs)
    tf32 = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False                       # a true fp32 oracle
    try:
        ref = oenc.gte_embed(state, cfg, ids, mask, device=DEV).cpu()
    finally:
        torch.backends.cuda.matmul.allow_tf32 = tf32
    refb = F.normalize(oenc.gte_embed(state, cfg, ids, mask, torch.bfloat16, device=DEV).cpu(), dim=1)
    model = Qwen2Encoder(cfg, state, device=DEV)
    _, ef = model.embed_packed(PackedBatch.from_padded(ids, mask, DEV))
    ef = ef.cpu()
    cos = F.cosine_similarity(ef, ref, dim=1)
    assert (cos > 1 - 1e-3).all(), cos
    floor = ((refb @ refb.T) - (ref @ ref.T)).abs().max().item()
    mine = F.normalize(ef, dim=1)
    err = ((mine @ mine.T) - (ref @ ref.T)).abs().max().item()
    _report("qwen2 encoder d=3584 2 layers", dict(min_cos=cos.min().item(), pairwise_err=err, bf16_floor=floor))
    assert err <= floor + 1e-3, f"pairwise cosine error {err:.2e} vs fp32; the reference's own bf16 floor is {floor:.2e}"
    _, ef0 = model.embed_packed(PackedBatch.from_lists(seqs, DEV))     # packed, positions from 0: RoPE is relative
    assert (F.cosine_similarity(ef0.cpu(), ref, dim=1) > 1 - 1e-3).all()


# ------------------------------------------------------------------------------------ dense search, dim 3584
N_ROWS, DIM, N_Q = 100_000, 3584, 700      # score rows of 671 queries fill the SIMT path's 256 MB block: 671 + 29


@pytest.fixture(scope="module")
def int_case():
    """Integer vectors in [-2, 2]: every dot product (|s| <= 4 * 3584) is exact in fp32, so any summation order
    gives the same score and ties are common."""
    g = _gen(80)
    c = torch.randint(-2, 3, (N_ROWS, DIM), generator=g, device=DEV).to(torch.bfloat16)
    q = torch.randint(-2, 3, (N_Q, DIM), generator=g, device=DEV).to(torch.bfloat16)
    sims = q.double() @ c.double().T
    return c, q, sims


def _dense(index, q, k, q_group=None):
    res = batched.dense_topk(index, q, k, q_group=q_group)
    torch.cuda.synchronize()
    assert _lib.lib().ezr_dense_last_kernel() == b"simt"       # dim 3584 is past the wgmma forms' 1024
    return res


@pytest.mark.parametrize("k", [10, 288])
def test_dense_3584_exact_integers_bit_exact(int_case, k):
    c, q, sims = int_case
    res = _dense(DenseIndex(c, device=DEV), q, k)
    ids, sc = canonical_topk(sims, k)
    assert (res.counts == k).all()
    assert torch.equal(res.ids.long(), ids)
    assert torch.equal(res.scores, sc.float())
    # the host oracle on queries from both query blocks (671 is the first of the second)
    pick = [0, 1, 670, 671, 699]
    ref_i, ref_s = ort.dense_topk(c.float().cpu().numpy(), q[pick].float().cpu().numpy(), k)
    assert np.array_equal(res.ids[pick].cpu().numpy(), ref_i)
    assert np.array_equal(res.scores[pick].cpu().numpy(), ref_s)


def test_dense_3584_group_filter_with_row_lo(int_case):
    c, q, sims = int_case
    k, lo = 10, 1000
    groups = synth.make_groups(N_ROWS, 4, 81).to(DEV)
    want = torch.tensor([i % 6 - 1 for i in range(N_Q)], dtype=torch.int32, device=DEV)
    want[want == 4] = -2                                              # a class no row has: empty result
    res = _dense(DenseIndex(c, device=DEV, doc_group=groups, row_lo=lo), q, k, q_group=want)
    allowed = (want[:, None] == -1) | (groups[None, :] == want[:, None])
    ids, sc = canonical_topk(sims, k, allowed)
    cnt = allowed.sum(1).clamp(max=k)
    assert torch.equal(res.counts.long(), cnt)
    assert (cnt == 0).any() and (cnt == k).any()
    live = torch.arange(k, device=DEV)[None, :] < cnt[:, None]
    assert torch.equal(res.ids.long(), torch.where(live, ids + lo, -1))
    assert torch.equal(res.scores[live], sc[live].float())


def test_dense_3584_unit_vectors_within_cos_tol():
    c = synth.make_dense_corpus(N_ROWS, DIM, 82, device=DEV)
    q = synth.make_dense_queries(c, N_Q, 83)
    k = 10
    res = _dense(DenseIndex(c, device=DEV), q, k)
    sims = q.double() @ c.double().T
    kth = sims.topk(k, dim=1).values[:, -1]
    got = res.ids.long()
    assert (res.counts == k).all()
    true = sims.gather(1, got)
    assert (res.scores.double() - true).abs().max().item() <= COS_TOL        # each score is its row's cosine
    assert (res.scores[:, 1:] <= res.scores[:, :-1]).all()                    # sorted descending
    assert (true >= kth[:, None] - COS_TOL).all()                              # the oracle's set up to the tolerance
    assert all(len(set(r)) == k for r in got.cpu().tolist())
