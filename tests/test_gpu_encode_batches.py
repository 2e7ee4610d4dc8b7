"""GPU: attention and the encoders on batches the size the encode benchmark runs, against fp64.

The encode benchmark (bench_encode.py) runs BertEncoder over packed batches of 512 sequences of U[64, 512] tokens, and
the cross-encoder reranker packs up to 65 535 pairs into one attention call.  The code that depends on the number of
sequences is the attention plan (attn_plan_kernel lists query blocks in sweeps of 256 sequences, carrying a running
base from one sweep to the next), the persistent CTAs that walk n_pairs x n_heads items one plan entry ahead, and the
per-call plan allocation.  So every case here packs hundreds to tens of thousands of sequences:

* attention at 255 / 256 / 257 (either side of one sweep), 512, 513 and 4 097 sequences, every row of every
  sequence against the fp64 reference and bound of tests/_attn_ref.py, at the head shapes of BERT-base, BGE-large
  and a 128-dim GQA model; the mma.sync kernel on the same batches; the causal form at 513 sequences;
* exact cases at the 65 535-sequence limit: length 1 (the output is the V row) and length 2 with zero logits (the
  output is the bf16 rounding of the mean of two V rows), and 65 536 sequences refused;
* plan reuse across batch sizes, two streams from one host thread, CUDA graph capture, device switches;
* negative controls, each rejected by the check that accepts the kernel;
* BertEncoder and Qwen2Encoder on a full 512-sequence batch against the fp64 oracle, and bit-exact packing
  invariance (alone, in the 6-sequence prefix, reversed, written into a DenseIndex).

The figures each check measures are printed (``pytest -s``).
"""
import math
import threading

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from _attn_ref import _attn_check, _attn_ref, _causal_check, _causal_ref, _kernel_tiles
from _bounds import rejects, round_bf16, ulp_bf16
from bench_encode import build_model, make_batches
from oracle import encoder as oenc
from easyrag_b200 import _lib, encoder as enc
from easyrag_b200.encoder import PackedBatch, Qwen2Config, Qwen2Encoder, random_state
from easyrag_b200.index import DenseIndex

pytestmark = pytest.mark.gpu
DEV = "cuda"
COS_TOL = 1e-3                 # the bar of test_bge_large_24_layers_vs_fp64 and bench_encode.oracle_parity
EZR_ERR_INVALID = -1
MAX_SEQ = 65535                # sequences one attention call takes
SHAPES = {"bert-base": (12, 12, 64), "bge-large": (16, 16, 64), "gqa-128": (28, 4, 128)}
COUNTS = [255, 256, 257, 512, 513, 4097]


@pytest.fixture(scope="module", autouse=True)
def _ready(lib_built):
    _lib.require_cuda()


def _report(what, info):
    print(f"\n[bounds] {what}: " + ", ".join(f"{k}={v:.5g}" if isinstance(v, float) else f"{k}={v}"
                                          for k, v in info.items()))


def _randn(*shape, seed, std=1.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(*shape, generator=g, device=DEV) * std).to(torch.bfloat16)


def _cu(lens):
    return torch.tensor(np.cumsum([0] + list(lens)), dtype=torch.int32, device=DEV)


def _lens(n, seed):
    """make_batches' U[64, 512] lengths with 1, 127, 128 and 129 at one place in 16 (the lengths where a sequence
    has one query block or starts its second).  Sequences 255 and 256, the last of the first sweep of the plan kernel
    and the first of the second, get different lengths.  Past 256 sequences the lengths repeat with period 256, so
    a reference of the first 256 sequences repeated has the batch's shape (a negative control)."""
    g = torch.Generator().manual_seed(seed)
    base = torch.randint(64, 513, (min(n, 256),), generator=g)
    pick = torch.randperm(base.numel(), generator=g)[:max(4, base.numel() // 16)]
    base[pick] = torch.tensor([1, 127, 128, 129]).repeat(pick.numel() // 4 + 1)[:pick.numel()]
    if n > 256 and base[255] == base[0]:
        base[0] = 129 if base[255] != 129 else 128
    return [int(base[i % base.numel()]) for i in range(n)]


def _batch(n, H, KV, hd, seed):
    lens = _lens(n, seed)
    qkv = _randn(sum(lens), (H + 2 * KV) * hd, seed=seed + 1, std=0.8)
    return lens, qkv


def _attn(qkv, lens, H, KV, hd, out=None, causal=False):
    return enc.attention(qkv, _cu(lens), max(lens), H, KV, hd, out=out, causal=causal)


def _check_all(got, qkv, lens, H, KV, hd, what, group=64):
    """Every row of every sequence of ``got`` [T, H * hd] against fp64 (tests/_attn_ref.py).
    -> (worst error / bound over all elements, worst rms ratio against the fp64 emulation)."""
    got = got.view(-1, H, hd)
    scale = 1.0 / math.sqrt(hd)
    offs = np.cumsum([0] + list(lens))
    stats = {}
    worst_elem = worst_rms = 0.0
    for b0 in range(0, len(lens), group):
        seqs = range(b0, min(b0 + group, len(lens)))
        ref = _attn_ref(qkv, lens, H, KV, hd, scale, seqs=seqs)
        for b in seqs:
            r = _attn_check(got[offs[b]:offs[b + 1]], ref[b], lens[b], f"{what}: seq {b} (len {lens[b]})", stats)
            worst_rms = max(worst_rms, r)
            worst_elem = max(worst_elem, stats["worst"])
    return worst_elem, worst_rms


def _control(got, qkv, lens, H, KV, hd, seqs, what):
    """A negative control: the reference of ``lens`` (which differ from the kernel's) on sequences ``seqs`` must be
    rejected.  -> worst error / bound among the rejected sequences."""
    got = got.view(-1, H, hd)
    offs = np.cumsum([0] + list(lens))
    ref = _attn_ref(qkv, lens, H, KV, hd, 1.0 / math.sqrt(hd), seqs=seqs)
    worst, rejected = 0.0, False
    for b in seqs:
        stats = {}
        if rejects(_attn_check, got[offs[b]:offs[b + 1]], ref[b], lens[b], what, stats):
            rejected = True
        worst = max(worst, stats.get("worst", 0.0))
    assert rejected, f"accepted {what}"
    return worst


# ------------------------------------------------------------------------------- a. bidirectional, batch scale
@pytest.mark.parametrize("n", COUNTS)
@pytest.mark.parametrize("shape", list(SHAPES), ids=list(SHAPES))
def test_attention_batch_scale_vs_fp64(shape, n):
    H, KV, hd = SHAPES[shape]
    lens, qkv = _batch(n, H, KV, hd, seed=1000 * hd + n)
    got = _attn(qkv, lens, H, KV, hd)
    torch.cuda.synchronize()
    assert _lib.lib().ezr_attn_last_kernel() == b"wgmma"
    worst, rms = _check_all(got, qkv, lens, H, KV, hd, f"{shape} n={n}")
    info = dict(sequences=n, tokens=sum(lens), worst_err_over_bound=worst, worst_rms_ratio=rms)
    if n == 513:
        # the mma.sync kernel: another launch structure (a CTA per 64 query rows of one (sequence, head)), same bound
        L = _lib.lib()
        try:
            _lib.check(L.ezr_attn_set_kernel(1))
            legacy = _attn(qkv, lens, H, KV, hd)
            torch.cuda.synchronize()
            assert L.ezr_attn_last_kernel() == b"mma.sync"
        finally:
            _lib.check(L.ezr_attn_set_kernel(0))
        info["mma_sync_worst_err_over_bound"], info["mma_sync_worst_rms_ratio"] = \
            _check_all(legacy, qkv, lens, H, KV, hd, f"{shape} n={n} mma.sync")
        info["mma_sync_share_equal_to_wgmma"] = (legacy == got).double().mean().item()
    _report(f"attention {shape} H={H} KV={KV} hd={hd}", info)


# ---------------------------------------------------------------------------------------- b. causal, batch scale
def test_causal_attention_batch_scale_vs_fp64():
    H, KV, hd = SHAPES["gqa-128"]
    n = 513
    lens, qkv = _batch(n, H, KV, hd, seed=77)
    got = _attn(qkv, lens, H, KV, hd, causal=True).view(-1, H, hd)
    torch.cuda.synchronize()
    assert _lib.lib().ezr_attn_last_kernel() == b"wgmma-causal"
    offs = np.cumsum([0] + lens)
    scale = 1.0 / math.sqrt(hd)
    worst = 0.0
    for b, m in enumerate(lens):
        r = torch.arange(m, device=DEV)
        ref = _causal_ref(qkv[offs[b]:offs[b + 1]], H, KV, hd, scale, r + 1)
        worst = max(worst, _causal_check(got[offs[b]:offs[b + 1]], ref, r + 1, _kernel_tiles(m), f"causal seq {b}"))
    _report("causal attention gqa-128", dict(sequences=n, tokens=sum(lens), worst_rms_ratio=worst))


# ------------------------------------------------------------------------------ c. exact cases at the limit
def _v_rows(qkv, H, KV, hd):
    """[T, H, hd]: the V row each head reads (GQA: head h reads KV head h // (H / KV))."""
    v = qkv[:, (H + KV) * hd:].view(qkv.shape[0], KV, hd)
    return v.repeat_interleave(H // KV, dim=1)


@pytest.mark.parametrize("shape", ["bert-base", "gqa-128"])
def test_length_one_sequences_at_the_limit_return_their_v_rows(shape):
    """A single key: P = 1 in bf16 and l = P, so O = V exactly and the output is V up to 1 / l, within an ulp of 1,
    which cannot move a bf16 value.  65 535 sequences are one call; 65 536 are refused."""
    H, KV, hd = SHAPES[shape]
    L = _lib.lib()
    qkv = _randn(MAX_SEQ + 1, (H + 2 * KV) * hd, seed=5 + hd)
    lens = [1] * MAX_SEQ
    for kernel in (0, 1) if hd == 64 else (0,):
        try:
            _lib.check(L.ezr_attn_set_kernel(kernel))
            got = _attn(qkv[:MAX_SEQ], lens, H, KV, hd).view(MAX_SEQ, H, hd)
            torch.cuda.synchronize()
        finally:
            _lib.check(L.ezr_attn_set_kernel(0))
        assert torch.equal(got, _v_rows(qkv[:MAX_SEQ], H, KV, hd)), f"kernel {kernel}: outputs differ from V"
    out = torch.empty(MAX_SEQ + 1, H * hd, dtype=torch.bfloat16, device=DEV)
    cu = _cu([1] * (MAX_SEQ + 1))
    rc = L.ezr_attn_bidir(_lib.ptr(qkv), MAX_SEQ + 1, qkv.stride(0), _lib.ptr(cu), MAX_SEQ + 1, 1, H, KV, hd,
                          1.0 / math.sqrt(hd), _lib.ptr(out), out.stride(0), _lib.stream_ptr())
    assert rc == EZR_ERR_INVALID
    assert b"grid too large" in L.ezr_last_error()


def _v_pairs(n_seq, width, seed):
    """bf16 values of magnitude in [0.25, 4): the fp32 sum of two is exact (their exponents differ by at most 4)."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    mag = torch.exp2(torch.rand(2 * n_seq, width, generator=g, device=DEV) * 4 - 2)
    sign = torch.where(torch.rand(2 * n_seq, width, generator=g, device=DEV) < 0.5, -1.0, 1.0)
    return (mag * sign).to(torch.bfloat16)


@pytest.mark.parametrize("shape", ["bert-base", "gqa-128"])
def test_length_two_sequences_with_equal_logits_return_the_rounded_mean(shape):
    """Two keys per sequence, 65 535 sequences.  Zero queries make every logit exactly 0: ex2(0) = 1, so P = 1 for
    both keys, l = 2, O = v0 + v1 exactly in fp32, and the output is bf16_rn((v0 + v1) / 2) -- ties included, since
    the mean of two bf16 values often lies halfway between two (tests/test_attn_exact_cpu.py checks this model).
    With random queries and equal keys the two logits are equal but not 0, so P may miss 1 by a few ulps: the output is
    then the rounded mean everywhere except on a tie, where it may be either neighbour."""
    H, KV, hd = SHAPES[shape]
    t = 2 * MAX_SEQ
    lens = [2] * MAX_SEQ
    v = _v_pairs(MAX_SEQ, KV * hd, seed=9 + hd)
    mean = (v[0::2].double() + v[1::2].double()) / 2                          # [MAX_SEQ, KV hd], exact
    want = round_bf16(mean).view(MAX_SEQ, KV, hd).repeat_interleave(H // KV, dim=1)
    ties = ((mean - round_bf16(mean)).abs() == ulp_bf16(mean) / 2).view(MAX_SEQ, KV, hd)
    ties = ties.repeat_interleave(H // KV, dim=1)
    assert ties.double().mean().item() > 0.2                                  # the rounding of ties is tested
    qkv = torch.zeros(t, (H + 2 * KV) * hd, dtype=torch.bfloat16, device=DEV)
    qkv[:, (H + KV) * hd:] = v
    k = _randn(MAX_SEQ, KV * hd, seed=10 + hd)
    qkv[:, H * hd:(H + KV) * hd] = k.repeat_interleave(2, dim=0)              # equal keys within each sequence
    got = _attn(qkv, lens, H, KV, hd).view(MAX_SEQ, 2, H, hd)
    torch.cuda.synchronize()
    assert torch.equal(got[:, 0], got[:, 1])                                  # both rows of a sequence see the same
    assert torch.equal(got[:, 0].double(), want), \
        f"{int((got[:, 0].double() != want).sum())} outputs are not the rounded mean of their two V rows"
    # random queries, equal keys
    qkv[:, :H * hd] = _randn(t, H * hd, seed=11 + hd, std=0.25)
    got = _attn(qkv, lens, H, KV, hd).view(MAX_SEQ, 2, H, hd).double()
    torch.cuda.synchronize()
    other = 2 * mean.view(MAX_SEQ, KV, hd).repeat_interleave(H // KV, dim=1) - want    # a tie's other neighbour
    off = got != want[:, None]
    assert not (off & ~ties[:, None]).any(), "an output off its rounded mean away from a tie"
    assert not (off & (got != other[:, None])).any(), "a tie rounded to neither neighbour"
    _report(f"length-2 sequences {shape}", dict(sequences=MAX_SEQ, tie_share=ties.double().mean().item(),
                                                ties_rounded_the_other_way=int(off.sum())))


# ----------------------------------------------------------------------- d. plan reuse across batch sizes
def test_plan_across_batch_sizes_from_one_thread():
    """4 097 sequences, then 7, then 513, then 4 097 again, all from this thread: each against fp64, and the second
    4 097-sequence run bit for bit equal to the first."""
    H, KV, hd = SHAPES["bert-base"]
    runs = {}
    for i, n in enumerate([4097, 7, 513, 4097]):
        lens, qkv = _batch(n, H, KV, hd, seed=300 + n)
        got = _attn(qkv, lens, H, KV, hd)
        torch.cuda.synchronize()
        if n in runs:
            assert torch.equal(got, runs[n]), f"run {i}: {n} sequences differ from the first run of the same batch"
            continue
        runs[n] = got
        worst, rms = _check_all(got, qkv, lens, H, KV, hd, f"run {i} n={n}")
        _report(f"plan reuse run {i}", dict(sequences=n, worst_err_over_bound=worst, worst_rms_ratio=rms))


# ------------------------------------------------------------------------------------ e. negative controls
def test_negative_controls_are_rejected():
    H, KV, hd = SHAPES["bert-base"]
    info = {}
    # sequences 255 and 256 (either side of the sweep boundary) swapped: the reference reads the two lengths in the
    # other order, over the same tokens
    lens, qkv = _batch(513, H, KV, hd, seed=1000 * hd + 513)
    got = _attn(qkv, lens, H, KV, hd)
    torch.cuda.synchronize()
    assert lens[255] != lens[256]
    sw = list(lens)
    sw[255], sw[256] = sw[256], sw[255]
    info["swap_255_256"] = _control(got, qkv, sw, H, KV, hd, [255, 256], "sequences 255 and 256 swapped")
    # one interior boundary of cu_seqlens moved by one token
    b = next(i for i in range(300, 513) if lens[i + 1] > 1)
    mv = list(lens)
    mv[b] += 1
    mv[b + 1] -= 1
    info["boundary_moved"] = _control(got, qkv, mv, H, KV, hd, [b, b + 1], f"boundary {b + 1} moved by one token")
    # the 4 097-sequence output against the reference of the first 256 sequences repeated (same lengths, the tokens
    # of sequence b % 256)
    lens, qkv = _batch(4097, H, KV, hd, seed=1000 * hd + 4097)
    got = _attn(qkv, lens, H, KV, hd).view(-1, H, hd)
    torch.cuda.synchronize()
    offs = np.cumsum([0] + lens)
    scale = 1.0 / math.sqrt(hd)
    worst, accepted = 0.0, []
    for b in range(256, 4097, 255):                      # one sequence in each later sweep, at varying offsets in it
        a = b % 256
        assert lens[a] == lens[b]
        ref = _attn_ref(qkv, lens, H, KV, hd, scale, seqs=[a])[a]
        stats = {}
        if not rejects(_attn_check, got[offs[b]:offs[b + 1]], ref, lens[b], "first 256 repeated", stats):
            accepted.append(b)
        worst = max(worst, stats.get("worst", 0.0))
    assert not accepted, f"the reference of sequence b % 256 accepted for sequences {accepted}"
    info["first_256_repeated"] = worst
    _report("negative controls (worst error / bound)", info)


# ----------------------------------------------------------------------------- f. the encode batch end to end
ENC_N = 512


def _seqs(batch):
    ids = batch.ids.cpu().tolist()
    cu = batch.cu.cpu().tolist()
    return [ids[cu[i]:cu[i + 1]] for i in range(batch.n_seq)]


def _encode_batch(vocab, seed):
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(64, 513, (ENC_N,), generator=g)                      # encode_block's chunk lengths
    return make_batches(lens, ENC_N, vocab, DEV, seed + 1)[0]


def _oracle_chunks(fn, seqs, chunk=128):
    return torch.cat([fn(seqs[i:i + chunk]) for i in range(0, len(seqs), chunk)])


def _pairwise(ef, ref, refb):
    mine = F.normalize(ef.double(), dim=1)
    ref, refb = ref.double(), F.normalize(refb.double(), dim=1)
    floor = ((refb @ refb.T) - (ref @ ref.T)).abs().max().item()
    err = ((mine @ mine.T) - (ref @ ref.T)).abs().max().item()
    return err, floor


@pytest.fixture(scope="module")
def bert_case():
    cfg, state, model = build_model("bert", 12, 768, DEV)                    # the encode benchmark's model
    batch = _encode_batch(cfg.vocab_size, 21)
    return cfg, state, model, batch


@pytest.fixture(scope="module")
def qwen2_case():
    cfg = Qwen2Config(vocab_size=32000, hidden_size=1536, intermediate_size=8960, num_hidden_layers=2,
                      num_attention_heads=12, num_key_value_heads=2, max_position_embeddings=1024)
    state = random_state("qwen2", cfg, 31)
    return cfg, state, Qwen2Encoder(cfg, state, device=DEV), _encode_batch(cfg.vocab_size, 32)


def test_bert_encode_batch_vs_fp64(bert_case):
    cfg, state, model, batch = bert_case
    _, ef = model.embed_packed(batch)
    ef = ef.cpu()
    seqs = _seqs(batch)
    ref = _oracle_chunks(lambda s: oenc.bert_embed(state, cfg, s, device=DEV, dtype=torch.float64), seqs)
    refb = _oracle_chunks(lambda s: oenc.bert_embed(state, cfg, s, device=DEV, dtype=torch.bfloat16), seqs)
    cos = F.cosine_similarity(ef.double(), ref.double(), dim=1)
    err, floor = _pairwise(ef, ref, refb)
    # control: every sequence shorter than the position table read with positions from 1
    lens = (batch.cu[1:] - batch.cu[:-1]).long()
    short = lens < cfg.max_position_embeddings
    shift = torch.repeat_interleave(short.int(), lens)
    wrong = PackedBatch(ids=batch.ids, cu=batch.cu, positions=batch.positions + shift, max_len=batch.max_len,
                        n_seq=batch.n_seq)
    _, ec = model.embed_packed(wrong)
    cos_c = F.cosine_similarity(ec.cpu().double(), ref.double(), dim=1)[short.cpu()]
    _report("bert-base 12 layers, 512 sequences", dict(min_cos=cos.min().item(), pairwise_err=err, bf16_floor=floor,
                                                       control_max_cos=cos_c.max().item(),
                                                       control_sequences=int(short.sum())))
    assert (cos > 1 - COS_TOL).all(), f"{int((cos <= 1 - COS_TOL).sum())} sequences below cosine 1 - 1e-3"
    assert err <= floor + COS_TOL, f"pairwise cosine error {err:.2e} vs fp64; the bf16 floor is {floor:.2e}"
    assert (cos_c < 1 - COS_TOL).all(), f"position offset off by one accepted: max cosine {cos_c.max().item()}"


def test_qwen2_encode_batch_vs_fp64(qwen2_case):
    cfg, state, model, batch = qwen2_case
    _, ef = model.embed_packed(batch)                                         # positions from 0: RoPE is relative
    ef = ef.cpu()
    seqs = _seqs(batch)

    def fp64(s):
        ids, mask = oenc.pad_left(s)
        h = oenc.qwen2_hidden(state, cfg, ids, mask, torch.float64, DEV)
        return torch.stack([F.normalize(h[:, -1], dim=1), F.normalize(h[:, -2], dim=1)], 1).cpu()

    both = _oracle_chunks(fp64, seqs)
    ref, wrong = both[:, 0], both[:, 1]                                       # last token; the one before (control)
    refb = _oracle_chunks(lambda s: oenc.gte_embed(state, cfg, *oenc.pad_left(s), torch.bfloat16, DEV).cpu(), seqs)
    cos = F.cosine_similarity(ef.double(), ref, dim=1)
    err, floor = _pairwise(ef, ref, refb)
    cos_c = F.cosine_similarity(ef.double(), wrong, dim=1)
    _report("qwen2 d=1536 12/2 heads of 128, 2 layers, 512 sequences",
            dict(min_cos=cos.min().item(), pairwise_err=err, bf16_floor=floor, control_max_cos=cos_c.max().item()))
    assert (cos > 1 - COS_TOL).all(), f"{int((cos <= 1 - COS_TOL).sum())} sequences below cosine 1 - 1e-3"
    assert err <= floor + COS_TOL, f"pairwise cosine error {err:.2e} vs fp64; the bf16 floor is {floor:.2e}"
    assert (cos_c < 1 - COS_TOL).all(), f"pooling the second-to-last token accepted: max cosine {cos_c.max().item()}"


# ------------------------------------------------------------------------------- g. packing invariance, exact
def _sub(batch, idx):
    """The sequences ``idx`` of a packed batch, in that order, as a batch of their own (positions as they were)."""
    cu = batch.cu.cpu().tolist()
    parts = [torch.arange(cu[i], cu[i + 1]) for i in idx]
    tok = torch.cat(parts).to(DEV)
    lens = [cu[i + 1] - cu[i] for i in idx]
    return PackedBatch(ids=batch.ids[tok], cu=_cu(lens), positions=batch.positions[tok], max_len=max(lens),
                       n_seq=len(idx))


@pytest.mark.parametrize("arch", ["bert", "qwen2"])
def test_embeddings_do_not_depend_on_packing(arch, bert_case, qwen2_case):
    """Every layer is row-local except attention, which reads only its own sequence's keys in the same tile order
    wherever the sequence sits: a sequence's embedding is the same bits alone, in the 6-sequence prefix
    bench_encode.oracle_parity encodes, in the batch reversed and written into a DenseIndex."""
    cfg, _, model, batch = bert_case if arch == "bert" else qwen2_case
    eb, ef = model.embed_packed(batch)
    n = batch.n_seq
    alone = torch.cat([model.embed_packed(_sub(batch, [i]))[1] for i in range(n)])
    assert torch.equal(alone, ef), f"{int((alone != ef).any(1).sum())} sequences differ alone"
    _, pre = model.embed_packed(_sub(batch, list(range(6))))
    assert torch.equal(pre, ef[:6])
    _, rev = model.embed_packed(_sub(batch, list(range(n - 1, -1, -1))))
    assert torch.equal(rev.flip(0), ef)
    # the rows embed_packed writes into the index matrix are the rows it returns; the index grows in between
    index = DenseIndex(None, device=DEV, dim=cfg.hidden_size, capacity=6)
    for part in (_sub(batch, list(range(6))), batch):
        lo = index.n_rows
        got, _ = model.embed_packed(part, out_bf16=index.rows_for_append(part.n_seq))
        index.commit(part.n_seq)
        assert torch.equal(index.vectors[lo:lo + part.n_seq], got)
    assert torch.equal(index.vectors[:6], eb[:6]) and torch.equal(index.vectors[6:], eb)


# ------------------------------------------------------------------------------------ h. streams and devices
def test_two_streams_from_one_thread_match_serial_results():
    """A 4 097-sequence call on stream A and a 513-sequence call on stream B right behind it, nothing ordering the
    two: each output equals its serial result bit for bit (each call's plan is its own)."""
    H, KV, hd = SHAPES["bert-base"]
    la, qa = _batch(4097, H, KV, hd, seed=501)
    lb, qb = _batch(513, H, KV, hd, seed=502)
    ca, cb = _cu(la), _cu(lb)
    want_a = enc.attention(qa, ca, max(la), H, KV, hd)
    want_b = enc.attention(qb, cb, max(lb), H, KV, hd)
    out_a, out_b = torch.empty_like(want_a), torch.empty_like(want_b)
    sa, sb = torch.cuda.Stream(), torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(sa):
        enc.attention(qa, ca, max(la), H, KV, hd, out=out_a)
    with torch.cuda.stream(sb):
        enc.attention(qb, cb, max(lb), H, KV, hd, out=out_b)
    torch.cuda.synchronize()
    assert torch.equal(out_a, want_a), f"stream A: {int((out_a != want_a).any(1).sum())} rows differ"
    assert torch.equal(out_b, want_b), f"stream B: {int((out_b != want_b).any(1).sum())} rows differ"


def test_graph_capture_on_a_fresh_thread():
    """ezr_attn_bidir captured into a CUDA graph on a thread's first call, and again after a larger batch ran on
    that thread; each replay equals the eager result."""
    H, KV, hd = SHAPES["bert-base"]
    ls, qs = _batch(257, H, KV, hd, seed=601)
    lg, qg = _batch(4097, H, KV, hd, seed=602)
    cs, cg = _cu(ls), _cu(lg)
    want = enc.attention(qs, cs, max(ls), H, KV, hd)
    torch.cuda.synchronize()
    res = {}

    def capture_and_replay():
        out = torch.empty_like(want)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            enc.attention(qs, cs, max(ls), H, KV, hd, out=out)
        graph.replay()
        torch.cuda.synchronize()
        return out

    def body():
        try:
            res["first"] = capture_and_replay()
            enc.attention(qg, cg, max(lg), H, KV, hd)
            torch.cuda.synchronize()
            res["after_growth"] = capture_and_replay()
        except Exception as e:                                                  # reported on the test's thread
            res["error"] = e

    t = threading.Thread(target=body)
    t.start()
    t.join()
    if "error" in res:
        raise res["error"]
    assert torch.equal(res["first"], want), "first-call capture: replay differs from the eager result"
    assert torch.equal(res["after_growth"], want), "capture after a larger batch: replay differs"


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_device_switches_do_not_leak():
    """One thread alternating between two devices, one attention call per switch (65 535 one-token sequences, so a
    plan is about 2 MB): the free memory of both devices returns to where it started."""
    H, KV, hd = SHAPES["bert-base"]
    cases = []
    for d in range(2):
        with torch.cuda.device(d):
            qkv = _randn(MAX_SEQ, (H + 2 * KV) * hd, seed=700 + d).to(f"cuda:{d}")
            cu = torch.arange(MAX_SEQ + 1, dtype=torch.int32, device=f"cuda:{d}")
            cases.append((qkv, cu, torch.empty(MAX_SEQ, H * hd, dtype=torch.bfloat16, device=f"cuda:{d}")))
    prev = torch.cuda.current_device()

    def call(d):
        torch.cuda.set_device(d)
        qkv, cu, out = cases[d]
        enc.attention(qkv, cu, 1, H, KV, hd, out=out)
        torch.cuda.synchronize(d)

    try:
        call(0)
        call(1)
        free0 = [torch.cuda.mem_get_info(d)[0] for d in range(2)]
        for i in range(200):
            call(i % 2)
        free1 = [torch.cuda.mem_get_info(d)[0] for d in range(2)]
    finally:
        torch.cuda.set_device(prev)
    lost = [(a - b) / 2 ** 20 for a, b in zip(free0, free1)]
    _report("device switches", dict(switches=200, lost_mib_dev0=lost[0], lost_mib_dev1=lost[1]))
    assert max(lost) < 32, f"free memory fell by {lost} MiB over 200 device switches"
