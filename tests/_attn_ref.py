"""Test infrastructure: fp64 references of the attention kernels (csrc/encoder/attention_tc.cuh) and the checks that
compare a kernel's output with them.

``_attn_ref`` / ``_attn_check``: bidirectional attention over packed sequences -- the fp64 result per (sequence,
head), the kernel's rounding points emulated in fp64, and a per-element bound derived from them plus a per-head rms
check against the emulation.  ``_causal_ref`` / ``_causal_check`` / ``_kernel_tiles``: the same for one sequence
where query row r sees keys 0 .. hi[r] - 1 (the causal form).  Every reference runs in float64 on the device on the
same bf16 inputs.  Used by tests/test_gpu_model_shapes.py, tests/test_gpu_attention_causal.py and
tests/test_gpu_encode_batches.py.
"""
import math

import numpy as np
import torch

from _bounds import U32, round_bf16, ulp_bf16

DEV = "cuda"
LAM = 4.0              # probabilistic accumulation bound (Higham & Mary 2019): |err| <= LAM sqrt(K) u sum|a_i b_i| fails
                       # with probability <= 2 exp(-LAM^2 / 2) per element under independent rounding errors


# ------------------------------------------------------------------------------------------ bidirectional
def _attn_ref(qkv, lens, H, KV, hd, scale, seqs=None, kv_of_head=None, drop=None):
    """fp64 attention per (sequence, head) with query rows chunked.  Returns {seq: (out, p_absv, emu, eps_p)}:
    out = softmax(q k^T scale) v; p_absv = the same applied to |v|; emu = the kernel's rounding points emulated in fp64
    (P rounded to bf16 for the numerator, the row sum of unrounded P, output rounded to bf16); eps_p = a bound on the
    relative error of each kernel P value.  ``kv_of_head`` / ``drop`` (a key range of one sequence) build controls."""
    kv_of_head = kv_of_head if kv_of_head is not None else [h // (H // KV) for h in range(H)]
    kvi = torch.tensor(kv_of_head, device=DEV)
    cu = np.cumsum([0] + list(lens))
    out = {}
    for b in (seqs if seqs is not None else range(len(lens))):
        lo, n = int(cu[b]), int(lens[b])
        rows = qkv[lo:lo + n].double()
        q = rows[:, :H * hd].view(n, H, hd).transpose(0, 1)
        k = rows[:, H * hd:(H + KV) * hd].view(n, KV, hd).index_select(1, kvi).transpose(0, 1)
        v = rows[:, (H + KV) * hd:(H + 2 * KV) * hd].view(n, KV, hd).index_select(1, kvi).transpose(0, 1)
        if drop is not None and drop[0] == b:
            keep = torch.ones(n, dtype=torch.bool, device=DEV)
            keep[drop[1]:drop[2]] = False
            k, v = k[:, keep], v[:, keep]
        o, pa, em = (torch.empty(H, n, hd, dtype=torch.float64, device=DEV) for _ in range(3))
        ep = torch.empty(H, n, 1, dtype=torch.float64, device=DEV)
        step = max(1, (1 << 25) // (H * k.shape[1]))
        for c0 in range(0, n, step):
            qc = q[:, c0:c0 + step]
            s = qc @ k.transpose(1, 2)
            m = s.amax(-1, keepdim=True)
            p = torch.exp((s - m) * scale)
            l = p.sum(-1, keepdim=True)
            o[:, c0:c0 + step] = (p @ v) / l
            pa[:, c0:c0 + step] = (p @ v.abs()) / l
            em[:, c0:c0 + step] = round_bf16((round_bf16(p) @ v) / l)
            qk = (qc.abs() @ k.abs().transpose(1, 2)).amax(-1, keepdim=True)
            ep[:, c0:c0 + step] = (scale * LAM * math.sqrt(hd) * U32 * qk     # fp32 accumulation of the logits
                                   + 3 * U32 * scale * (s.abs().amax(-1, keepdim=True) + m.abs())
                                   # fma(s, scale log2 e, -m scale log2 e) and its rounded operands
                                   + 2.0 ** -22)                               # ex2.approx.ftz (2 ulp)
            del s, p
        out[b] = (o.transpose(0, 1), pa.transpose(0, 1), em.transpose(0, 1), ep.transpose(0, 1))
    return out


def _attn_check(got, ref, n, what, stats=None):
    """got [n, H, hd] (bf16) against one sequence's reference: a per-element bound and a per-head rms ratio.
    Returns the worst rms ratio (kernel error / emulated error); ``stats["worst"]`` receives the worst error / bound
    (set before the checks, so a rejected negative control reports it as well)."""
    o, pa, em, ep = ref
    g = got.double()
    n_tiles = (n + 63) // 64
    main = 2.0 ** -8 * pa                          # P rounded to bf16 before P V (relative 2^-9 per term, doubled)
    bound = (main
             + (2 * ep                             # the P values' own error, in the numerator and in the row sum
                + (2 * n_tiles                     # O and the row sum rescaled by alpha once per key tile (fp32)
                   + LAM * math.sqrt(n)            # fp32 accumulation of P V over the keys
                   + 2) * U32)                     # 1 / l and O * (1 / l)
             * (pa + o.abs())
             + ulp_bf16(o.abs() + main))           # the bf16 output rounding
    err = (g - o).abs()
    worst = int(torch.argmax(err / bound))
    if stats is not None:
        stats["worst"] = (err.reshape(-1)[worst] / bound.reshape(-1)[worst]).item()
    assert (err <= bound).all(), (f"{what}: worst element {worst}: |err| {err.reshape(-1)[worst].item():.3g} vs bound "
                                  f"{bound.reshape(-1)[worst].item():.3g}")
    # per head: relative rms error vs fp64 <= 1.5 x that of the fp64 emulation of the kernel's rounding points
    den = o.pow(2).sum((0, 2)).sqrt().clamp_min(1e-300)
    e_got = (g - o).pow(2).sum((0, 2)).sqrt() / den
    e_emu = (em - o).pow(2).sum((0, 2)).sqrt() / den
    ratio = e_got / e_emu.clamp_min(1e-300)
    bad = e_got > 1.5 * e_emu + 1e-12
    assert not bad.any(), (f"{what}: rms error of heads {torch.nonzero(bad).flatten().tolist()}: "
                           f"{e_got[bad].tolist()} vs emulation {e_emu[bad].tolist()}")
    return torch.where(e_emu > 0, ratio, torch.zeros_like(ratio)).max().item()


# ------------------------------------------------------------------------------------------------ causal
def _causal_ref(rows, H, KV, hd, scale, hi):
    """fp64 attention of one sequence ([n, (H + 2 KV) hd] bf16 rows) where query row r sees keys 0 .. hi[r] - 1.
    -> (out, p_absv, emu, eps_p), each [n, H, *]: out = softmax(q k^T scale) v over the visible keys; p_absv the same
    applied to |v|; emu the kernel's rounding points in fp64 (P rounded to bf16 for the numerator, the row sum of the
    unrounded P, output rounded to bf16); eps_p a bound on the relative error of each kernel P value."""
    n = rows.shape[0]
    kvi = torch.tensor([h // (H // KV) for h in range(H)], device=DEV)
    r = rows.double()
    q = r[:, :H * hd].view(n, H, hd).transpose(0, 1)
    k = r[:, H * hd:(H + KV) * hd].view(n, KV, hd).index_select(1, kvi).transpose(0, 1)
    v = r[:, (H + KV) * hd:(H + 2 * KV) * hd].view(n, KV, hd).index_select(1, kvi).transpose(0, 1)
    hi = torch.as_tensor(hi, device=DEV)
    o, pa, em = (torch.empty(H, n, hd, dtype=torch.float64, device=DEV) for _ in range(3))
    ep = torch.empty(H, n, 1, dtype=torch.float64, device=DEV)
    step = max(1, (1 << 25) // (H * n))
    cols = torch.arange(n, device=DEV)
    for c0 in range(0, n, step):
        vis = (cols[None, :] < hi[c0:c0 + step, None])[None]            # [1, rows, n]
        qc = q[:, c0:c0 + step]
        s = (qc @ k.transpose(1, 2)).masked_fill(~vis, -math.inf)
        m = s.amax(-1, keepdim=True)
        p = torch.exp((s - m) * scale)
        l = p.sum(-1, keepdim=True)
        o[:, c0:c0 + step] = (p @ v) / l
        pa[:, c0:c0 + step] = (p @ v.abs()) / l
        em[:, c0:c0 + step] = round_bf16((round_bf16(p) @ v) / l)
        qk = (qc.abs() @ k.abs().transpose(1, 2)).masked_fill(~vis, 0).amax(-1, keepdim=True)
        sa = s.abs().masked_fill(~vis, 0).amax(-1, keepdim=True)
        ep[:, c0:c0 + step] = (scale * LAM * math.sqrt(hd) * U32 * qk    # fp32 accumulation of the logits
                               + 3 * U32 * scale * (sa + m.abs())        # fma(s, scale log2 e, -m scale log2 e)
                               + 2.0 ** -22)                             # ex2.approx.ftz (2 ulp)
        del s, p
    return tuple(t.transpose(0, 1) for t in (o, pa, em, ep))


def _kernel_tiles(n):
    """Key tiles the kernel walks for each row's 128-row item: min(ceil(n / 64), q0 / 64 + 2)."""
    r = torch.arange(n, device=DEV)
    return torch.clamp((r // 128) * 2 + 2, max=(n + 63) // 64).double()


def _causal_check(got, ref, keys, tiles, what):
    """got [n, H, hd] bf16 against a reference: per-element bound (row r accumulates keys[r] terms over tiles[r] key
    tiles) and per-head rms error at most 1.5 x that of the fp64 emulation.  Returns the worst rms ratio."""
    o, pa, em, ep = ref
    g = got.double()
    keys = keys.double()[:, None, None]
    tiles = tiles[:, None, None]
    main = 2.0 ** -8 * pa                          # P rounded to bf16 before P V (relative 2^-9 per term, doubled)
    bound = (main
             + (2 * ep                             # the P values' own error, in the numerator and in the row sum
                + (2 * tiles                       # O and the row sum rescaled by alpha once per key tile (fp32)
                   + LAM * keys.sqrt()             # fp32 accumulation of P V over the visible keys
                   + 2) * U32)                     # 1 / l and O * (1 / l)
             * (pa + o.abs())
             + ulp_bf16(o.abs() + main))           # the bf16 output rounding
    err = (g - o).abs()
    worst = int(torch.argmax(err / bound))
    assert (err <= bound).all(), (f"{what}: worst element {worst}: |err| {err.reshape(-1)[worst].item():.3g} vs bound "
                                  f"{bound.reshape(-1)[worst].item():.3g}")
    den = o.pow(2).sum((0, 2)).sqrt().clamp_min(1e-300)
    e_got = (g - o).pow(2).sum((0, 2)).sqrt() / den
    e_emu = (em - o).pow(2).sum((0, 2)).sqrt() / den
    bad = e_got > 1.5 * e_emu + 1e-12
    assert not bad.any(), (f"{what}: rms error of heads {torch.nonzero(bad).flatten().tolist()}: "
                           f"{e_got[bad].tolist()} vs emulation {e_emu[bad].tolist()}")
    return torch.where(e_emu > 0, e_got / e_emu.clamp_min(1e-300), torch.zeros_like(e_got)).max().item()
