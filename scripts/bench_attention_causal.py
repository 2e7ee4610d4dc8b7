#!/usr/bin/env python
"""Causal against bidirectional wgmma attention (ezr_attn_causal / ezr_attn_bidir) on one GPU, in the same run.

    python scripts/bench_attention_causal.py --out DIR [--rounds 5]

Writes DIR/bench_attention_causal.json and prints it.  For each head shape (gte-Qwen2-7B: 28 query / 4 KV heads of
128; MiniCPM-2B: 36 heads of 64) and each packed batch of about 147k tokens (U[64, 512]-token sequences, the
bench_encode.py mix; 1024-token sequences, a reranker pair; 8192-token sequences) it reports the kernel time of each
form (CUDA events around back-to-back launches, median over --rounds rounds that alternate the two kernels) and
TFLOP/s.  FLOPs count the keys each query row sees: 4 n^2 hd per (sequence, head) bidirectional, 2 n (n + 1) hd
causal.  Each case also checks that the last row of every sequence is the same in both forms (it sees every key).
GPU name and power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

SHAPES = [("gte-qwen2-7b", 28, 4, 128), ("minicpm-2b", 36, 36, 64)]
TOKENS = 147_456


def gpu_info() -> dict:
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    return {"nvidia_smi": r.stdout.strip(), "torch_name": torch.cuda.get_device_name()}


def batches() -> dict:
    g = torch.Generator().manual_seed(11)
    mix, total = [], 0
    while total < TOKENS:
        n = int(torch.randint(64, 513, (1,), generator=g))
        mix.append(n)
        total += n
    return {"mix U[64,512]": mix, "1024": [1024] * (TOKENS // 1024), "8192": [8192] * (TOKENS // 8192)}


def _event_ms(fn, reps: int) -> float:
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def run_case(lens, H, KV, hd, rounds: int) -> dict:
    from easyrag_b200 import _lib, encoder as enc
    dev = "cuda"
    t = sum(lens)
    g = torch.Generator(device=dev).manual_seed(t + H)
    qkv = (torch.randn(t, (H + 2 * KV) * hd, generator=g, device=dev) * 0.8).to(torch.bfloat16)
    cu = torch.tensor([0] + lens, dtype=torch.int64).cumsum(0).to(torch.int32).to(dev)
    out_b = torch.empty(t, H * hd, dtype=torch.bfloat16, device=dev)
    out_c = torch.empty_like(out_b)
    f_b = lambda: enc.attention(qkv, cu, max(lens), H, KV, hd, out=out_b)
    f_c = lambda: enc.attention(qkv, cu, max(lens), H, KV, hd, out=out_c, causal=True)
    for f in (f_b, f_c):                                       # warm-up: module load, function attributes, the plan pool
        f()
    torch.cuda.synchronize()
    assert _lib.lib().ezr_attn_last_kernel() == b"wgmma-causal"
    ends = cu[1:].long() - 1
    same_last = bool((out_b[ends] == out_c[ends]).all())
    reps = max(3, int(200.0 / max(_event_ms(f_b, 1), 1e-3)))   # about 0.2 s of bidirectional work per sample
    tb, tc = [], []
    for _ in range(rounds):
        tb.append(_event_ms(f_b, reps))
        tc.append(_event_ms(f_c, reps))
    mb, mc = sorted(tb)[len(tb) // 2], sorted(tc)[len(tc) // 2]
    fl_b = sum(4.0 * n * n * hd * H for n in lens)
    fl_c = sum(2.0 * n * (n + 1) * hd * H for n in lens)
    return dict(tokens=t, sequences=len(lens), reps=reps, bidir_ms=mb, causal_ms=mc, causal_over_bidir=mc / mb,
                bidir_tflops=fl_b / mb / 1e9, causal_tflops=fl_c / mc / 1e9,
                bidir_ms_all=tb, causal_ms_all=tc, last_rows_equal=same_last)


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--out", required=True)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_attention_causal needs a CUDA device (sm_90a)")
    from easyrag_b200 import _lib
    _lib.require_cuda()
    res = {"gpu": gpu_info(), "cases": []}
    for name, H, KV, hd in SHAPES:
        for bname, lens in batches().items():
            r = run_case(lens, H, KV, hd, args.rounds)
            r.update(shape=name, heads=H, kv_heads=KV, head_dim=hd, batch=bname)
            res["cases"].append(r)
            print(f"{name:13s} {bname:13s} bidir {r['bidir_ms']:8.3f} ms {r['bidir_tflops']:6.1f} TF/s   "
                  f"causal {r['causal_ms']:8.3f} ms {r['causal_tflops']:6.1f} TF/s   ratio {r['causal_over_bidir']:.3f}",
                  flush=True)
    out = Path(args.out)
    out.mkdir(parents=True, exist_ok=True)
    (out / "bench_attention_causal.json").write_text(json.dumps(res, indent=1))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
