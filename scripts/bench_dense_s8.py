"""Dense top-k on a quantized index (int8 candidate pass + exact rescoring) against ezr_dense_topk on the bf16 rows.

    python scripts/bench_dense_s8.py --out DIR [--steps 10] [--warmup 3]

Shapes: 1M x 768 at 10k and at 64 queries, 4M x 1024 at 64 queries, k = 10, the synthetic corpus and queries of
bench.py (unit rows of N(0, 1); each query is a corpus row plus noise).  The two paths alternate step by step in the
same run, on the same corpus buffer.  The 64-query shapes read a corpus far larger than the L2, but each step is
still timed on its own with a 512 MB write in between (as bench.py does for small batches), so every step starts
from a cold L2.  Per step: CUDA events around the call; per part: the library's kernel timing slots.  Reported
figures are medians over the timed steps.  Writes DIR/bench_dense_s8.json and prints it.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

from easyrag_b200 import _lib, batched, synth  # noqa: E402
from easyrag_b200.index import DenseIndex  # noqa: E402

SHAPES = [(1_000_000, 768, 10_000), (1_000_000, 768, 64), (4_000_000, 1024, 64)]
CAP = 4096          # the default candidate capacity per query (csrc/dense_s8.cu)


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in out.split(",")]
        return dict(name=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:                    # the figures are still valid; say what could not be read
        return dict(name=torch.cuda.get_device_name(0), power_limit=f"unknown ({e})", max_sm_clock="unknown")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--k", type=int, default=10)
    args = ap.parse_args()
    _lib.require_cuda()
    L = _lib.lib()
    dev = torch.device("cuda:0")
    flush = torch.empty(512 << 20, dtype=torch.uint8, device=dev)
    results = dict(gpu=gpu_info(), k=args.k, steps=args.steps, warmup=args.warmup, shapes=[])
    for n, dim, nq in SHAPES:
        c = synth.make_dense_corpus(n, dim, 1002, device=dev)
        q = synth.make_dense_queries(c, nq, 1003)
        plain = DenseIndex(c, device=dev)                   # shares the bf16 buffer with the quantized index
        quant = DenseIndex(c, device=dev, quantized=True)
        ws_a, ws_b = batched.Workspace(dev), batched.Workspace(dev)
        cc = torch.empty(nq, dtype=torch.int32, device=dev)
        flush_each = nq <= 64

        def one(fn):
            if flush_each:
                flush.fill_(1)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            torch.cuda.synchronize()
            return a.elapsed_time(b)

        run_bf16 = lambda: batched.dense_topk(plain, q, args.k, ws=ws_a)
        run_s8 = lambda: batched.dense_topk(quant, q, args.k, ws=ws_b, cand_counts=cc)
        for _ in range(args.warmup):
            one(run_bf16)
            one(run_s8)
        bf16_kernel = L.ezr_dense_last_kernel().decode()
        t_bf16, t_s8, parts = [], [], {"dense_s8_scan": [], "dense_s8_rescore": [], "dense_s8_full": []}
        for _ in range(args.steps):
            t_bf16.append(one(run_bf16))
            L.ezr_profile_reset()
            L.ezr_profile_enable(1)
            t_s8.append(one(run_s8))
            L.ezr_profile_enable(0)
            for name in parts:
                parts[name].append(_lib.profile_read(name)[0])
        ref = batched.dense_topk(plain, q, args.k, ws=ws_a)
        got = batched.dense_topk(quant, q, args.k, ws=ws_b)
        torch.cuda.synchronize()
        row = dict(rows=n, dim=dim, queries=nq, l2_flush_each_step=flush_each,
                   bf16_kernel=bf16_kernel, bf16_ms=statistics.median(t_bf16), s8_ms=statistics.median(t_s8),
                   s8_parts_ms={k: statistics.median(v) for k, v in parts.items()},
                   cand_mean=float(cc.float().mean()), cand_max=int(cc.max()), overflowed=int((cc > CAP).sum()),
                   bf16_index_bytes=plain.index_bytes(), s8_index_bytes=quant.index_bytes(),
                   same_ids_as_bf16=float((ref.ids == got.ids).float().mean()))
        print(json.dumps(row), flush=True)
        results["shapes"].append(row)
        del c, q, plain, quant, ws_a, ws_b, ref, got
        torch.cuda.empty_cache()
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "bench_dense_s8.json"), "w") as f:
        json.dump(results, f, indent=1)
    print(json.dumps(results["gpu"]))


if __name__ == "__main__":
    main()
