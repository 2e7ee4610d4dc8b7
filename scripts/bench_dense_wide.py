"""Dense top-k at gte-Qwen2-7B's width: form 6 of ezr_dense_topk (wgmma score rows + select) against form 1 (the SIMT
score rows the automatic choice runs there).

    python scripts/bench_dense_wide.py --out DIR [--steps 5] [--warmup 2]

Seeded unit vectors (synth.make_dense_corpus / make_dense_queries).  Where a form-1 step takes well under a second, the
two forms alternate step by step on the same buffers: 1M x 3584 at 1 and 64 queries (k 10 and 288), and 100k x 3584 at
700 queries (k 288).  Past that (1M x 3584 at 700 and 4096 queries, 1M x 768 at 10 000) form 6 runs alone, and form 1
is "not run".  Per call: CUDA events around it, medians over the timed steps; per part: the library's kernel timing
slots (dense_wide / dense_simt = the score kernel, merge = the select), taken in separate profiled calls.  TFLOP/s
counts 2 n d Q over the score kernel's time; corpus GB/s counts one read of the corpus per query block; the bound is
the score kernel's least time, the larger of flops / 989 TFLOP/s and bytes / 3.35 TB/s (H100 SXM data sheet), bytes
being its corpus reads plus the score rows it writes (the select reads them back).  Writes DIR/bench_dense_wide.json and prints each row.
"""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

from easyrag_b200 import _lib, batched, synth  # noqa: E402
from easyrag_b200.index import DenseIndex  # noqa: E402
from _bounds import dense_delta_max  # noqa: E402

PEAK_FLOPS, PEAK_BYTES = 989e12, 3.35e12
# (rows, dim, queries, k, block_queries, run form 1)
SHAPES = [
    (1_000_000, 3584, 1, 10, None, True),
    (1_000_000, 3584, 1, 288, None, True),
    (1_000_000, 3584, 64, 10, None, True),
    (1_000_000, 3584, 64, 288, None, True),
    (100_000, 3584, 700, 288, None, True),
    (1_000_000, 3584, 700, 288, None, False),
    (1_000_000, 3584, 4096, 288, None, False),
    (1_000_000, 3584, 4096, 288, 512, False),
    (1_000_000, 768, 10_000, 288, None, False),
]


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in out.split(",")]
        return dict(name=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:                    # the figures are still valid; say what could not be read
        return dict(name=torch.cuda.get_device_name(0), power_limit=f"unknown ({e})", max_sm_clock="unknown")


def block_of(L, n, dim, nq, k, block_queries):
    """The query block form 6 runs: the largest whose ezr_dense_wide_workspace fits the bytes it is given."""
    if block_queries is not None:
        return min(block_queries, nq)
    have = L.ezr_dense_topk_workspace(n, dim, nq, k)
    qb = min(nq, 65535, have // (4 * n))
    while qb > 0 and L.ezr_dense_wide_workspace(n, nq, k, qb) > have:
        qb -= 1
    return qb


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def profiled(L, fn, slots, steps):
    got = {s: [] for s in slots}
    for _ in range(steps):
        L.ezr_profile_reset()
        L.ezr_profile_enable(1)
        fn()
        torch.cuda.synchronize()
        L.ezr_profile_enable(0)
        for s in slots:
            got[s].append(_lib.profile_read(s)[0])
    return {s: statistics.median(v) for s, v in got.items()}


def figures(n, dim, nq, qb, ms, score_ms):
    flops = 2.0 * n * dim * nq
    corpus = math.ceil(nq / qb) * n * dim * 2.0
    rows = 4.0 * nq * n
    t_flop, t_mem = flops / PEAK_FLOPS, (corpus + rows) / PEAK_BYTES
    return dict(ms=ms, qps=nq / ms * 1e3, score_tflops=flops / score_ms / 1e9, corpus_gbps=corpus / score_ms / 1e6,
                bound="compute" if t_flop >= t_mem else "memory",
                score_share_of_bound=max(t_flop, t_mem) * 1e3 / score_ms)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    _lib.require_cuda()
    L = _lib.lib()
    dev = torch.device("cuda:0")
    results = dict(gpu=gpu_info(), steps=args.steps, warmup=args.warmup, shapes=[])
    corpus_key, c, index = None, None, None
    for n, dim, nq, k, bq, with_simt in SHAPES:
        if corpus_key != (n, dim):
            c = index = None
            torch.cuda.empty_cache()
            c = synth.make_dense_corpus(n, dim, 2001, device=dev)
            index, corpus_key = DenseIndex(c, device=dev), (n, dim)
        q = synth.make_dense_queries(c, nq, 2002 + nq)
        ws1, ws6 = batched.Workspace(dev), batched.Workspace(dev)
        run6 = lambda: batched.dense_topk(index, q, k, ws=ws6, form=6, block_queries=bq)
        run1 = lambda: batched.dense_topk(index, q, k, ws=ws1, form=1)
        for _ in range(args.warmup):
            timed(run6)
            if with_simt:
                timed(run1)
        t6, t1 = [], []
        for _ in range(args.steps):
            t6.append(timed(run6))
            if with_simt:
                t1.append(timed(run1))
        qb = block_of(L, n, dim, nq, k, bq)
        p6 = profiled(L, run6, ("dense_wide", "merge"), args.steps)
        row = dict(rows=n, dim=dim, queries=nq, k=k, block_queries=qb, blocks=math.ceil(nq / qb),
                   form6=dict(figures(n, dim, nq, qb, statistics.median(t6), p6["dense_wide"]),
                              score_ms=p6["dense_wide"], select_ms=p6["merge"]))
        if with_simt:
            p1 = profiled(L, run1, ("dense_simt", "merge"), args.steps)
            qb1 = max(1, min(nq, 1024, (256 << 20) // (4 * n)))       # the SIMT block: 256 MB of score rows
            row["form1"] = dict(figures(n, dim, nq, qb1, statistics.median(t1), p1["dense_simt"]),
                                score_ms=p1["dense_simt"], select_ms=p1["merge"])
            row["speedup"] = row["form1"]["ms"] / row["form6"]["ms"]
            # both forms' k-th scores lie within their own error bound of the fp64 k-th score of every rank, so
            # rank-wise they differ by at most the sum of the two bounds: wgmma (dense_delta_max) and a sequential
            # fp32 FMA chain over dim terms (gamma_dim * ||q|| ||c||)
            a, b = run6(), run1()
            torch.cuda.synchronize()
            cmax = max(c[i:i + 131072].double().norm(dim=1).max().item() for i in range(0, n, 131072))
            qn = q.double().norm(dim=1)
            u = 2.0 ** -24
            bound = dense_delta_max(q, cmax) + dim * u / (1 - dim * u) * qn * cmax
            diff = (a.scores.double() - b.scores.double()).abs()
            row["agreement"] = dict(ids_equal_share=(a.ids == b.ids).double().mean().item(),
                                    max_rank_score_diff=diff.max().item(),
                                    worst_diff_over_bound=(diff / bound[:, None]).max().item(),
                                    within_bound=bool((diff <= bound[:, None]).all()))
        else:
            row["form1"] = "not run"
        print(json.dumps(row), flush=True)
        results["shapes"].append(row)
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_dense_wide.json"), "w") as f:      # rewritten after every shape
            json.dump(results, f, indent=1)
        del q, ws1, ws6
        torch.cuda.empty_cache()
    print(json.dumps(results["gpu"]))


if __name__ == "__main__":
    main()
