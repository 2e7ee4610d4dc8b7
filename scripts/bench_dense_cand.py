"""Dense top-k at the pipeline's depths: the candidate form (``batched.dense_topk_cand``, csrc/dense_cand.cu) against
form 6 (wgmma score rows + select), whose results it must reproduce bit for bit.

    python scripts/bench_dense_cand.py --out DIR [--steps 5] [--warmup 2]

Seeded unit vectors (synth.make_dense_corpus / make_dense_queries); the "clustered" corpus lays its rows out cluster
by cluster, as the chunks of one document sit next to each other (clusters of CLUSTER rows around a random centre).
The two forms alternate step by step on the same inputs; per call: CUDA events around it, medians over the timed
steps.  Per part: the library's kernel timing slots, in separate profiled calls -- candidate GEMM (dense_cand_gemm),
bound steps (dense_cand_bound), fallback (dense_wide + merge: form 6 on the overflowed queries; nothing else in the
candidate form uses those slots); form 6's score kernel (dense_wide) and select (merge).  TFLOP/s counts 2 n d Q over
the GEMM time; the bound is the GEMM's least time, the larger of flops / 989 TFLOP/s and bytes / 3.35 TB/s (H100 SXM
data sheet), the bytes being one corpus read per query block plus the query rows (form 6: plus its score rows).
Equality: counts and ids byte-equal in full, scores byte-equal wherever a result is listed.  Writes
DIR/bench_dense_cand.json with the card's name and power limit, and prints each row.
"""
import argparse
import json
import math
import statistics
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from easyrag_b200 import _lib, batched, synth  # noqa: E402
from easyrag_b200.index import DenseIndex  # noqa: E402

PEAK_FLOPS, PEAK_BYTES = 989e12, 3.35e12
CAND_BLOCK_BYTES = 16 << 20      # the candidate form's query block (csrc/dense_cand.cu)
CLUSTER = 512
# (rows, dim, queries, k, form 6's block_queries, clustered)
SHAPES = [
    (1_000_000, 768, 10_000, 288, None, False),
    (1_000_000, 768, 10_000, 1024, None, False),
    (1_000_000, 768, 64, 288, None, False),
    (1_000_000, 3584, 4096, 288, None, False),
    (1_000_000, 3584, 4096, 288, 512, False),
    (4_000_000, 1024, 64, 288, None, False),
    (1_000_000, 768, 10_000, 288, None, True),
]


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in out.split(",")]
        return dict(name=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:                    # the figures are still valid; say what could not be read
        return dict(name=torch.cuda.get_device_name(0), power_limit=f"unknown ({e})", max_sm_clock="unknown")


def clustered_corpus(n, dim, seed, dev, spread=0.5):
    g = torch.Generator(device=dev).manual_seed(seed)
    centres = torch.randn((n + CLUSTER - 1) // CLUSTER, dim, generator=g, device=dev)
    out = torch.empty(n, dim, dtype=torch.bfloat16, device=dev)
    step = 1 << 17
    for s in range(0, n, step):
        e = min(n, s + step)
        x = centres[torch.arange(s, e, device=dev) // CLUSTER]
        x = torch.nn.functional.normalize(x, dim=1) + spread * torch.nn.functional.normalize(
            torch.randn(e - s, dim, generator=g, device=dev), dim=1)
        out[s:e] = torch.nn.functional.normalize(x, dim=1).to(torch.bfloat16)
    return out


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


def bound(flops, nbytes, ms):
    t_flop, t_mem = flops / PEAK_FLOPS, nbytes / PEAK_BYTES
    return dict(tflops=flops / ms / 1e9, bound="compute" if t_flop >= t_mem else "memory",
                share_of_bound=max(t_flop, t_mem) * 1e3 / ms)


def wide_block(L, n, dim, nq, k, block_queries):
    """The query block form 6 runs: the largest whose ezr_dense_wide_workspace fits the bytes it is given."""
    if block_queries is not None:
        return min(block_queries, nq)
    have = L.ezr_dense_topk_workspace(n, dim, nq, k)
    qb = min(nq, 65535, have // (4 * n))
    while qb > 0 and L.ezr_dense_wide_workspace(n, nq, k, qb) > have:
        qb -= 1
    return qb


def same(a, b):
    k = a.ids.shape[1]
    valid = torch.arange(k, device=a.ids.device)[None, :] < a.counts[:, None].long()
    sb = (a.scores.view(torch.int32) != b.scores.view(torch.int32)) & valid
    return dict(counts_equal=bool(torch.equal(a.counts, b.counts)), ids_equal=bool(torch.equal(a.ids, b.ids)),
                scores_equal=not bool(sb.any()))


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
    print(json.dumps(results["gpu"]), flush=True)
    corpus_key, c, index = None, None, None
    for n, dim, nq, k, bq, clustered in SHAPES:
        if corpus_key != (n, dim, clustered):
            c = index = None
            torch.cuda.empty_cache()
            c = clustered_corpus(n, dim, 3001, dev) if clustered else synth.make_dense_corpus(n, dim, 3001, device=dev)
            index, corpus_key = DenseIndex(c, device=dev), (n, dim, clustered)
        q = synth.make_dense_queries(c, nq, 3002 + nq)
        ws_c, ws_6 = batched.Workspace(dev), batched.Workspace(dev)
        out_c = batched.TopK(torch.empty(nq, k, device=dev), torch.empty(nq, k, dtype=torch.int32, device=dev),
                             torch.empty(nq, dtype=torch.int32, device=dev))
        out_6 = batched.TopK(torch.empty(nq, k, device=dev), torch.empty(nq, k, dtype=torch.int32, device=dev),
                             torch.empty(nq, dtype=torch.int32, device=dev))
        cc = torch.empty(nq, dtype=torch.int32, device=dev)
        run_c = lambda: batched.dense_topk_cand(index, q, k, ws=ws_c, out=out_c, cand_counts=cc)
        run_6 = lambda: batched.dense_topk(index, q, k, ws=ws_6, out=out_6, form=6, block_queries=bq)
        for _ in range(args.warmup):
            run_c()
            run_6()
        torch.cuda.synchronize()
        t_c, t_6 = [], []
        for _ in range(args.steps):
            t_c.append(timed(run_c))
            t_6.append(timed(run_6))
        ms_c, ms_6 = statistics.median(t_c), statistics.median(t_6)
        eq = same(out_c, out_6)
        pc = profiled(L, run_c, ("dense_cand_gemm", "dense_cand_bound", "dense_wide", "merge"), 2)
        p6 = profiled(L, run_6, ("dense_wide", "merge"), 2)
        flops = 2.0 * n * dim * nq
        qb_c = min(nq, max(128, CAND_BLOCK_BYTES // (2 * dim) // 128 * 128))
        qb_6 = wide_block(L, n, dim, nq, k, bq)
        bytes_c = math.ceil(nq / qb_c) * n * dim * 2.0 + nq * dim * 2.0
        bytes_6 = math.ceil(nq / qb_6) * n * dim * 2.0 + nq * dim * 2.0 + 4.0 * nq * n
        ws_bytes_6 = (L.ezr_dense_wide_workspace(n, nq, k, bq) if bq is not None
                      else L.ezr_dense_topk_workspace(n, dim, nq, k))
        ccf = cc.float()
        row = dict(
            rows=n, dim=dim, queries=nq, k=k, corpus="clustered" if clustered else "random", form6_block_queries=qb_6,
            cand=dict(ms=ms_c, qps=nq / ms_c * 1e3, gemm_ms=pc["dense_cand_gemm"], bound_ms=pc["dense_cand_bound"],
                      fallback_ms=pc["dense_wide"] + pc["merge"], query_block=qb_c,
                      **{f"gemm_{a}": b for a, b in bound(flops, bytes_c, pc["dense_cand_gemm"]).items()},
                      cand_per_query_mean=float(ccf[cc >= 0].mean()) if bool((cc >= 0).any()) else None,
                      cand_per_query_max=int(cc.max()), overflowed=int((cc < 0).sum()),
                      workspace_bytes=L.ezr_dense_cand_topk_workspace(n, dim, nq, k)),
            form6=dict(ms=ms_6, qps=nq / ms_6 * 1e3, score_ms=p6["dense_wide"], select_ms=p6["merge"],
                       **{f"score_{a}": b for a, b in bound(flops, bytes_6, p6["dense_wide"]).items()},
                       workspace_bytes=ws_bytes_6),
            speedup=ms_6 / ms_c, **eq)
        results["shapes"].append(row)
        print(json.dumps(row), flush=True)
        del out_c, out_6, ws_c, ws_6, q, cc
    out = Path(args.out)
    out.mkdir(parents=True, exist_ok=True)
    (out / "bench_dense_cand.json").write_text(json.dumps(results, indent=1))
    ok = all(r["counts_equal"] and r["ids_equal"] and r["scores_equal"] for r in results["shapes"])
    print(json.dumps(dict(all_equal=ok)))
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
