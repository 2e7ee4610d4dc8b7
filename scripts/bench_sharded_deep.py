#!/usr/bin/env python
"""Row-sharded coarse ranking at the pipeline's depths: dense top-288 + BM25 top-192 + RRF to 256 per shard, merged
with ezr_merge_sorted_parts.

    python scripts/bench_sharded_deep.py --out DIR [--rounds 5]
    torchrun --nproc-per-node N scripts/bench_sharded_deep.py --out DIR

Writes DIR/bench_sharded_deep.json and prints it.  bench.py's corpus (1M x 768 rows, 200k vocabulary, float64 Okapi,
bench.py's seeds), cut as bench.py cuts it (align 64), at Q = 10000 and Q = 64.

One process simulates G in {1, 2, 8} shards in sequence on one GPU: each shard's two routes write into its slice of
one gathered buffer (the record layout of ShardedCoarseRanker.pipeline_hybrid); there is no collective.  Per case:
the per-shard route times (max and median over the shards, CUDA events, median over --rounds) and the dense kernel
form the dispatcher picked; the merge time of each route and the RRF time; the record and gathered bytes; and an A/B,
alternating within each round, of the in-place merge against copying each route's G lists into a contiguous
[Q, G * k] array + ezr_merge_topk (the select kernel).  The two merges must return the same bytes: the run fails
otherwise.  ``estimate_step_ms`` (the slowest shard's routes + both merges + RRF, no collective) is a sum of separately
timed parts, not a measured step.

Under torchrun with N processes each rank holds one shard of N and runs the whole ``pipeline_hybrid`` step (routes,
NCCL all-gather, merges, RRF); that step time is measured on N GPUs.  GPU name and power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
from pathlib import Path
from types import SimpleNamespace

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

K_DENSE, K_SPARSE, K_OUT = 288, 192, 256
QS = (10_000, 64)
GS = (1, 2, 8)
ALIGN = 64
DATA = SimpleNamespace(rows=1_000_000, dim=768, vocab=200_000, queries=max(QS))


def gpu_info() -> dict:
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    return {"nvidia_smi": r.stdout.strip(), "torch_name": torch.cuda.get_device_name()}


def event_ms(fn, rounds):
    """Median over ``rounds`` of CUDA-event time around ``fn()`` on the current stream."""
    out = []
    for _ in range(rounds):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b))
    return statistics.median(out)


def same_bytes(a, b) -> bool:
    bits = lambda t: t.contiguous().view(torch.int64 if t.element_size() == 8 else torch.int32)
    return (torch.equal(a.counts, b.counts) and torch.equal(a.ids.contiguous(), b.ids.contiguous())
            and torch.equal(bits(a.scores), bits(b.scores)))


def simulated(data, nq, G, rounds):
    from easyrag_b200 import _lib, batched
    from easyrag_b200 import dist as ezdist
    from easyrag_b200.index import Bm25Index, DenseIndex
    L = _lib.lib()
    dev = "cuda"
    qv = data["qvec"][:nq].contiguous()
    qp_all, qt_all = data["queries"].term_ptr.to(dev), data["queries"].terms.to(dev)
    qp, qt = qp_all[:nq + 1].contiguous(), qt_all[:int(qp_all[nq])].contiguous()
    layout = ezdist.RecordLayout(nq, K_DENSE, 8, k_sparse=K_SPARSE)
    nb = layout.nbytes
    gathered = torch.zeros(G * nb, dtype=torch.uint8, device=dev)
    ws_d, ws_s = batched.Workspace(dev), batched.Workspace(dev)
    dense_ms, sparse_ms, forms = [], [], set()
    for r in range(G):
        lo, hi = ezdist.shard_bounds(DATA.rows, G, r, align=ALIGN)
        dix = DenseIndex(data["vec"][lo:hi], device=dev, row_lo=lo)
        six = Bm25Index(data["stats"], device=dev, doc_lo=lo, doc_hi=hi)
        ds, di, ss, si = ezdist.record_views(layout, gathered[r * nb:(r + 1) * nb])
        d_out = batched.TopK(ds, di, torch.empty(nq, dtype=torch.int32, device=dev))
        s_out = batched.TopK(ss, si, torch.empty(nq, dtype=torch.int32, device=dev))
        run_d = lambda: batched.dense_topk(dix, qv, K_DENSE, ws=ws_d, out=d_out)
        run_s = lambda: batched.bm25_topk(six, qp, qt, K_SPARSE, ws=ws_s, out=s_out)
        run_d(), run_s()                                          # warm-up of this shard's shapes
        torch.cuda.synchronize()
        forms.add(L.ezr_dense_last_kernel().decode())
        dense_ms.append(event_ms(run_d, rounds))
        sparse_ms.append(event_ms(run_s, rounds))
        del dix, six
    g_ds, g_di, g_ss, g_si = ezdist.record_views(layout, gathered[:nb])
    W = max(K_DENSE, K_SPARSE)
    mk = lambda dt: batched.TopK(torch.empty(nq, W, dtype=dt, device=dev),
                                 torch.empty(nq, W, dtype=torch.int32, device=dev),
                                 torch.empty(nq, dtype=torch.int32, device=dev))
    m_d, m_s, fused = mk(torch.float32), mk(torch.float64), None

    def in_place(route):
        if route == "dense":
            return batched.merge_sorted_parts(g_ds, g_di, G, nb, K_DENSE, out=m_d)
        return batched.merge_sorted_parts(g_ss, g_si, G, nb, K_SPARSE, out=m_s)

    part_views = [ezdist.record_views(layout, gathered[p * nb:(p + 1) * nb]) for p in range(G)]

    def copy_select(route, k):
        j = 0 if route == "dense" else 2
        cs = torch.cat([v[j] for v in part_views], dim=1)          # the copy into a contiguous [Q, G * k]
        ci = torch.cat([v[j + 1] for v in part_views], dim=1)
        return batched.merge_topk(cs, ci, k)

    cases = {}
    for route, k in (("dense", K_DENSE), ("sparse", K_SPARSE)):
        a = in_place(route)
        b = copy_select(route, k)
        torch.cuda.synchronize()
        a_k = batched.TopK(a.scores[:, :k], a.ids[:, :k], a.counts)
        if not same_bytes(a_k, b):
            raise SystemExit(f"Q={nq} G={G} {route}: merge_sorted_parts and copy + merge_topk differ")
        ta, tb = [], []
        for _ in range(rounds):                                   # alternating A / B
            ta.append(event_ms(lambda: in_place(route), 1))
            tb.append(event_ms(lambda: copy_select(route, k), 1))
        cases[route] = dict(merge_sorted_parts_ms=statistics.median(ta), copy_plus_merge_topk_ms=statistics.median(tb),
                            equal=True)
    fused_fn = lambda: batched.rrf_fuse(m_s.ids, m_s.counts, m_d.ids, m_d.counts, K_OUT)
    fused = fused_fn()
    rrf_ms = event_ms(fused_fn, rounds)
    est = max(d + s for d, s in zip(dense_ms, sparse_ms)) + cases["dense"]["merge_sorted_parts_ms"] + \
        cases["sparse"]["merge_sorted_parts_ms"] + rrf_ms
    return dict(queries=nq, shards=G, dense_form=sorted(forms),
                dense_ms_max=max(dense_ms), dense_ms_median=statistics.median(dense_ms),
                sparse_ms_max=max(sparse_ms), sparse_ms_median=statistics.median(sparse_ms),
                merge_dense=cases["dense"], merge_sparse=cases["sparse"], rrf_ms=rrf_ms,
                record_bytes=nb, gathered_bytes=G * nb, fused_full=int((fused.counts == K_OUT).sum()),
                estimate_step_ms=est, estimate_note="sum of separately timed parts on one GPU, no collective",
                step_ms_on_G_gpus="not measured" if G > 1 else None)


def distributed(data, rounds):
    import torch.distributed as dist
    from easyrag_b200 import batched
    from easyrag_b200 import dist as ezdist
    from easyrag_b200.index import Bm25Index, DenseIndex
    world, rank = dist.get_world_size(), dist.get_rank()
    dev = torch.device("cuda", torch.cuda.current_device())
    lo, hi = ezdist.shard_bounds(DATA.rows, world, rank, align=ALIGN)
    ranker = batched.CoarseRanker(DenseIndex(data["vec"][lo:hi], device=dev, row_lo=lo),
                                  Bm25Index(data["stats"], device=dev, doc_lo=lo, doc_hi=hi))
    sh = ezdist.ShardedCoarseRanker(ranker)
    out = []
    qp_all, qt_all = data["queries"].term_ptr.to(dev), data["queries"].terms.to(dev)
    for nq in QS:
        qv = data["qvec"][:nq].contiguous()
        qp, qt = qp_all[:nq + 1].contiguous(), qt_all[:int(qp_all[nq])].contiguous()
        step = lambda: sh.pipeline_hybrid(qv, qp, qt, K_DENSE, K_SPARSE, K_OUT)
        step()
        torch.cuda.synchronize()
        out.append(dict(queries=nq, gpus=world, step_ms=event_ms(step, rounds),
                        gathered_bytes=int(sh._state[("deep", nq, K_DENSE, K_SPARSE, K_OUT)]["gathered"].numel())))
    return out


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--out", required=True)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    import bench
    from easyrag_b200 import _lib
    _lib.require_cuda()
    _lib.lib()
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if world > 1:
        import torch.distributed as dist
        local = int(os.environ.get("LOCAL_RANK", "0"))
        torch.cuda.set_device(local)
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    data = bench.make_data(DATA, torch.device("cuda"))
    out = dict(gpu=gpu_info(), corpus=dict(rows=DATA.rows, dim=DATA.dim, vocab=DATA.vocab, align=ALIGN),
               depths=dict(k_dense=K_DENSE, k_sparse=K_SPARSE, k_out=K_OUT), rounds=args.rounds)
    try:
        if world > 1:
            out["measured_on_gpus"] = world
            out["steps"] = distributed(data, args.rounds)
            if torch.distributed.get_rank() != 0:
                return
        else:
            out["simulated"] = []
            for nq in QS:
                for G in GS:
                    case = simulated(data, nq, G, args.rounds)
                    out["simulated"].append(case)
                    print(json.dumps(case), flush=True)
        d = Path(args.out)
        d.mkdir(parents=True, exist_ok=True)
        (d / "bench_sharded_deep.json").write_text(json.dumps(out, indent=1))
        print(json.dumps(out, indent=1))
    finally:
        if world > 1:
            torch.distributed.destroy_process_group()


if __name__ == "__main__":
    main()
