#!/usr/bin/env python
"""Cross-encoder reranking with the pairs split across GPUs (ShardedCrossEncoderReranker), beside the one-GPU
CrossEncoderReranker on the same inputs in the same run.

Workload: the one of scripts/bench_rerank.py -- Q queries x k = 192 coarse candidates, top_n = 6, max_length 512;
passages U[64, 480] tokens, queries U[8, 48], seeded; XLM-R-large and XLM-R-base shapes with random bf16-representable
weights.  Every rank builds the same model and the same candidate lists from the seed, as replicated coarse results
would give it.

Reported by rank 0 per (model, Q): pairs/s of the split path (median wall time of a rerank call, all ranks started
together, ending in a device synchronise) and of the one-GPU reranker on rank 0 in the same run; per-rank encoder
milliseconds (CUDA events around the rank's encoder run) and token share (largest / smallest share of the pairs' tokens
a rank encodes); the card name and power limit; parity: rank 0's output equals the one-GPU output bit for bit (score
bits, ids, counts and all_scores).  The run exits non-zero if parity fails.

    torchrun --standalone --nproc-per-node N scripts/bench_rerank_dist.py --out DIR [--models large,base]
        [--queries 16,64] [--reps 3]
"""
import argparse
import json
import os
import sys
import time
from pathlib import Path

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent))
from bench_rerank import CLS, MAX_LENGTH, PAD, SEP, SHAPES, card, workload        # noqa: E402
from easyrag_b200 import _lib                                                     # noqa: E402
from easyrag_b200.batched import TopK                                             # noqa: E402
from easyrag_b200.dist import ShardedCrossEncoderReranker, token_balanced_ranges  # noqa: E402
from easyrag_b200.encoder import BertConfig                                       # noqa: E402
from easyrag_b200.rerank import CrossEncoderModel, CrossEncoderReranker, random_cross_encoder_state   # noqa: E402


def timed(fn, reps, together=True):
    """Median wall seconds and median stage times (ms) of ``fn(events)`` over ``reps`` calls after one warm-up;
    ``together``: every rank starts each call at the same time (a barrier first)."""
    fn(None)
    torch.cuda.synchronize()
    walls, stages = [], []
    for _ in range(reps):
        if together:
            dist.barrier()
        torch.cuda.synchronize()
        ev = []
        t0 = time.perf_counter()
        res = fn(ev)
        torch.cuda.synchronize()
        walls.append(time.perf_counter() - t0)
        stages.append([ev[i].elapsed_time(ev[i + 1]) for i in range(3)])
    return float(np.median(walls)), np.median(np.array(stages), axis=0), res


def bits_equal(a, b):
    (ta, sa), (tb, sb) = a, b
    f = lambda t: t.contiguous().view(torch.int32).cpu()
    return bool(torch.equal(ta.ids, tb.ids) and torch.equal(ta.counts, tb.counts)
                and torch.equal(f(ta.scores), f(tb.scores)) and torch.equal(f(sa), f(sb)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--models", default="large,base")
    ap.add_argument("--queries", default="16,64")
    ap.add_argument("--k", type=int, default=192)
    ap.add_argument("--top-n", type=int, default=6)
    ap.add_argument("--docs", type=int, default=20000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_rerank_dist: no CUDA device (this benchmark measures the GPU path only)")
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    rank, world = dist.get_rank(), dist.get_world_size()
    _lib.require_cuda()
    info = card() if rank == 0 else None
    results, failed = [], False
    try:
        for name in a.models.split(","):
            cfg = BertConfig(vocab_size=250002, max_position_embeddings=514, layer_norm_eps=1e-5, **SHAPES[name])
            model = CrossEncoderModel("roberta", cfg, random_cross_encoder_state("roberta", cfg, a.seed), CLS, SEP,
                                      PAD, device=dev)
            rng = np.random.default_rng(a.seed)
            for nq in [int(x) for x in a.queries.split(",")]:
                passages, queries, ids = workload(rng, cfg.vocab_size, a.docs, nq, a.k)
                rr = CrossEncoderReranker(model, passages, max_length=MAX_LENGTH)
                sh = ShardedCrossEncoderReranker(rr)
                cand = TopK(torch.zeros(nq, a.k, device=dev), torch.from_numpy(ids).to(dev),
                            torch.full((nq,), a.k, dtype=torch.int32, device=dev))
                q_ptr = torch.tensor(np.cumsum([0] + [len(q) for q in queries]), dtype=torch.int32, device=dev)
                q_tok = torch.tensor([t for q in queries for t in q], dtype=torch.int32, device=dev)
                cu = rr.pack(cand.ids, cand.counts, q_ptr, q_tok).cu_h
                n_pairs, n_tok = cu.size - 1, int(cu[-1])
                lo, hi = token_balanced_ranges(cu, world)[rank]
                wall, st, out = timed(lambda ev: sh.rerank(cand, q_ptr, q_tok, a.top_n, events=ev), a.reps)
                per_rank = [None] * world
                dist.all_gather_object(per_rank, {"rank": rank, "pairs": hi - lo, "tokens": int(cu[hi] - cu[lo]),
                                                  "encoder_ms": float(st[1]), "wall_s": wall})
                # the one-GPU reranker on rank 0, same inputs; the other ranks wait
                if rank == 0:
                    wall1, st1, out1 = timed(lambda ev: rr.rerank(cand, q_ptr, q_tok, a.top_n, events=ev), a.reps,
                                             together=False)
                    same = bits_equal(out, out1)
                    failed |= not same
                    share = [r["tokens"] / n_tok for r in per_rank]
                    rec = {"model": f"xlm-roberta-{name}", "gpus": world, "queries": nq, "k": a.k, "top_n": a.top_n,
                           "pairs": n_pairs, "tokens": n_tok, "wall_s": wall, "pairs_per_s": n_pairs / wall,
                           "stage_ms_rank0": {"pack_check": float(st[0]), "encoder": float(st[1]),
                                              "head_exchange_order": float(st[2])},
                           "per_rank": per_rank, "token_share_max": max(share), "token_share_min": min(share),
                           "one_gpu": {"wall_s": wall1, "pairs_per_s": n_pairs / wall1,
                                       "encoder_ms": float(st1[1])},
                           "speedup_vs_one_gpu": wall1 / wall, "parity_bit_exact": same, "reps": a.reps,
                           "card": info}
                    print(json.dumps(rec), flush=True)
                    results.append(rec)
                dist.barrier()
                del rr, sh
                torch.cuda.empty_cache()
            del model
            torch.cuda.empty_cache()
        if rank == 0:
            out_dir = Path(a.out)
            out_dir.mkdir(parents=True, exist_ok=True)
            (out_dir / "bench_rerank_dist.json").write_text(json.dumps(results, indent=1))
    finally:
        dist.destroy_process_group()
    if failed:
        sys.exit("bench_rerank_dist: the split output differs from the one-GPU output")


if __name__ == "__main__":
    main()
