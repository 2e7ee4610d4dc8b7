#!/usr/bin/env python
"""Rerank fusion (``CrossEncoderReranker.rerank_fusion``) against the two-call route it replaces, in the same run.

Workload: pipeline.py's rerank fusion -- per query a sparse list of 192 (f_topk_2) and a dense list of 288 (f_topk_1)
candidates, each reranked to top_n = 6 (r_topk), the two fused by RRF to 6 (r_topk_1), max_length 512.  A fraction of
each sparse list (0 / 25 / 50 / 100 %) is drawn from the same query's dense list: that overlap is what the union saves,
and the benchmark's random corpus has none of its own.  Passages U[64, 480] tokens, queries U[8, 48], seeded, as in
bench_rerank.py; XLM-R-large (24 L / 1024 d / 16 H / ffn 4096) and XLM-R-base (12 L / 768 d / 12 H / ffn 3072) shapes
with random bf16-representable weights (speed does not depend on the values).

Per (model, Q, overlap), the two routes alternate in one run (after a warm-up of both per model):
  fused: ``rerank_fusion`` (one union, one pack, one encoder run, two mapped orders, RRF);
  two calls: ``rerank(sparse)`` + ``rerank(dense)`` + ``rrf_fuse``.
Reported: pairs encoded and wall ms of both (each ends in a device synchronise), their stage times from CUDA events,
pairs/s on one GPU (the two lists' pairs over the wall time), the ``ezr_pair_union`` and the two
``ezr_cross_order_topk_mapped`` launches timed alone with CUDA events, whether every output is byte-equal, and the
card name and power limit read in this run.

    python scripts/bench_rerank_fusion.py --out DIR [--models large,base] [--queries 1,16,64] [--overlaps 0,0.25,0.5,1]
"""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from easyrag_b200 import _lib, batched                                            # noqa: E402
from easyrag_b200.batched import TopK                                             # noqa: E402
from easyrag_b200.encoder import BertConfig                                       # noqa: E402
from easyrag_b200.rerank import CrossEncoderModel, CrossEncoderReranker, random_cross_encoder_state   # noqa: E402

SHAPES = {"large": dict(hidden_size=1024, num_hidden_layers=24, num_attention_heads=16, intermediate_size=4096),
          "base": dict(hidden_size=768, num_hidden_layers=12, num_attention_heads=12, intermediate_size=3072)}
CLS, PAD, SEP = 0, 1, 2          # XLM-R <s> <pad> </s>
MAX_LENGTH = 512
KERNEL_REPS = 20


def card():
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=60)
        name, power, clk = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": power, "sm_max_clock": clk}
    except Exception as e:            # the device name still comes from torch
        return {"name": torch.cuda.get_device_name(0), "power_limit": f"unavailable ({e})"}


def routes(rng, n_docs, nq, k_s, k_d, overlap):
    """Sparse [Q, k_s] and dense [Q, k_d] lists of distinct ids, round(overlap * k_s) of each sparse list drawn from
    its dense list, at random ranks."""
    n_shared = int(round(overlap * k_s))
    s, d = np.empty((nq, k_s), np.int32), np.empty((nq, k_d), np.int32)
    for q in range(nq):
        perm = rng.choice(n_docs, k_d + k_s, replace=False)
        d[q] = perm[:k_d]
        s[q] = rng.permutation(np.concatenate([rng.choice(perm[:k_d], n_shared, replace=False),
                                               perm[k_d:k_d + k_s - n_shared]]))
    mk = lambda ids: TopK(torch.zeros(ids.shape, device="cuda"), torch.from_numpy(ids).cuda(),
                          torch.full((nq,), ids.shape[1], dtype=torch.int32, device="cuda"))
    return mk(s), mk(d)


def two_calls(rr, sparse, dense, q_ptr, q_tok, top_n, k_out, events=None):
    ev_s, ev_d = ([], []) if events is not None else (None, None)
    s, s_all = rr.rerank(sparse, q_ptr, q_tok, top_n, events=ev_s)
    d, d_all = rr.rerank(dense, q_ptr, q_tok, top_n, events=ev_d)
    fused = batched.rrf_fuse(s.ids, s.counts, d.ids, d.counts, k_out)
    if events is not None:
        events.extend([ev_s, ev_d])
    return fused, s, d, s_all, d_all


def stage_ms(ev):
    return [ev[i].elapsed_time(ev[i + 1]) for i in range(len(ev) - 1)]


def byte_equal(res, ref):
    fused, s, d, s_all, d_all = ref
    pairs = [(res.sparse_all, s_all), (res.dense_all, d_all)]
    for a, b in ((res.fused, fused), (res.sparse, s), (res.dense, d)):
        pairs += [(a.ids, b.ids), (a.scores, b.scores), (a.counts, b.counts)]
    return all(x.cpu().numpy().tobytes() == y.cpu().numpy().tobytes() for x, y in pairs)


def kernel_ms(rr, sparse, dense, q_ptr, q_tok, top_n):
    """ezr_pair_union alone, and the two mapped orders alone, over KERNEL_REPS launches each (CUDA events)."""
    L = _lib.lib()
    u = batched.pair_union(sparse.ids, sparse.counts, dense.ids, dense.counts)
    pairs = rr.pack(u.ids, u.counts, q_ptr, q_tok)
    nq = pairs.n_queries
    sig = torch.rand(max(pairs.n_pairs, 1), device="cuda")
    outs = [(torch.empty(nq, c.ids.shape[1], device="cuda"), torch.empty(nq, top_n, device="cuda"),
             torch.empty(nq, top_n, dtype=torch.int32, device="cuda"), torch.empty(nq, dtype=torch.int32, device="cuda"))
            for c in (sparse, dense)]

    def orders():
        for c, m, o in zip((sparse, dense), (u.map_a, u.map_b), outs):
            _lib.check(L.ezr_cross_order_topk_mapped(_lib.ptr(sig), _lib.ptr(pairs.pair_off), nq, c.ids.shape[1],
                                                     _lib.ptr(m), m.stride(0), _lib.ptr(c.ids), c.ids.stride(0),
                                                     top_n, *[_lib.ptr(x) for x in o], _lib.stream_ptr()))

    res = {}
    for name, fn in (("union", lambda: batched.pair_union(sparse.ids, sparse.counts, dense.ids, dense.counts)),
                     ("mapped_orders", orders)):
        fn()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(KERNEL_REPS):
            fn()
        t1.record()
        torch.cuda.synchronize()
        res[name] = t0.elapsed_time(t1) / KERNEL_REPS
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--models", default="large,base")
    ap.add_argument("--queries", default="1,16,64")
    ap.add_argument("--overlaps", default="0,0.25,0.5,1")
    ap.add_argument("--k-sparse", type=int, default=192)
    ap.add_argument("--k-dense", type=int, default=288)
    ap.add_argument("--top-n", type=int, default=6)
    ap.add_argument("--k-out", type=int, default=6)
    ap.add_argument("--docs", type=int, default=20000)
    ap.add_argument("--reps", type=int, default=1)
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_rerank_fusion: no CUDA device (this benchmark measures the GPU path only)")
    _lib.require_cuda()
    out_dir = Path(a.out)
    out_dir.mkdir(parents=True, exist_ok=True)
    info = card()
    results = []
    for name in a.models.split(","):
        cfg = BertConfig(vocab_size=250002, max_position_embeddings=514, layer_norm_eps=1e-5, **SHAPES[name])
        model = CrossEncoderModel("roberta", cfg, random_cross_encoder_state("roberta", cfg, a.seed), CLS, SEP, PAD,
                                  device="cuda")
        rng = np.random.default_rng(a.seed)
        passages = [rng.integers(4, cfg.vocab_size, int(n)).tolist() for n in rng.integers(64, 481, a.docs)]
        rr = CrossEncoderReranker(model, passages, max_length=MAX_LENGTH)
        warm = False
        for nq in [int(x) for x in a.queries.split(",")]:
            queries = [rng.integers(4, cfg.vocab_size, int(n)).tolist() for n in rng.integers(8, 49, nq)]
            q_ptr = torch.tensor(np.cumsum([0] + [len(q) for q in queries]), dtype=torch.int32).cuda()
            q_tok = torch.tensor([t for q in queries for t in q], dtype=torch.int32).cuda()
            if not warm:                   # both routes once per model, at its first batch size
                sparse, dense = routes(rng, a.docs, nq, a.k_sparse, a.k_dense, 0.5)
                rr.rerank_fusion(sparse, dense, q_ptr, q_tok, a.top_n, a.k_out)
                two_calls(rr, sparse, dense, q_ptr, q_tok, a.top_n, a.k_out)
                torch.cuda.synchronize()
                warm = True
            for overlap in [float(x) for x in a.overlaps.split(",")]:
                sparse, dense = routes(rng, a.docs, nq, a.k_sparse, a.k_dense, overlap)
                walls = {"fused": [], "two_calls": []}
                stages = {"fused": [], "two_calls": []}
                equal = True
                for _ in range(a.reps):
                    ev = []
                    t0 = time.perf_counter()
                    res = rr.rerank_fusion(sparse, dense, q_ptr, q_tok, a.top_n, a.k_out, events=ev)
                    torch.cuda.synchronize()
                    walls["fused"].append(time.perf_counter() - t0)
                    stages["fused"].append(stage_ms(ev))
                    ev = []
                    t0 = time.perf_counter()
                    ref = two_calls(rr, sparse, dense, q_ptr, q_tok, a.top_n, a.k_out, events=ev)
                    torch.cuda.synchronize()
                    walls["two_calls"].append(time.perf_counter() - t0)
                    stages["two_calls"].append(np.add(stage_ms(ev[0]), stage_ms(ev[1])).tolist())
                    equal = equal and byte_equal(res, ref)
                n_route = res.n_route_pairs
                wall = {k: float(np.median(v)) * 1e3 for k, v in walls.items()}
                st = {k: dict(zip(("pack", "encoder", "head_order"), np.median(np.array(v), axis=0).tolist()))
                      for k, v in stages.items()}
                rec = {"model": f"xlm-roberta-{name}", "queries": nq, "k_sparse": a.k_sparse, "k_dense": a.k_dense,
                       "overlap": overlap, "top_n": a.top_n, "k_out": a.k_out,
                       "pairs_encoded": {"fused": res.n_pairs, "two_calls": n_route},
                       "wall_ms": wall, "stage_ms": st,
                       "pairs_per_s": {k: n_route / (v * 1e-3) for k, v in wall.items()},
                       "speedup": wall["two_calls"] / wall["fused"],
                       "kernel_ms": kernel_ms(rr, sparse, dense, q_ptr, q_tok, a.top_n),
                       "byte_equal": bool(equal), "reps": a.reps, "card": info}
                print(json.dumps(rec), flush=True)
                results.append(rec)
        del rr, model
        torch.cuda.empty_cache()
    (out_dir / "bench_rerank_fusion.json").write_text(json.dumps(results, indent=1))
    bad = [(r["model"], r["queries"], r["overlap"]) for r in results if not r["byte_equal"]]
    if bad:
        sys.exit(f"bench_rerank_fusion: outputs differ from the two-call route at {bad}")


if __name__ == "__main__":
    main()
