#!/usr/bin/env python
"""BM25 top-k for k > 32: the deep two-phase path (ezr_bm25_topk) against score rows in Python blocks, in one run.

    python scripts/bench_bm25_deep.py --out DIR [--rounds 5]

Writes DIR/bench_bm25_deep.json and prints it.  bench.py's corpus and query seeds (1M chunks, 200k vocabulary,
float64 Okapi index with packed postings), at Q in {64, 1000, 10000} and k in {32, 33, 192, 288, 1024}.  Per case:
median call time and q/s of each route over --rounds rounds that alternate the two (a host clock around a call that
ends in a device synchronise), the candidate-pass, bound and rescore kernel times from the EZR_PROF_BM25_* slots in
a separate profiled call, the score-row launches that answered overflowed queries, the workspace bytes of each
route, and whether the two routes return the same bytes.  k = 32 runs the k <= 32 fused path for comparison.  The
score-row route is bm25_scores + select_rows(positive_only=True) over blocks of 256 queries.  GPU name and power
limit are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
import time
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

SEED = 20240922 + 3            # bench.py
N_DOCS, VOCAB = 1_000_000, 200_000
QS = (64, 1000, 10_000)
KS = (32, 33, 192, 288, 1024)
BLOCK = 256


def gpu_info() -> dict:
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    return {"nvidia_smi": r.stdout.strip(), "torch_name": torch.cuda.get_device_name()}


def rows_route(batched, ix, qp, qt, k):
    parts = []
    nq = qp.numel() - 1
    for b in range(0, nq, BLOCK):
        e = min(nq, b + BLOCK)
        rows = batched.bm25_scores(ix, qp[b:e + 1] - qp[b], qt[int(qp[b]):max(int(qp[e]), int(qp[b]) + 1)])
        parts.append(batched.select_rows(rows, k, positive_only=True))
        del rows
    return batched.TopK(torch.cat([p.scores for p in parts]), torch.cat([p.ids for p in parts]),
                        torch.cat([p.counts for p in parts]))


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, r


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--out", required=True)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    from easyrag_b200 import _lib, batched, synth
    from easyrag_b200.index import Bm25Index, Bm25Stats
    _lib.require_cuda()
    L = _lib.lib()
    dev = "cuda"
    corpus = synth.make_sparse_corpus(N_DOCS, VOCAB, SEED, device=dev)
    queries = synth.make_queries(corpus, max(QS), SEED + 1)
    stats = Bm25Stats.from_tokens(corpus.tokens, corpus.doc_ptr, VOCAB, bm25_type=0)
    ix = Bm25Index(stats, device=dev, packed=True)
    assert ix.post_pk is not None
    del corpus
    qp_all = queries.term_ptr.to(device=dev, dtype=torch.int32)
    qt_all = queries.terms.to(device=dev, dtype=torch.int32)
    ws = batched.Workspace(dev)
    cases = []
    for nq in QS:
        qp, qt = qp_all[:nq + 1], qt_all[:int(qp_all[nq])]
        for k in KS:
            fast = lambda: batched.bm25_topk(ix, qp, qt, k, ws=ws)
            slow = lambda: rows_route(batched, ix, qp, qt, k)
            a, b = fast(), slow()                                  # warm-up of every shape
            same = (torch.equal(a.counts, b.counts) and torch.equal(a.ids, b.ids)
                    and torch.equal(a.scores.view(torch.int64), b.scores.view(torch.int64)))
            tf, ts = [], []
            for _ in range(args.rounds):
                tf.append(timed(fast)[0])
                ts.append(timed(slow)[0])
            L.ezr_profile_reset()
            L.ezr_profile_enable(1)
            timed(fast)
            L.ezr_profile_enable(0)
            prof = {n: _lib.profile_read(n) for n in ("bm25_cand", "bm25_bound", "bm25_rescore", "bm25_score",
                                                      "merge")}
            mf, ms = statistics.median(tf), statistics.median(ts)
            rows_ws = min(nq, BLOCK) * N_DOCS * 8 + L.ezr_select_rows_workspace(min(nq, BLOCK), N_DOCS, k, _lib.F64)
            case = dict(queries=nq, k=k, deep_ms=mf * 1e3, deep_qps=nq / mf, rows_ms=ms * 1e3, rows_qps=nq / ms,
                        speedup=ms / mf, equal=same,
                        cand_ms=prof["bm25_cand"][0] - prof["bm25_bound"][0], bound_ms=prof["bm25_bound"][0],
                        rescore_ms=prof["bm25_rescore"][0], select_ms=prof["merge"][0],
                        overflow_score_launches=prof["bm25_score"][1],
                        deep_workspace_bytes=int(L.ezr_bm25_topk_workspace(ix.struct, nq, k)),
                        rows_workspace_bytes=int(rows_ws))
            cases.append(case)
            print(json.dumps(case), flush=True)
    out = dict(gpu=gpu_info(), corpus=dict(docs=N_DOCS, vocab=VOCAB, postings=ix.n_postings, seed=SEED),
               rounds=args.rounds, cases=cases)
    d = Path(args.out)
    d.mkdir(parents=True, exist_ok=True)
    (d / "bench_bm25_deep.json").write_text(json.dumps(out, indent=1))
    print(json.dumps(out["gpu"]))


if __name__ == "__main__":
    main()
