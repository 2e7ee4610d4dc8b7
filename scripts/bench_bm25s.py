"""BM25 top-k on a bm25s (float32) index: the two-phase path over packed postings (``Bm25Index(packed=True)``)
against the route it replaces on the same arrays (``ordered_view()``: the ordered kernel for k <= 32, score rows in
blocks + select above), whose results it must reproduce byte for byte.

    python scripts/bench_bm25s.py --out DIR [--steps 5] [--warmup 2]

bench.py's corpus and queries (make_sparse_corpus(SEED), make_queries(SEED + 1), 1M documents, 200k vocabulary)
with bm25s statistics.  The two routes alternate step by step on the same inputs; per call: CUDA events around it,
medians over the timed steps.  Per case, in separate profiled calls: the library's kernel timing slots of the
packed path -- candidate launches (bm25_cand, which includes the bound steps between range chunks), bound steps
alone (bm25_bound), rescoring (bm25_rescore), the ordered kernel and select/merge (bm25_score, merge: overflowed
queries and the deep form's select) -- and of the ordered route (bm25_score, merge).  Candidates per query (mean and
max over the queries that did not overflow) and the overflowed queries are read from the call's workspace.
Equality: counts and ids byte-equal in full, scores byte-equal wherever a result is listed.  Writes
DIR/bench_bm25s.json with the card's name and power limit, and prints each row.
"""
import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from easyrag_b200 import _lib, batched, synth  # noqa: E402
from easyrag_b200.index import Bm25Index, Bm25Stats  # noqa: E402

SEED = 20240922 + 3              # bench.py
N_DOCS, VOCAB = 1_000_000, 200_000
QUERIES = (64, 1_000, 10_000)
KS = (10, 32, 192, 288, 1024)
SLOTS_PK = ("bm25_cand", "bm25_bound", "bm25_rescore", "bm25_score", "merge")
SLOTS_ORD = ("bm25_score", "merge")


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in out.split(",")]
        return dict(name=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:                    # the figures are still valid; say what could not be read
        return dict(name=torch.cuda.get_device_name(0), power_limit=f"unknown ({e})", max_sm_clock="unknown")


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


def cand_stats(ws, nq, k, n_ranges):
    """Candidates per query and overflowed queries of the last call, from its workspace (``pk_carve`` in
    csrc/bm25.cu: thr_key, thr_q, cand_cnt, ovf, ... [Q] each, after the k <= 32 path's float32 candidate lists,
    at offset 0 in the deep form)."""
    align = lambda x: (x + 255) // 256 * 256
    n = nq * n_ranges * k
    base = align(n * 4) + align(n * 4) if k <= 32 else 0
    words = ws.buf[base:base + 4 * (6 * nq + 1)].view(torch.int32)
    cnt, ovf = words[2 * nq:3 * nq], words[3 * nq:4 * nq]
    n_ovf = int(words[6 * nq])
    ok = ovf == 0
    c = cnt[ok].float()
    return dict(cand_per_query_mean=float(c.mean()) if c.numel() else None,
                cand_per_query_max=int(cnt[ok].max()) if c.numel() else None, overflowed=n_ovf)


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
    results = dict(gpu=gpu_info(), steps=args.steps, warmup=args.warmup, docs=N_DOCS, vocab=VOCAB, cases=[])
    print(json.dumps(results["gpu"]), flush=True)
    corpus = synth.make_sparse_corpus(N_DOCS, VOCAB, SEED, device=dev)
    stats = Bm25Stats.from_tokens(corpus.tokens, corpus.doc_ptr, VOCAB, bm25_type=1)
    packed = Bm25Index(stats, device=dev, packed=True)
    ordered = packed.ordered_view()
    assert packed.post_pk is not None and ordered.post_pk is None
    results.update(index_bytes_packed=packed.index_bytes(), index_bytes_ordered=ordered.index_bytes(),
                   postings=packed.n_postings, ranges=packed.n_ranges)
    print(json.dumps({k: results[k] for k in ("index_bytes_packed", "index_bytes_ordered", "postings", "ranges")}),
          flush=True)
    for nq in QUERIES:
        qs = synth.make_queries(corpus, nq, SEED + 1)
        qp, qt = qs.term_ptr.to(dev), qs.terms.to(dev)
        for k in KS:
            ws_p, ws_o = batched.Workspace(dev), batched.Workspace(dev)
            mk = lambda: batched.TopK(torch.empty(nq, k, device=dev), torch.empty(nq, k, dtype=torch.int32, device=dev),
                                      torch.empty(nq, dtype=torch.int32, device=dev))
            out_p, out_o = mk(), mk()
            run_p = lambda: batched.bm25_topk(packed, qp, qt, k, ws=ws_p, out=out_p)
            run_o = lambda: batched.bm25_topk(ordered, qp, qt, k, ws=ws_o, out=out_o)
            for _ in range(args.warmup):
                run_p()
                run_o()
            torch.cuda.synchronize()
            t_p, t_o = [], []
            for _ in range(args.steps):
                t_p.append(timed(run_p))
                t_o.append(timed(run_o))
            ms_p, ms_o = statistics.median(t_p), statistics.median(t_o)
            eq = same(out_p, out_o)
            cs = cand_stats(ws_p, nq, k, packed.n_ranges)
            pp = profiled(L, run_p, SLOTS_PK, 2)
            po = profiled(L, run_o, SLOTS_ORD, 2)
            row = dict(queries=nq, k=k,
                       packed=dict(ms=ms_p, qps=nq / ms_p * 1e3, cand_ms=pp["bm25_cand"], bound_ms=pp["bm25_bound"],
                                   rescore_ms=pp["bm25_rescore"], fallback_score_ms=pp["bm25_score"],
                                   select_merge_ms=pp["merge"], **cs,
                                   workspace_bytes=L.ezr_bm25_topk_workspace(packed.struct, nq, k)),
                       ordered=dict(ms=ms_o, qps=nq / ms_o * 1e3, score_ms=po["bm25_score"], select_merge_ms=po["merge"],
                                    workspace_bytes=L.ezr_bm25_topk_workspace(ordered.struct, nq, k)),
                       speedup=ms_o / ms_p, **eq)
            results["cases"].append(row)
            print(json.dumps(row), flush=True)
            del out_p, out_o, ws_p, ws_o
            torch.cuda.empty_cache()
    out = Path(args.out)
    out.mkdir(parents=True, exist_ok=True)
    (out / "bench_bm25s.json").write_text(json.dumps(results, indent=1))
    ok = all(r["counts_equal"] and r["ids_equal"] and r["scores_equal"] for r in results["cases"])
    print(json.dumps(dict(all_equal=ok)))
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
