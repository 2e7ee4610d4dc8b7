"""String interning: the host dict loops (compress.pack, retrievers._encode_corpus, retrievers._canon_ids, a dict
lookup of query tokens) against the device interner (easyrag_b200.vocab.Vocabulary) on the same inputs, in one run,
alternating.

Workloads: compress packs at 1 000 and 10 000 contexts (scripts/bench_compress.py's generator), a 1M-document corpus
of about 300 multi-byte pseudo-Chinese tokens each, _canon_ids over 1M chunk texts, and 10 000 queries looked up in
that corpus's vocabulary.  Per workload: the host join (planner + "\\0".join + encode, timed on its own), the bytes
copied to the device, the interner's kernel time (torch.profiler, in a run of its own), the bytes read back, the
total wall time of each route, the vocabulary size and whether ids, dicts and first indices are equal.  Also
ContextCompressor.compress_batch end to end with the host pack (before) and the device pack (after).

    python scripts/bench_vocab.py --out DIR      (writes DIR/bench_vocab.json)
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time
from itertools import chain
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent))
from bench_compress import Tok, card, contexts  # noqa: E402
from easyrag_b200 import _lib  # noqa: E402
from easyrag_b200.compress import ContextCompressor, pack, pack_device  # noqa: E402
from easyrag_b200.retrievers import BM25Retriever, _canon_ids, _encode_corpus  # noqa: E402
from easyrag_b200.schema import TextNode  # noqa: E402
from easyrag_b200.vocab import CHUNK_BYTES, CHUNK_STRINGS, Vocabulary, iter_chunks  # noqa: E402

MB = 1 << 20


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, (time.perf_counter() - t0) * 1e3


def join_cost(groups, flat=False):
    """(ms, bytes) of the host side of the device route alone: the chunk planner, the join and the encode."""
    counts = np.ones(len(groups), np.int64) if flat else np.fromiter(map(len, groups), np.int64, len(groups))
    t0 = time.perf_counter()
    nb = sum(len(d) for _, _, d, _ in iter_chunks(groups, counts, CHUNK_STRINGS, CHUNK_BYTES, flat))
    return (time.perf_counter() - t0) * 1e3, nb


def kernel_ms(fn):
    """Summed device time of the interner's kernels in one run of ``fn`` under torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    names = ("vocab_", "scan_tiles", "scan_top", "scan_emit")
    return sum(e.self_device_time_total for e in prof.key_averages() if any(n in e.key for n in names)) / 1e3


def pseudo_chinese_pool(n):
    return [chr(0x4E00 + i % 4000) + chr(0x4E00 + i // 4000) + "的" * (i % 3) for i in range(n)]


def corpus(rng, n_docs, mean_len, pool):
    lens = rng.integers(mean_len // 2, mean_len * 3 // 2 + 1, n_docs)
    pid = np.minimum(rng.zipf(1.1, int(lens.sum())) - 1, len(pool) - 1)
    flat = np.asarray(pool, dtype=object)[pid].tolist()
    off = np.concatenate([[0], np.cumsum(lens)])
    return [flat[off[i]:off[i + 1]] for i in range(n_docs)]


def row(name, rounds, host_fn, dev_fn, compare, groups, flat=False, d2h=0):
    """Alternate the two routes ``rounds`` times; keep the best of each."""
    best_h = best_d = None
    for _ in range(rounds):
        h, ms_h = timed(host_fn)
        best_h = ms_h if best_h is None else min(best_h, ms_h)
        d, ms_d = timed(dev_fn)
        best_d = ms_d if best_d is None else min(best_d, ms_d)
    eq = compare(h, d)
    j_ms, nb = join_cost(groups, flat)
    k_ms = kernel_ms(dev_fn)
    r = dict(workload=name, strings=int(sum(1 for _ in (groups if flat else chain.from_iterable(groups)))),
             host_total_ms=round(best_h, 1), device_total_ms=round(best_d, 1), host_join_ms=round(j_ms, 1),
             h2d_mb=round(nb / MB, 1), kernel_ms=round(k_ms, 2), d2h_mb=round(d2h(d) / MB, 2) if callable(d2h) else d2h,
             **eq)
    print(json.dumps(r), flush=True)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--docs", type=int, default=1_000_000)
    ap.add_argument("--doc-len", type=int, default=300)
    ap.add_argument("--texts", type=int, default=1_000_000)
    ap.add_argument("--contexts", default="1000,10000")
    ap.add_argument("--rounds", type=int, default=2)
    # --contexts "" / --docs 0 / --texts 0 skip a workload (the 1M-document one can run alone)
    a = ap.parse_args()
    _lib.require_cuda()
    info = card()
    rng = np.random.default_rng(0)
    rows = []
    Vocabulary().intern([["warm", "up"]])

    # compress packs (sentence tokens interned, query tokens looked up)
    comp = ContextCompressor("bm25_extract", 0.5, BM25Retriever([TextNode(text="seed", id_="n0")], Tok(),
                                                                stopwords=["the"]), splitter=lambda c: c.split("\n"))
    for g in (int(x) for x in a.contexts.split(",") if x):
        qs, cs = contexts(rng, g)
        sents = comp.split(cs)
        qt, st = comp.tokenize(qs, sents)
        dev = comp.bm25_retriever.bm25.device

        def cmp_pack(p, d):
            return dict(vocab=len(p.vocab), ids_equal=bool(np.array_equal(p.tokens, d.tokens.cpu().numpy())
                                                           and np.array_equal(p.q_tokens, d.q_tokens.cpu().numpy())),
                        dict_equal=list(p.vocab.items()) == list(d.vocab.to_dict().items()), first_equal=None)
        rows.append(row(f"compress pack, {g} contexts", a.rounds, lambda: pack(qt, st, sents, cs),
                        lambda: pack_device(qt, st, sents, cs, dev), cmp_pack,
                        [t for s in st for t in s] + list(qt), d2h=0))
        # compress_batch end to end: host pack (before) and device pack (after)
        ms = {}
        for rnd in range(a.rounds):
            for route in ("before", "after"):
                def go():
                    if route == "after":
                        return comp.compress_batch(qs, cs)
                    s2 = comp.split(cs)
                    q2, t2 = comp.tokenize(qs, s2)
                    return comp.join(s2, comp.run(pack(q2, t2, s2, cs))[0])
                out, t = timed(go)
                ms[route] = min(ms.get(route, t), t)
                ms[route + "_out"] = out
        r = dict(workload=f"compress_batch end to end, {g} contexts",
                 before_contexts_per_s=round(g / ms["before"] * 1e3, 1),
                 after_contexts_per_s=round(g / ms["after"] * 1e3, 1),
                 strings_equal=ms["before_out"] == ms["after_out"])
        print(json.dumps(r), flush=True)
        rows.append(r)

    if a.docs:
        # a 1M-document corpus
        pool = pseudo_chinese_pool(200_000)
        docs = corpus(rng, a.docs, a.doc_len, pool)

        def dev_corpus():                                   # BM25Retriever's route: ids on the device, the dict on the host
            v = Vocabulary()
            ids, ptr = v.intern(docs)
            return v, ids, ptr, v.to_dict()

        def cmp_corpus(h, d):
            vocab, tokens, doc_ptr = h
            v, ids, ptr, dd = d
            return dict(vocab=len(vocab), ids_equal=bool(torch.equal(tokens, ids.cpu()) and torch.equal(doc_ptr, ptr)),
                        dict_equal=list(vocab.items()) == list(dd.items()), first_equal=None)
        rows.append(row(f"BM25 corpus, {a.docs} documents", max(1, a.rounds - 1), lambda: _encode_corpus(docs),
                        dev_corpus, cmp_corpus, docs,
                        d2h=lambda d: int(d[0]._state[1]) + 8 * (len(d[0]) + 1)))          # to_dict's arena read
        v_corpus, _, _, host_vocab = dev_corpus()

        # 10k-query lookups in that vocabulary
        queries = [[pool[int(i)] for i in np.minimum(rng.zipf(1.1, int(rng.integers(3, 16))) - 1, len(pool) - 1)]
                   + ["未知词"] for _ in range(10_000)]

        def host_lookup():
            ids = [host_vocab.get(t, -1) for q in queries for t in q]
            ptr = np.concatenate([[0], np.cumsum([len(q) for q in queries])])
            return torch.tensor(ids, dtype=torch.int32), ptr

        rows.append(row("10k-query lookup", a.rounds, host_lookup, lambda: v_corpus.lookup(queries),
                        lambda h, d: dict(vocab=len(host_vocab), ids_equal=bool(torch.equal(h[0], d[0].cpu())),
                                          dict_equal=None, first_equal=None), queries, d2h=0))
        del docs, v_corpus

    if a.texts:
        # _canon_ids over 1M chunk texts (about 10 % repeated)
        words = pseudo_chinese_pool(20_000)
        base = [" ".join(words[int(j)] for j in rng.integers(0, len(words), int(n))) for n in rng.integers(20, 200, a.texts)]
        dup = rng.integers(0, a.texts, a.texts // 10)
        texts = base[:]
        for i, j in zip(rng.integers(0, a.texts, dup.size), dup):
            texts[int(i)] = base[int(j)]
        rows.append(row(f"_canon_ids, {a.texts} texts", a.rounds, lambda: _canon_ids(texts),
                        lambda: Vocabulary().first_index(texts).cpu(),
                        lambda h, d: dict(vocab=None, ids_equal=None, dict_equal=None,
                                          first_equal=bool(np.array_equal(h, d.numpy()))),
                        texts, flat=True, d2h=round(8 * a.texts / MB, 2)))
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "bench_vocab.json"), "w") as f:
        json.dump(dict(card=info, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
