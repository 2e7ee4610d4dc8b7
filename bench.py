#!/usr/bin/env python
"""Benchmark of the coarse-ranking hot path: queries/sec, dense + BM25 + RRF top-10 over 1M x 768 chunks.

    python bench.py [--gpus N] [--steps K] [--warmup W] [--impl ours|reference] [--workload retrieve|encode]
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port P \
        bench.py --gpus N --steps K --warmup W

Workload = BASELINE.json configs[2] ("dense+BM25 dual-route + RRF fusion top-10, 1M chunks, 10k queries",
the configuration the metric is quoted on); at N > 1 the SAME corpus is row-sharded (configs[3]) -> strong
scaling.  One step = one pass of the hot path over the whole batch of synthetic queries (10k by default;
``--queries 64`` is the HBM-bound small-batch regime of SURVEY.md 8(d), configs[4] adds ``--rows 4000000 --dim 1024``).

  value : whole-job queries/s with query vectors + term ids resident in HBM when the timed region starts; the
          two routes run on two streams (``--overlap 1``, the product default) and the K timed steps are submitted
          back to back (``--pipeline 1``: the join of step i -- all-gather, merges, RRF -- runs under the routes of
          step i+1; the bracket closes after ``join()``.  ``--pipeline 0`` joins every step to the caller's stream).
  e2e   : same metric through the public host-buffer API (``batched.HostPipeline``): pinned HOST inputs, H2D of
          the queries / term ids and D2H of the fused (id, score) lists inside the timed region, every step.
  roofline : dominant kernel, algorithmic FLOPs or bytes / CUDA-event duration on its launch stream, taken from
          ``--cal-steps`` NON-overlapped calibration steps of the same run (with the routes co-resident a kernel's
          event time would include the other route's share of the SM); the overlapped durations are listed too.
  parity_full_size : after timing, the first ``--parity-queries`` queries of the measured workload are compared with
          the CPU oracle over the FULL corpus: BM25 ids + float64 score bits identical, dense scores within 1e-3 of
          the fp32 cosine (ids equal outside near-ties), RRF identical; a digest of all fused results pins N>1 == N=1.
  cpu_baseline : the oracle port of the reference's CPU retrievers (numpy BM25Okapi restatement + full argsort,
          fp32 BLAS cosine, Python RRF) on a bounded query sample over the same corpus, on this box's cores.

``--impl reference`` prints the CPU arm as its own line (rank 0 only under torchrun).
``--workload encode`` measures the chunk-embedding forward pass (configs[1]) instead; see bench_encode.py.
Nothing here reads the reference checkout.
"""
from __future__ import annotations

import argparse
import hashlib
import json
import os
import statistics
import subprocess
import sys
import threading
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent
sys.path.insert(0, str(ROOT))

SEED = 20240922 + 3
METRIC = "queries/sec dense+BM25+RRF top-10 over 1M x 768 chunks"
DENSE_TOL = 1e-3            # north star: cosine scores within 1e-3 for bf16 embeddings
DIGEST_FILE = ROOT / "tests" / "golden" / "bench_digest.json"


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--workload", default="retrieve", choices=["retrieve", "encode"])
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--vocab", type=int, default=200_000)
    ap.add_argument("--queries", type=int, default=10_000)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--cpu-queries", type=int, default=256, help="bounded sample for the CPU baseline (~12 s a step)")
    ap.add_argument("--ref-queries", type=int, default=64,
                    help="--impl reference: queries per step (a bounded sample so that K + W steps end in minutes)")
    ap.add_argument("--no-cpu", action="store_true", help="skip the cpu_baseline leg (parity still runs)")
    ap.add_argument("--parity-queries", type=int, default=256,
                    help="queries compared with the CPU oracle over the full corpus after timing (0 = off)")
    ap.add_argument("--dense-kernel", type=int, default=0,
                    help="0 auto, 1 simt, 2 wgmma with 128-query blocks (dim <= 768), 3 wgmma with 64-query blocks, "
                         "4 the same with 128-row corpus tiles, 5 = 4 in cluster pairs (multicast corpus tiles)")
    ap.add_argument("--overlap", type=int, default=1, help="1 (default): dense and BM25 routes on two streams")
    ap.add_argument("--bm25-span", type=int, default=4, help="document ranges in the first candidate launch (tuning)")
    ap.add_argument("--serial-routes", type=int, default=0,
                    help="1 (with --overlap 1 --pipeline 1): both routes on ONE side stream, dense kernel with its full "
                         "shared-memory ring (cluster-pair form); the join still runs under the next step's routes")
    ap.add_argument("--pipeline", type=int, default=1,
                    help="1 (default, needs --overlap 1): steps are submitted, not joined -- the join of step i (all-gather, "
                         "merges, RRF) runs under the route kernels of step i+1; 0: every step joins the caller's stream")
    ap.add_argument("--cal-steps", type=int, default=5, help="non-overlapped calibration steps for per-kernel times")
    ap.add_argument("--self-check", type=int, default=64,
                    help="after timing: first N queries through both BM25 kernel paths at full size, compared bit for bit")
    ap.add_argument("--bm25-skip", type=int, default=0, help="1: candidate pass skips non-essential terms (A/B)")
    ap.add_argument("--bm25-plan", type=int, default=1, help="0: candidate CTAs resolve their posting segments themselves (A/B)")
    ap.add_argument("--dense-probe", type=int, default=0, help="measurement probe of the dense kernel (results invalid)")
    ap.add_argument("--dense-stages", type=int, default=0,
                    help="cap of the dense kernel's TMA ring (0 = all smem, the default: with the query block resident the "
                         "dense CTA fills the SM's shared memory, so a cap frees no room for BM25 CTAs; 3 stages measured "
                         "41.6 vs 31.9 ms per 10k-query launch on H100)")
    ap.add_argument("--enc-chunks", type=int, default=100_000,
                    help="chunks of the `encode` block (configs[1]: GTE-base-shaped encoder); 0 = skip the block")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write the fused / sparse / dense (scores, ids, counts) of the last timed "
                         "step as DIR/<route>_<field>.npy (float64; entries past a query's count set to -1 / 0; at most "
                         "64 MB: a fixed seeded sample of query rows above that, listed in DIR/query_rows.npy)")
    ap.add_argument("--l2-flush", type=int, default=-1,
                    help="1: write a 512 MB buffer between steps and time each step on its own (default for <= 512 queries)")
    return ap.parse_args()


# ----------------------------------------------------------------------------------- data
def make_data(args, dev):
    """Synthetic config-3 data, generated on the GPU (3e8 tokens), identical on every rank (same seed)."""
    from easyrag_b200 import synth
    from easyrag_b200.index import Bm25Stats
    t0 = time.time()
    corpus = synth.make_sparse_corpus(args.rows, args.vocab, SEED, device=dev)
    queries = synth.make_queries(corpus, args.queries, SEED + 1)
    stats = Bm25Stats.from_tokens(corpus.tokens, corpus.doc_ptr, args.vocab, bm25_type=0)
    n_tokens = int(corpus.tokens.numel())
    del corpus
    vec = synth.make_dense_corpus(args.rows, args.dim, SEED + 2, device=dev)
    qvec = synth.make_dense_queries(vec, args.queries, SEED + 3)
    torch.cuda.synchronize()
    return dict(stats=stats, queries=queries, vec=vec, qvec=qvec, n_tokens=n_tokens, gen_s=time.time() - t0)


# --------------------------------------------------------------------------------- clocks
class ClockSampler:
    FIELDS = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,"
              "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
              "clocks_event_reasons.sw_power_cap")

    def __init__(self, index: int):
        self.index = index
        self.lines = []          # (arrival time, csv line)
        self.windows = []        # [t_begin, t_end] of the timed regions
        self.proc = None

    def begin(self):
        self.windows.append([time.perf_counter(), None])

    def end(self):
        self.windows[-1][1] = time.perf_counter()

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "-i", str(self.index), f"--query-gpu={self.FIELDS}",
                                          "--format=csv,noheader,nounits", "-lms", "50"], stdout=subprocess.PIPE,
                                         stderr=subprocess.DEVNULL, text=True)
            threading.Thread(target=self._pump, daemon=True).start()
        except Exception:
            self.proc = None

    def _pump(self):
        for line in self.proc.stdout:
            self.lines.append((time.perf_counter(), line.strip()))

    def stop(self):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        time.sleep(0.15)
        self.proc.terminate()
        sm, mx, reasons = [], [], set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        # nvidia-smi is started before the warm-up (its start-up takes longer than a short timed region); only
        # samples that arrived while a timed region was running count (a line arrives a few ms after its sample)
        inside = [ln for t, ln in self.lines if any(a <= t <= (b or t) + 0.03 for a, b in self.windows)]
        for ln in inside:
            parts = [p.strip() for p in ln.split(",")]
            if len(parts) < 7:
                continue
            try:
                sm.append(float(parts[0]))
                mx.append(float(parts[1]))
            except ValueError:
                continue
            for nm, v in zip(names, parts[3:7]):
                if v.lower().startswith("active"):
                    reasons.add(nm)
        return {"sm_mhz": statistics.median(sm) if sm else None, "sm_max_mhz": max(mx) if mx else None,
                "reasons": sorted(reasons), "samples": len(sm)}


# -------------------------------------------------------------------------- CPU reference
def canonical_topk(score: np.ndarray, k: int, positive_only: bool):
    """Top-k of a score vector under the canonical order (score desc, id desc) without a full sort, plus the tie
    flags SURVEY.md 8(c) asks for: (ids, scores, tie inside the top-k, tie straddling the k-th / (k+1)-th place)."""
    n = score.shape[0]
    kk = min(k + 1, n)
    top = np.sort(score[np.argpartition(score, n - kk)[n - kk:]])[::-1]     # the k+1 largest values, descending
    v_k = top[min(k, n) - 1]
    cand = np.nonzero(score >= v_k)[0]                                      # everything tied with the k-th or better
    order = cand[np.lexsort((-cand, -score[cand]))][:k]
    sc = score[order]
    if positive_only:                                                       # retrievers.py:195-196
        keep = sc > 0
        order, sc = order[keep], sc[keep]
    inside = bool(sc.size > 1 and np.any(sc[1:] == sc[:-1]))
    straddle = bool(kk > k and top[k] == top[k - 1] and (top[k - 1] > 0 or not positive_only) and sc.size == k)
    return order.astype(np.int64), sc, inside, straddle


class CpuReference:
    """Oracle port of the reference's CPU retrievers over the full corpus (kind = "port").

    BM25: rank_bm25.BM25Okapi.get_scores restated on CSR postings with numpy (oracle/bm25.py evaluation
    order; the literal reference loops over all N documents in Python per query term and is far slower),
    then BM25Retriever.filter's full ``argsort()[::-1]`` (retrievers.py:192).  Dense: exact fp32 cosine with
    the host BLAS on all cores + argpartition (qdrant local mode).  Fusion: Python RRF (retrievers.py:256-274).
    """

    def __init__(self, data, args):
        from oracle import retrieve as ort
        self.ort = ort
        st = data["stats"]
        self.indptr = st.indptr.cpu().numpy()
        self.post_doc = st.post_doc.cpu().numpy()
        self.post_tf = st.post_tf.cpu().numpy().astype(np.float64)
        self.idf = st.idf
        dl = st.doc_len.cpu().numpy()
        self.K_d = 1.5 * ((1 - 0.75) + (0.75 * dl) / st.avgdl)
        self.n = st.n_docs
        self.vec = data["vec"].float().cpu()
        self.qvec = data["qvec"].float().cpu()
        self.term_lists = data["queries"].term_lists()
        self.k = args.k
        self.cores = os.cpu_count()
        torch.set_num_threads(self.cores)

    def bm25_scores(self, qi: int) -> np.ndarray:
        score = np.zeros(self.n)
        for t in self.term_lists[qi]:
            if t < 0 or self.idf[t] == 0.0:
                continue
            s, e = self.indptr[t], self.indptr[t + 1]
            tf = self.post_tf[s:e]
            d = self.post_doc[s:e]
            score[d] += self.idf[t] * (tf * 2.5 / (tf + self.K_d[d]))
        return score

    def run(self, lo: int, hi: int):
        """The timed CPU arm: literal control flow of the reference (full argsort per query)."""
        k = self.k
        sims = (self.qvec[lo:hi] @ self.vec.T).numpy()
        out = []
        for j, qi in enumerate(range(lo, hi)):
            score = self.bm25_scores(qi)
            order = score.argsort()[::-1]                                   # retrievers.py:192
            sparse = [int(i) for i in order[:k] if score[i] > 0]
            part = np.argpartition(-sims[j], k)[:k]
            dense = [int(i) for i in part[np.argsort(-sims[j][part], kind="stable")]]
            out.append(self.ort.rrf_ids([sparse, dense], None, K=60, topk=k))
        return out

    def collect(self, lo: int, hi: int):
        """The parity arm (untimed): the same arithmetic with the canonical tie order and everything the comparison
        with the GPU lists needs.  Returns per query a dict(sparse_ids, sparse_sc, dense_ids, dense_sc, fused_ids,
        fused_sc, ties) and the fp32 similarity matrix of these queries."""
        k = self.k
        sims = (self.qvec[lo:hi] @ self.vec.T).numpy()
        out = []
        for j, qi in enumerate(range(lo, hi)):
            s_ids, s_sc, inside, straddle = canonical_topk(self.bm25_scores(qi), k, positive_only=True)
            d_ids, d_sc, d_in, d_str = canonical_topk(sims[j], k, positive_only=False)
            f_ids, f_sc = self.ort.rrf_ids([s_ids, d_ids], None, K=60, topk=k)
            out.append(dict(sparse_ids=s_ids, sparse_sc=s_sc, dense_ids=d_ids, dense_sc=d_sc, fused_ids=f_ids,
                            fused_sc=f_sc, bm25_tie=inside or straddle, dense_tie=d_in or d_str))
        return out, sims

    def measure(self, n_queries: int, steps: int = 1, warmup: int = 0):
        n_queries = min(n_queries, len(self.term_lists))
        for _ in range(warmup):
            self.run(0, n_queries)
        t0 = time.perf_counter()
        for _ in range(steps):
            self.run(0, n_queries)
        dt = time.perf_counter() - t0
        return steps * n_queries / dt, dt / steps


def parity_full_size(ref: CpuReference, nq: int, fused, sparse, dense, k: int):
    """GPU lists (torch tensors, first ``nq`` queries over the full corpus, global ids) against the CPU oracle."""
    ora, sims = ref.collect(0, nq)
    f_ids, f_sc, f_cnt = fused.ids.cpu().numpy(), fused.scores.cpu().numpy(), fused.counts.cpu().numpy()
    s_ids, s_sc, s_cnt = sparse.ids.cpu().numpy(), sparse.scores.cpu().numpy(), sparse.counts.cpu().numpy()
    d_ids, d_sc = dense.ids.cpu().numpy(), dense.scores.cpu().numpy()
    bm25_ok = dense_ids_equal = rrf_ok = lists_identical = near_tie_swaps = 0
    dense_max_abs, dense_ok = 0.0, True
    first_bad = None
    for i, o in enumerate(ora):
        c = int(s_cnt[i])
        b_ok = (c == o["sparse_ids"].size and np.array_equal(s_ids[i, :c], o["sparse_ids"])
                and s_sc[i, :c].tobytes() == o["sparse_sc"].tobytes())
        bm25_ok += b_ok
        g = d_ids[i]
        diff = float(np.abs(d_sc[i].astype(np.float64) - sims[i][g].astype(np.float64)).max())
        dense_max_abs = max(dense_max_abs, diff)
        same = np.array_equal(g, o["dense_ids"])
        dense_ids_equal += same
        if not same:
            # allowed only as a near-tie: every oracle id the GPU list lacks scores within tol of the GPU's k-th,
            # every GPU id the oracle list lacks scores within tol of the oracle's k-th
            miss = np.setdiff1d(o["dense_ids"], g)
            extra = np.setdiff1d(g, o["dense_ids"])
            ok = (np.all(sims[i][miss] <= d_sc[i].min() + DENSE_TOL) and np.all(sims[i][extra] >= o["dense_sc"].min() - DENSE_TOL)
                  and set(g.tolist()) - set(extra.tolist()) == set(o["dense_ids"].tolist()) - set(miss.tolist()))
            near_tie_swaps += int(ok)
            dense_ok &= bool(ok)
        dense_ok &= diff <= DENSE_TOL
        # fusion at full size: the oracle's RRF over the lists the GPU produced must equal the GPU's fused list
        r_ids, r_sc = ref.ort.rrf_ids([s_ids[i, :c], g], None, K=60, topk=k)
        fc = int(f_cnt[i])
        r_ok = fc == r_ids.size and np.array_equal(f_ids[i, :fc], r_ids) and f_sc[i, :fc].tobytes() == r_sc.tobytes()
        rrf_ok += r_ok
        ident = b_ok and same
        lists_identical += ident
        if ident and r_ok:
            assert np.array_equal(r_ids, o["fused_ids"])
        if first_bad is None and not (b_ok and r_ok):
            first_bad = i
    res = {"queries": nq, "corpus_rows": ref.n, "bm25_bit_exact": bm25_ok == nq, "bm25_queries_bit_exact": int(bm25_ok),
           "dense_max_abs": dense_max_abs, "dense_tol": DENSE_TOL, "dense_within_tol": bool(dense_ok),
           "dense_ids_equal": int(dense_ids_equal), "dense_near_tie_swaps": int(near_tie_swaps),
           "rrf_equal": rrf_ok == nq, "fused_lists_identical_to_oracle": int(lists_identical),
           "ties_in_or_straddling_topk": {"bm25": int(sum(o["bm25_tie"] for o in ora)),
                                          "dense": int(sum(o["dense_tie"] for o in ora))},
           "oracle": "oracle port (numpy BM25Okapi restatement, fp32 BLAS cosine, Python RRF), canonical tie order"}
    res["ok"] = bool(res["bm25_bit_exact"] and res["dense_within_tol"] and res["rrf_equal"])
    if first_bad is not None:
        res["first_bad_query"] = int(first_bad)
    return res


def fused_digest(fused) -> str:
    """sha256 over (counts, ids, float64 score bits) of every fused list of the step."""
    h = hashlib.sha256()
    for t in (fused.counts, fused.ids, fused.scores):
        h.update(np.ascontiguousarray(t.cpu().numpy()).tobytes())
    return h.hexdigest()


DUMP_CAP_BYTES = 64 << 20


def dump_outputs(out_dir, routes) -> None:
    """Writes (scores, ids, counts) of the fused / sparse / dense lists as float64 .npy files; list entries past a
    query's count are set to id -1 and score 0 so that two runs compare element for element.  All query rows are
    written while the files stay within 64 MB in all; above that, a fixed seeded sample of rows (sorted).
    ``query_rows.npy`` holds the query index of every written row."""
    torch.cuda.synchronize()
    d = Path(out_dir)
    d.mkdir(parents=True, exist_ok=True)
    nq = int(routes[0].ids.shape[0])
    row_bytes = 8 * (1 + sum(2 * int(t.ids.shape[1]) + 1 for t in routes))     # float64 values per query row
    keep = min(nq, (DUMP_CAP_BYTES - 4096) // row_bytes)            # 4 KB for the ten .npy headers
    rows = np.arange(nq) if keep == nq else np.sort(np.random.default_rng(SEED).choice(nq, keep, replace=False))
    np.save(d / "query_rows.npy", rows.astype(np.float64))
    sel = torch.from_numpy(rows)
    for name, t in zip(("fused", "sparse", "dense"), routes):
        counts = t.counts.cpu()[sel].numpy().astype(np.int64)
        ids, sc = t.ids.cpu()[sel].numpy(), t.scores.cpu()[sel].numpy()
        valid = np.arange(ids.shape[1])[None, :] < counts[:, None]
        np.save(d / f"{name}_ids.npy", np.where(valid, ids, -1).astype(np.float64))
        np.save(d / f"{name}_scores.npy", np.where(valid, sc.astype(np.float64), 0.0))
        np.save(d / f"{name}_counts.npy", counts.astype(np.float64))


def digest_key(args) -> str:
    return f"rows={args.rows},dim={args.dim},vocab={args.vocab},queries={args.queries},k={args.k},seed={SEED}"


# ------------------------------------------------------------------------------ our arm
def algorithmic_bytes(args, data, index, n_rows_local):
    """Per-step algorithmic bytes of the two dominant kernels (DESIGN.md section 'Measurement')."""
    q = data["queries"]
    terms = q.terms.to(index.device).long()
    valid = (terms >= 0) & (terms < index.vocab)
    df = (index.indptr[1:] - index.indptr[:-1])
    postings = int(df[terms[valid]].sum())
    bm25 = postings * (4 + index.post_w.element_size()) + args.queries * args.k * 12
    # two-phase path: the candidate pass reads one packed 4-byte word per posting (+ the candidate ids it emits)
    bm25_cand = postings * 4 + args.queries * args.k * 4
    passes = -(-args.queries // 128)
    dense = passes * n_rows_local * args.dim * 2 + args.queries * args.dim * 2 + args.queries * args.k * 8
    return {"bm25_score": bm25, "bm25_cand": bm25_cand, "dense_tc": dense, "postings_per_step": postings,
            "dense_passes": passes}


PROF_NAMES = ("bm25_cand", "bm25_rescore", "bm25_score", "dense_tc", "dense_simt", "merge", "fuse")


def run_ours(args):
    import torch.distributed as dist
    from easyrag_b200 import _lib, batched
    from easyrag_b200 import dist as ezdist
    from easyrag_b200.index import Bm25Index, DenseIndex

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if world != args.gpus:
        raise SystemExit(f"--gpus {args.gpus} but WORLD_SIZE={world}: launch with torch.distributed.run")
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("nccl", device_id=dev)
    _lib.require_cuda()
    L = _lib.lib()
    small_batch = args.queries <= 512
    overlap = bool(args.overlap)
    serial_routes = bool(args.serial_routes) and overlap and bool(args.pipeline)
    stage_cap = args.dense_stages
    l2_flush = bool(args.l2_flush) if args.l2_flush >= 0 else small_batch
    _lib.check(L.ezr_dense_set_kernel(args.dense_kernel))
    _lib.check(L.ezr_dense_set_stage_cap(stage_cap))
    _lib.check(L.ezr_dense_set_probe(args.dense_probe))
    _lib.check(L.ezr_bm25_set_skipping(args.bm25_skip))
    _lib.check(L.ezr_bm25_set_plan(args.bm25_plan))
    _lib.check(L.ezr_bm25_set_span(args.bm25_span))

    data = make_data(args, dev)
    lo, hi = ezdist.shard_bounds(args.rows, world, rank, align=64)
    t0 = time.time()
    sparse = Bm25Index(data["stats"], device=dev, doc_lo=lo, doc_hi=hi)
    dense = DenseIndex(data["vec"][lo:hi], device=dev, row_lo=lo)
    torch.cuda.synchronize()
    build_s = time.time() - t0
    ranker = batched.CoarseRanker(dense, sparse, canon=None, overlap=overlap, serial_routes=serial_routes)
    ranker_seq = batched.CoarseRanker(dense, sparse, canon=None, overlap=False)       # calibration: one stream
    sharded = ezdist.ShardedCoarseRanker(ranker) if world > 1 else None
    sharded_seq = ezdist.ShardedCoarseRanker(ranker_seq) if world > 1 else None
    k = args.k
    q = data["queries"]
    d_qvec = data["qvec"].contiguous()
    d_ptr, d_terms = q.term_ptr.to(dev), q.terms.to(dev)
    h_qvec = d_qvec.cpu().pin_memory()
    h_ptr, h_terms = q.term_ptr.cpu().pin_memory(), q.terms.cpu().pin_memory()
    h_ids = torch.empty(args.queries, k, dtype=torch.int32).pin_memory()
    h_sc = torch.empty(args.queries, k, dtype=torch.float64).pin_memory()
    pipe = batched.HostPipeline(sharded if sharded is not None else ranker, args.queries, args.dim,
                                int(h_terms.numel()), k, k, pipelined=bool(args.pipeline) and overlap)

    def hybrid(r, s, qv, qp, qt):
        if s is not None:
            return s.hybrid(qv, qp, qt, k=k, k_out=k)
        return r.hybrid(qv, qp, qt, k, k, k)

    pipelined = bool(args.pipeline) and overlap
    top = sharded if sharded is not None else ranker

    last_step = {}          # (fused, sparse, dense) of the most recent step_device(): what --dump-outputs writes

    def step_device():
        if pipelined:
            t = top.submit(d_qvec, d_ptr, d_terms, k=k, k_out=k)
            last_step["out"] = (t.fused, t.sparse, t.dense)
            return t
        out = hybrid(ranker, sharded, d_qvec, d_ptr, d_terms)
        last_step["out"] = out
        return out[0]

    def step_cal():
        return hybrid(ranker_seq, sharded_seq, d_qvec, d_ptr, d_terms)[0]

    def step_e2e():
        pipe.step(h_qvec, h_ptr, h_terms, h_ids, h_sc)

    flush_buf = torch.empty(512 << 20, dtype=torch.uint8, device=dev) if l2_flush else None

    def timed(fn, steps, drain=None):
        """K steps bracketed by barrier + synchronize, max over ranks.  With --l2-flush every step is timed on its
        own (CUDA events around it) and a 512 MB write between steps evicts the L2; the sum of the steps counts."""
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()
        if flush_buf is None:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(steps):
                fn()
            if drain is not None:
                drain()
            b.record()
            torch.cuda.synchronize()
            per = None
            total = a.elapsed_time(b)
        else:
            evs = []
            for _ in range(steps):
                flush_buf.fill_(1)
                if world > 1:
                    dist.barrier()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                fn()
                if drain is not None:
                    drain()
                b.record()
                evs.append((a, b))
            torch.cuda.synchronize()
            per = [x.elapsed_time(y) for x, y in evs]
            total = sum(per)
        ms = torch.tensor([total], device=dev)
        if world > 1:
            dist.barrier()
            dist.all_reduce(ms, op=dist.ReduceOp.MAX)
        return float(ms.item()), per

    def read_prof():
        return {name: _lib.profile_read(name) for name in PROF_NAMES}

    sampler = ClockSampler(local)
    if rank == 0:
        sampler.start()
    n_warm = max(args.warmup, 3)
    for _ in range(n_warm):
        step_cal()
        step_device()
    top.join()
    torch.cuda.synchronize()
    # ---- calibration: the routes back to back on one stream, per-kernel CUDA events (roofline durations)
    _lib.check(L.ezr_profile_reset())
    _lib.check(L.ezr_profile_enable(1))
    ms_cal, _ = timed(step_cal, max(args.cal_steps, 1))
    prof = read_prof()
    dense_kernel_name = L.ezr_dense_last_kernel().decode()
    # the one collective on its own (scaling_terms.all_gather_ms): the exchange record of a step, 10 launches
    ag_ms, rec_bytes = None, None
    if sharded is not None:
        st_ = sharded._buffers(args.queries, k, sparse.score_dtype)
        rec_bytes = int(st_["layout"].nbytes)
        dist.all_gather_into_tensor(st_["gathered"], st_["record"])
        torch.cuda.synchronize()
        ea, eb = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        dist.barrier()
        ea.record()
        for _ in range(10):
            dist.all_gather_into_tensor(st_["gathered"], st_["record"])
        eb.record()
        torch.cuda.synchronize()
        ag_ms = ea.elapsed_time(eb) / 10
    # ---- timed region 1: device-resident inputs, product path
    _lib.check(L.ezr_profile_reset())
    launches0 = L.ezr_launch_count()
    sampler.begin()
    ms, per_step = timed(step_device, args.steps, drain=top.join)
    sampler.end()
    launches_timed = L.ezr_launch_count() - launches0
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, last_step["out"])      # before later submits reuse the result buffers
    prof_timed = read_prof()
    _lib.check(L.ezr_profile_enable(0))
    last = hybrid(ranker, sharded, d_qvec, d_ptr, d_terms)      # results of the measured configuration, all queries
    torch.cuda.synchronize()
    digest = fused_digest(last[0])
    hi_ = hashlib.sha256()                                      # what the digest was computed FROM
    for t in (q.term_ptr, q.terms, d_qvec.view(torch.int16)):
        hi_.update(np.ascontiguousarray(t.cpu().numpy()).tobytes())
    hi_.update(str((int(data["vec"].view(torch.int16).to(torch.int64).sum()), data["n_tokens"],
                    int(data["stats"].post_doc.to(torch.int64).sum()))).encode())
    inputs_sha = hi_.hexdigest()
    # ---- timed region 2: host buffers in, host buffers out, through the public pipeline API
    for _ in range(2):
        step_e2e()
    pipe.drain()
    sampler.begin()
    ms_e2e, per_step_e2e = timed(step_e2e, args.steps, drain=pipe.drain)
    sampler.end()
    clocks = sampler.stop() if rank == 0 else None
    # what the host-buffer API delivered must be what the device path computed
    e2e_digest_ok = bool(np.array_equal(h_ids.numpy(), last[0].ids.cpu().numpy())
                         and h_sc.numpy().tobytes() == last[0].scores.cpu().numpy().tobytes())

    # ---- full-size parity against the CPU oracle (outside the timed regions; every rank joins the GPU call)
    parity, ref = None, None
    if args.parity_queries > 0 and args.dense_probe == 0:
        nq = min(args.parity_queries, args.queries)
        qp = q.term_ptr[:nq + 1].to(dev)
        f, s, d = hybrid(ranker, sharded, d_qvec[:nq], qp, d_terms)
        torch.cuda.synchronize()
        if rank == 0:
            ref = CpuReference(data, args)
            parity = parity_full_size(ref, nq, f, s, d, k)

    # Full-size property check: the two-phase path (integer candidates + exact rescoring) and the ordered float64
    # kernel are independent implementations; on this shard they must return the same ids, scores and counts.
    self_check = None
    if args.self_check > 0 and sparse.post_pk is not None and args.dense_probe == 0:
        nq = min(args.self_check, args.queries)
        qp = q.term_ptr[:nq + 1].to(dev)
        a = batched.bm25_topk(sparse, qp, d_terms, k)
        b = batched.bm25_topk(sparse.ordered_view(), qp, d_terms, k)
        torch.cuda.synchronize()
        same = bool(torch.equal(a.ids, b.ids) and torch.equal(a.counts, b.counts)
                    and torch.equal(a.scores.view(torch.int64), b.scores.view(torch.int64)))
        self_check = {"bm25_two_phase_equals_ordered": same, "queries": nq, "postings_local": sparse.n_postings}
        if not same:
            raise SystemExit(f"bench.py self-check FAILED on rank {rank}: BM25 kernel paths disagree")
    # ---- configs[1]: the chunk-embedding forward pass (every rank encodes its share of the chunks)
    encode = None
    if rank == 0 and world == 1 and not args.no_cpu and ref is None:
        ref = CpuReference(data, args)                  # host copies for the cpu_baseline leg, before HBM is freed
    if args.enc_chunks > 0 and args.dense_probe == 0 and not small_batch:
        import bench_encode
        index_bytes = sparse.index_bytes()
        postings_local, n_rows_local = sparse.n_postings, dense.n_rows
        alg = algorithmic_bytes(args, data, sparse, dense.n_rows)
        del ranker, ranker_seq, sharded, sharded_seq, pipe, sparse, dense, last, flush_buf
        data["vec"] = data["qvec"] = None
        torch.cuda.empty_cache()
        encode = bench_encode.encode_block(dev, "bert", args.enc_chunks, 1000, 512, 12, 768, 3, rank, world)
    else:
        index_bytes = sparse.index_bytes()
        postings_local, n_rows_local = sparse.n_postings, dense.n_rows
        alg = algorithmic_bytes(args, data, sparse, dense.n_rows)
    if rank != 0:
        if world > 1:
            dist.barrier()
            dist.destroy_process_group()
        return

    peaks = {}
    pk_file = ROOT / "MEASURED_PEAKS.json"
    if pk_file.exists():
        peaks = json.loads(pk_file.read_text())
    hbm_peak = float(peaks.get("hbm_gbs", 3350.0))
    peak_src = "measured (MEASURED_PEAKS.json hbm_gbs)" if "hbm_gbs" in peaks else "H100 SXM data sheet 3350 GB/s"
    long_step = ms > 2000.0          # a seconds-long loop settles at the sustained clock
    tf_key = "bf16_tflops_sustained" if long_step else "bf16_tflops"
    tf_peak = float(peaks.get(tf_key, 989.0))                   # H100 SXM data sheet, dense bf16
    tf_src = (f"measured (MEASURED_PEAKS.json {tf_key}: "
              + ("kernel timed inside a seconds-long loop)" if long_step else "burst figure, the timed loop lasts well under 2 s)")
              if tf_key in peaks else "H100 SXM data sheet 989 TFLOP/s")
    dense_flops = 2.0 * n_rows_local * args.dim * args.queries          # per launch: every query x every local row
    kernels = {}
    two_phase = prof["bm25_cand"][1] > 0
    for name in ("bm25_cand", "bm25_score", "dense_tc"):
        tot, n = prof[name]
        if n and not (name == "bm25_score" and two_phase):     # two-phase: bm25_score only sees overflowed queries
            avg_ms = tot / n
            kernels[name] = {"launches": n, "avg_ms": avg_ms, "alg_bytes_per_launch": alg[name],
                             "GBps": alg[name] / (avg_ms * 1e-3) / 1e9}
            t2, n2 = prof_timed[name]
            if n2:
                kernels[name]["avg_ms_in_timed_region"] = t2 / n2       # routes co-resident: includes the other route's share
    others = {name: {"launches": prof[name][1], "avg_ms": prof[name][0] / prof[name][1]}
              for name in ("bm25_rescore", "bm25_score", "merge", "fuse") if prof[name][1] and name not in kernels}
    if "dense_tc" in kernels:
        kernels["dense_tc"]["flops_per_launch"] = dense_flops
        kernels["dense_tc"]["TFLOPs"] = dense_flops / (kernels["dense_tc"]["avg_ms"] * 1e-3) / 1e12
        kernels["dense_tc"]["queries_per_corpus_pass"] = min(args.queries, 128)
    dom = max(kernels, key=lambda n_: kernels[n_]["avg_ms"]) if kernels else None
    timing_note = (f"per-kernel durations: CUDA events on the launch stream over {max(args.cal_steps, 1)} calibration "
                   f"steps with the two routes back to back on one stream (same kernels, same launch shapes as the "
                   f"timed region); avg_ms_in_timed_region = the same events over the {args.steps} timed steps"
                   + (", where the routes share the SMs" if overlap else ""))
    roofline = None
    # SURVEY.md 8(d): the dense scan is HBM-bound while queries per corpus pass stay below the H100 ridge
    # (989 TFLOP/s / 3.35 TB/s, about 295 flop/byte)
    dense_hbm_bound = args.queries <= 295
    if dom == "dense_tc" and not dense_hbm_bound:
        roofline = {"bound": "tensor", "kernel": dom, "achieved": kernels[dom]["TFLOPs"], "peak": tf_peak,
                    "unit": "TFLOP/s", "frac": kernels[dom]["TFLOPs"] / tf_peak,
                    "peak_source": tf_src, "timing": timing_note, "kernels": kernels}
    elif dom:
        note = {"dense_tc": "algorithmic bytes = one pass over the corpus shard (N_s x D x 2) + queries + outputs "
                            "(SURVEY.md 8(d)); B = queries per pass is in config",
                "bm25_cand": "algorithmic bytes = postings touched (4 B packed word each) + candidate ids",
                "bm25_score": "algorithmic bytes = postings touched (12 B each) + outputs"}[dom]
        roofline = {"bound": "hbm", "kernel": dom, "achieved": kernels[dom]["GBps"], "peak": hbm_peak, "unit": "GB/s",
                    "frac": kernels[dom]["GBps"] / hbm_peak, "peak_source": peak_src,
                    "timing": timing_note, "kernels": kernels, "note": note}
    if roofline:
        roofline["other_kernels"] = others
    value = args.steps * args.queries / (ms * 1e-3)
    e2e_v = args.steps * args.queries / (ms_e2e * 1e-3)
    h2d = h_qvec.numel() * 2 + h_ptr.numel() * 4 + h_terms.numel() * 4
    d2h = h_ids.numel() * 4 + h_sc.numel() * 8
    cpu = None
    if world == 1 and not args.no_cpu:
        v, dt = ref.measure(args.cpu_queries, steps=1, warmup=0 if parity is not None else 1)
        cpu = {"value": v, "unit": "queries/s", "cores": ref.cores, "kind": "port",
               "sample": f"first {min(args.cpu_queries, args.queries)} of the {args.queries} queries over the full "
                         f"{args.rows} x {args.dim} corpus, 1 step of {dt:.1f} s after a warm-up pass; numpy BM25Okapi "
                         f"restatement + full argsort, fp32 BLAS cosine, Python RRF"}
    # digest of every fused list of the step: identical for every N (configs[3]: "must equal C3 bit-for-bit")
    dig = {"fused_sha256": digest, "inputs_sha256": inputs_sha, "key": digest_key(args),
           "e2e_results_equal_device_results": e2e_digest_ok, "matches_committed_n1": None}
    if DIGEST_FILE.exists():
        want = json.loads(DIGEST_FILE.read_text()).get(dig["key"])
        if want is not None and want.get("inputs_sha256") == inputs_sha:
            # same synthetic inputs (same generator stream on this box) -> the fused lists must be the committed ones
            dig["matches_committed_n1"] = bool(want["fused_sha256"] == digest)
            dig["committed_from"] = want.get("from")
        elif want is not None:
            dig["note"] = "the committed digest was taken on different synthetic inputs (generator stream differs); not compared"
    max_rows = max(b - a for a, b in (ezdist.shard_bounds(args.rows, world, r, align=64) for r in range(world)))
    step_ms = ms / args.steps
    seq_ms = ms_cal / max(args.cal_steps, 1)
    scaling_terms = {
        "max_shard_rows": max_rows, "ideal_shard_rows": args.rows / world, "imbalance": max_rows / (args.rows / world),
        "dense_TFLOPs": kernels.get("dense_tc", {}).get("TFLOPs"), "dense_ms": kernels.get("dense_tc", {}).get("avg_ms"),
        "bm25_cand_ms": kernels.get("bm25_cand", {}).get("avg_ms"),
        "fixed_ms": seq_ms - sum(kernels[n_]["avg_ms"] for n_ in kernels),
        "sequential_step_ms": seq_ms, "overlapped_step_ms": step_ms, "all_gather_ms": ag_ms,
        "record_bytes_per_rank": rec_bytes,
        "note": "fixed_ms = one-stream step minus dense and candidate kernels (rescore, merges, fusion, all-gather, gaps); "
                "compare the terms across N: imbalance -> 1.0 is balanced, dense_TFLOPs falling = shorter units per CTA"}
    line = {
        "metric": METRIC, "value": value, "unit": "queries/s", "n_gpus": world, "steps": args.steps,
        "warmup": n_warm, "ms_per_step": step_ms, "higher_is_better": True,
        "scaling": "strong", "vs_baseline": None, "dtype": "bf16 dense / f64 bm25", "data": "synthetic",
        "config": {"workload": (f"configs[4] shape: {args.rows} x {args.dim} chunks (BGE-large width) + BM25 + RRF top-{k}, "
                                f"batch-{args.queries} queries"
                                if args.rows >= 4_000_000 and args.dim == 1024 else
                                f"configs[2]: dense+BM25 dual-route + RRF top-{k}, {args.rows} x {args.dim} chunks, "
                                f"{args.queries} queries/step")
                               + (f", row-sharded over {world} GPUs" + (" (configs[3])" if args.rows < 4_000_000 else "")
                                  if world > 1 else ""),
                   "rows": args.rows, "dim": args.dim, "vocab": args.vocab, "queries_per_step": args.queries,
                   "k": k, "rrf_K": 60, "tokens": data["n_tokens"], "postings_local": postings_local,
                   "queries_per_corpus_pass": min(args.queries, 128), "routes_overlapped": overlap,
                   "steps_pipelined": pipelined, "routes_serial_on_side_stream": serial_routes,
                   "dense_ring_stages_cap": stage_cap, "timed_region_starts_from": "query vectors + term ids",
                   "l2": ("explicit flush: 512 MB written between steps, every step timed on its own" if l2_flush else
                          "inputs larger than L2 (corpus shard and postings >> 50 MB), no explicit flush"),
                   "parallelism": f"rows{world}"},
        "e2e": {"value": e2e_v, "unit": "queries/s", "h2d_bytes_per_step": h2d, "d2h_bytes_per_step": d2h,
                "ms_per_step": ms_e2e / args.steps,
                "api": "batched.HostPipeline.step: pinned host inputs -> H2D -> both routes -> (all-gather, merge) -> "
                       "RRF -> D2H into pinned host outputs, every step; copies of step i+1 overlap the kernels of step i"},
        "gpu_launches": int(launches_timed),
        "clocks": clocks, "roofline": roofline, "cpu_baseline": cpu,
        "parity_full_size": parity, "digest": dig, "scaling_terms": scaling_terms, "encode": encode,
        "setup": {"generate_s": round(data["gen_s"], 1), "index_build_s": round(build_s, 1),
                  "index_bytes": index_bytes, "dense_kernel": dense_kernel_name,
                  "self_check": self_check},
    }
    if per_step is not None:
        line["latency_ms"] = {"median": statistics.median(per_step), "min": min(per_step), "max": max(per_step),
                              "e2e_median": statistics.median(per_step_e2e) if per_step_e2e else None}
    print(json.dumps(line))
    sys.stdout.flush()
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()
    if parity is not None and not parity["ok"]:
        raise SystemExit(f"bench.py parity_full_size FAILED: {json.dumps(parity)}")
    if dig["matches_committed_n1"] is False:
        raise SystemExit(f"bench.py digest differs from the committed N=1 digest: {json.dumps(dig)}")


def run_reference(args):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", "0")))     # data generation only
    data = make_data(args, dev)
    ref = CpuReference(data, args)
    n = min(args.ref_queries, args.queries)
    v, dt = ref.measure(n, steps=args.steps, warmup=args.warmup)
    sample = (f"each step = first {n} of the {args.queries} queries over the full {args.rows} x {args.dim} corpus; "
              f"numpy BM25Okapi restatement + full argsort, fp32 BLAS cosine ({ref.cores} threads), Python RRF")
    line = {
        "impl": "reference", "metric": METRIC, "value": v, "unit": "queries/s", "n_gpus": args.gpus,
        "steps": args.steps, "warmup": args.warmup, "ms_per_step": dt * 1e3, "higher_is_better": True,
        "scaling": "strong", "vs_baseline": None, "dtype": "f32 dense / f64 bm25", "data": "synthetic",
        "config": {"workload": f"configs[2]: dense+BM25 dual-route + RRF top-{args.k}, {args.rows} x {args.dim} chunks "
                               f"(bounded query sample)",
                   "rows": args.rows, "dim": args.dim, "vocab": args.vocab, "queries_per_step": n, "k": args.k},
        "cpu_baseline": {"value": v, "unit": "queries/s", "cores": ref.cores, "kind": "port", "sample": sample},
        "e2e": {"value": v, "unit": "queries/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
        "gpu_launches": 0,
    }
    print(json.dumps(line))


if __name__ == "__main__":
    a = parse()
    if a.workload == "encode":
        import bench_encode
        bench_encode.main(from_bench=a)
    elif a.impl == "reference":
        run_reference(a)
    else:
        run_ours(a)
