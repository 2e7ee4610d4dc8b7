"""GPU, world_size 2, NCCL: the row-sharded path must return exactly the 1-GPU rank lists (SURVEY.md 8(e)).

Needs two GPUs; skipped on a single-GPU machine.
"""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, ret):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    try:
        from easyrag_b200 import batched, synth
        from easyrag_b200 import dist as ezdist
        from easyrag_b200.index import Bm25Index, Bm25Stats, DenseIndex
        n, vocab, dim, nq, k = 40_000, 8_000, 256, 300, 10
        corpus = synth.make_sparse_corpus(n, vocab, 5)
        queries = synth.make_queries(corpus, nq, 6)
        stats = Bm25Stats.from_tokens(corpus.tokens, corpus.doc_ptr, vocab)
        g = torch.Generator().manual_seed(7)
        vec = torch.randint(-2, 3, (n, dim), generator=g).to(torch.bfloat16)       # exact dot products
        qv = torch.randint(-2, 3, (nq, dim), generator=g).to(torch.bfloat16)
        canon = synth.make_duplicates(n, 0.03, 8)
        groups = synth.make_groups(n, 4, 9)
        want = torch.tensor([i % 5 - 1 for i in range(nq)], dtype=torch.int32)
        lo, hi = ezdist.shard_bounds(n, world, rank, align=8192)
        ranker = batched.CoarseRanker(DenseIndex(vec[lo:hi], device=dev, row_lo=lo, doc_group=groups[lo:hi]),
                                      Bm25Index(stats, device=dev, doc_lo=lo, doc_hi=hi, doc_group=groups), canon=canon)
        sharded = ezdist.ShardedCoarseRanker(ranker)
        args = (qv.to(dev), queries.term_ptr.to(dev), queries.terms.to(dev))
        ok = True
        for qg in (None, want):
            f, s, d = sharded.hybrid(*args, k=k, k_out=k, q_group=qg)
            torch.cuda.synchronize()
            if rank == 0:
                full = batched.CoarseRanker(DenseIndex(vec, device=dev, doc_group=groups),
                                            Bm25Index(stats, device=dev, doc_group=groups), canon=canon)
                f1, s1, d1 = full.hybrid(*args, k, k, k, q_group=qg)
                torch.cuda.synchronize()
                for a, b in ((f, f1), (s, s1), (d, d1)):
                    ok &= torch.equal(a.ids, b.ids) and torch.equal(a.counts, b.counts)
                    ok &= a.scores.cpu().numpy().tobytes() == b.scores.cpu().numpy().tobytes()
        # submitted (pipelined) batches: four different batches in flight over two result slots, never joined to the
        # caller's stream, must equal the joined path batch by batch
        ranker_o = batched.CoarseRanker(ranker.dense, ranker.sparse, canon=canon, overlap=True)
        sh_o = ezdist.ShardedCoarseRanker(ranker_o)
        qd = qv.to(dev)
        batches = [torch.roll(qd, 7 * i, 0).contiguous() for i in range(4)]
        want_f = []
        for b in batches:
            f, _, _ = sharded.hybrid(b, args[1], args[2], k=k, k_out=k)
            want_f.append((f.ids.clone(), f.scores.clone(), f.counts.clone()))
        torch.cuda.synchronize()
        side = torch.cuda.Stream(device=dev)
        got_f = []
        for b in batches:
            t = sh_o.submit(b, args[1], args[2], k=k, k_out=k)
            with torch.cuda.stream(side):
                t.wait(side)
                got_f.append((t.fused.ids.clone(), t.fused.scores.clone(), t.fused.counts.clone()))
                t.release(side)
        sh_o.join()
        torch.cuda.synchronize()
        for a, b in zip(got_f, want_f):
            ok &= all(torch.equal(x, y) for x, y in zip(a, b))
        ok &= not torch.equal(want_f[0][0], want_f[1][0])
        ret[rank] = bool(ok)
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpu_sharded_equals_single_gpu(lib_built):
    world = 2
    mgr = mp.get_context("spawn").Manager()
    ret = mgr.dict()
    mp.spawn(_worker, args=(world, _free_port(), ret), nprocs=world, join=True)
    assert dict(ret) == {0: True, 1: True}
