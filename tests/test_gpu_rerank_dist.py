"""GPU: cross-encoder reranking with the pairs split across ranks (ShardedCrossEncoderReranker).

The two-launch head (ezr_cross_pair_scores + ezr_cross_order_topk) against the fused ezr_cross_score_topk, and the
sharded reranker against the one-GPU CrossEncoderReranker: with no process group, with a one-rank NCCL group, with two
ranks over gloo sharing one GPU (the split, the exchange and the input check run for real on a one-GPU machine) and
with two ranks over NCCL on two GPUs.  Every comparison is bit for bit.
"""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from easyrag_b200 import _lib
from easyrag_b200.batched import TopK

pytestmark = pytest.mark.gpu
DEV = "cuda"
SPECIAL = {"bert": dict(cls_id=2, sep_id=3, pad_id=0), "roberta": dict(cls_id=0, sep_id=2, pad_id=1)}


@pytest.fixture(scope="module", autouse=True)
def _ready(lib_built):
    _lib.require_cuda()


def _bits(t):
    return t.contiguous().view(torch.int32).cpu()


def _same(a, b):
    """(TopK, all_scores) pairs equal bit for bit."""
    (ta, sa), (tb, sb) = a, b
    return (torch.equal(ta.ids, tb.ids) and torch.equal(ta.counts, tb.counts)
            and torch.equal(_bits(ta.scores), _bits(tb.scores)) and torch.equal(_bits(sa), _bits(sb)))


# ------------------------------------------------------------------------------------------------- kernels
def _head_case(d, seed):
    """Dense head rows for 7 queries at k = 192 (full, short and empty lists), with exact ties and sigmoids that
    saturate to exactly 1.0f and 0.0f."""
    g = torch.Generator().manual_seed(seed)
    counts = [192, 1, 0, 5, 192, 37, 191]
    n_pairs = sum(counts)
    w = torch.randn(d, generator=g) * 0.2
    dense = (torch.randn(n_pairs, d, generator=g) * 0.5).to(torch.bfloat16)
    for p in range(0, n_pairs, 11):
        dense[p] = (torch.sign(w) * 3).to(torch.bfloat16)         # logit ~ +130: sigmoid == 1.0f
    for p in range(5, n_pairs, 13):
        dense[p] = (-torch.sign(w) * 3).to(torch.bfloat16)        # logit ~ -130: sigmoid == +0.0f
    for p in range(3, n_pairs - 2, 17):
        dense[p + 2] = dense[p]                                   # an exact tie two ranks apart
    k, k_stride = 192, 200
    ids = torch.full((len(counts), k_stride), -1, dtype=torch.int32)
    for q, c in enumerate(counts):
        ids[q, :c] = torch.randperm(5000, generator=g)[:c].to(torch.int32)
    pair_off = torch.tensor(np.concatenate([[0], np.cumsum(counts)]), dtype=torch.int32)
    return (dense.to(DEV), w.to(DEV), 0.25, pair_off.to(DEV), ids.to(DEV), len(counts), k)


def _outputs(nq, k, top_n):
    return (torch.empty(nq, k, device=DEV), torch.empty(nq, top_n, device=DEV),
            torch.empty(nq, top_n, dtype=torch.int32, device=DEV), torch.empty(nq, dtype=torch.int32, device=DEV))


@pytest.mark.parametrize("d", [768, 1024], ids=["bert-base-head", "xlmr-large-head"])
@pytest.mark.parametrize("top_n", [6, 192, 250])
def test_two_launch_head_equals_the_fused_kernel(d, top_n):
    L, st = _lib.lib(), _lib.stream_ptr()
    dense, w, b, pair_off, ids, nq, k = _head_case(d, 100 + d + top_n)
    n_pairs = dense.shape[0]
    a_all, a_sc, a_ids, a_cnt = _outputs(nq, k, top_n)
    _lib.check(L.ezr_cross_score_topk(_lib.ptr(dense), d, _lib.ptr(pair_off), nq, k, _lib.ptr(ids), ids.stride(0),
                                      _lib.ptr(w), b, d, top_n, _lib.ptr(a_all), _lib.ptr(a_sc), _lib.ptr(a_ids),
                                      _lib.ptr(a_cnt), st))
    # scored in three runs as three ranks would (one of them empty), each into its slice of one buffer
    sig = torch.zeros(n_pairs, device=DEV)
    for lo, hi in ((0, 300), (300, 300), (300, n_pairs)):
        _lib.check(L.ezr_cross_pair_scores(_lib.ptr(dense[lo:]), d, hi - lo, _lib.ptr(w), b, _lib.ptr(sig[lo:]), st))
    b_all, b_sc, b_ids, b_cnt = _outputs(nq, k, top_n)
    _lib.check(L.ezr_cross_order_topk(_lib.ptr(sig), _lib.ptr(pair_off), nq, k, _lib.ptr(ids), ids.stride(0), top_n,
                                      _lib.ptr(b_all), _lib.ptr(b_sc), _lib.ptr(b_ids), _lib.ptr(b_cnt), st))
    torch.cuda.synchronize()
    assert torch.equal(a_ids, b_ids) and torch.equal(a_cnt, b_cnt)
    assert torch.equal(_bits(a_sc), _bits(b_sc)) and torch.equal(_bits(a_all), _bits(b_all))
    # the case covers what it claims: saturated scores on both ends, sorted ties, short and empty lists
    assert int((sig == 1.0).sum()) >= 30 and int((sig == 0.0).sum()) >= 30
    assert not torch.signbit(sig).any()
    assert a_cnt.cpu().tolist() == [min(c, top_n) for c in (192, 1, 0, 5, 192, 37, 191)]
    row = a_all[0].cpu()
    assert row[3] == row[5] and row[0] == 1.0
    assert torch.isneginf(a_all[1, 1:]).all() and torch.isneginf(a_all[2]).all()


def test_two_launch_head_rejects_bad_arguments():
    L, st = _lib.lib(), _lib.stream_ptr()
    assert L.ezr_cross_pair_scores(None, 0, 4, None, 0.0, None, st) != 0
    assert b"cross_pair_scores" in L.ezr_last_error()
    assert L.ezr_cross_pair_scores(None, 768, 0, None, 0.0, None, st) == 0           # nothing to score
    assert L.ezr_cross_order_topk(None, None, 1, 1025, None, 1025, 6, None, None, None, None, st) != 0
    assert b"cross_order_topk" in L.ezr_last_error()


# ------------------------------------------------------------------------------------------ sharded reranker
def _model(family, d=256, layers=2, vocab=800, seed=7):
    from easyrag_b200.encoder import BertConfig
    from easyrag_b200.rerank import CrossEncoderModel, random_cross_encoder_state
    cfg = BertConfig(vocab_size=vocab, hidden_size=d, intermediate_size=4 * d, num_hidden_layers=layers,
                     num_attention_heads=d // 64, max_position_embeddings=514 if family == "roberta" else 512,
                     layer_norm_eps=1e-5 if family == "roberta" else 1e-12)
    return CrossEncoderModel(family, cfg, random_cross_encoder_state(family, cfg, seed, std=0.03), device=DEV,
                             **SPECIAL[family])


def _inputs(seed, n_docs, counts, k, vocab):
    rng = np.random.default_rng(seed)
    passages = [rng.integers(4, vocab, int(n)).tolist() for n in rng.integers(0, 600, n_docs)]
    queries = [rng.integers(4, vocab, int(n)).tolist() for n in rng.integers(1, 60, len(counts))]
    ids = np.full((len(counts), k), -1, np.int32)
    for q, c in enumerate(counts):
        ids[q, :c] = rng.choice(n_docs, c, replace=False)
        if c >= 4:
            ids[q, 3] = ids[q, 1]                              # an exact tie
    cand = TopK(torch.zeros(len(counts), k, device=DEV), torch.from_numpy(ids).to(DEV),
                torch.tensor(counts, dtype=torch.int32, device=DEV))
    q_ptr = torch.tensor(np.cumsum([0] + [len(q) for q in queries]), dtype=torch.int32, device=DEV)
    q_tok = torch.tensor([t for q in queries for t in q], dtype=torch.int32, device=DEV)
    return passages, cand, q_ptr, q_tok


@pytest.mark.parametrize("family", ["bert", "roberta"])
def test_without_a_process_group_equals_one_gpu(family):
    from easyrag_b200.dist import ShardedCrossEncoderReranker
    from easyrag_b200.rerank import CrossEncoderReranker
    assert not dist.is_initialized()
    model = _model(family, d=768 if family == "bert" else 1024, vocab=3000)
    passages, cand, q_ptr, q_tok = _inputs(31, 150, [40, 0, 13, 40, 1], 40, 3000)
    rr = CrossEncoderReranker(model, passages, max_tokens=2048)
    sh = ShardedCrossEncoderReranker(rr)
    assert (sh.world, sh.rank) == (1, 0)
    for top_n in (6, 40):
        assert _same(sh.rerank(cand, q_ptr, q_tok, top_n), rr.rerank(cand, q_ptr, q_tok, top_n))


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, backend, port, ret):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    gpu = rank if backend == "nccl" else 0               # gloo: every rank on the one GPU
    torch.cuda.set_device(gpu)
    dev = torch.device("cuda", gpu)
    if backend == "nccl":
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    else:
        dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from easyrag_b200 import batched, synth
        from easyrag_b200 import dist as ezdist
        from easyrag_b200.index import Bm25Index, Bm25Stats, DenseIndex
        from easyrag_b200.rerank import CrossEncoderReranker
        fails = []

        def expect(name, a, b):
            if not _same(a, b):
                fails.append(name)

        # a coarse result with short lists: a 24-document corpus asked for k = 32
        n, vocab, dim, nq = 24, 300, 128, 6
        corpus = synth.make_sparse_corpus(n, vocab, 1)
        qs = synth.make_queries(corpus, nq, 2)
        g = torch.Generator().manual_seed(4)
        c = torch.randn(n, dim, generator=g).to(torch.bfloat16)
        qv = torch.randn(nq, dim, generator=g).to(torch.bfloat16).to(dev)
        stats = Bm25Stats.from_tokens(corpus.tokens, corpus.doc_ptr, vocab)
        args = (qv, qs.term_ptr.to(dev), qs.terms.to(dev))
        if backend == "nccl":                           # the product pairing: the row-sharded coarse ranker's output
            lo, hi = ezdist.shard_bounds(n, world, rank)
            coarse = ezdist.ShardedCoarseRanker(batched.CoarseRanker(
                DenseIndex(c[lo:hi], device=dev, row_lo=lo), Bm25Index(stats, device=dev, doc_lo=lo, doc_hi=hi)))
            fused, _, _ = coarse.hybrid(*args, k=32, k_out=32, K=60)
        else:
            coarse = batched.CoarseRanker(DenseIndex(c, device=dev), Bm25Index(stats, device=dev))
            fused, _, _ = coarse.hybrid(*args, 32, 32, 32, 60)
        cnt = fused.counts.cpu().numpy()
        if not np.all((cnt > 0) & (cnt < 32)):
            fails.append("coarse lists are not short")

        model = _model("roberta", vocab=800)
        rng = np.random.default_rng(41)
        passages = [rng.integers(4, 800, int(x)).tolist() for x in rng.integers(5, 300, n)]
        queries = [rng.integers(4, 800, int(x)).tolist() for x in rng.integers(3, 30, nq)]
        q_ptr = torch.tensor(np.cumsum([0] + [len(q) for q in queries]), dtype=torch.int32, device=dev)
        q_tok = torch.tensor([t for q in queries for t in q], dtype=torch.int32, device=dev)
        rr = CrossEncoderReranker(model, passages, max_tokens=1024)
        sh = ezdist.ShardedCrossEncoderReranker(rr)
        if (sh.world, sh.rank) != (world, rank):
            fails.append("world / rank")
        expect("hybrid", sh.rerank(fused, q_ptr, q_tok, 6), rr.rerank(fused, q_ptr, q_tok, 6))
        pairs = rr.pack(fused.ids, fused.counts, q_ptr, q_tok)
        runs = ezdist.token_balanced_ranges(pairs.cu_h, world)
        if world > 1 and any(hi == lo for lo, hi in runs):
            fails.append("a rank got no pairs in the main case")

        # fewer pairs than ranks, and no pairs at all
        big = CrossEncoderReranker(model, [rng.integers(4, 800, 200).tolist() for _ in range(20)])
        sh_big = ezdist.ShardedCrossEncoderReranker(big)
        for counts in ([1, 0, 0], [0, 0, 0]):
            ids = torch.full((3, 8), -1, dtype=torch.int32, device=dev)
            ids[0, 0] = 17
            cand = TopK(torch.zeros(3, 8, device=dev), ids, torch.tensor(counts, dtype=torch.int32, device=dev))
            p3 = torch.tensor([0, 5, 9, 12], dtype=torch.int32, device=dev)
            t3 = torch.arange(4, 16, dtype=torch.int32, device=dev)
            expect(f"counts {counts}", sh_big.rerank(cand, p3, t3, 4), big.rerank(cand, p3, t3, 4))

        # inputs that differ across ranks are refused on every rank, before any encoder work
        k_bad = 32 if rank == 0 else 31
        bad = TopK(fused.scores[:, :k_bad], fused.ids[:, :k_bad].contiguous(), fused.counts.clamp(max=k_bad))
        try:
            sh.rerank(bad, q_ptr, q_tok, 6)
            if world > 1:
                fails.append("mismatched inputs were accepted")
        except ValueError as e:
            if world == 1 or "differ across ranks" not in str(e):
                fails.append(f"unexpected error: {e}")
        torch.cuda.synchronize()
        ret[rank] = fails
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("backend,world", [
    pytest.param("nccl", 1, id="nccl-1"),
    pytest.param("gloo", 2, id="gloo-2-on-one-gpu"),
    pytest.param("nccl", 2, id="nccl-2", marks=pytest.mark.skipif(torch.cuda.device_count() < 2,
                                                                 reason="needs 2 GPUs")),
])
def test_sharded_reranker_equals_one_gpu(backend, world):
    mgr = mp.get_context("spawn").Manager()
    ret = mgr.dict()
    mp.spawn(_worker, args=(world, backend, _free_port(), ret), nprocs=world, join=True)
    assert dict(ret) == {r: [] for r in range(world)}
