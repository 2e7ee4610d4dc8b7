"""GPU: rerank fusion (``CrossEncoderReranker.rerank_fusion``, pipeline.py:393-452).

``ezr_pair_union`` against the numpy union of oracle/rerank_fusion.py; ``ezr_cross_order_topk_mapped`` against
``ezr_cross_order_topk`` on each list alone; ``rerank_fusion`` against two ``rerank`` calls plus ``rrf_fuse`` (bit for
bit), on saturated scores and against the CPU oracle; the sharded form against one GPU.
"""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import rerank_fusion as orf
from oracle import retrieve as ort
from easyrag_b200 import _lib, batched, synth
from easyrag_b200.batched import TopK

pytestmark = pytest.mark.gpu
DEV = "cuda"
SPECIAL = {"bert": dict(cls_id=2, sep_id=3, pad_id=0), "roberta": dict(cls_id=0, sep_id=2, pad_id=1)}
K_SPARSE, K_DENSE = 192, 288          # pipeline.py's f_topk_2 / f_topk_1


@pytest.fixture(scope="module", autouse=True)
def _ready(lib_built):
    _lib.require_cuda()


def _bits(t):
    return t.contiguous().view(torch.int32).cpu() if t.element_size() == 4 else t.contiguous().view(torch.int64).cpu()


def _same_topk(a, b):
    return (torch.equal(a.ids.cpu(), b.ids.cpu()) and torch.equal(a.counts.cpu(), b.counts.cpu())
            and torch.equal(_bits(a.scores), _bits(b.scores)))


def _same(res, ref):
    """A RerankFusion against another one, bit for bit."""
    return (_same_topk(res.fused, ref.fused) and _same_topk(res.sparse, ref.sparse) and _same_topk(res.dense, ref.dense)
            and torch.equal(_bits(res.sparse_all), _bits(ref.sparse_all))
            and torch.equal(_bits(res.dense_all), _bits(ref.dense_all)) and res.n_pairs == ref.n_pairs)


def _routes(seed, nq, n_docs, overlap, k_s=K_SPARSE, k_d=K_DENSE, short=True):
    """Sparse [Q, k_s] and dense [Q, k_d] lists of distinct ids; ``overlap`` of each sparse list is drawn from the
    dense list of the same query.  ``short``: some lists are cut short, some emptied."""
    rng = np.random.default_rng(seed)
    ids_s = np.full((nq, k_s), -1, np.int32)
    ids_d = np.full((nq, k_d), -1, np.int32)
    n_shared = int(round(overlap * k_s))
    for q in range(nq):
        perm = rng.permutation(n_docs)
        ids_d[q] = perm[:k_d]
        s = np.concatenate([rng.choice(perm[:k_d], n_shared, replace=False), perm[k_d:k_d + k_s - n_shared]])
        ids_s[q] = rng.permutation(s)
    cnt_s, cnt_d = np.full(nq, k_s, np.int32), np.full(nq, k_d, np.int32)
    if short:
        cnt_s[3::7] = rng.integers(1, k_s, cnt_s[3::7].size)
        cnt_d[5::11] = rng.integers(1, k_d, cnt_d[5::11].size)
        cnt_s[6::13] = 0
        cnt_d[9::17] = 0
        ids_s[np.arange(k_s)[None] >= cnt_s[:, None]] = -1
        ids_d[np.arange(k_d)[None] >= cnt_d[:, None]] = -1
    return ids_s, cnt_s, ids_d, cnt_d


def _dev(*arrays):
    return [torch.from_numpy(np.ascontiguousarray(a)).to(DEV) for a in arrays]


def _check_union(ids_a, cnt_a, ids_b, cnt_b, **views):
    got = batched.pair_union(*_dev(ids_a, cnt_a, ids_b, cnt_b), **views)
    torch.cuda.synchronize()
    want = orf.pair_union(ids_a, cnt_a, ids_b, cnt_b)
    for name, g, w in zip(("ids", "counts", "map_a", "map_b"), (got.ids, got.counts, got.map_a, got.map_b), want):
        assert np.array_equal(g.cpu().numpy(), w), name
    return got


# ------------------------------------------------------------------------------------------------- union
@pytest.mark.parametrize("overlap", [0.0, 0.25, 1.0])
def test_union_matches_reference_at_pipeline_widths(overlap):
    a, ca, b, cb = _routes(1, 300, 2000, overlap)
    cnt = _check_union(a, ca, b, cb).counts.cpu().numpy()
    full = (ca == K_SPARSE) & (cb == K_DENSE)
    assert full.sum() > 200 and (cnt[full] == K_SPARSE + K_DENSE - round(overlap * K_SPARSE)).all()
    assert (cnt[ca + cb == 0] == 0).all()


def test_union_disjoint_identical_and_empty():
    rng = np.random.default_rng(2)
    k = 64
    a = np.stack([rng.permutation(500)[:k] for _ in range(6)]).astype(np.int32)
    b = np.stack([rng.permutation(500)[:k] for _ in range(6)]).astype(np.int32)
    b[0] = a[0] + 1000                                             # disjoint lists
    b[1] = a[1]                                                    # identical lists
    b[2] = a[2][::-1]                                              # identical sets, other order
    b[3] = np.concatenate([a[3][40:], 1000 + np.arange(40)])       # partly shared, at other ranks
    a[4, :] = -1                                                   # list a empty
    ca = np.array([k, k, k, k, 0, 0], np.int32)
    cb = np.array([k, k, k, k, k, 0], np.int32)                    # query 5: both empty
    u = _check_union(a, ca, b, cb)
    cnt = u.counts.cpu().tolist()
    assert cnt[1] == cnt[2] == k and cnt[4] == k and cnt[5] == 0
    ids = u.ids.cpu().numpy()
    assert np.array_equal(ids[0], np.concatenate([a[0], b[0]]))    # disjoint: list a, then list b
    assert (ids[5] == -1).all() and (u.map_a.cpu().numpy()[4:] == -1).all()


def test_union_total_1024_strided_views_repeats_and_refusal():
    nq = 40
    a, ca, b, cb = _routes(4, nq, 5000, 0.02, k_s=1000, k_d=24)    # 20 of list a's ids in list b
    a[0, 7] = a[0, 2]                                              # a repeated id inside list a
    b[1, 20] = b[1, 3]                                             # ... and inside list b
    b[2, :] = a[2, :24]                                            # list b a prefix of list a
    ca[:3], cb[:3] = 1000, 24
    _check_union(a, ca, b, cb)
    _check_union(b, cb, a[:, :1000], ca)                           # the other way round: 24 + 1000
    # row strides wider than k (the [Q, W] buffers of the sharded merge); the padding must not be read
    wa = np.full((nq, 1100), 777777, np.int32)
    wa[:, :1000] = a
    wb = np.full((nq, 30), 888888, np.int32)
    wb[:, :24] = b
    ta, tb = _dev(wa, wb)
    got = batched.pair_union(ta[:, :1000], torch.from_numpy(ca).to(DEV), tb[:, :24], torch.from_numpy(cb).to(DEV))
    want = orf.pair_union(a, ca, b, cb)
    assert all(np.array_equal(g.cpu().numpy(), w) for g, w in zip((got.ids, got.counts, got.map_a, got.map_b), want))
    # a repeated id maps both slots to one entry, which holds that id
    assert got.map_a[0, 7].item() == got.map_a[0, 2].item() and got.ids[0, got.map_a[0, 2]].item() == a[0, 2]
    with pytest.raises(ValueError, match="1024"):
        batched.pair_union(*_dev(a, ca), *_dev(np.zeros((nq, 25), np.int32), cb))
    L = _lib.lib()
    t = torch.zeros(1025, dtype=torch.int32, device=DEV)
    assert L.ezr_pair_union(_lib.ptr(t), _lib.ptr(t), 1000, 1000, _lib.ptr(t), _lib.ptr(t), 25, 25, 1, _lib.ptr(t),
                            _lib.ptr(t), _lib.ptr(t), _lib.ptr(t), _lib.stream_ptr()) == -1
    assert b"1024" in L.ezr_last_error()


def test_union_at_10000_queries():
    a, ca, b, cb = _routes(5, 10_000, 20_000, 0.25)
    _check_union(a, ca, b, cb)


# ------------------------------------------------------------------------------------------ mapped order
@pytest.mark.parametrize("top_n", [6, 192, 300])
def test_mapped_order_equals_the_order_of_each_list_alone(top_n):
    """Scores given per union entry, with exact ties and values saturated at 1.0f and 0.0f: each list ordered through
    its map equals ezr_cross_order_topk over that list's own packed scores."""
    L, st = _lib.lib(), _lib.stream_ptr()
    nq = 50
    a, ca, b, cb = _routes(6, nq, 800, 0.5)
    u = batched.pair_union(*_dev(a, ca, b, cb))
    cnt_u = u.counts.cpu().numpy()
    pair_off = torch.tensor(np.concatenate([[0], np.cumsum(cnt_u)]), dtype=torch.int32, device=DEV)
    g = torch.Generator().manual_seed(top_n)
    sig = torch.sigmoid(torch.randn(int(cnt_u.sum()), generator=g) * 4)
    sig[::9], sig[4::13] = 1.0, 0.0
    sig[2::17] = sig[1::17][:sig[2::17].numel()]
    sig = sig.to(DEV)
    for ids, cnt, slot_map in ((a, ca, u.map_a), (b, cb, u.map_b)):
        k = ids.shape[1]
        ids_t, = _dev(ids)
        mapped = [torch.empty(nq, k, device=DEV), torch.empty(nq, top_n, device=DEV),
                  torch.empty(nq, top_n, dtype=torch.int32, device=DEV), torch.empty(nq, dtype=torch.int32, device=DEV)]
        _lib.check(L.ezr_cross_order_topk_mapped(_lib.ptr(sig), _lib.ptr(pair_off), nq, k, _lib.ptr(slot_map),
                                                 slot_map.stride(0), _lib.ptr(ids_t), k, top_n,
                                                 *[_lib.ptr(x) for x in mapped], st))
        # the list's own pairs: its scores gathered through the map, packed as the reranker packs one list
        m = slot_map.cpu().numpy()
        valid = m >= 0
        own_sig_t, = _dev(sig.cpu().numpy()[(pair_off[:-1, None].cpu().numpy() + m)[valid]])
        own_off = torch.tensor(np.concatenate([[0], np.cumsum(valid.sum(1))]), dtype=torch.int32, device=DEV)
        plain = [torch.empty_like(x) for x in mapped]
        _lib.check(L.ezr_cross_order_topk(_lib.ptr(own_sig_t), _lib.ptr(own_off), nq, k, _lib.ptr(ids_t), k, top_n,
                                          *[_lib.ptr(x) for x in plain], st))
        torch.cuda.synchronize()
        assert torch.equal(mapped[2], plain[2]) and torch.equal(mapped[3], plain[3])
        assert torch.equal(_bits(mapped[0]), _bits(plain[0])) and torch.equal(_bits(mapped[1]), _bits(plain[1]))
    assert int((sig == 1.0).sum()) > 100 and int((sig == 0.0).sum()) > 100


def test_mapped_order_rejects_bad_arguments():
    L, st = _lib.lib(), _lib.stream_ptr()
    assert L.ezr_cross_order_topk_mapped(None, None, 1, 1025, None, 1025, None, 1025, 6, None, None, None, None,
                                         st) != 0
    assert b"cross_order_topk_mapped" in L.ezr_last_error()
    assert L.ezr_cross_order_topk_mapped(None, None, 1, 8, None, 4, None, 8, 6, None, None, None, None, st) != 0


# ------------------------------------------------------------------------------------------ rerank_fusion
def _model(family, d=256, layers=2, vocab=800, seed=7):
    from easyrag_b200.encoder import BertConfig
    from easyrag_b200.rerank import CrossEncoderModel, random_cross_encoder_state
    cfg = BertConfig(vocab_size=vocab, hidden_size=d, intermediate_size=4 * d, num_hidden_layers=layers,
                     num_attention_heads=d // 64, max_position_embeddings=514 if family == "roberta" else 512,
                     layer_norm_eps=1e-5 if family == "roberta" else 1e-12)
    return CrossEncoderModel(family, cfg, random_cross_encoder_state(family, cfg, seed, std=0.03), device=DEV,
                             **SPECIAL[family])


def _setup(family, seed, n_docs, nq, vocab=800, max_tokens=65536):
    from easyrag_b200.rerank import CrossEncoderReranker
    rng = np.random.default_rng(seed)
    passages = [rng.integers(4, vocab, int(n)).tolist() for n in rng.integers(0, 120, n_docs)]
    queries = [rng.integers(4, vocab, int(n)).tolist() for n in rng.integers(1, 40, nq)]
    q_ptr = torch.tensor(np.cumsum([0] + [len(q) for q in queries]), dtype=torch.int32, device=DEV)
    q_tok = torch.tensor([t for q in queries for t in q], dtype=torch.int32, device=DEV)
    return CrossEncoderReranker(_model(family, vocab=vocab), passages, max_tokens=max_tokens), q_ptr, q_tok


def _topks(a, ca, b, cb):
    ta, tca, tb, tcb = _dev(a, ca, b, cb)
    return TopK(torch.zeros(ta.shape, device=DEV), ta, tca), TopK(torch.zeros(tb.shape, device=DEV), tb, tcb)


def _two_calls(rr, sparse, dense, q_ptr, q_tok, top_n, k_out, canon):
    s, s_all = rr.rerank(sparse, q_ptr, q_tok, top_n)
    d, d_all = rr.rerank(dense, q_ptr, q_tok, top_n)
    return s, d, s_all, d_all, batched.rrf_fuse(s.ids, s.counts, d.ids, d.counts, k_out, K=60, canon=canon)


@pytest.mark.parametrize("family", ["bert", "roberta"])
@pytest.mark.parametrize("overlap", [0.0, 0.5, 1.0])
def test_rerank_fusion_equals_two_rerank_calls(family, overlap):
    nq, n_docs, top_n, k_out = 64, 3000, 6, 6
    rr, q_ptr, q_tok = _setup(family, 20 + int(overlap * 10), n_docs, nq)
    a, ca, b, cb = _routes(7, nq, n_docs, overlap)
    sparse, dense = _topks(a, ca, b, cb)
    canon = synth.make_duplicates(n_docs, 0.2, 9).to(DEV)
    events = []
    res = rr.rerank_fusion(sparse, dense, q_ptr, q_tok, top_n, k_out, canon=canon, events=events)
    s, d, s_all, d_all, fused = _two_calls(rr, sparse, dense, q_ptr, q_tok, top_n, k_out, canon)
    torch.cuda.synchronize()
    assert len(events) == 4
    assert _same_topk(res.sparse, s) and _same_topk(res.dense, d) and _same_topk(res.fused, fused)
    assert torch.equal(_bits(res.sparse_all), _bits(s_all)) and torch.equal(_bits(res.dense_all), _bits(d_all))
    want = orf.pair_union(a, ca, b, cb)
    assert res.n_pairs == int(want[1].sum())
    assert res.n_route_pairs == int(ca.sum() + cb.sum())
    full = (ca == K_SPARSE) & (cb == K_DENSE)
    assert (want[1][full] == K_SPARSE + K_DENSE - round(overlap * K_SPARSE)).all()
    # a wider top_n, with k_out past what the two lists hold
    res = rr.rerank_fusion(sparse, dense, q_ptr, q_tok, 200, 420)
    s, d, s_all, d_all, fused = _two_calls(rr, sparse, dense, q_ptr, q_tok, 200, 420, None)
    assert _same_topk(res.sparse, s) and _same_topk(res.dense, d) and _same_topk(res.fused, fused)


def test_rerank_fusion_refusals():
    rr, q_ptr, q_tok = _setup("bert", 3, 100, 4)
    a, ca, b, cb = _routes(8, 4, 100, 0.5, k_s=10, k_d=20)
    sparse, dense = _topks(a, ca, b, cb)
    for top_n, k_out in ((0, 6), (6, 0)):
        with pytest.raises(ValueError, match=">= 1"):
            rr.rerank_fusion(sparse, dense, q_ptr, q_tok, top_n, k_out)
    with pytest.raises(ValueError, match="queries"):
        rr.rerank_fusion(sparse, TopK(dense.scores[:3], dense.ids[:3], dense.counts[:3]), q_ptr, q_tok, 6, 6)
    wide = TopK(torch.zeros(4, 1015, device=DEV), torch.full((4, 1015), -1, dtype=torch.int32, device=DEV),
                torch.zeros(4, dtype=torch.int32, device=DEV))
    with pytest.raises(ValueError, match="1024"):
        rr.rerank_fusion(sparse, wide, q_ptr, q_tok, 6, 6)


def test_saturated_scores_keep_coarse_order():
    """A head bias that drives every sigmoid to exactly 1.0f: each route's order is its coarse order, and the fused
    list is the RRF of the coarse prefixes."""
    nq, n_docs, top_n, k_out = 16, 1500, 6, 6
    rr, q_ptr, q_tok = _setup("roberta", 30, n_docs, nq)
    rr.model.b2 = 200.0
    a, ca, b, cb = _routes(9, nq, n_docs, 0.5)
    sparse, dense = _topks(a, ca, b, cb)
    canon = synth.make_duplicates(n_docs, 0.3, 11)
    res = rr.rerank_fusion(sparse, dense, q_ptr, q_tok, top_n, k_out, canon=canon.to(DEV))
    torch.cuda.synchronize()
    assert (res.sparse_all.cpu()[torch.from_numpy(a) >= 0] == 1.0).all()
    for q in range(nq):
        ns, nd = min(ca[q], top_n), min(cb[q], top_n)
        assert res.sparse.ids[q, :ns].cpu().tolist() == a[q, :ns].tolist()
        assert res.dense.ids[q, :nd].cpu().tolist() == b[q, :nd].tolist()
        assert (res.sparse.scores[q, :ns].cpu() == 1.0).all() and (res.dense.scores[q, :nd].cpu() == 1.0).all()
        ids, sc = ort.rrf_ids([a[q, :ns], b[q, :nd]], canon.numpy(), K=60, topk=k_out)
        c = int(res.fused.counts[q])
        assert c == ids.size and res.fused.ids[q, :c].cpu().tolist() == ids.tolist()
        assert res.fused.scores[q, :c].cpu().numpy().tobytes() == sc.tobytes()


def test_fused_list_matches_the_oracle_on_texts():
    """The reference's control flow on node texts, where ``canon`` duplicates share a text: per-pair scores are the
    GPU's own (the encoder is checked against transformers in test_gpu_rerank.py), so order and fusion must match
    exactly."""
    nq, n_docs, top_n, k_out = 24, 1200, 120, 256
    rr, q_ptr, q_tok = _setup("bert", 40, n_docs, nq)
    a, ca, b, cb = _routes(10, nq, n_docs, 0.5)
    sparse, dense = _topks(a, ca, b, cb)
    canon = synth.make_duplicates(n_docs, 0.4, 12)
    res = rr.rerank_fusion(sparse, dense, q_ptr, q_tok, top_n, k_out, canon=canon.to(DEV))
    torch.cuda.synchronize()
    nodes = [ort.ONode(text=f"chunk {int(canon[i])}", idx=i) for i in range(n_docs)]
    s_all, d_all = res.sparse_all.cpu().numpy(), res.dense_all.cpu().numpy()
    shared_texts = 0
    for q in range(nq):
        fused, s, d = orf.rerank_fusion([nodes[i] for i in a[q, :ca[q]]], [nodes[i] for i in b[q, :cb[q]]],
                                        s_all[q, :ca[q]].tolist(), d_all[q, :cb[q]].tolist(), top_n, k_out)
        for got, want in ((res.sparse, s), (res.dense, d)):
            c = int(got.counts[q])
            assert got.ids[q, :c].cpu().tolist() == [i for i, _ in want]
            assert got.scores[q, :c].cpu().numpy().tobytes() == np.array([x for _, x in want], np.float32).tobytes()
        c = int(res.fused.counts[q])
        assert res.fused.ids[q, :c].cpu().tolist() == [i for i, _ in fused]
        assert res.fused.scores[q, :c].cpu().numpy().tobytes() == np.array([x for _, x in fused]).tobytes()
        s_ids, d_ids = {i for i, _ in s}, {i for i, _ in d}
        shared_texts += sum(int(canon[i]) == int(canon[j]) for i in s_ids for j in d_ids if i != j)
    assert shared_texts >= 10                     # the case merges different ids of one text across the two lists


# ------------------------------------------------------------------------------------------ sharded
def test_sharded_without_a_process_group_equals_one_gpu():
    from easyrag_b200.dist import ShardedCrossEncoderReranker
    assert not dist.is_initialized()
    rr, q_ptr, q_tok = _setup("roberta", 50, 1000, 12, max_tokens=4096)
    sparse, dense = _topks(*_routes(11, 12, 1000, 0.5))
    sh = ShardedCrossEncoderReranker(rr)
    assert _same(sh.rerank_fusion(sparse, dense, q_ptr, q_tok, 6, 6), rr.rerank_fusion(sparse, dense, q_ptr, q_tok, 6, 6))


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
        from easyrag_b200 import dist as ezdist
        fails = []
        nq, n_docs = 16, 1500
        rr, q_ptr, q_tok = _setup("bert", 60, n_docs, nq, max_tokens=8192)
        sh = ezdist.ShardedCrossEncoderReranker(rr)
        if (sh.world, sh.rank) != (world, rank):
            fails.append("world / rank")
        canon = synth.make_duplicates(n_docs, 0.2, 13).to(dev)
        for overlap in (0.0, 0.5, 1.0):
            sparse, dense = _topks(*_routes(12, nq, n_docs, overlap))
            got = sh.rerank_fusion(sparse, dense, q_ptr, q_tok, 6, 6, canon=canon)
            if not _same(got, rr.rerank_fusion(sparse, dense, q_ptr, q_tok, 6, 6, canon=canon)):
                fails.append(f"overlap {overlap}")
        u = batched.pair_union(sparse.ids, sparse.counts, dense.ids, dense.counts)
        pairs = rr.pack(u.ids, u.counts, q_ptr, q_tok)
        if world > 1 and any(hi == lo for lo, hi in ezdist.token_balanced_ranges(pairs.cu_h, world)):
            fails.append("a rank got no pairs")
        # fewer pairs than ranks, and no pairs at all
        for cs, cd in (([1, 0, 0], [0, 0, 0]), ([0, 0, 0], [0, 0, 0])):
            a = torch.full((3, 4), -1, dtype=torch.int32, device=dev)
            a[0, 0] = 17
            sp = TopK(torch.zeros(3, 4, device=dev), a, torch.tensor(cs, dtype=torch.int32, device=dev))
            de = TopK(torch.zeros(3, 5, device=dev), torch.full((3, 5), -1, dtype=torch.int32, device=dev),
                      torch.tensor(cd, dtype=torch.int32, device=dev))
            got = sh.rerank_fusion(sp, de, q_ptr[:4], q_tok, 3, 4)
            if not _same(got, rr.rerank_fusion(sp, de, q_ptr[:4], q_tok, 3, 4)):
                fails.append(f"counts {cs}")
        # inputs that differ across ranks are refused on every rank
        sparse, dense = _topks(*_routes(12, nq, n_docs, 0.5))
        if rank == 0:
            dense = TopK(dense.scores, dense.ids, dense.counts.clamp(max=100))
        try:
            sh.rerank_fusion(sparse, dense, q_ptr, q_tok, 6, 6)
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
    pytest.param("gloo", 3, id="gloo-3-on-one-gpu"),
    pytest.param("nccl", 2, id="nccl-2", marks=pytest.mark.skipif(torch.cuda.device_count() < 2,
                                                                 reason="needs 2 GPUs")),
    pytest.param("nccl", 3, id="nccl-3", marks=pytest.mark.skipif(torch.cuda.device_count() < 3,
                                                                 reason="needs 3 GPUs")),
])
def test_sharded_rerank_fusion_equals_one_gpu(backend, world):
    mgr = mp.get_context("spawn").Manager()
    ret = mgr.dict()
    mp.spawn(_worker, args=(world, backend, _free_port(), ret), nprocs=world, join=True)
    assert dict(ret) == {r: [] for r in range(world)}
