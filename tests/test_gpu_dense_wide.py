"""GPU: form 6 of ezr_dense_topk (csrc/dense_wide.cu) -- wgmma score rows of a query block, then the generic select.

Every score of form 6 is one fp32 accumulator chain over the same k16 products, in the same increasing k order, as the
wgmma forms 2-4, so on shapes those forms take the two must agree bit for bit.  At gte-Qwen2-7B's width (3584) it is
checked against fp64: exactly on integer vectors (every dot product is exact in fp32, ties are common), and within the
derived bound of ``_bounds.dense_score_bound`` on unit vectors.  The figures measured are printed (``pytest -s``).
"""
import asyncio

import pytest
import torch

from _bounds import check_dense_topk, dense_delta_max, dense_score_bound
from _topk_ref import canonical_topk, fp64_top
from easyrag_b200 import _lib, batched, synth
from easyrag_b200.index import DenseIndex
from easyrag_b200.retrievers import B200VectorStore, QdrantRetriever
from easyrag_b200.schema import BaseEmbedding, QueryBundle, TextNode, build_qdrant_filters

pytestmark = pytest.mark.gpu
DEV = "cuda"
EZR_ERR_WORKSPACE, EZR_ERR_UNSUPPORTED = -3, -4
FORM_NAMES = {1: b"simt", 2: b"wgmma", 3: b"wgmma-q64", 4: b"wgmma-q64-n128", 6: b"wgmma-scores"}


@pytest.fixture(scope="module", autouse=True)
def _ready(lib_built):
    _lib.require_cuda()


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _ints(n, d, seed, lo=-2, hi=2):
    return torch.randint(lo, hi + 1, (n, d), generator=_gen(seed), device=DEV).to(torch.bfloat16)


def _unit(n, d, seed):
    x = torch.randn(n, d, generator=_gen(seed), device=DEV)
    return torch.nn.functional.normalize(x, dim=1).to(torch.bfloat16)


def _report(what, info):
    print(f"\n[dense wide] {what}: " + ", ".join(f"{k}={v:.5g}" if isinstance(v, float) else f"{k}={v}"
                                               for k, v in info.items()))


def _run(form, index, q, k, q_group=None, **kw):
    """batched.dense_topk with a forced form; checks the kernel that ran."""
    res = batched.dense_topk(index, q, k, q_group=q_group, form=form, **kw)
    torch.cuda.synchronize()
    assert _lib.lib().ezr_dense_last_kernel() == FORM_NAMES[form]
    return res


def _raw(c, q, k, doc_group=None, q_group=None, id_base=0, ws_bytes=None, form=6):
    """ezr_dense_topk under ``form`` on any (possibly strided) views, with exactly ``ws_bytes`` of workspace (default:
    ezr_dense_topk_workspace).  -> (status, TopK)."""
    L = _lib.lib()
    n, d = c.shape
    nq = q.shape[0]
    out = batched.TopK(torch.full((nq, k), 7.0, device=DEV), torch.full((nq, k), 7, dtype=torch.int32, device=DEV),
                       torch.full((nq,), 7, dtype=torch.int32, device=DEV))
    if ws_bytes is None:
        ws_bytes = L.ezr_dense_topk_workspace(n, d, nq, k)
    buf = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=DEV)
    _lib.check(L.ezr_dense_set_kernel(form))
    try:
        rc = L.ezr_dense_topk(_lib.ptr(c), n, d, c.stride(0), _lib.ptr(q), nq, q.stride(0), k, _lib.ptr(doc_group),
                              _lib.ptr(q_group), id_base, _lib.ptr(out.scores), _lib.ptr(out.ids), _lib.ptr(out.counts),
                              _lib.ptr(buf), ws_bytes, _lib.stream_ptr())
        torch.cuda.synchronize()
        if rc == 0 and n > 0:
            assert L.ezr_dense_last_kernel() == FORM_NAMES[form]
    finally:
        L.ezr_dense_set_kernel(0)
    return rc, out


def _assert_same(a, b):
    assert torch.equal(a.counts, b.counts)
    assert torch.equal(a.ids, b.ids)
    assert torch.equal(a.scores.view(torch.int32), b.scores.view(torch.int32))


def _assert_canonical(res, sims, k, allowed=None, id_base=0):
    """res equals the (score desc, id desc) top-k of exact integer scores sims [Q, n] (fp64), -1 padded."""
    kk = min(k, sims.shape[1])
    ids, sc = canonical_topk(sims, kk, allowed)
    valid = torch.ones_like(ids, dtype=torch.bool) if allowed is None else allowed.gather(1, ids)
    cnt = valid.sum(1)
    assert torch.equal(res.counts.long(), cnt)
    want_ids = torch.full((sims.shape[0], k), -1, dtype=torch.int64, device=DEV)
    want_ids[:, :kk] = torch.where(valid, ids + id_base, torch.full_like(ids, -1))
    assert torch.equal(res.ids.long(), want_ids)
    got = res.scores[:, :kk]
    assert torch.equal(got[valid], sc[valid].float())


# ------------------------------------------------------------ bit identity with the wgmma forms (dim <= 1024)
_UNIT = {}


def _unit_case(d):
    if d not in _UNIT:
        c = _unit(200_000, d, 10 + d)
        _UNIT[d] = (DenseIndex(c, device=DEV), _unit(1000, d, 20 + d))
    return _UNIT[d]


@pytest.mark.parametrize("d", [64, 768, 1024])
@pytest.mark.parametrize("k", [1, 10, 16])
def test_bit_identical_to_wgmma_forms(d, k):
    index, q = _unit_case(d)
    wide = _run(6, index, q, k)
    assert (wide.counts == k).all()
    for form in [3, 4] + ([2] if d <= 768 else []):
        _assert_same(wide, _run(form, index, q, k))


# ------------------------------------------------------------ gte-Qwen2-7B width, exact integers
N_INT, D_INT, Q_INT = 100_000, 3584, 700       # the default workspace holds 671 queries of score rows: 671 + 29


@pytest.fixture(scope="module")
def int_case():
    c = _ints(N_INT, D_INT, 80)
    q = _ints(Q_INT, D_INT, 81)
    return dict(c=c, q=q, index=DenseIndex(c, device=DEV), sims=q.double() @ c.double().T)


@pytest.mark.parametrize("k", [1, 10, 288, 1024])
def test_exact_integers_at_3584(int_case, k):
    res = _run(6, int_case["index"], int_case["q"], k)
    _assert_canonical(res, int_case["sims"], k)
    _assert_same(res, _run(1, int_case["index"], int_case["q"], k))


def test_block_size_does_not_change_results(int_case):
    L = _lib.lib()
    c, q, index, k = int_case["c"], int_case["q"], int_case["index"], 288
    rc, ref = _raw(c, q, k)                               # the default workspace of ezr_dense_topk_workspace
    assert rc == 0
    _assert_canonical(ref, int_case["sims"], k)
    for bq in (1, 7, 64, 700):
        _assert_same(_run(6, index, q, k, block_queries=bq), ref)
    one = L.ezr_dense_wide_workspace(N_INT, 65, k, 1)
    assert one > 0 and L.ezr_dense_wide_workspace(N_INT, 65, k, 65) > one
    rc, res = _raw(c, q[:65], k, ws_bytes=one)
    assert rc == 0
    _assert_same(res, batched.TopK(ref.scores[:65], ref.ids[:65], ref.counts[:65]))
    rc, _ = _raw(c, q[:65], k, ws_bytes=one - 1)
    assert rc == EZR_ERR_WORKSPACE
    assert b"workspace" in L.ezr_last_error()


def test_simt_blocks_fit_the_default_workspace(int_case):
    # form 1 runs SIMT blocks of 671 + 29 queries here.  The 29-query block's select splits each row into more parts
    # and needs more workspace than the 671-query block's; it sits right behind the block's own rows, so exactly
    # ezr_dense_topk_workspace holds it.
    c, q, k = int_case["c"], int_case["q"], 288
    rc, simt = _raw(c, q, k, form=1)
    assert rc == 0
    rc, wide = _raw(c, q, k)
    assert rc == 0
    _assert_same(simt, wide)


def test_block_queries_needs_form_6(int_case):
    with pytest.raises(ValueError):
        batched.dense_topk(int_case["index"], int_case["q"][:4], 10, block_queries=4)
    with pytest.raises(ValueError):
        batched.dense_topk(int_case["index"], int_case["q"][:4], 10, form=1, block_queries=4)


def test_filters_row_lo_and_short_classes(int_case):
    c, q, sims, k = int_case["c"], int_case["q"], int_case["sims"], 288
    groups = synth.make_groups(N_INT, 3, 82).to(DEV)
    groups[torch.randperm(N_INT, generator=_gen(83), device=DEV)[:100]] = 3     # class 3: 100 rows, fewer than k
    want = torch.tensor([i % 6 - 1 for i in range(Q_INT)], dtype=torch.int32, device=DEV)   # -1 .. 4
    want[want == 4] = 7                                            # a class no row has: count 0, all -1
    base = (1 << 31) - 1 - N_INT                                   # the largest row_lo whose ids stay int32
    rc, res = _raw(c, q, k, doc_group=groups, q_group=want, id_base=base)
    assert rc == 0
    allowed = (want[:, None] == -1) | (groups[None, :] == want[:, None])
    _assert_canonical(res, sims, k, allowed, id_base=base)
    assert int(res.counts[want == 7].max()) == 0 and (res.ids[want == 7] == -1).all()
    assert (res.counts[want == 3] == int((groups == 3).sum())).all()
    assert int(res.ids.max()) <= (1 << 31) - 2


# ------------------------------------------------------------ unit vectors at width, derived bound
@pytest.mark.parametrize("d", [3584, 4096])
def test_unit_vectors_within_derived_bound(d):
    n, nq, k = 100_000, 256, 288
    c = synth.make_dense_corpus(n, d, 90 + d, device=DEV)
    q = synth.make_dense_queries(c, nq, 91 + d)
    res = _run(6, DenseIndex(c, device=DEV), q, k)
    assert (res.counts == k).all()
    top_i, top_s, _ = fp64_top(q, c, k + 32, integer=False)
    exact, delta = dense_score_bound(q, c, res.ids.long(), chunk=64)
    dmax = dense_delta_max(q, c.double().norm(dim=1).max().item())
    info = check_dense_topk(res.scores, res.ids, exact, delta, top_s, top_i, dmax, n, f"unit d={d}")
    _report(f"unit vectors d={d} k={k}", info)


# ------------------------------------------------------------ edges
@pytest.mark.parametrize("n", [1, 127, 128, 129, 100_003])
@pytest.mark.parametrize("nq", [1, 63, 65, 257])
def test_row_and_query_counts(n, nq):
    c, q = _ints(n, 64, 100 + n), _ints(nq, 64, 200 + nq)
    sims = q.double() @ c.double().T
    for k in (10, 288):
        rc, res = _raw(c, q, k)
        assert rc == 0
        _assert_canonical(res, sims, k)


@pytest.mark.parametrize("d", [64, 1088, 8192])
def test_dims(d):
    c, q = _ints(5000, d, 300 + d), _ints(65, d, 301 + d)
    rc, res = _raw(c, q, 50)
    assert rc == 0
    _assert_canonical(res, q.double() @ c.double().T, 50)


def test_row_strides_larger_than_dim():
    n, nq, d, ld, k = 20_000, 130, 3584, 3600, 288
    cb, qb = _ints(n, ld, 400), _ints(nq, ld, 401)
    c, q = cb[:, :d], qb[:, :d]
    assert c.stride(0) == ld and q.stride(0) == ld
    rc, res = _raw(c, q, k)
    assert rc == 0
    _assert_canonical(res, q.double() @ c.double().T, k)
    rc, dense = _raw(c.contiguous(), q.contiguous(), k)
    _assert_same(res, dense)


def test_zero_query_and_negative_scores():
    n, d, k = 3000, 256, 300
    c = _ints(n, d, 500)
    q = _ints(3, d, 501)
    q[0] = 0                                                       # all-zero query: every score is +0.0
    rc, res = _raw(c, q, k)
    assert rc == 0
    assert (res.scores[0].view(torch.int32) == 0).all()            # sign bit clear, not -0.0
    _assert_canonical(res, q.double() @ c.double().T, k)
    cn, qp = -_ints(n, d, 502, 1, 2), _ints(4, d, 503, 1, 2)      # every score negative
    rc, res = _raw(cn, qp, k)
    assert rc == 0 and (res.scores < 0).all()
    _assert_canonical(res, qp.double() @ cn.double().T, k)


def test_empty_corpus():
    c = torch.empty(0, 128, dtype=torch.bfloat16, device=DEV)
    rc, res = _raw(c, _ints(5, 128, 600), 12)
    assert rc == 0
    assert (res.counts == 0).all() and (res.ids == -1).all()


def test_forced_on_unsupported_shapes_is_refused():
    L = _lib.lib()
    n, k = 1000, 10
    assert _raw(_ints(n, 3588, 700), _ints(4, 3588, 701), k)[0] == EZR_ERR_UNSUPPORTED          # dim % 64 != 0
    assert b"wgmma-scores" in L.ezr_last_error()
    flat = _ints(1, n * 3584 + 8, 702)[0]
    mis = flat[1:1 + n * 3584].view(n, 3584)                                                    # 2-byte offset
    assert _raw(mis, _ints(4, 3584, 703), k)[0] == EZR_ERR_UNSUPPORTED
    wide = _ints(n, 3588, 704)[:, :3584]                                                        # ld % 8 != 0
    assert _raw(wide, _ints(4, 3584, 705), k)[0] == EZR_ERR_UNSUPPORTED
    assert _raw(_ints(n, 3584, 706), _ints(4, 3588, 707)[:, :3584], k)[0] == EZR_ERR_UNSUPPORTED


# ------------------------------------------------------------ drop-in vector store
class _TableEmbedding(BaseEmbedding):
    """Query embedding looked up from a fixed table (query text = row index)."""

    def __init__(self, table):
        super().__init__(model_name="table", embed_batch_size=8)
        self._table = table

    def _get_query_embedding(self, query):
        return self._table[int(query)].tolist()

    _get_text_embedding = _get_query_embedding


def _plus_minus_rows(n, d, nnz, seed):
    """Rows with nnz entries of +-1, the rest 0: unit norm after the store's normalisation is exact in bf16 when nnz
    is a power of 4, and so is every score (a multiple of 1 / nnz)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.zeros(n, d)
    pos = torch.rand(n, d, generator=g).argsort(1)[:, :nnz]
    x.scatter_(1, pos, torch.randint(0, 2, (n, nnz), generator=g).float() * 2 - 1)
    return x


def test_vector_store_form_6_matches_default_store():
    n, d, k, dirs = 3000, 256, 288, ["director", "emsplus", "rcp", "umac"]
    emb = _plus_minus_rows(n, d, 16, 800)
    g = torch.Generator().manual_seed(801)
    nodes = [TextNode(text=f"chunk {i}", id_=f"node-{i}", metadata={"dir": dirs[int(torch.randint(4, (1,), generator=g))]},
                      embedding=emb[i].tolist()) for i in range(n)]
    queries = _TableEmbedding(_plus_minus_rows(8, d, 16, 802))
    default, wide = B200VectorStore(nodes), B200VectorStore(nodes, dense_form=6)
    for qi in range(8):
        lists = []
        for store in (default, wide):
            r = QdrantRetriever(store, queries, similarity_top_k=k)
            r.filters = build_qdrant_filters(dirs[qi % 4]) if qi % 2 else None
            lists.append([(x.node.node_id, x.score) for x in asyncio.run(r.aretrieve(QueryBundle(str(qi))))])
        assert lists[0] == lists[1]
        assert len(lists[0]) == (k if qi % 2 == 0 else min(k, sum(nd.metadata["dir"] == dirs[qi % 4] for nd in nodes)))
    assert _lib.lib().ezr_dense_last_kernel() == b"wgmma-scores"
