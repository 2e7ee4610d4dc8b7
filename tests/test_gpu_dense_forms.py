"""The 128-query dense kernel (form 2: query chunks held in registers, 128-row corpus tiles) against the 64-query
kernel with both operands in shared memory (form 3): every score is the fp32 sum of the same k16 products in the same
order, so ids, counts and score bits must be identical."""
import pytest
import torch

from easyrag_b200 import _lib, batched, synth
from easyrag_b200.index import DenseIndex

pytestmark = pytest.mark.gpu
DEV = "cuda"
N_ROWS = 200_000


def _unit_rows(n, d, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, d, generator=g)
    return (x / x.norm(dim=1, keepdim=True)).to(torch.bfloat16)


def _run(form, index, qv, k, q_group=None):
    L = _lib.lib()
    _lib.check(L.ezr_dense_set_kernel(form))
    try:
        res = batched.dense_topk(index, qv, k, q_group=q_group)
        torch.cuda.synchronize()
        assert L.ezr_dense_last_kernel() == {2: b"wgmma", 3: b"wgmma-q64"}[form]
    finally:
        L.ezr_dense_set_kernel(0)
    return res


def _assert_same(a, b):
    assert torch.equal(a.counts, b.counts)
    assert torch.equal(a.ids, b.ids)
    assert torch.equal(a.scores.view(torch.int32), b.scores.view(torch.int32))


@pytest.mark.parametrize("nq", [129, 1000, 10_000])
@pytest.mark.parametrize("d", [64, 128, 256, 512, 768])
def test_register_query_form_matches_smem_form(d, nq):
    c = _unit_rows(N_ROWS, d, 10 + d)
    qv = _unit_rows(nq, d, 20 + d + nq).to(DEV)
    index = DenseIndex(c, device=DEV)
    _assert_same(_run(2, index, qv, 10), _run(3, index, qv, 10))


@pytest.mark.parametrize("k", [4, 8, 12, 16])
def test_register_query_form_filter_and_id_base(k):
    d, nq = 768, 300
    c = _unit_rows(N_ROWS, d, 31)
    qv = _unit_rows(nq, d, 32).to(DEV)
    groups = synth.make_groups(N_ROWS, 4, 33)
    want = torch.tensor([i % 6 - 1 for i in range(nq)], dtype=torch.int32)
    want[want == 4] = -2
    index = DenseIndex(c, device=DEV, doc_group=groups, row_lo=1000)
    a, b = _run(2, index, qv, k, q_group=want), _run(3, index, qv, k, q_group=want)
    _assert_same(a, b)
    assert int(a.ids[a.ids >= 0].min()) >= 1000
