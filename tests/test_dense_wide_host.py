"""Host side of form 6 of ezr_dense_topk (csrc/dense_wide.cu): the switch, the workspace arithmetic and the Python
refusals.  No GPU needed."""
import pytest

from easyrag_b200 import _lib, batched
from easyrag_b200.retrievers import B200VectorStore


def _align(x):
    return (x + 255) // 256 * 256


def test_form_6_is_a_valid_switch(lib_built):
    L = _lib.lib()
    assert L.ezr_dense_set_kernel(6) == 0
    assert L.ezr_dense_set_kernel(7) == -1
    assert b"6 wgmma score rows" in L.ezr_last_error()
    assert L.ezr_dense_set_kernel(0) == 0


@pytest.mark.parametrize("n,nq,k,bq", [(100_000, 700, 288, 671), (100_000, 700, 288, 1), (1_000_000, 4096, 288, 512),
                                       (1_000_003, 65, 10, 64), (129, 257, 1024, 7)])
def test_workspace_covers_every_block(lib_built, n, nq, k, bq):
    L = _lib.lib()

    def block(m):
        return _align(m * n * 4) + L.ezr_select_rows_workspace(m, n, k, _lib.F32)

    want = block(bq) if nq % bq == 0 else max(block(bq), block(nq % bq))
    assert L.ezr_dense_wide_workspace(n, nq, k, bq) == want
    assert L.ezr_dense_wide_workspace(n, nq, k, nq + 5) == L.ezr_dense_wide_workspace(n, nq, k, nq)
    assert L.ezr_dense_wide_workspace(n, nq, k, 0) == 0 and L.ezr_dense_wide_workspace(0, nq, k, bq) == 0


def test_default_workspace_holds_the_simt_block(lib_built):
    # 100k rows: the SIMT block is 671 queries (256 MB of score rows), and 700 = 671 + 29
    L = _lib.lib()
    n, nq, k = 100_000, 700, 288
    assert L.ezr_dense_topk_workspace(n, 3584, nq, k) >= L.ezr_dense_wide_workspace(n, nq, k, 671)


@pytest.mark.parametrize("n,nq,k", [(100_000, 700, 288), (1_000_000, 100, 288), (129, 1025, 1024), (5000, 1500, 10),
                                    (100_000, 671, 288)])
def test_default_workspace_covers_every_simt_block(lib_built, n, nq, k):
    # form 1 / the SIMT fallback runs blocks of up to 1024 queries and 256 MB of score rows; each block's select
    # workspace follows its own rows, so a smaller last block counts on its own (no wgmma form at dim 3584)
    L = _lib.lib()

    def block(m):
        return _align(m * n * 4) + L.ezr_select_rows_workspace(m, n, k, _lib.F32)

    qb = min(nq, 1024, max(1, (256 << 20) // (n * 4)))
    want = block(qb) if nq % qb == 0 else max(block(qb), block(nq % qb))
    assert L.ezr_dense_topk_workspace(n, 3584, nq, k) == want


def test_block_queries_refusals():
    class _Index:
        quantized = True

    with pytest.raises(ValueError, match="form=6"):
        batched.dense_topk(_Index(), None, 10, block_queries=64)
    with pytest.raises(ValueError, match="quantized"):
        batched.dense_topk(_Index(), None, 10, form=6, block_queries=64)
    _Index.quantized = False
    with pytest.raises(ValueError, match=">= 1"):
        batched.dense_topk(_Index(), None, 10, form=6, block_queries=0)
    with pytest.raises(ValueError, match="dense_form=6"):
        B200VectorStore(block_queries=64)
    with pytest.raises(ValueError, match="dense_form=6"):
        B200VectorStore(dense_form=6, block_queries=64, quantize=True)
