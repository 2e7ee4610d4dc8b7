"""CPU: the whole-tensor restatement of the reranker pair packers (tests/_pack_ref.py) against the per-pair oracles --
``oracle/rerank.py::cross_encoder_inputs`` (pinned to a real fast tokenizer in test_rerank_host.py) for both
cross-encoder templates, and ``oracle/retrieve.py::rerank_inputs`` for the LLM reranker's ``get_inputs``.  The GPU
tests (test_gpu_rerank_scale.py) compare the kernels with this restatement at pipeline scale."""
import numpy as np
import pytest
import torch

import _pack_ref as pr
from oracle import rerank as orr
from oracle import retrieve as ort
from easyrag_b200.handoff import PackedRerankInput

CLS = {"bert": (2, 3, 0), "roberta": (0, 2, 2)}          # family -> (cls, sep, pos_offset)


def _csr(seqs):
    ptr = torch.tensor(np.cumsum([0] + [len(s) for s in seqs]), dtype=torch.int64)
    tok = torch.tensor([t for s in seqs for t in s], dtype=torch.int32)
    return ptr, tok


def _case(rng, nq, k, n_docs, max_length, id_base=0, extra_cols=0, q_hi=None, p_hi=None):
    """Random queries / passages / candidate lists with every edge the packers have: empty query and passage,
    queries beyond room / 2, room and 3/4 max_length, passages beyond max_length, counts 0 and k, -1 padding, the
    same document twice in one list, and (``extra_cols``) a [Q, k] view of a wider list with junk past column k."""
    q_hi = q_hi or 2 * max_length
    p_hi = p_hi or 2 * max_length
    passages = [rng.integers(4, 900, int(rng.integers(0, p_hi + 1))).tolist() for _ in range(n_docs)]
    passages[0] = []
    passages[1] = rng.integers(4, 900, max_length + 3).tolist()
    queries = [rng.integers(4, 900, int(rng.integers(0, q_hi + 1))).tolist() for _ in range(nq)]
    queries[0] = []
    queries[1] = rng.integers(4, 900, max_length // 2 + 1).tolist()
    queries[2] = rng.integers(4, 900, max_length + 1).tolist()
    queries[3] = rng.integers(4, 900, max_length * 3 // 4 + 2).tolist()
    counts = rng.integers(0, k + 1, nq)
    counts[0], counts[1], counts[2] = k, 0, k
    ids = np.full((nq, k + extra_cols), -1, np.int64)
    ids[:, k:] = rng.integers(-5, 10 ** 6, (nq, extra_cols))
    for q in range(nq):
        c = int(counts[q])
        ids[q, :c] = rng.integers(0, n_docs, c) + id_base                  # duplicates happen
        if c >= 3:
            ids[q, 2] = ids[q, 0]                                          # and one for sure
        ids[q, c:min(c + 1, k)] = id_base                                  # ignored: past the count
    ids[0, :2] = np.array([0, 1]) + id_base                                # empty passage, too-long passage
    return queries, passages, torch.from_numpy(ids.astype(np.int32)), torch.from_numpy(counts.astype(np.int32))


@pytest.mark.parametrize("family", ["bert", "roberta"])
@pytest.mark.parametrize("max_length", ["min", 9, 33, 64])
def test_cross_pack_matches_the_pair_oracle(family, max_length):
    n_mid, type_b = orr.TEMPLATES[family]
    cls, sep, pos_offset = CLS[family]
    max_length = 2 + n_mid if max_length == "min" else max_length
    rng = np.random.default_rng([n_mid, max_length])
    nq, k, n_docs, id_base = 40, 70, 300, 12345
    queries, passages, cand, counts = _case(rng, nq, k, n_docs, max_length, id_base=id_base, extra_cols=5)
    (qp, qt), (pp, pt) = _csr(queries), _csr(passages)
    got = pr.cross_pack(qp, qt, pp, pt, cand, counts, k, id_base, n_mid, type_b, cls, sep, pos_offset, max_length)
    assert got["pair_off"].tolist() == np.concatenate([[0], np.cumsum(counts.numpy())]).tolist()
    assert got["P"] == int(counts.sum()) and got["T"] == got["ids"].numel() == int(got["cu"][-1])
    cu, ids, types, pos = got["cu"], got["ids"].tolist(), got["types"].tolist(), got["positions"].tolist()
    p, n = 0, 0
    for q in range(nq):
        for r in range(int(counts[q])):
            want = orr.cross_encoder_inputs(queries[q], passages[int(cand[q, r]) - id_base], max_length, family, cls,
                                            sep, pad_id=pos_offset - 1 if family == "roberta" else 0)
            s = slice(int(cu[p]), int(cu[p + 1]))
            assert (ids[s], types[s], pos[s]) == want, (q, r)
            assert int(got["slot_len"][q, r]) == len(want[0]) <= max_length
            p += 1
            n += 1
        assert got["slot_len"][q, int(counts[q]):].eq(0).all()
    assert n == got["P"] and n > 1000


@pytest.mark.parametrize("sep_prompt", [(1, 9), (2, 5), (0, 4), (1, 0), (0, 0)])
@pytest.mark.parametrize("max_length", ["min", 16, 50, 64])
def test_llm_pack_matches_get_inputs(sep_prompt, max_length):
    n_sep, n_prompt = sep_prompt
    max_length = pr.llm_min_max_length(n_sep) if max_length == "min" else max_length
    rng = np.random.default_rng([n_sep, n_prompt, max_length])
    nq, k, n_docs, id_base = 36, 45, 250, 7
    queries, passages, cand, counts = _case(rng, nq, k, n_docs, max_length, id_base=id_base, extra_cols=3)
    sep, prompt, bos = rng.integers(4, 900, n_sep).tolist(), rng.integers(4, 900, n_prompt).tolist(), 1
    (qp, qt), (pp, pt) = _csr(queries), _csr(passages)
    got = pr.llm_pack(qp, qt, pp, pt, cand, counts, k, id_base, torch.tensor(sep, dtype=torch.int32),
                      torch.tensor(prompt, dtype=torch.int32), bos, max_length)
    cu, ids, qlen = got["cu"], got["ids"].tolist(), got["query_len"].tolist()
    assert cu.numel() == nq * k + 1 and got["T"] == len(ids) == int(cu[-1])
    n = 0
    for q in range(nq):
        c = int(counts[q])
        want, want_ql, _ = ort.rerank_inputs(queries[q], [passages[int(d) - id_base] for d in cand[q, :c]], sep,
                                             prompt, bos, max_length)
        for r in range(k):
            p = q * k + r
            s = ids[int(cu[p]):int(cu[p + 1])]
            if r < c:
                assert s == want[r] and qlen[p] == want_ql[r], (q, r)
                n += 1
            else:
                assert s == [] and qlen[p] == 0
    assert n > 600
    out = PackedRerankInput(ids=got["ids"], cu=cu.to(torch.int32), query_len=got["query_len"],
                            prompt_len=n_sep + n_prompt, n_queries=nq, k=k)
    assert list(out.slices(32)) == pr.llm_slices(nq, k)


def test_slices_and_smallest_max_lengths():
    assert pr.llm_slices(2, 70) == [(0, 0, 32), (0, 32, 64), (0, 64, 70), (1, 70, 102), (1, 102, 134),
                                    (1, 134, 140)]
    assert pr.llm_slices(3, 32) == [(0, 0, 32), (1, 32, 64), (2, 64, 96)]
    assert [pr.llm_min_max_length(s) for s in (0, 1, 2, 3, 6)] == [8, 8, 9, 13, 25]
    one = torch.zeros(2, dtype=torch.int64)
    cand, cnt = torch.zeros(1, 1, dtype=torch.int32), torch.ones(1, dtype=torch.int32)
    for n_sep in (0, 1, 2, 3, 6):
        m = pr.llm_min_max_length(n_sep)
        pr.llm_plan(one[:2], one[:2], cand, cnt, 1, 0, n_sep, 0, m)
        with pytest.raises(ValueError, match="no room"):
            pr.llm_plan(one[:2], one[:2], cand, cnt, 1, 0, n_sep, 0, m - 1)
    pr.cross_plan(one, one, cand, cnt, 1, 0, 2, 4)
    with pytest.raises(ValueError, match="no room"):
        pr.cross_plan(one, one, cand, cnt, 1, 0, 2, 3)


def test_out_of_range_ids_are_refused_inside_the_count_only():
    qp, pp = torch.tensor([0, 2, 3]), torch.tensor([0, 4, 9, 9])                 # 2 queries, 3 passages
    base = 100
    for bad in (base - 1, base + 3, -1):
        cand = torch.tensor([[base, bad], [base + 2, base + 1]], dtype=torch.int32)
        for plan in (lambda c, n: pr.cross_plan(qp, pp, c, n, 2, base, 1, 16),
                     lambda c, n: pr.llm_plan(qp, pp, c, n, 2, base, 1, 0, 16)):
            with pytest.raises(ValueError, match="outside"):
                plan(cand, torch.tensor([2, 2]))
            plan(cand, torch.tensor([1, 2]))                                      # padding past the count
    got = pr.cross_plan(qp[:2], pp, torch.tensor([[base, base + 3]], dtype=torch.int32), torch.tensor([1]), 2, base,
                        1, 16)
    assert got["P"] == 1 and got["slot_len"].tolist() == [[3 + 2 + 4, 0]]
