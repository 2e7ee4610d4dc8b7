"""Host side of the device interner (easyrag_b200/vocab.py): the NUL join and its fallback triggers, the chunk
planner, and the dict restatement the GPU tests use as their oracle, pinned to the host functions it restates."""
from itertools import chain

import numpy as np
import pytest

from easyrag_b200 import vocab as vocab_mod
from easyrag_b200.compress import pack
from easyrag_b200.retrievers import _canon_ids, _encode_corpus
from easyrag_b200.vocab import NotJoinable, iter_chunks, join_strings, plan_chunks

import _vocab_ref as ref


def test_join_round_trips_multibyte_and_empty_strings():
    strings = ["", "a", "", "词语", "ß", "😀x", ""]
    data, n = join_strings(strings)
    assert n == len(strings)
    assert data == "\0".join(strings).encode("utf-8")
    assert [s.decode("utf-8") for s in data.split(b"\0")] == strings
    assert join_strings([]) == (b"", 0)
    assert join_strings([""]) == (b"", 1)            # one empty string: same bytes as no string, told apart by n


@pytest.mark.parametrize("bad", [["a", "b\0c"], ["\0"], ["a", 3], [b"bytes"], ["ok", "\ud800"]])
def test_join_refuses_what_it_cannot_represent(bad):
    with pytest.raises(NotJoinable):
        join_strings(bad)


def test_plan_covers_groups_in_order_and_keeps_the_bound():
    rng = np.random.default_rng(0)
    for trial in range(300):
        counts = rng.integers(0, 12, int(rng.integers(0, 60)))
        if trial % 5 == 0 and counts.size:
            counts[int(rng.integers(0, counts.size))] = 40             # a group larger than the bound
        cap = int(rng.integers(1, 30))
        plan = plan_chunks(counts, cap)
        assert [a for a, _ in plan] == ([0] + [b for _, b in plan[:-1]] if plan else [])    # consecutive, in order
        assert (plan[-1][1] if plan else 0) == counts.size
        for a, b in plan:
            assert b > a
            assert counts[a:b].sum() <= cap or b - a == 1


def test_chunks_never_split_a_group_and_keep_the_byte_bound():
    rng = np.random.default_rng(1)
    words = ["", "x", "词", "长" * 50, "abc"]
    for _ in range(100):
        groups = [[words[int(i)] for i in rng.integers(0, len(words), int(rng.integers(0, 9)))]
                  for _ in range(int(rng.integers(0, 40)))]
        counts = np.asarray([len(g) for g in groups], dtype=np.int64)
        max_strings, max_bytes = int(rng.integers(1, 20)), int(rng.integers(1, 400))
        parts, nxt = [], 0
        for a, b, data, n in iter_chunks(groups, counts, max_strings, max_bytes):
            assert a == nxt and b > a
            nxt = b
            assert n == counts[a:b].sum() and data == "\0".join(chain.from_iterable(groups[a:b])).encode()
            assert (len(data) <= max_bytes and n <= max_strings) or b - a == 1
            parts.append((a, b))
        assert nxt == len(groups)
    flat = ["a", "bb", "词"] * 7
    got = [(a, b) for a, b, _, _ in iter_chunks(flat, np.ones(len(flat), np.int64), 4, 5, flat=True)]
    assert got[0][0] == 0 and got[-1][1] == len(flat) and all(b - a <= 4 for a, b in got)


def test_the_oracle_restates_the_host_functions():
    rng = np.random.default_rng(2)
    pool = ["", "a", "词", "词语", "b", "the", "x" * 40]
    docs = [[pool[int(i)] for i in rng.integers(0, len(pool), int(rng.integers(0, 12)))] for _ in range(50)]
    ids, ptr, d, first, seen = ref.intern(docs)
    vocab, tokens, doc_ptr = _encode_corpus(docs)
    assert list(d.items()) == list(vocab.items())
    assert np.array_equal(ids, tokens.numpy()) and np.array_equal(ptr, doc_ptr.numpy())
    flat = list(chain.from_iterable(docs))
    assert seen == len(flat)
    assert np.array_equal(np.asarray(first)[ids], ref.first_index(flat))
    assert np.array_equal(ref.first_index(flat), _canon_ids(flat))
    # continuing a call equals one call over both halves
    a = ref.intern(docs[:20])
    b = ref.intern(docs[20:], a[2], a[3], a[4])
    assert np.array_equal(np.concatenate([a[0], b[0]]), ids) and b[2] == d and b[3] == first
    # compress.pack: interned sentence tokens, then the queries looked up without inserting
    queries = [["a", "zz", "词语"], [], ["the", "a"]]
    sents = [docs[0:3], [docs[3]], docs[4:9]]
    p = pack(queries, sents, [[""] * len(s) for s in sents], ["", "", ""])
    s_ids, s_ptr, s_d, _, _ = ref.intern([t for s in sents for t in s])
    assert np.array_equal(p.tokens, s_ids) and np.array_equal(p.tok_ptr, s_ptr) and p.vocab == s_d
    assert np.array_equal(p.q_tokens, ref.lookup(queries, s_d))


def test_the_oracle_tells_orders_apart():
    """Negative control: a vocabulary numbered in sorted order is a different answer."""
    docs = [["b", "a", "c"], ["a", "d"]]
    ids, _, d, _, _ = ref.intern(docs)
    sorted_ids = {s: i for i, s in enumerate(sorted(d))}
    assert not np.array_equal(ids, [sorted_ids[s] for s in chain.from_iterable(docs)])


@pytest.mark.parametrize("flat", [False, True])
def test_no_join_covers_more_than_one_bounded_chunk(monkeypatch, flat):
    """The byte bound is planned before joining: every join is one yielded chunk, within the bound unless it is one
    group, and each string is joined once (several-KB texts, one per group, as first_index plans them)."""
    calls = []

    def spy(strings):
        out = join_strings(strings)
        calls.append((len(out[0]), out[1]))
        return out
    monkeypatch.setattr(vocab_mod, "join_strings", spy)
    rng = np.random.default_rng(3)
    texts = ["词" * int(n) if n % 2 else "a" * int(n) for n in rng.integers(0, 6000, 400)]
    groups = texts if flat else [texts[i:i + int(k)] for i, k in zip(range(0, 400, 4), rng.integers(0, 5, 100))]
    counts = np.ones(len(groups), np.int64) if flat else np.asarray([len(g) for g in groups], np.int64)
    max_bytes = 20_000
    got = list(iter_chunks(groups, counts, 1000, max_bytes, flat))
    assert len(calls) == len(got) and sum(n for _, n in calls) == counts.sum()
    for (nb, n), (a, b, data, n2) in zip(calls, got):
        assert nb == len(data) and n == n2
        assert nb <= max_bytes or b - a == 1
    whole = list(groups if flat else chain.from_iterable(groups))
    joined = [x for _, _, d, n in got for x in (d.decode().split("\0") if n else [])]
    assert joined == whole
