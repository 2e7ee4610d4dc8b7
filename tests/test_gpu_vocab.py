"""GPU: the device interner (csrc/vocab.cu, easyrag_b200/vocab.py) against the dict restatement in _vocab_ref, and
the two call sites that use it (BM25Retriever, ContextCompressor.compress_batch) against their host paths."""
import copy
from itertools import chain

import numpy as np
import pytest
import torch

from easyrag_b200 import _lib
from easyrag_b200.compress import ContextCompressor, pack, pack_device
from easyrag_b200.retrievers import BM25Retriever, _canon_ids, _encode_corpus
from easyrag_b200.schema import QueryBundle, TextNode
from easyrag_b200.vocab import HostFallbackWarning, Vocabulary, join_strings

import _vocab_ref as ref

pytestmark = pytest.mark.gpu


@pytest.fixture
def hash_bits():
    """Set the hash bits of vocabularies made in the test; back to the default 64 afterwards."""
    def set_bits(n):
        _lib.check(_lib.lib().ezr_vocab_set_hash_bits(n), "ezr_vocab_set_hash_bits")
    yield set_bits
    set_bits(64)


def pseudo_chinese(n, rng, max_chars=4):
    """n distinct-ish multi-byte tokens: 1..max_chars CJK characters (3 UTF-8 bytes each), some ASCII mixed in."""
    out = []
    for i in range(n):
        k = int(rng.integers(1, max_chars + 1))
        s = "".join(chr(0x4E00 + int(c)) for c in rng.integers(0, 2000, k))
        out.append(s if i % 7 else s + f"{i}")
    return list(dict.fromkeys(out))


def zipf_docs(rng, n_docs, mean_len, pool):
    lens = rng.poisson(mean_len, n_docs)
    ids = np.minimum(rng.zipf(1.2, int(lens.sum())) - 1, len(pool) - 1)
    flat = np.asarray(pool, dtype=object)[ids].tolist()
    off = np.concatenate([[0], np.cumsum(lens)])
    return [flat[off[i]:off[i + 1]] for i in range(n_docs)]


def check_same(v, groups, ids, ptr, want):
    """ids / ptr / dict of one fresh intern against the oracle ``want`` = ref.intern(groups)."""
    assert np.array_equal(ptr.numpy(), want[1])
    assert np.array_equal(ids.cpu().numpy(), want[0]), "ids differ"
    assert len(v) == len(want[2])
    assert list(v.to_dict().items()) == list(want[2].items())


def test_zipf_multibyte_corpus():
    rng = np.random.default_rng(0)
    docs = zipf_docs(rng, 3000, 40, pseudo_chinese(20000, rng))
    v = Vocabulary()
    ids, ptr = v.intern(docs)
    check_same(v, docs, ids, ptr, ref.intern(docs))


def test_empty_strings_groups_and_long_strings():
    rng = np.random.default_rng(1)
    lengths = [0, 1, 2, 31, 32, 33, 63, 64, 65, 1000, 4096, 16384]
    base = ["".join(chr(97 + int(c)) for c in rng.integers(0, 3, n)) for n in lengths]
    near = [s[:-1] + ("b" if s.endswith("a") else "a") for s in base if s]          # same length, last byte differs
    pool = base + near + ["é" * 5000, "é" * 4999 + "e"]
    groups = [[], [""], ["", ""], []]
    for _ in range(60):
        groups.append([pool[int(i)] for i in rng.integers(0, len(pool), int(rng.integers(0, 8)))])
        if rng.random() < 0.2:
            groups.append([])
    groups.append([])
    v = Vocabulary()
    ids, ptr = v.intern(groups)
    check_same(v, groups, ids, ptr, ref.intern(groups))
    assert Vocabulary().intern([])[0].numel() == 0
    e = Vocabulary()
    ids, ptr = e.intern([[], []])
    assert ids.numel() == 0 and ptr.tolist() == [0, 0, 0] and len(e) == 0 and e.to_dict() == {}


def test_chunk_boundaries_at_every_position():
    strings = ["b", "a", "", "b", "词", "a", "", "长" * 40, "c", "词", "b", "长" * 40, "d"]
    want = ref.intern([strings])
    for cut in range(len(strings) + 1):                     # two calls on one vocabulary
        v = Vocabulary()
        i1, _ = v.intern([strings[:cut]])
        i2, _ = v.intern([strings[cut:]])
        assert torch.cat([i1, i2]).cpu().tolist() == want[0].tolist(), cut
        assert v.to_dict() == want[2]
    groups = [[s] for s in strings]
    for chunk in range(1, len(strings) + 1):                # one call, chunked by the planner
        v = Vocabulary(chunk_strings=chunk)
        ids, ptr = v.intern(groups)
        check_same(v, groups, ids, ptr, ref.intern(groups))
    v = Vocabulary(chunk_bytes=3)                           # byte bound: about a string per chunk
    ids, ptr = v.intern(groups)
    check_same(v, groups, ids, ptr, ref.intern(groups))


def test_table_grows_mid_stream():
    rng = np.random.default_rng(2)
    pool = [f"t{i}" for i in range(60000)]
    docs = [[pool[int(i)] for i in rng.integers(0, len(pool), 30)] for _ in range(4000)]
    v = Vocabulary(chunk_strings=5000)
    cap0 = v._cap
    ids, ptr = v.intern(docs)
    assert v._cap > 8 * cap0                                # several rehashes between chunks
    check_same(v, docs, ids, ptr, ref.intern(docs))


@pytest.mark.parametrize("bits", [64, 16, 4])
def test_hash_bits_keep_results_exact(hash_bits, bits):
    rng = np.random.default_rng(3)
    hash_bits(bits)
    pool = pseudo_chinese(1500, rng, 3) + [s * 20 for s in pseudo_chinese(100, rng, 2)]    # short and warp-path
    docs = zipf_docs(rng, 300, 20, pool)
    v = Vocabulary(chunk_strings=700)
    ids, ptr = v.intern(docs)
    assert int(v._table.view(torch.int64)[1]) == bits       # the table header records the knob
    hash_bits(64)                                           # a table keeps the bits it was made with
    want = ref.intern(docs)
    check_same(v, docs, ids, ptr, want)
    queries = [[pool[int(i)] for i in rng.integers(0, len(pool), 5)] + ["nowhere", "词" * 40] for _ in range(50)]
    q, qp = v.lookup(queries)
    assert np.array_equal(q.cpu().numpy(), ref.lookup(queries, want[2]))
    assert len(v) == len(want[2])                           # lookup inserted nothing


def test_lookup_oov_and_first_index():
    rng = np.random.default_rng(4)
    pool = pseudo_chinese(3000, rng)
    docs = zipf_docs(rng, 500, 30, pool[:2000])
    v = Vocabulary()
    v.intern(docs)
    want = ref.intern(docs)
    queries = [[pool[int(i)] for i in rng.integers(0, len(pool), int(rng.integers(0, 12)))] for _ in range(2000)]
    queries[3] = []
    q, qp = v.lookup(queries)
    assert np.array_equal(q.cpu().numpy(), ref.lookup(queries, want[2]))
    assert np.array_equal(qp.numpy(), np.concatenate([[0], np.cumsum([len(x) for x in queries])]))
    texts = [f"chunk text {int(i)} " * int(1 + i % 300) for i in rng.integers(0, 400, 3000)]   # up to several KB
    got = Vocabulary().first_index(texts)
    assert np.array_equal(got.cpu().numpy(), _canon_ids(texts))
    # a second call on the same vocabulary counts on from the first
    v2 = Vocabulary()
    v2.first_index(texts[:100])
    assert np.array_equal(v2.first_index(texts[100:]).cpu().numpy(), ref.first_index(texts)[100:])


@pytest.mark.parametrize("bad", ["nul", "int"])
def test_unjoinable_tokens_take_the_host_fallback(bad):
    tok = "a\0b" if bad == "nul" else 7
    docs = [["x", "y", "x"], ["z", tok, "x"], ["q", "y"]]
    v = Vocabulary(chunk_strings=3)                         # the first chunk runs on the device, then the fallback
    with pytest.warns(HostFallbackWarning):
        ids, ptr = v.intern(docs)
    check_same(v, docs, ids, ptr, ref.intern(docs))
    assert v._host is not None
    more = [["q", "new"]]
    ids2, _ = v.intern(more)
    want = ref.intern(docs)
    assert ids2.cpu().tolist() == ref.intern(more, want[2], want[3], want[4])[0].tolist()
    q, _ = v.lookup([["x", tok, "none"]])
    assert q.cpu().tolist() == [0, 3, -1]


def test_unjoinable_lookup_falls_back_for_that_call_only():
    docs = [["x", "y", "x"], ["z", "w"]]
    v = Vocabulary()
    v.intern(docs)
    want = ref.intern(docs)
    queries = [["x", "nope"], ["z", "a\0b", "y"], ["w"]]
    q, _ = v.lookup(queries)
    assert q.cpu().tolist() == ref.lookup(queries, want[2]).tolist()
    assert v._host is None                                  # still on the device
    more = [["new", "x"]]
    ids, _ = v.intern(more)
    assert ids.cpu().tolist() == ref.intern(more, want[2], want[3], want[4])[0].tolist()


def test_refused_chunk_leaves_the_table_as_it_was():
    """An insert whose new ids or bytes do not fit the caller's buffers returns EZR_ERR_WORKSPACE and empties the slots
    it claimed; the same vocabulary then interns on exactly as the dict does."""
    L = _lib.lib()
    docs = [[f"s{i}" for i in range(300)], ["词" * 20, "x" * 100]]
    v = Vocabulary()
    v.intern(docs)
    want = ref.intern(docs)
    chunk = ["s5", "new1", "x" * 100, "new2" * 30, "new1", "s7"]          # old and new, short and warp-path strings
    data, n = join_strings(chunk)
    v._reserve(n, len(data))
    buf = torch.frombuffer(bytearray(data), dtype=torch.uint8).to(v.device)
    ws = torch.empty(L.ezr_vocab_workspace(n, len(data)), dtype=torch.uint8, device=v.device)
    out = torch.empty(n, dtype=torch.int32, device=v.device)
    n_ids, used = int(v._state[0]), int(v._state[1])
    for id_cap, arena_cap in ((n_ids + 1, v._arena.numel()), (v._id_first.numel(), used + 3)):
        rc = L.ezr_vocab_insert(_lib.ptr(v._table), v._cap, _lib.ptr(buf), len(data), n, v._seen, _lib.ptr(v._arena),
                                arena_cap, _lib.ptr(v._arena_off), _lib.ptr(v._id_first), id_cap, v._state,
                                _lib.ptr(out), None, _lib.ptr(ws), ws.numel(), _lib.stream_ptr())
        assert rc == -3, L.ezr_last_error()
        assert (int(v._state[0]), int(v._state[1])) == (n_ids, used)
    q, _ = v.lookup([chunk])
    assert q.cpu().tolist() == ref.lookup([chunk], want[2]).tolist()          # the new strings are absent again
    ids, _ = v.intern([chunk])
    assert ids.cpu().tolist() == ref.intern([chunk], want[2], want[3], want[4])[0].tolist()
    assert list(v.to_dict().items()) == list(want[2].items())


def test_wrong_order_fails_the_comparison():
    """Negative control: the same ids with two of them swapped, or numbered in sorted order, must not pass."""
    rng = np.random.default_rng(5)
    docs = zipf_docs(rng, 200, 20, pseudo_chinese(500, rng))
    v = Vocabulary()
    ids, ptr = v.intern(docs)
    want = ref.intern(docs)
    check_same(v, docs, ids, ptr, want)
    swapped = ids.clone()
    swapped[ids == 0], swapped[ids == 1] = 1, 0
    with pytest.raises(AssertionError, match="ids differ"):
        check_same(v, docs, swapped, ptr, want)
    order = {s: i for i, s in enumerate(sorted(want[2]))}
    sorted_ids = torch.tensor([order[s] for s in chain.from_iterable(docs)], dtype=torch.int32)
    with pytest.raises(AssertionError, match="ids differ"):
        check_same(v, docs, sorted_ids, ptr, want)


def test_configs2_scale_over_1e8_tokens():
    """1M documents of about 110 tokens (1.1e8 tokens) from 200k multi-byte pool strings, in the default chunks.
    The pool strings are distinct, so the dict order is the order of each pool id's first occurrence."""
    rng = np.random.default_rng(6)
    pool = [chr(0x4E00 + i % 4000) + chr(0x4E00 + i // 4000) + "的" * (i % 3) for i in range(200000)]
    n_docs = 1_000_000
    lens = rng.integers(80, 141, n_docs)
    pid = np.minimum(rng.zipf(1.1, int(lens.sum())) - 1, len(pool) - 1)
    pid = np.where(rng.random(pid.size) < 0.3, rng.integers(0, len(pool), pid.size), pid)
    flat = np.asarray(pool, dtype=object)[pid].tolist()
    off = np.concatenate([[0], np.cumsum(lens)])
    docs = [flat[off[i]:off[i + 1]] for i in range(n_docs)]
    assert off[-1] > 1e8
    v = Vocabulary()
    ids, ptr = v.intern(docs)
    uniq, first = np.unique(pid, return_index=True)
    order = uniq[np.argsort(first)]                         # pool ids in first-seen order
    rank = np.full(len(pool), -1, dtype=np.int64)
    rank[order] = np.arange(order.size)
    assert np.array_equal(ptr.numpy(), off)
    assert np.array_equal(ids.cpu().numpy(), rank[pid])
    d = v.to_dict()
    assert len(d) == order.size and list(d) == [pool[i] for i in order]


# ------------------------------------------------------------------ call sites
class Tok:
    @staticmethod
    def cut(text):
        return [w for w in text.split(" ") if w]


def corpus_nodes(rng, n):
    pool = pseudo_chinese(3000, rng, 3) + ["the", "of"]
    texts = [" ".join(pool[int(i)] for i in np.minimum(rng.zipf(1.3, int(rng.integers(0, 40))) - 1, len(pool) - 1))
             for _ in range(n)]
    texts[5] = texts[2]                                     # duplicate texts share a canon id
    texts[9] = ""
    return [TextNode(text=t, id_=f"n{i}", metadata={"g": i % 3}) for i, t in enumerate(texts)], pool


@pytest.mark.parametrize("bm25_type", [0, 1])
def test_bm25_retriever_with_and_without_the_interner(bm25_type):
    rng = np.random.default_rng(7)
    nodes, pool = corpus_nodes(rng, 2000)
    r = BM25Retriever(nodes, Tok(), similarity_top_k=20, stopwords=["the", "of"], bm25_type=bm25_type)
    vocab, tokens, doc_ptr = _encode_corpus(r._corpus)
    assert list(r._vocab.items()) == list(vocab.items())
    assert r.canon.dtype == torch.int32 and r.canon.device.type == "cpu"
    assert np.array_equal(r.canon.numpy(), _canon_ids([n.get_content() for n in nodes]))
    host = copy.copy(r)
    host.bm25 = r._build(tokens, doc_ptr, len(vocab))
    host._vocab = vocab
    for name in ("indptr", "post_doc", "post_w", "range_off"):
        a, b = getattr(r.bm25, name), getattr(host.bm25, name)
        assert a.dtype == b.dtype and a.cpu().numpy().tobytes() == b.cpu().numpy().tobytes(), name
    for name in ("post_pk", "term_max"):
        a, b = getattr(r.bm25, name), getattr(host.bm25, name)
        assert (a is None and b is None) or a.cpu().numpy().tobytes() == b.cpu().numpy().tobytes(), name
    for i in range(40):
        q = " ".join(pool[int(j)] for j in rng.integers(0, len(pool), 4)) + " nowhere"
        got = [(n.node.node_id, n.score) for n in r.retrieve(QueryBundle(q))]
        want = [(n.node.node_id, n.score) for n in host.retrieve(QueryBundle(q))]
        assert got == want, q


@pytest.mark.parametrize("bm25_type", [0, 1])
def test_compress_batch_matches_pack_and_run(bm25_type):
    rng = np.random.default_rng(8)
    retr = BM25Retriever([TextNode(text="seed words", id_="n0")], Tok(), stopwords=["the"], bm25_type=bm25_type)
    comp = ContextCompressor("bm25_extract", 0.5, retr, splitter=lambda c: c.split("\n"))
    pool = pseudo_chinese(4000, rng, 3) + ["the"]
    queries, contexts = [], []
    for g in range(300):
        sents = [" ".join(pool[int(i)] for i in np.minimum(rng.zipf(1.3, int(rng.integers(1, 30))) - 1, len(pool) - 1))
                 for _ in range(int(rng.integers(1, 60)))]
        if g % 10 == 0:
            sents.append("the the")                           # a sentence without tokens
        contexts.append("\n".join(sents))
        queries.append(" ".join(pool[int(i)] for i in rng.integers(0, len(pool), 5)) + " nowhere")
    sents = comp.split(contexts)
    qt, st = comp.tokenize(queries, sents)
    p, d = pack(qt, st, sents, contexts), pack_device(qt, st, sents, contexts, retr.bm25.device)
    for name in ("sent_ptr", "tok_ptr", "sent_chars", "ctx_chars", "q_ptr"):
        assert np.array_equal(getattr(p, name), getattr(d, name)), name
    assert d.tokens.is_cuda and d.q_tokens.is_cuda
    assert np.array_equal(p.tokens, d.tokens.cpu().numpy()) and np.array_equal(p.q_tokens, d.q_tokens.cpu().numpy())
    assert list(p.vocab.items()) == list(d.vocab.to_dict().items())
    keep, _ = comp.run(p)
    assert comp.compress_batch(queries, contexts) == comp.join(sents, keep)
