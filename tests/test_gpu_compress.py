"""GPU: BM25-Extract compression (csrc/bm25_extract.cu) against BM25Retriever.get_scores(query, sentences) and the
oracle (oracle/compress.py), byte for byte, for both bm25_type values."""
import numpy as np
import pytest
import torch

from easyrag_b200 import batched
from easyrag_b200.compress import ContextCompressor, pack
from easyrag_b200.retrievers import BM25Retriever
from easyrag_b200.schema import TextNode
from oracle import compress as oc

pytestmark = pytest.mark.gpu
STOP = ["the", "of"]


class Tok:
    @staticmethod
    def cut(text):
        return [w for w in text.split(" ") if w]


def retriever(bt):
    return BM25Retriever([TextNode(text="seed words", id_="n0")], Tok(), stopwords=STOP, bm25_type=bt)


def compressor(bt, rate=0.5):
    return ContextCompressor("bm25_extract", rate, retriever(bt), splitter=lambda c: c.split("\n"))


def synth(rng, G, max_sents=400, max_tok=60, vocab=3000):
    queries, contexts = [], []
    for g in range(G):
        n = int(rng.integers(1, max_sents + 1))
        words = rng.integers(0, vocab, int(rng.integers(5, 200)))
        sents = []
        for i in range(n):
            u = rng.random()
            if u < 0.08:
                sents.append(" ".join(rng.choice(STOP, int(rng.integers(1, 4)))))      # no tokens left
            elif u < 0.13 and sents:
                sents.append(sents[int(rng.integers(0, len(sents)))])                 # a duplicate sentence
            else:
                k = int(rng.integers(1, max_tok + 1))
                sents.append(" ".join(f"w{w}" for w in rng.choice(words, k)))
        q = [f"w{w}" for w in rng.choice(words, int(rng.integers(1, 8)))]
        q = q + q[:1] + ["nowhere", f"w{int(rng.integers(0, vocab))}", "the"]       # duplicate, unknown, stop word
        rng.shuffle(q)
        queries.append(" ".join(q))
        contexts.append("\n".join(sents) + " " * int(rng.integers(0, 5)))
    return queries, contexts


def run(comp, queries, contexts):
    sents = comp.split(contexts)
    qt, st = comp.tokenize(queries, sents)
    p = pack(qt, st, sents, contexts)
    keep, counts, sc = comp.run(p, scores=True)
    return sents, qt, st, p, keep, counts, sc.cpu().numpy()


def check_groups(comp, queries, contexts, literal=True, get_scores=True):
    sents, qt, st, p, keep, counts, sc = run(comp, queries, contexts)
    bt = comp.bm25_retriever.bm25_type
    out = comp.join(sents, keep)
    for g in range(len(contexts)):
        s0, s1 = p.sent_ptr[g], p.sent_ptr[g + 1]
        got = comp.bm25_retriever.get_scores(queries[g], sents[g]) if get_scores or not any(st[g]) else None
        # no token at all: rank_bm25 raises (idf_sum / 0); the result is get_scores(query, docs)'s zeros
        ref = oc.scores(qt[g], st[g], bt) if any(st[g]) else got
        assert sc[s0:s1].tobytes() == ref.tobytes(), g
        if got is not None:
            assert sc[s0:s1].tobytes() == got.tobytes(), g
        want = oc.kept(ref, sents[g], len(contexts[g]), comp.rate)
        assert np.nonzero(keep[s0:s1])[0].tolist() == want and counts[g] == len(want), g
        assert out[g] == "".join(sents[g][i] for i in want)
        if literal and np.unique(ref).size == ref.size:
            assert oc.kept(ref, sents[g], len(contexts[g]), comp.rate, literal=True) == want
    return sc, keep


@pytest.mark.parametrize("bt", [0, 1])
def test_scores_keep_and_strings_on_2000_groups(bt):
    rng = np.random.default_rng(100 + bt)
    q, c = synth(rng, 2000)
    check_groups(compressor(bt, 0.5), q, c)


@pytest.mark.parametrize("bt", [0, 1])
def test_edge_cases(bt):
    # idf exactly 0 (N = 2n), a negative mean idf (every term in every sentence), rates 0, 1 and above 1
    cases = [("a", "a b\nc d"), ("a b", "a b\nb a\na a b"), ("a", "a\na\na b")]
    for rate in (0.0, 0.3, 1.0, 1.7):
        comp = compressor(bt, rate)
        check_groups(comp, [x for x, _ in cases], [y for _, y in cases])
    sc = run(compressor(bt), ["a b"], ["a b\nb a\na a b"])[-1]
    if bt == 0:
        assert (sc < 0).all()                                 # epsilon * negative mean idf
    # no sentence: ZeroDivisionError in compress, count -1 in the batched call
    with pytest.raises(ZeroDivisionError):
        compressor(bt).compress("a", " \n  ")
    res = batched.bm25_extract(np.array([0, 0, 1]), np.array([0, 1]), np.array([0]), np.array([1]), np.array([0, 1]),
                               np.array([0, 0, 1]), np.array([0]), 1, bm25_type=bt)
    assert res.counts.cpu().tolist() == [-1, 1] and res.keep.cpu().tolist() == [1]
    # sentences that all tokenize to nothing: get_scores(query, docs) returns zeros (rank_bm25 itself would raise);
    # recorded on the H100: zeros, kept in index-descending order until 17 * 0.5 characters
    comp = compressor(bt)
    sents, _, _, _, keep, counts, sc = run(comp, ["a the"], ["the\nof the\nthe of"])
    assert sc.tolist() == [0.0, 0.0, 0.0]
    assert sc.tobytes() == comp.bm25_retriever.get_scores("a the", sents[0]).tobytes()
    assert keep.tolist() == [0, 1, 1] and counts.tolist() == [2]
    assert comp.compress("a the", "the\nof the\nthe of") == "of thethe of"


@pytest.mark.parametrize("bt", [0, 1])
def test_cap_boundaries(bt):
    cap_t, cap_s = batched.extract_caps()
    rng = np.random.default_rng(7)
    qs, cs = [], []
    for t in (cap_t - 1, cap_t, cap_t + 1):
        n = 97
        lens = np.full(n, t // n)
        lens[: t - lens.sum()] += 1
        cs.append("\n".join(" ".join(f"w{w}" for w in rng.integers(0, 400, k)) for k in lens))
        qs.append("w1 w2 w3 w2 w399")
    for n in (cap_s - 1, cap_s, cap_s + 1):
        cs.append("\n".join(f"w{w}" for w in rng.integers(0, 300, n)))
        qs.append("w5 w7 w11 nowhere")
    check_groups(compressor(bt, 0.5), qs, cs, literal=True)


@pytest.mark.parametrize("bt", [0, 1])
def test_batch_independence(bt):
    rng = np.random.default_rng(9)
    q, c = synth(rng, 40, max_sents=60)
    comp = compressor(bt)
    _, _, _, p, keep, _, sc = run(comp, q, c)
    perm = rng.permutation(40)
    idx = list(perm) + list(perm[:10])                         # shuffled, with repeats
    _, _, _, p2, keep2, _, sc2 = run(comp, [q[i] for i in idx], [c[i] for i in idx])
    for j, g in enumerate(idx):
        a, b = slice(p.sent_ptr[g], p.sent_ptr[g + 1]), slice(p2.sent_ptr[j], p2.sent_ptr[j + 1])
        assert sc[a].tobytes() == sc2[b].tobytes() and keep[a].tobytes() == keep2[b].tobytes()
    for g in (0, 17, 39):
        _, _, _, _, k1, _, s1 = run(comp, [q[g]], [c[g]])
        a = slice(p.sent_ptr[g], p.sent_ptr[g + 1])
        assert s1.tobytes() == sc[a].tobytes() and k1.tobytes() == keep[a].tobytes()


@pytest.mark.parametrize("bt", [0, 1])
def test_scale_10000_groups(bt):
    """Joined top-6 chunks: about 200 sentences and 6k tokens per group, ids generated directly."""
    rng = np.random.default_rng(50 + bt)
    G, V = 10_000, 60_000
    n_sent = rng.integers(180, 221, G)
    sent_ptr = np.concatenate([[0], np.cumsum(n_sent)]).astype(np.int64)
    lens = rng.integers(0, 61, int(sent_ptr[-1]))
    tok_ptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    tokens = np.minimum(rng.zipf(1.3, int(tok_ptr[-1])) - 1, V - 1).astype(np.int32)
    chars = (lens * 5 + rng.integers(1, 9, lens.size)).astype(np.int64)
    ctx = np.array([chars[sent_ptr[g]:sent_ptr[g + 1]].sum() + 200 for g in range(G)], dtype=np.int64)
    nq = rng.integers(3, 16, G)
    q_ptr = np.concatenate([[0], np.cumsum(nq)]).astype(np.int64)
    q_tok = np.minimum(rng.zipf(1.3, int(q_ptr[-1])) - 1, V - 1).astype(np.int32)
    q_tok[rng.random(q_tok.size) < 0.05] = -1
    res = batched.bm25_extract(sent_ptr, tok_ptr, tokens, chars, ctx, q_ptr, q_tok, V, rate=0.5, bm25_type=bt,
                               scores=True)
    sc, keep, counts = res.scores.cpu().numpy(), res.keep.cpu().numpy(), res.counts.cpu().numpy()
    r = retriever(bt)
    for i, g in enumerate(rng.choice(G, 60, replace=False)):
        s0, s1 = sent_ptr[g], sent_ptr[g + 1]
        sents = [tokens[tok_ptr[s]:tok_ptr[s + 1]].tolist() for s in range(s0, s1)]
        q = q_tok[q_ptr[g]:q_ptr[g + 1]].tolist()
        ref = oc.scores(q, sents, bt)
        assert sc[s0:s1].tobytes() == ref.tobytes(), g
        if i < 20:
            docs = [" ".join(f"w{t}" for t in s) for s in sents]
            got = r.get_scores(" ".join(f"w{t}" if t >= 0 else "nowhere" for t in q), docs)
            assert sc[s0:s1].tobytes() == got.tobytes(), g
        texts = ["x" * int(c) for c in chars[s0:s1]]
        want = oc.kept(ref, texts, int(ctx[g]), 0.5)
        assert np.nonzero(keep[s0:s1])[0].tolist() == want and counts[g] == len(want), g


@pytest.mark.parametrize("bt", [0, 1])
def test_drop_in_compress_and_compress_batch(bt):
    rng = np.random.default_rng(31)
    q, c = synth(rng, 12, max_sents=30)
    comp = compressor(bt, 0.4)
    outs = comp.compress_batch(q, c)
    for g in range(12):
        sents = comp.split([c[g]])[0]
        qt, st = comp.tokenize([q[g]], [sents])
        want = oc.compress(qt[0], st[0], sents, len(c[g]), 0.4, bt)
        assert outs[g] == want == comp.compress(q[g], c[g])
