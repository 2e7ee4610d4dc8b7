"""CPU: the BM25-Extract compressor's oracle against a published vector, the exact idf table the kernel reads, the
host packing, the overlay, and negative controls: a numpy restatement of csrc/bm25_extract.cu's steps that matches
the oracle, and four mistakes a kernel could make, each of which changes a constructed answer."""
import math
import subprocess
import sys
import textwrap
from pathlib import Path

import numpy as np
import pytest

from easyrag_b200 import batched
from easyrag_b200.compress import ContextCompressor, pack, split_sentences
from oracle import compress as oc

ROOT = Path(__file__).resolve().parent.parent
K1, B, EPS = 1.5, 0.75, 0.25

# rank_bm25's README: corpus, query "windy London", get_scores -> [0, 0.93729472, 0]
README = ["Hello there good man!", "It is quite windy in London", "How is the weather today?"]
README_TOKS = [s.split(" ") for s in README]
README_Q = "windy London".split(" ")


def test_oracle_matches_the_rank_bm25_readme_vector():
    sc = oc.scores(README_Q, README_TOKS, 0)
    assert np.allclose(sc, [0.0, 0.93729472, 0.0], rtol=0, atol=5e-9)
    ctx = " ".join(README)                                       # 75 characters; sentences 21 / 27 / 25
    assert len(ctx) == 75
    # order: sentence 1 (0.937), then the zero scores by index descending: 2, 0; running sums 27, 52, 73
    for rate, want in [(0.0, [1]), (0.3, [1]), (0.5, [1, 2]), (0.9, [0, 1, 2]), (1.0, [0, 1, 2]), (1.5, [0, 1, 2])]:
        for literal in (False, True):
            out = oc.compress(README_Q, README_TOKS, README, len(ctx), rate, 0, literal)
            assert out == "".join(README[i] for i in want), (rate, literal)
    # an exact boundary: 54 * 0.5 == 27.0 == the first sentence's characters, so it alone is kept
    assert oc.kept(sc, README, 54, 0.5) == [1]


def test_log_half_table_gives_python_idf_exactly():
    L = batched.log_half_table(5001)
    for N in range(1, 5001):
        n = np.arange(1, N + 1)
        want = np.array([math.log(N - k + 0.5) - math.log(k + 0.5) for k in range(1, N + 1)])
        assert (L[N - n] - L[n]).tobytes() == want.tobytes(), N


# ------------------------------------------------------------------ numpy restatement of the kernel's steps
def model(q_ids, sents, chars, ctx_len, rate, bm25_type=0, strict=False, ties_ascending=False,
          idf_for_absent=False, sorted_idf_sum=False):
    """Scores and kept indices of one group, as bm25_extract_kernel computes them (ids of a batch vocabulary)."""
    N = len(sents)
    T = sum(len(x) for x in sents)
    df, first = {}, {}
    pos = 0
    for s, toks in enumerate(sents):
        for t in toks:
            first.setdefault(t, pos)
            pos += 1
        for t in set(toks):
            df[t] = df.get(t, 0) + 1
    L = batched.log_half_table(N + 2)
    terms = sorted(df) if sorted_idf_sum else sorted(df, key=first.get)
    extra = [t for t in dict.fromkeys(q_ids) if t >= 0 and t not in df] if idf_for_absent else []
    idf_sum = 0.0
    for t in terms:
        idf_sum += L[N - df[t]] - L[df[t]]
    for t in extra:
        idf_sum += L[N] - L[0]
    avg = idf_sum / (len(terms) + len(extra)) if terms else 0.0
    avgdl = T / N
    kd = [K1 * ((1 - B) + (B * len(x)) / avgdl) for x in sents]
    acc = np.zeros(N, dtype=np.float64 if bm25_type == 0 else np.float32)
    for t in q_ids:
        if t < 0 or t not in df:
            continue
        if bm25_type == 0:
            idf = L[N - df[t]] - L[df[t]]
            idf = EPS * avg if idf < 0 else idf
        else:
            idf = float(np.float32(math.log(1 + (N - df[t] + 0.5) / (df[t] + 0.5))))
        for s, toks in enumerate(sents):
            tf = toks.count(t)
            if tf:
                w = idf * ((tf * (K1 + 1 if bm25_type == 0 else 1.0)) / (tf + kd[s]))
                acc[s] = acc[s] + (w if bm25_type == 0 else np.float32(w))
    order = sorted(range(N), key=lambda s: (-acc[s], s if ties_ascending else -s))
    thr = ctx_len * rate
    run, keep = 0, []
    for s in order:
        keep.append(s)
        run += chars[s]
        if (run > thr) if strict else (run >= thr):
            break
    return acc, sorted(keep)


def _ids(groups):
    vocab = {}
    return [[[vocab.setdefault(w, len(vocab)) for w in s] for s in g] for g in groups], vocab


def test_model_matches_the_oracle_on_random_groups():
    rng = np.random.default_rng(5)
    for case in range(150):
        n = int(rng.integers(1, 30))
        words = [f"w{i}" for i in range(int(rng.integers(2, 25)))]
        sents = [[words[j] for j in rng.integers(0, len(words), int(rng.integers(0, 12)))] for _ in range(n)]
        if not any(sents):
            sents[0] = ["w0"]
        query = [words[j] for j in rng.integers(0, len(words), int(rng.integers(1, 6)))] + ["unknown"]
        texts = ["x" * int(rng.integers(1, 40)) for _ in range(n)]
        ctx = int(sum(len(t) for t in texts) + rng.integers(0, 20))
        rate = float(rng.choice([0.0, 0.25, 0.5, 0.7, 1.0, 1.2]))
        [ids], vocab = _ids([sents])
        q_ids = [vocab.get(w, -1) for w in query]
        for bt in (0, 1):
            acc, keep = model(q_ids, ids, [len(t) for t in texts], ctx, rate, bt)
            ref = oc.scores(query, sents, bt)
            assert acc.tobytes() == ref.tobytes(), (case, bt)
            assert keep == oc.kept(ref, texts, ctx, rate), (case, bt)


def test_negative_controls_change_constructed_answers():
    [ids], vocab = _ids([README_TOKS])
    q = [vocab[w] for w in README_Q]
    chars = [len(s) for s in README]
    # '>' instead of '>=' at an exact boundary: 54 * 0.5 == 27 == the best sentence's characters
    assert model(q, ids, chars, 54, 0.5)[1] == [1] == oc.kept(oc.scores(README_Q, README_TOKS), README, 54, 0.5)
    assert model(q, ids, chars, 54, 0.5, strict=True)[1] == [1, 2]
    # ties ordered by index ascending: all scores 0, rate 0 keeps one sentence, the last one
    assert model([], ids, chars, 75, 0.0)[1] == [2]
    assert model([], ids, chars, 75, 0.0, ties_ascending=True)[1] == [0]
    # idf for a query term of the batch vocabulary that this group lacks: "a" is in every sentence (negative idf,
    # floored to epsilon * mean idf); counting absent "z" among the group's terms moves the mean
    sents = [["a", "b"], ["a", "c"], ["a", "a", "d"]]
    [g_ids], v2 = _ids([sents])
    v2["z"] = len(v2)
    qa = [v2["a"], v2["z"]]
    ch = [10, 10, 10]
    right = model(qa, g_ids, ch, 30, 0.5)[0]
    assert right.tobytes() == oc.scores(["a", "z"], sents).tobytes()
    assert model(qa, g_ids, ch, 30, 0.5, idf_for_absent=True)[0].tobytes() != right.tobytes()
    # idf_sum in sorted rather than first-seen term order: the float64 sum rounds differently for some group
    rng = np.random.default_rng(11)
    for trial in range(2000):
        n = int(rng.integers(3, 12))
        perm = rng.permutation(60)                        # term ids unrelated to first-seen order
        sents = [[int(perm[j]) for j in rng.integers(0, 40, int(rng.integers(1, 9)))] for _ in range(n)]
        common = int(perm[0])
        sents = [s + [common] for s in sents]             # in every sentence: negative idf, floored
        a = model([common], sents, [5] * n, 10, 0.5)[0]
        b = model([common], sents, [5] * n, 10, 0.5, sorted_idf_sum=True)[0]
        if a.tobytes() != b.tobytes():
            ref = oc.scores([str(common)], [[str(t) for t in s] for s in sents])
            assert a.tobytes() == ref.tobytes()
            break
    else:
        pytest.fail("no group found where the idf summation order changes a score")


def test_pack_matches_a_per_group_restatement_and_ignores_neighbours():
    rng = np.random.default_rng(3)
    words = [f"t{i}" for i in range(40)]
    groups = []
    for g in range(12):
        sents = [[words[j] for j in rng.integers(0, 40, int(rng.integers(0, 7)))] for _ in range(int(rng.integers(1, 6)))]
        texts = [" ".join(s) + "." for s in sents]
        query = [words[j] for j in rng.integers(0, 40, 4)] + ["nowhere"]
        groups.append((query, sents, texts, "  ".join(texts)))

    def decode(p, g):
        inv = {v: k for k, v in p.vocab.items()}
        s0, s1 = p.sent_ptr[g], p.sent_ptr[g + 1]
        sents = [[inv[int(t)] for t in p.tokens[p.tok_ptr[s]:p.tok_ptr[s + 1]]] for s in range(s0, s1)]
        q = [inv.get(int(t)) for t in p.q_tokens[p.q_ptr[g]:p.q_ptr[g + 1]]]
        return sents, q, p.sent_chars[s0:s1].tolist(), int(p.ctx_chars[g])

    qs, ss, ts, cs = zip(*groups)
    p = pack(qs, ss, ts, cs)
    assert p.tokens.dtype == np.int32 and p.tok_ptr[-1] == p.tokens.size and p.sent_ptr[-1] == p.tok_ptr.size - 1
    for g, (query, sents, texts, ctx) in enumerate(groups):
        alone = pack([query], [sents], [texts], [ctx])
        d_all, d_one = decode(p, g), decode(alone, 0)
        assert d_all[0] == d_one[0] == sents
        assert d_all[2] == d_one[2] == [len(t) for t in texts] and d_all[3] == d_one[3] == len(ctx)
        own = {w for s in sents for w in s}
        # a query token keeps its string when its group has it; otherwise it has no postings in the group
        for w, a, o in zip(query, d_all[1], d_one[1]):
            assert o == (w if w in own else None)
            assert a == (w if w in p.vocab else None)


def test_compressor_construction_and_splitting():
    with pytest.raises(NotImplementedError):
        ContextCompressor("llmlingua", 0.5)
    with pytest.raises(NotImplementedError):
        ContextCompressor("longllmlingua", 0.5)
    c = ContextCompressor("bm25_extract", 0.5, None, splitter=lambda t: t.split("|"))
    assert c.split(["a| b |  |c"]) == [["a", "b", "c"]]
    assert split_sentences(" | ", c.splitter) == []
    assert ContextCompressor.join([["a", "b", "c"], ["d"]], np.array([1, 0, 1, 1], dtype=np.uint8)) == ["ac", "d"]


def test_overlay_resolves_compressors_to_easyrag_b200(tmp_path):
    ref = tmp_path / "src" / "easyrag"
    for d in (ref, ref / "custom", ref / "pipeline"):
        d.mkdir(parents=True, exist_ok=True)
        (d / "__init__.py").write_text("")
    (ref / "custom" / "compressors.py").write_text("WHO = 'reference'\nclass ContextCompressor: pass\n")
    (ref / "custom" / "rerankers.py").write_text("WHO = 'reference'\n")
    (ref / "pipeline" / "rag.py").write_text("def cut_sent(para):\n    return para.split('#')\n")
    (ref / "pipeline" / "pipeline.py").write_text(textwrap.dedent('''
        from ..custom.compressors import ContextCompressor
        from ..custom.rerankers import WHO
    '''))
    code = textwrap.dedent(f'''
        import sys
        sys.path[:0] = [{str(ROOT / "shim")!r}, {str(tmp_path / "src")!r}, {str(ROOT)!r}]
        import easyrag.pipeline.pipeline as p
        import easyrag_b200.compress as ours
        assert p.ContextCompressor is ours.ContextCompressor and p.WHO == "reference"
        c = p.ContextCompressor("bm25_extract", 0.5, None)
        assert c.split(["x# y#"]) == [["x", "y"]]        # the reference's own cut_sent, found lazily
        print("overlay-ok")
    ''')
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "overlay-ok" in r.stdout, r.stderr[-2000:]
