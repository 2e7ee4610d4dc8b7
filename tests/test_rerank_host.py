"""CPU: the cross-encoder reranker's host-side contract -- pair encoding vs a real fast tokenizer, the reference's
order, chunking under a token budget, argument checks, and the failure mode without a GPU."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import rerank as orr
from easyrag_b200 import _lib, rerank
from easyrag_b200.encoder import BertConfig
from easyrag_b200.schema import NodeWithScore, QueryBundle, TextNode

N_WORDS = 64


def _fast_tokenizer(family):
    """A real ``tokenizers`` fast tokenizer built offline: WordLevel vocab of w0..w63 + the family's specials."""
    from tokenizers import Tokenizer, models, pre_tokenizers, processors
    from transformers import PreTrainedTokenizerFast
    if family == "bert":
        specials = ["[PAD]", "[UNK]", "[CLS]", "[SEP]"]
    else:
        specials = ["<s>", "<pad>", "</s>", "<unk>"]
    vocab = {t: i for i, t in enumerate(specials)}
    vocab.update({f"w{i}": len(specials) + i for i in range(N_WORDS)})
    unk = specials[1] if family == "bert" else specials[3]
    tk = Tokenizer(models.WordLevel(vocab, unk_token=unk))
    tk.pre_tokenizer = pre_tokenizers.WhitespaceSplit()
    if family == "bert":
        tk.post_processor = processors.TemplateProcessing(
            single="[CLS] $A [SEP]", pair="[CLS] $A [SEP] $B:1 [SEP]:1",
            special_tokens=[("[CLS]", vocab["[CLS]"]), ("[SEP]", vocab["[SEP]"])])
        tok = PreTrainedTokenizerFast(tokenizer_object=tk, cls_token="[CLS]", sep_token="[SEP]", pad_token="[PAD]",
                                      unk_token="[UNK]")
    else:
        tk.post_processor = processors.RobertaProcessing(sep=("</s>", vocab["</s>"]), cls=("<s>", vocab["<s>"]))
        tok = PreTrainedTokenizerFast(tokenizer_object=tk, bos_token="<s>", cls_token="<s>", eos_token="</s>",
                                      sep_token="</s>", pad_token="<pad>", unk_token="<unk>")
    return tok


@pytest.mark.parametrize("family", ["bert", "roberta"])
def test_pair_encoding_matches_a_fast_tokenizer(family):
    tok = _fast_tokenizer(family)
    rng = np.random.default_rng(3)
    lengths = [0, 1, 2, 3, 4, 5, 7, 8, 9, 15, 16, 17, 23, 31, 39]
    for max_length in (8, 9, 16, 17, 33):
        qs, ps = [], []
        for a in lengths:
            for b in lengths:
                qs.append(" ".join(f"w{x}" for x in rng.integers(0, N_WORDS, a)))
                ps.append(" ".join(f"w{x}" for x in rng.integers(0, N_WORDS, b)))
        # the batch pair form CrossEncoder.predict uses
        enc = tok(qs, ps, padding=True, truncation="longest_first", max_length=max_length,
                  return_token_type_ids=True)
        q_ids = tok(qs, add_special_tokens=False)["input_ids"]
        p_ids = tok(ps, add_special_tokens=False)["input_ids"]
        for i in range(len(qs)):
            n = sum(enc["attention_mask"][i])
            want_ids, want_types = enc["input_ids"][i][:n], enc["token_type_ids"][i][:n]
            ids, types, pos = orr.cross_encoder_inputs(q_ids[i], p_ids[i], max_length, family, tok.cls_token_id,
                                                       tok.sep_token_id, pad_id=tok.pad_token_id)
            assert ids == want_ids, (max_length, len(q_ids[i]), len(p_ids[i]))
            assert types == want_types, (max_length, len(q_ids[i]), len(p_ids[i]))
            off = tok.pad_token_id + 1 if family == "roberta" else 0
            assert pos == list(range(off, off + n))


def _kernel_order(scores, top_n):
    """The ordering rule of csrc/rerank.cu: rank = #(s_j > s_r) + #(s_j == s_r, j < r)."""
    n = len(scores)
    rank = [sum(1 for j in range(n) if scores[j] > scores[r] or (scores[j] == scores[r] and j < r)) for r in range(n)]
    out = [None] * n
    for r, p in enumerate(rank):
        out[p] = r
    return out[:top_n]


@pytest.mark.parametrize("scores", [
    [0.5, 0.9, 0.5, 0.1, 0.9],
    [0.0, 0.3, 0.0, 1.0, 1.0, 1.0, 2.0 ** -149],
    [1.0] * 6,
    [0.0, 0.0],
    [0.7],
    [],
])
@pytest.mark.parametrize("top_n", [1, 2, 6, 10])
def test_rerank_order_is_the_reference_sort(scores, top_n):
    scores = [float(np.float32(s)) for s in scores]
    nodes = [NodeWithScore(TextNode(f"t{i}", id_=str(i)), s) for i, s in enumerate(scores)]
    ref = sorted(nodes, key=lambda x: -x.score if x.score else 0)[:top_n]        # rerankers.py:94-96
    want = [int(n.node.node_id) for n in ref]
    assert orr.rerank_order(scores, top_n) == want
    assert _kernel_order(scores, top_n) == want


def test_truncation_closed_form_spends_the_whole_budget():
    for room in range(0, 40):
        for a in range(0, 45):
            for b in range(0, 45):
                na, nb = orr.truncate_longest_first(a, b, room)
                assert 0 <= na <= a and 0 <= nb <= b
                assert na + nb == min(a + b, room)


def test_chunks_hold_whole_pairs_under_the_budget():
    rng = np.random.default_rng(5)
    lens = rng.integers(3, 513, 300)
    cu = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    for budget in (512, 513, 1000, 4096, 10 ** 9):
        parts = rerank.CrossEncoderReranker.chunks(SimpleNamespace(max_tokens=budget), cu)
        assert parts[0][0] == 0 and parts[-1][1] == lens.size
        assert all(a[1] == b[0] for a, b in zip(parts, parts[1:]))
        assert all(cu[p1] - cu[p0] <= budget for p0, p1 in parts)
        # greedy: the next pair would not have fit
        assert all(cu[p1 + 1] - cu[p0] > budget for p0, p1 in parts[:-1])
    assert len(rerank.CrossEncoderReranker.chunks(SimpleNamespace(max_tokens=10 ** 9), cu)) == 1


def test_chunks_stay_within_the_attention_sequence_limit():
    """Many short pairs under a large budget: a chunk holds at most MAX_CHUNK_PAIRS pairs, the sequences one attention
    launch takes."""
    cu = np.arange(0, 3 * 20 * rerank.MAX_CHUNK_PAIRS + 1, 20, dtype=np.int64)          # 3 * MAX_CHUNK_PAIRS pairs
    parts = rerank.CrossEncoderReranker.chunks(SimpleNamespace(max_tokens=1 << 22), cu)
    assert parts == [(i * rerank.MAX_CHUNK_PAIRS, (i + 1) * rerank.MAX_CHUNK_PAIRS) for i in range(3)]
    parts = rerank.CrossEncoderReranker.chunks(SimpleNamespace(max_tokens=20 * 1000), cu)
    assert all(p1 - p0 == 1000 for p0, p1 in parts[:-1])


def test_model_rejects_multi_label_heads_and_unsupported_head_dims():
    cfg = BertConfig(vocab_size=50, hidden_size=128, intermediate_size=256, num_hidden_layers=1,
                     num_attention_heads=2, max_position_embeddings=64)
    st = rerank.random_cross_encoder_state("bert", cfg, 1)
    st["classifier.weight"] = torch.zeros(3, 128)
    st["classifier.bias"] = torch.zeros(3)
    with pytest.raises(ValueError, match="num_labels"):
        rerank.CrossEncoderModel("bert", cfg, st, 2, 3)
    mini = BertConfig(vocab_size=50, hidden_size=384, intermediate_size=1536, num_hidden_layers=1,
                      num_attention_heads=12, max_position_embeddings=64)          # MiniLM-L6 shape: head_dim 32
    with pytest.raises(ValueError, match="head_dim"):
        rerank.CrossEncoderModel("roberta", mini, rerank.random_cross_encoder_state("roberta", mini, 1), 0, 2)
    with pytest.raises(ValueError, match="family"):
        rerank.CrossEncoderModel("gpt", cfg, st, 2, 3)


def test_random_state_loads_into_the_transformers_classifiers():
    """The oracle's models accept the state dicts the GPU model is built from (names and shapes agree)."""
    cfg = BertConfig(vocab_size=40, hidden_size=64, intermediate_size=128, num_hidden_layers=1,
                     num_attention_heads=1, max_position_embeddings=40)
    for family in ("bert", "roberta"):
        st = rerank.random_cross_encoder_state(family, cfg, 2)
        ids, types, _ = orr.cross_encoder_inputs([5, 6, 7], [8, 9], 16, family, 0 if family == "roberta" else 2,
                                                 2 if family == "roberta" else 3)
        logits, scores = orr.cross_encoder_scores(family, cfg, st, [(ids, types)] * 3)
        assert logits.shape == (3,) and np.all((scores > 0) & (scores < 1))
        assert np.array_equal(scores, torch.sigmoid(torch.from_numpy(logits)).numpy())


def test_postprocessor_stand_in_surface():
    from easyrag_b200.schema import BaseNodePostprocessor, MetadataMode

    class Echo(BaseNodePostprocessor):
        def _postprocess_nodes(self, nodes, query_bundle=None):
            return [(n.node.get_content(metadata_mode=MetadataMode.NONE), query_bundle.query_str) for n in nodes]

    nodes = [NodeWithScore(TextNode("a"), 1.0)]
    assert Echo().postprocess_nodes(nodes, query_str="q") == [("a", "q")]
    assert Echo().postprocess_nodes(nodes, QueryBundle("r")) == [("a", "r")]


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")
def test_reranker_fails_loudly_without_cuda(lib_built):
    with pytest.raises(_lib.EzrError):
        rerank.CrossEncoderReranker(SimpleNamespace(), [[1, 2, 3]])
    cfg = BertConfig(vocab_size=50, hidden_size=128, intermediate_size=256, num_hidden_layers=1,
                     num_attention_heads=2, max_position_embeddings=64)
    with pytest.raises(_lib.EzrError):
        rerank.CrossEncoderModel("bert", cfg, rerank.random_cross_encoder_state("bert", cfg, 1), 2, 3, device="cpu")
