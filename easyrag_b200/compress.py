"""Context compression: the reference's ``ContextCompressor`` (src/easyrag/custom/compressors.py) with its
``bm25_extract`` method on the GPU.

The reference compresses one (query, context) pair per call: it cuts the context into sentences, builds a
throw-away BM25 index over them (``BM25Retriever.get_scores(query, sentences)``), walks the sentences best-first
until their characters reach ``rate * len(context)`` and joins the kept ones in their original order.
:meth:`ContextCompressor.compress_batch` does the same for many contexts with one launch of ``ezr_bm25_extract``
(csrc/bm25_extract.cu): every context is one group, scored bit for bit as ``get_scores(query, sentences)`` scores it.

Host work that stays in Python: sentence splitting (the reference's own ``cut_sent`` unless a ``splitter`` is given),
tokenisation with the retriever's tokenizer and stop words (as ``get_scores`` does) and joining the kept sentences.
``compress_batch`` packs the batch into CSR arrays over one vocabulary on the device (:func:`pack_device`, through
:class:`easyrag_b200.vocab.Vocabulary`); :func:`pack` is the same packing as a host loop.

Ties between equal scores are broken by sentence index, higher first (the project's canonical order); the
reference's ``argsort()[::-1]`` leaves that order to numpy's unstable sort.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Callable, Dict, List, Optional, Sequence, Union

import numpy as np
import torch

from . import batched
from .retrievers import BM25Retriever, tokenize_and_remove_stopwords
from .vocab import Vocabulary


def _reference_cut_sent() -> Callable[[str], List[str]]:
    try:
        from easyrag.pipeline.rag import cut_sent          # the reference package (through the shim/ overlay)
    except ImportError as e:
        raise ImportError("ContextCompressor splits sentences with easyrag.pipeline.rag.cut_sent: put the reference's "
                          "src/ on sys.path or pass splitter=") from e
    return cut_sent


def split_sentences(context: str, splitter: Callable[[str], List[str]]) -> List[str]:
    """compressors.py:35-40: the splitter's pieces, stripped, empty ones dropped."""
    return [s for s in (r.strip() for r in splitter(context)) if s != ""]


@dataclass
class Packed:
    """A batch of groups over one vocabulary (CSR, host arrays): sentences ``sent_ptr[g]:sent_ptr[g+1]``, tokens of
    sentence s ``tokens[tok_ptr[s]:tok_ptr[s+1]]``, query tokens ``q_tokens[q_ptr[g]:q_ptr[g+1]]`` (-1 = no sentence of
    the batch has it), character counts of every sentence and context.  From :func:`pack_device`, ``tokens`` and
    ``q_tokens`` are int32 device tensors and ``vocab`` is a :class:`~easyrag_b200.vocab.Vocabulary`."""
    sent_ptr: np.ndarray     # int64 [G+1]
    tok_ptr: np.ndarray      # int64 [S+1]
    tokens: np.ndarray       # int32 [T]
    sent_chars: np.ndarray   # int64 [S]
    ctx_chars: np.ndarray    # int64 [G]
    q_ptr: np.ndarray        # int64 [G+1]
    q_tokens: np.ndarray     # int32
    vocab: Union[Dict[str, int], Vocabulary]     # pack: the dict; pack_device: the device vocabulary


def pack(query_tokens: Sequence[Sequence[str]], sentence_tokens: Sequence[Sequence[Sequence[str]]],
         sentences: Sequence[Sequence[str]], contexts: Sequence[str]) -> Packed:
    vocab: Dict[str, int] = {}
    flat: List[int] = []
    tok_ptr = [0]
    sent_ptr = [0]
    for sents in sentence_tokens:
        for toks in sents:
            flat.extend([vocab.setdefault(w, len(vocab)) for w in toks])
            tok_ptr.append(len(flat))
        sent_ptr.append(len(tok_ptr) - 1)
    q_flat: List[int] = []
    q_ptr = [0]
    for toks in query_tokens:
        q_flat.extend([vocab.get(w, -1) for w in toks])
        q_ptr.append(len(q_flat))
    return Packed(sent_ptr=np.asarray(sent_ptr, dtype=np.int64), tok_ptr=np.asarray(tok_ptr, dtype=np.int64),
                  tokens=np.asarray(flat, dtype=np.int32),
                  sent_chars=np.asarray([len(s) for sents in sentences for s in sents], dtype=np.int64),
                  ctx_chars=np.asarray([len(c) for c in contexts], dtype=np.int64),
                  q_ptr=np.asarray(q_ptr, dtype=np.int64), q_tokens=np.asarray(q_flat, dtype=np.int32), vocab=vocab)


def pack_device(query_tokens: Sequence[Sequence[str]], sentence_tokens: Sequence[Sequence[Sequence[str]]],
                sentences: Sequence[Sequence[str]], contexts: Sequence[str], device="cuda") -> Packed:
    """:func:`pack` with the term ids made on the device: the same ids, with ``tokens`` and ``q_tokens`` left there for
    :func:`easyrag_b200.batched.bm25_extract`.  Pointers and character counts stay on the host."""
    vocab = Vocabulary(device)
    tokens, tok_ptr = vocab.intern([toks for sents in sentence_tokens for toks in sents])
    q_tokens, q_ptr = vocab.lookup(query_tokens)
    return Packed(sent_ptr=np.concatenate([[0], np.cumsum([len(s) for s in sentence_tokens])]).astype(np.int64),
                  tok_ptr=tok_ptr.numpy(), tokens=tokens,
                  sent_chars=np.asarray([len(s) for sents in sentences for s in sents], dtype=np.int64),
                  ctx_chars=np.asarray([len(c) for c in contexts], dtype=np.int64),
                  q_ptr=q_ptr.numpy(), q_tokens=q_tokens, vocab=vocab)


class ContextCompressor:
    """compressors.py:6-66.  ``method="bm25_extract"`` only: the LLMLingua methods need a Qwen2-7B-Instruct language
    model this package does not provide.  ``splitter``: sentence splitter (default: the reference's ``cut_sent``)."""

    def __init__(self, method="bm25_extract", rate=0.5, bm25_retriever=None, *,
                 splitter: Optional[Callable[[str], List[str]]] = None):
        if "llmlingua" in method:
            raise NotImplementedError(f"compress_method {method!r} (an LLMLingua language model) is not provided by "
                                      "easyrag_b200")
        if method != "bm25_extract":
            raise ValueError(f"unknown compress_method {method!r}")
        self.rate = rate
        self.method = method
        self.bm25_retriever = bm25_retriever
        self._splitter = splitter

    @property
    def splitter(self) -> Callable[[str], List[str]]:
        if self._splitter is None:
            self._splitter = _reference_cut_sent()
        return self._splitter

    def compress(self, query, context) -> str:
        """compressors.py:27-55.  A context without sentences raises ZeroDivisionError, as the reference does."""
        return self.compress_batch([query], [context])[0]

    def compress_batch(self, queries: Sequence[str], contexts: Sequence[str]) -> List[str]:
        """``[compress(q, c) for q, c in zip(queries, contexts)]`` with one kernel launch for the batch."""
        if len(queries) != len(contexts):
            raise ValueError("compress_batch: one query per context")
        sentences = self.split(contexts)
        if any(not s for s in sentences):
            raise ZeroDivisionError("division by zero")     # get_scores(query, []): rank_bm25's avgdl
        r = self.bm25_retriever
        if not isinstance(r, BM25Retriever):
            keep = [batched._select_host(np.asarray(r.get_scores(q, s)), [len(x) for x in s], len(c), self.rate)
                    for q, s, c in zip(queries, sentences, contexts)]
            return self.join(sentences, np.concatenate(keep))
        q_toks, s_toks = self.tokenize(queries, sentences)
        keep, _ = self.run(pack_device(q_toks, s_toks, sentences, contexts, r.bm25.device))
        return self.join(sentences, keep)

    # ---- the steps of compress_batch, separately callable (scripts/bench_compress.py times each)
    def split(self, contexts: Sequence[str]) -> List[List[str]]:
        return [split_sentences(c, self.splitter) for c in contexts]

    def tokenize(self, queries: Sequence[str], sentences: Sequence[Sequence[str]]):
        """Query and sentence tokens exactly as ``BM25Retriever.get_scores(query, docs)`` makes them."""
        r = self.bm25_retriever
        tok = lambda text: tokenize_and_remove_stopwords(r._tokenizer, text, stopwords=r.stopwords)   # noqa: E731
        return [tok(q) for q in queries], [[tok(s) for s in sents] for sents in sentences]

    def run(self, p: Packed, scores: bool = False):
        """-> (keep uint8 [S], counts int32 [G]) on the host, plus the score rows (device) when asked for."""
        r = self.bm25_retriever
        res = batched.bm25_extract(p.sent_ptr, p.tok_ptr, p.tokens, p.sent_chars, p.ctx_chars, p.q_ptr, p.q_tokens,
                                   max(len(p.vocab), 1), rate=self.rate, bm25_type=1 if r.bm25_type == 1 else 0,
                                   k1=r.k1, b=r.b, epsilon=r.epsilon, scores=scores, device=r.bm25.device)
        keep, counts = res.keep.cpu().numpy(), res.counts.cpu().numpy()
        if (counts < -1).any():
            raise ValueError("bm25_extract: bad input in group %d" % int(np.nonzero(counts < -1)[0][0]))
        return (keep, counts, res.scores) if scores else (keep, counts)

    @staticmethod
    def join(sentences: Sequence[Sequence[str]], keep: np.ndarray) -> List[str]:
        """compressors.py:51-54: the kept sentences in their original order, no separator."""
        out, s = [], 0
        for sents in sentences:
            k = keep[s:s + len(sents)]
            out.append("".join(x for x, f in zip(sents, k) if f))
            s += len(sents)
        return out
