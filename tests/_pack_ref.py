"""Test infrastructure: the two reranker pair packers of csrc/handoff.cu restated in plain torch integer ops, for CPU
and CUDA tensors alike.

The per-pair oracles (``oracle/rerank.py::cross_encoder_inputs``, ``oracle/retrieve.py::rerank_inputs``) build one
Python list per pair, which is far too slow for the pipeline's millions of pairs.  This module computes the same
arrays with whole-tensor ops -- lengths from the truncation rules, offsets from cumulative sums, tokens from segment
gathers (``repeat_interleave`` plus ``arange`` offsets) -- so the GPU tests can compare the kernels' full outputs at
scale; tests/test_pack_ref_cpu.py pins it to the per-pair oracles.

Inputs are CSR arrays on one device: queries ``q_ptr`` [Q + 1] / ``q_tok``, passages ``p_ptr`` [n_docs + 1] /
``p_tok`` (passage ``id_base + i`` is row i), candidate ids ``cand`` [Q, >= k] (only the first k columns are read, so
a view of a wider top-k works) and ``counts`` [Q].  Every length and offset is int64; token arrays are int32.
The plans raise ``ValueError`` where the kernels' plans return EZR_ERR_INVALID: an id outside
``[id_base, id_base + n_docs)`` among a query's first ``count`` candidates, or a ``max_length`` with no room.

A plan is a dict; ``*_tokens(plan, ..., p0, p1)`` builds the tokens of pairs ``[p0, p1)`` only, so a caller can walk
a large pack in bounded memory.
"""
import torch

I64 = torch.int64


def _long(x):
    return x.to(I64)


def _lens(ptr):
    ptr = _long(ptr)
    return ptr[1:] - ptr[:-1]


def _segments(lens):
    """``lens`` int64 [n] -> (segment of each element, index inside its segment), both int64 [lens.sum()]."""
    dev = lens.device
    seg = torch.repeat_interleave(torch.arange(lens.numel(), device=dev), lens)
    start = torch.cumsum(lens, 0) - lens
    return seg, torch.arange(seg.numel(), device=dev) - start[seg]


def _doc_lens(p_ptr, doc):
    """Passage lengths of ``doc`` (any valid row; zeros when there are no passages)."""
    lens = _lens(p_ptr)
    return lens[doc] if lens.numel() else torch.zeros_like(doc)


def _cu(lens):
    return torch.cat([torch.zeros(1, dtype=I64, device=lens.device), torch.cumsum(lens, 0)])


def _gather(src, idx):
    """``src[idx]`` where ``idx`` may be out of range in lanes a ``torch.where`` discards (src may be empty)."""
    if src.numel() == 0:
        return torch.zeros_like(idx, dtype=torch.int32)
    return src[idx.clamp(0, src.numel() - 1)].to(torch.int32)


def _candidates(cand, counts, k, id_base, n_docs, clamp_counts):
    """-> (valid [Q, k]: the slot is among the query's first count; doc [Q, k] int64: row index, 0 where invalid)."""
    q = counts.numel()
    cnt = _long(counts)
    if clamp_counts:
        cnt = cnt.clamp(0, k)
    r = torch.arange(k, device=cand.device)
    valid = r[None, :] < cnt[:, None]
    doc = _long(cand[:q, :k]) - id_base
    bad = valid & ((doc < 0) | (doc >= n_docs))
    if bool(bad.any()):
        raise ValueError(f"{int(bad.sum())} candidate ids outside [id_base, id_base + n_docs) = "
                         f"[{id_base}, {id_base + n_docs})")
    return valid, torch.where(valid, doc, torch.zeros_like(doc))


# --------------------------------------------------------------------------------------------- cross-encoder pack
def longest_first(a, b, room):
    """The fast tokenizer's ``truncation="longest_first"`` on int64 tensors: kept lengths (na, nb) of a query of ``a``
    and a passage of ``b`` tokens with ``room`` tokens for both.  Both fit, or the shorter side keeps
    min(its length, room // 2) and the longer side takes the rest."""
    half = room // 2
    fits = a + b <= room
    a_longer = a > b
    nb = torch.where(fits, b, torch.where(a_longer, torch.minimum(b, half), room - torch.minimum(a, half)))
    na = torch.where(fits, a, torch.where(a_longer, room - torch.minimum(b, half), torch.minimum(a, half)))
    return na, nb


def cross_plan(q_ptr, p_ptr, cand, counts, k, id_base, n_mid, max_length):
    """``ezr_cross_pack_plan``: -> dict(pair_off [Q + 1], cu [P + 1], slot_len [Q, k], and per pair q, doc, na, nb),
    T and P.  Only real pairs (candidate r < count, counts clamped to [0, k]) are packed, in query order."""
    if n_mid not in (1, 2) or max_length < 2 + n_mid:
        raise ValueError(f"max_length={max_length} leaves no room for the {2 + n_mid} special tokens")
    n_docs = p_ptr.numel() - 1
    valid, doc = _candidates(cand, counts, k, id_base, n_docs, clamp_counts=True)
    qa = _lens(q_ptr)[:, None].expand_as(doc)
    pb = _doc_lens(p_ptr, doc)
    na, nb = longest_first(qa, pb, torch.full_like(qa, max_length - 2 - n_mid))
    slot_len = torch.where(valid, 2 + n_mid + na + nb, torch.zeros_like(na))
    per_query = valid.sum(1)
    qidx = torch.arange(valid.shape[0], device=valid.device)[:, None].expand_as(valid)
    lens = slot_len[valid]
    cu = _cu(lens)
    return dict(pair_off=_cu(per_query), cu=cu, slot_len=slot_len, len=lens, q=qidx[valid], doc=doc[valid],
                na=na[valid], nb=nb[valid], n_mid=n_mid, T=int(cu[-1]), P=int(lens.numel()))


def cross_tokens(plan, q_ptr, q_tok, p_ptr, p_tok, cls, sep, type_b, pos_offset, p0=0, p1=None):
    """ids, types, positions (int32) of pairs [p0, p1): ``[cls] q' [sep] x n_mid p' [sep]``, token type 0 through
    the first [sep] and ``type_b`` after it, positions ``pos_offset + i``."""
    p1 = plan["P"] if p1 is None else p1
    seg, i = _segments(plan["len"][p0:p1])
    seg = seg + p0
    na, nb = plan["na"][seg], plan["nb"][seg]
    b0 = 1 + na + plan["n_mid"]                                   # first passage token
    q_at = _gather(q_tok, _long(q_ptr)[plan["q"][seg]] + i - 1)
    p_at = _gather(p_tok, _long(p_ptr)[plan["doc"][seg]] + i - b0)
    ids = torch.where(i == 0, cls, torch.where(i <= na, q_at, torch.where(
        i < b0, sep, torch.where(i < b0 + nb, p_at, sep)))).to(torch.int32)
    types = torch.where(i < na + 2, 0, type_b).to(torch.int32)
    return ids, types, (pos_offset + i).to(torch.int32)


def cross_pack(q_ptr, q_tok, p_ptr, p_tok, cand, counts, k, id_base, n_mid, type_b, cls, sep, pos_offset,
               max_length):
    """Plan and every token at once (small inputs)."""
    plan = cross_plan(q_ptr, p_ptr, cand, counts, k, id_base, n_mid, max_length)
    plan["ids"], plan["types"], plan["positions"] = cross_tokens(plan, q_ptr, q_tok, p_ptr, p_tok, cls, sep, type_b,
                                                                 pos_offset)
    return plan


# ------------------------------------------------------------------------------------------------ LLM reranker pack
def llm_min_max_length(n_sep):
    """The smallest max_length ``ezr_rerank_pack_plan`` accepts: >= 8 and room for bos + 3/4 of it + sep."""
    m = 8
    while 1 + m * 3 // 4 + n_sep > m:
        m += 1
    return m


def llm_plan(q_ptr, p_ptr, cand, counts, k, id_base, n_sep, n_prompt, max_length):
    """``ezr_rerank_pack_plan``: pair p = q * k + r for every slot (empty past the count).  Per pair, as
    ``get_inputs``: first = [bos] + query[: 3/4 max_length]; second = (sep + passage[: max_length]) cut to
    max_length - len(first) ('only_second'); then sep + prompt.  -> dict(len, cu, query_len = len(first) + n_sep, and
    per pair q, doc, head = len(first), second = len(second)), T."""
    if max_length < 8 or 1 + max_length * 3 // 4 + n_sep > max_length:
        raise ValueError(f"max_length={max_length} leaves no room for bos + query + sep ({n_sep} sep ids)")
    n_docs = p_ptr.numel() - 1
    valid, doc = _candidates(cand, counts, k, id_base, n_docs, clamp_counts=False)
    valid, doc = valid.reshape(-1), doc.reshape(-1)
    q = torch.arange(counts.numel(), device=doc.device).repeat_interleave(k)
    head = 1 + torch.clamp(_lens(q_ptr), max=max_length * 3 // 4)[q]
    second = torch.minimum(n_sep + torch.clamp(_doc_lens(p_ptr, doc), max=max_length),
                           torch.clamp(max_length - head, min=0))
    zero = torch.zeros_like(head)
    head, second = torch.where(valid, head, zero), torch.where(valid, second, zero)
    lens = torch.where(valid, head + second + n_sep + n_prompt, zero)
    cu = _cu(lens)
    return dict(len=lens, cu=cu, query_len=torch.where(valid, head + n_sep, zero).to(torch.int32), q=q, doc=doc,
                head=head, second=second, n_sep=n_sep, T=int(cu[-1]))


def llm_tokens(plan, q_ptr, q_tok, p_ptr, p_tok, sep, prompt, bos, p0=0, p1=None):
    """Packed ids (int32) of pairs [p0, p1): [bos] q' | sep p' (second part) | sep prompt."""
    p1 = plan["len"].numel() if p1 is None else p1
    seg, i = _segments(plan["len"][p0:p1])
    seg = seg + p0
    head, second, n_sep = plan["head"][seg], plan["second"][seg], plan["n_sep"]
    j = i - head                                                   # index inside the second part
    t = j - second                                                 # index inside the tail
    q_at = _gather(q_tok, _long(q_ptr)[plan["q"][seg]] + i - 1)
    s_at = torch.where(j < n_sep, _gather(sep, j), _gather(p_tok, _long(p_ptr)[plan["doc"][seg]] + j - n_sep))
    tail = torch.where(t < n_sep, _gather(sep, t), _gather(prompt, t - n_sep))
    return torch.where(i == 0, bos, torch.where(i < head, q_at, torch.where(j < second, s_at, tail))).to(torch.int32)


def llm_pack(q_ptr, q_tok, p_ptr, p_tok, cand, counts, k, id_base, sep, prompt, bos, max_length):
    """Plan and every token at once (small inputs); ``sep`` / ``prompt`` int tensors."""
    plan = llm_plan(q_ptr, p_ptr, cand, counts, k, id_base, sep.numel(), prompt.numel(), max_length)
    plan["ids"] = llm_tokens(plan, q_ptr, q_tok, p_ptr, p_tok, sep, prompt, bos)
    return plan


def llm_slices(n_queries, k, batch_size=32):
    """(query, first pair, last pair + 1) of every slice ``LLMRerank._postprocess_nodes`` forms, in its order."""
    return [(q, q * k + r, q * k + min(r + batch_size, k)) for q in range(n_queries) for r in range(0, k, batch_size)]
