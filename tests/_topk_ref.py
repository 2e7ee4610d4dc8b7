"""Test infrastructure: the canonical dense top-k (score descending, id descending) in fp64, for the GPU tests.

Exact integer scores (small-integer inputs, where every dot product is exact in fp32 and ties are common) are ranked
with one int64 key per (score, id): ``score * 2^id_bits + id``.  ``id_bits`` is ``ID_BITS = 20`` (corpora of up to
2^20 rows, 1 000 077 in tests/test_gpu_dense_scale.py) or as many bits as the corpus's last row id needs (22 for the
4M rows of tests/test_gpu_configs4.py); every key is checked to fit in int64.  No TF32 anywhere: the
references are float64 matmuls, which ``torch.backends.cuda.matmul.allow_tf32`` does not touch.
"""
import torch

ID_BITS = 20
I64_MIN = torch.iinfo(torch.int64).min


def id_bits_for(n_rows: int) -> int:
    """The id field of the keys of a corpus of ``n_rows`` rows: ID_BITS, or more when its last id needs them."""
    return max(ID_BITS, (max(n_rows, 1) - 1).bit_length())


def canonical_keys(sims: torch.Tensor, ids: torch.Tensor, ids_asc: bool = False,
                   id_bits: int = ID_BITS) -> torch.Tensor:
    """int64 keys of exact integer scores ``sims`` [Q, m] (fp64) for column ids ``ids`` [m]; ``ids_asc`` reverses
    the tie order (a negative control).  Keys compare only between calls with the same ``id_bits``."""
    n_max = int(ids.max()) + 1
    assert n_max <= 1 << id_bits, f"{n_max} rows do not fit the {id_bits}-bit id field"
    assert torch.equal(sims, sims.round()), "canonical_keys needs exact integer scores"
    assert sims.abs().max().item() * 2.0 ** id_bits + n_max < 2.0 ** 63, f"score * 2^{id_bits} + id overflows int64"
    tie = ((1 << id_bits) - 1 - ids) if ids_asc else ids
    return sims.long() * (1 << id_bits) + tie


def canonical_topk(sims: torch.Tensor, k: int, allowed=None):
    """(score desc, id desc) top-k of exact integer scores [Q, n] -> (column ids, scores)."""
    key = canonical_keys(sims, torch.arange(sims.shape[1], device=sims.device), id_bits=id_bits_for(sims.shape[1]))
    if allowed is not None:
        key = torch.where(allowed, key, torch.full_like(key, I64_MIN))
    top = key.topk(k, dim=1).indices
    return top, sims.gather(1, top)


def fp64_top(q: torch.Tensor, c: torch.Tensor, kmax: int, integer: bool, allowed=None, ids_asc: bool = False,
             drop_dims: int = 0, q_chunk: int = 1024, c_chunk: int = 131072):
    """The fp64 top-``kmax`` of every query over the whole corpus, from plain float64 matmuls on the device, chunked
    so that the extra memory stays near 3 GB (one fp64 corpus chunk, one score block and its keys).
    -> (ids [Q, kmax] int64, scores [Q, kmax] fp64, valid [Q, kmax] bool).
    ``integer``: exact integer scores, canonical order (id descending on ties); otherwise plain fp64 scores (ties
    between distinct unit vectors do not occur).  ``allowed(q0, q1, c0, c1)`` -> bool mask of the rows a query may
    return.  ``ids_asc`` / ``drop_dims`` (the last dims left out) build negative controls."""
    nq, d = q.shape
    n = c.shape[0]
    bits = id_bits_for(n)
    dev = q.device
    qd = q[:, :d - drop_dims].double()
    low = I64_MIN if integer else -float("inf")
    best_k = torch.full((nq, kmax), low, dtype=torch.int64 if integer else torch.float64, device=dev)
    best_i = torch.full((nq, kmax), -1, dtype=torch.int64, device=dev)
    best_s = torch.zeros(nq, kmax, dtype=torch.float64, device=dev)
    for c0 in range(0, n, c_chunk):
        c1 = min(n, c0 + c_chunk)
        cd = c[c0:c1, :d - drop_dims].double()
        ids = torch.arange(c0, c1, device=dev)
        for q0 in range(0, nq, q_chunk):
            q1 = min(nq, q0 + q_chunk)
            s = qd[q0:q1] @ cd.T
            key = canonical_keys(s, ids, ids_asc, bits) if integer else s
            if allowed is not None:
                key = torch.where(allowed(q0, q1, c0, c1), key, torch.full_like(key, low))
            kv, ki = key.topk(min(kmax, c1 - c0), dim=1)
            ck = torch.cat([best_k[q0:q1], kv], 1)
            ci = torch.cat([best_i[q0:q1], ki + c0], 1)
            cs = torch.cat([best_s[q0:q1], s.gather(1, ki)], 1)
            top = ck.topk(kmax, dim=1).indices
            best_k[q0:q1], best_i[q0:q1], best_s[q0:q1] = ck.gather(1, top), ci.gather(1, top), cs.gather(1, top)
            del s, key
    return best_i, best_s, best_k != low
