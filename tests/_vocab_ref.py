"""The interning contract restated as plain dict loops (the oracle of tests/test_vocab_cpu.py and
tests/test_gpu_vocab.py)."""
from itertools import chain

import numpy as np


def intern(groups, d=None, first=None, seen=0):
    """-> (ids, group pointer, dict, first index per id, strings seen): ``d.setdefault(s, len(d))`` over the strings
    in order; ``first[i]`` is the global index of id i's first occurrence.  ``d`` / ``first`` / ``seen`` continue an
    earlier call."""
    d = {} if d is None else d
    first = [] if first is None else first
    ids, ptr = [], [0]
    for g in groups:
        for s in g:
            i = d.setdefault(s, len(d))
            if i == len(first):
                first.append(seen)
            seen += 1
            ids.append(i)
        ptr.append(len(ids))
    return np.asarray(ids, dtype=np.int64), np.asarray(ptr, dtype=np.int64), d, first, seen


def lookup(groups, d):
    return np.asarray([d.get(s, -1) for s in chain.from_iterable(groups)], dtype=np.int64)


def first_index(strings):
    """retrievers._canon_ids restated: the index of each string's first occurrence."""
    seen = {}
    return np.asarray([seen.setdefault(s, i) for i, s in enumerate(strings)], dtype=np.int64)
