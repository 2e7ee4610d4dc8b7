"""String interning on the GPU (csrc/vocab.cu): token strings to term ids, as a Python dict filled in first-seen
order numbers them, without a Python loop over the tokens.

A :class:`Vocabulary` takes groups of strings (documents, sentences, queries).  Groups stream through the device in
chunks of at most ``chunk_strings`` strings and ``chunk_bytes`` bytes (a group is never split: one group larger than
that is a chunk of its own).  The host's only work per chunk is ``"\\0".join`` and ``str.encode``, both at C speed, and
one copy through a pinned buffer.  For every list of strings, any chunking and any hash-bits setting:

* ``intern`` ids equal ``[d.setdefault(s, len(d)) for s in flat]``, and ``to_dict()`` equals ``d``;
* ``lookup`` ids equal ``d.get(s, -1)`` (it inserts nothing);
* ``first_index`` of a fresh vocabulary equals ``retrievers._canon_ids``.

Fallback: the join cannot represent a token that is not a ``str``, a string containing NUL, or one UTF-8 cannot encode
(a lone surrogate).  ``lookup`` answers the rest of such a call with a host dict read from :meth:`to_dict`, and the
vocabulary stays on the device.  ``intern`` / ``first_index`` must give such a token an id that the device table cannot
hold, so the vocabulary becomes a host dict from that chunk on, seeded from :meth:`to_dict` so that ids stay the same,
and every later call runs the same host loop as ``retrievers._encode_corpus``.  That switch warns once
(:class:`HostFallbackWarning`).
"""
from __future__ import annotations

import ctypes
import warnings
from itertools import chain
from typing import Dict, Iterator, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib

CHUNK_STRINGS = 1 << 22
CHUNK_BYTES = 1 << 26
_MIN_SLOTS = 1 << 12


class NotJoinable(ValueError):
    """The NUL join cannot stand for these strings (see the module docstring)."""


class HostFallbackWarning(RuntimeWarning):
    """A vocabulary interned a token the device table cannot hold and runs as a host dict from then on."""


def join_strings(strings: Sequence) -> Tuple[bytes, int]:
    """-> (UTF-8 bytes of the strings joined by single NULs, number of strings), or :class:`NotJoinable`."""
    try:
        text = "\0".join(strings)
    except TypeError as e:
        raise NotJoinable(f"a token is not a str: {e}") from None
    n = len(strings)
    if text.count("\0") != max(n - 1, 0):
        raise NotJoinable("a string contains NUL")
    try:
        return text.encode("utf-8"), n
    except UnicodeEncodeError as e:
        raise NotJoinable(f"a string has no UTF-8 encoding: {e}") from None


def _ranges(cum: np.ndarray, cap: int) -> List[Tuple[int, int]]:
    """Consecutive ranges [a, b) over the groups of the cumulative sizes ``cum`` ([G + 1]), in order: each totals at
    most ``cap``, or is one group that alone totals more."""
    out, a, g = [], 0, len(cum) - 1
    while a < g:
        b = int(np.searchsorted(cum, cum[a] + cap, side="right")) - 1
        b = min(max(b, a + 1), g)
        out.append((a, b))
        a = b
    return out


def plan_chunks(counts: np.ndarray, max_strings: int) -> List[Tuple[int, int]]:
    """Consecutive group ranges [a, b) covering every group in order.  Each holds at most ``max_strings`` strings, or
    is one group that alone holds more."""
    return _ranges(np.concatenate([[0], np.cumsum(np.asarray(counts, dtype=np.int64))]), max_strings)


def iter_chunks(groups: Sequence, counts: np.ndarray, max_strings: int, max_bytes: int,
                flat: bool = False) -> Iterator[Tuple[int, int, bytes, int]]:
    """Yield (a, b, joined bytes, strings) for consecutive group ranges, in order.  Each range holds at most
    ``max_strings`` strings and ``max_bytes`` bytes, or is one group.  The byte bound is planned from character counts
    before anything is joined (a character is at most 4 UTF-8 bytes), so every join covers exactly one yielded range.
    ``flat``: every item of ``groups`` is one string (a group of one)."""
    counts = np.asarray(counts, dtype=np.int64)
    for a, b in plan_chunks(counts, max_strings):
        strings = groups[a:b] if flat else list(chain.from_iterable(groups[a:b]))
        try:
            lens = np.fromiter(map(len, strings), dtype=np.int64, count=len(strings))
        except TypeError as e:
            raise NotJoinable(f"a token is not a str: {e}") from None
        if 4 * int(lens.sum()) <= max_bytes or b - a == 1:
            yield (a, b, *join_strings(strings))
            continue
        off = np.concatenate([[0], np.cumsum(counts[a:b])])                 # string offsets of the range's groups
        chars = np.concatenate([[0], np.cumsum(lens)])[off]                # cumulative characters per group
        for x, y in _ranges(chars, max_bytes // 4):
            yield (a + x, a + y, *join_strings(strings[off[x]:off[y]]))


def _pow2_at_least(x: int) -> int:
    return 1 << max(int(x) - 1, 1).bit_length()


class Vocabulary:
    """Device string -> id table in first-seen order (module docstring).  ``device``: a CUDA device."""

    def __init__(self, device="cuda", chunk_strings: int = CHUNK_STRINGS, chunk_bytes: int = CHUNK_BYTES):
        _lib.require_cuda()
        dev = torch.device(device)
        self.device = torch.device("cuda", torch.cuda.current_device()) if dev.index is None else dev
        self.chunk_strings = int(chunk_strings)
        self.chunk_bytes = int(chunk_bytes)
        self._L = _lib.lib()
        self._cap = _MIN_SLOTS
        self._table = self._new_table(self._cap)
        with torch.cuda.device(self.device):
            _lib.check(self._L.ezr_vocab_table_init(_lib.ptr(self._table), self._cap, _lib.stream_ptr()),
                       "ezr_vocab_table_init")
        self._arena = torch.empty(1 << 16, dtype=torch.uint8, device=self.device)
        self._arena_off = torch.zeros(_MIN_SLOTS + 1, dtype=torch.int64, device=self.device)
        self._id_first = torch.empty(_MIN_SLOTS, dtype=torch.int64, device=self.device)
        self._state = (ctypes.c_int64 * 2)(0, 0)      # ids, arena bytes used
        self._seen = 0                                # strings interned so far: the next one's global index
        self._bytes = torch.empty(0, dtype=torch.uint8, device=self.device)
        self._pinned = torch.empty(0, dtype=torch.uint8, pin_memory=True)
        self._ws = torch.empty(0, dtype=torch.uint8, device=self.device)
        self._host: Optional[Dict[str, int]] = None   # the host dict after a fallback
        self._host_first: List[int] = []

    # ---------------------------------------------------------------- public
    def intern(self, groups: Sequence[Sequence[str]]) -> Tuple[torch.Tensor, torch.Tensor]:
        """-> (ids int32 [T] on the device, group pointer int64 [G + 1] on the host), inserting unseen strings."""
        ids, _, ptr = self._run(groups, insert=True, want_first=False, flat=False)
        return ids, ptr

    def lookup(self, groups: Sequence[Sequence[str]]) -> Tuple[torch.Tensor, torch.Tensor]:
        """As :meth:`intern`, but inserts nothing: -1 for a string the vocabulary does not hold."""
        ids, _, ptr = self._run(groups, insert=False, want_first=False, flat=False)
        return ids, ptr

    def first_index(self, strings: Sequence[str]) -> torch.Tensor:
        """Interns ``strings`` and returns int64 [n] on the device: the global index (counted over every string this
        vocabulary has interned) of each string's first occurrence.  On a fresh vocabulary this is
        ``retrievers._canon_ids(strings)``."""
        _, first, _ = self._run(strings, insert=True, want_first=True, flat=True)
        return first

    def __len__(self) -> int:
        return len(self._host) if self._host is not None else int(self._state[0])

    def to_dict(self) -> Dict[str, int]:
        """The ``str -> id`` dict, in id order (read back from the device arena)."""
        if self._host is not None:
            return dict(self._host)
        n, used = int(self._state[0]), int(self._state[1])
        off = np.empty(n + 1, dtype=np.int64)
        raw = np.empty(max(used, 1), dtype=np.uint8)
        with torch.cuda.device(self.device):
            _lib.check(self._L.ezr_vocab_read(_lib.ptr(self._arena), _lib.ptr(self._arena_off), 0, n, raw.ctypes.data,
                                              raw.nbytes, off.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)),
                                              _lib.stream_ptr()), "ezr_vocab_read")
        data, o = raw.tobytes(), off.tolist()
        return {data[o[i]:o[i + 1]].decode("utf-8"): i for i in range(n)}

    # -------------------------------------------------------------- internals
    def _new_table(self, cap: int) -> torch.Tensor:
        return torch.empty(self._L.ezr_vocab_table_bytes(cap), dtype=torch.uint8, device=self.device)

    def _run(self, groups, insert: bool, want_first: bool, flat: bool):
        groups = groups if isinstance(groups, list) else list(groups)
        if flat:
            counts = np.ones(len(groups), dtype=np.int64)
        else:
            counts = np.fromiter(map(len, groups), dtype=np.int64, count=len(groups))
        cum = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
        total = int(cum[-1])
        ids = torch.empty(total, dtype=torch.int32, device=self.device)
        first = torch.empty(total, dtype=torch.int64, device=self.device) if want_first else None
        start = 0
        if self._host is None:
            try:
                for a, b, data, n in iter_chunks(groups, counts, self.chunk_strings, self.chunk_bytes, flat):
                    lo = int(cum[a])
                    self._chunk(data, n, ids[lo:lo + n], None if first is None else first[lo:lo + n], insert)
                    start = b
            except NotJoinable:
                if insert:
                    warnings.warn("a token that is not a str, contains NUL or has no UTF-8 encoding was interned: this "
                                  "vocabulary runs as a host dict from now on", HostFallbackWarning, stacklevel=3)
                    self._to_host()
        if start < len(groups):
            d, firsts = (self._host, self._host_first) if self._host is not None else (self.to_dict(), [])
            self._host_run(groups[start:], flat, insert, d, firsts, ids[int(cum[start]):],
                           None if first is None else first[int(cum[start]):])
        return ids, first, torch.from_numpy(cum)

    def _reserve(self, n: int, nb: int) -> None:
        n_ids, used = int(self._state[0]), int(self._state[1])
        if 2 * (n_ids + n) > self._cap:                   # grow before the load factor passes 1/2
            cap = max(_pow2_at_least(2 * (n_ids + n)), 2 * self._cap)
            table = self._new_table(cap)
            _lib.check(self._L.ezr_vocab_table_grow(_lib.ptr(self._table), self._cap, _lib.ptr(table), cap,
                                                    _lib.stream_ptr()), "ezr_vocab_table_grow")
            self._table, self._cap = table, cap
        if self._id_first.numel() < n_ids + n:
            size = max(n_ids + n, 2 * self._id_first.numel())
            id_first = torch.empty(size, dtype=torch.int64, device=self.device)
            id_first[:n_ids] = self._id_first[:n_ids]
            arena_off = torch.empty(size + 1, dtype=torch.int64, device=self.device)
            arena_off[:n_ids + 1] = self._arena_off[:n_ids + 1]
            self._id_first, self._arena_off = id_first, arena_off
        if self._arena.numel() < used + nb:
            arena = torch.empty(max(used + nb, 2 * self._arena.numel()), dtype=torch.uint8, device=self.device)
            arena[:used] = self._arena[:used]
            self._arena = arena

    def _chunk(self, data: bytes, n: int, out_ids: torch.Tensor, out_first: Optional[torch.Tensor],
               insert: bool) -> None:
        L, nb = self._L, len(data)
        with torch.cuda.device(self.device):
            if insert:
                self._reserve(n, nb)
            need = L.ezr_vocab_workspace(n, nb)
            if self._ws.numel() < need:
                self._ws = torch.empty(need, dtype=torch.uint8, device=self.device)
            if self._pinned.numel() < nb:
                self._pinned = torch.empty(max(nb, 2 * self._pinned.numel()), dtype=torch.uint8, pin_memory=True)
                self._bytes = torch.empty(self._pinned.numel(), dtype=torch.uint8, device=self.device)
            if nb:
                # both calls below synchronise the stream, so the pinned buffer is free again when they return
                self._pinned[:nb].numpy()[:] = np.frombuffer(data, dtype=np.uint8)
                self._bytes[:nb].copy_(self._pinned[:nb], non_blocking=True)
            st = _lib.stream_ptr()
            if insert:
                _lib.check(L.ezr_vocab_insert(
                    _lib.ptr(self._table), self._cap, _lib.ptr(self._bytes), nb, n, self._seen, _lib.ptr(self._arena),
                    self._arena.numel(), _lib.ptr(self._arena_off), _lib.ptr(self._id_first), self._id_first.numel(),
                    self._state, _lib.ptr(out_ids), _lib.ptr(out_first), _lib.ptr(self._ws), self._ws.numel(), st),
                    "ezr_vocab_insert")
                self._seen += n
            else:
                _lib.check(L.ezr_vocab_lookup(
                    _lib.ptr(self._table), self._cap, _lib.ptr(self._bytes), nb, n, _lib.ptr(self._arena),
                    _lib.ptr(self._arena_off), _lib.ptr(self._id_first), _lib.ptr(out_ids), _lib.ptr(out_first),
                    _lib.ptr(self._ws), self._ws.numel(), st), "ezr_vocab_lookup")

    def _to_host(self) -> None:
        n = int(self._state[0])
        self._host = self.to_dict()
        self._host_first = self._id_first[:n].tolist()

    def _host_run(self, groups, flat: bool, insert: bool, d: Dict, firsts: List[int], out_ids: torch.Tensor,
                  out_first: Optional[torch.Tensor]) -> None:
        """The host loop over ``groups``: ``d`` / ``firsts`` are the dict and the first index per id it continues."""
        ids: List[int] = []
        for s in (groups if flat else chain.from_iterable(groups)):
            if insert:
                i = d.setdefault(s, len(d))
                if i == len(firsts):
                    firsts.append(self._seen)
                self._seen += 1
            else:
                i = d.get(s, -1)
            ids.append(i)
        if ids:
            out_ids.copy_(torch.tensor(ids, dtype=torch.int32))
            if out_first is not None:
                out_first.copy_(torch.tensor([firsts[i] if i >= 0 else -1 for i in ids], dtype=torch.int64))
