"""Test infrastructure: G simulated ranks of the row-sharded coarse ranker in one process, on one GPU.

Each rank runs in its own host thread with its own shard-local ``CoarseRanker`` and ``ShardedCoarseRanker``; the
product classes run unchanged.  Their collective goes through :class:`Loopback`: ``torch.distributed.get_world_size``,
``get_rank`` and ``all_gather_into_tensor`` are patched so that, when the ``group`` argument is a :class:`Rank`
handle, the loopback answers, and otherwise the original function does.  easyrag_b200/dist.py looks these functions
up on the module at every call, so the patch reaches it.

The all-gather blocks: each rank synchronises its current stream (its record is complete), all ranks meet at a
barrier, each copies the G records into its ``out`` in rank order and synchronises again, and a second barrier keeps
every rank from rewriting its record while another rank may still be copying it.  The barrier has a timeout, and a
rank that raises aborts it, so a failing rank ends the run with an error instead of a hang.

The library's kernel switches are per host thread (``ezr_dense_set_kernel``, ``ezr_dense_s8_set_capacity``): set a
forced form inside each rank's function.
"""
import threading

import torch
import torch.distributed as tdist


class Rank:
    """The ``group`` handle of one simulated rank."""

    def __init__(self, loop, rank):
        self.loop, self.rank = loop, rank


class Loopback:
    def __init__(self, world: int, timeout: float = 300.0):
        self.world = world
        self.barrier = threading.Barrier(world, timeout=timeout)
        self.records = [None] * world
        self.n_gathers = 0

    def handles(self):
        return [Rank(self, r) for r in range(self.world)]

    def all_gather(self, out: torch.Tensor, inp: torch.Tensor, rank: int) -> None:
        n = inp.numel()
        assert out.numel() == self.world * n and out.dtype == inp.dtype
        torch.cuda.current_stream(inp.device).synchronize()
        self.records[rank] = inp
        self.barrier.wait()
        flat = out.view(-1)
        for p, rec in enumerate(self.records):
            flat[p * n:(p + 1) * n].copy_(rec.reshape(-1))
        torch.cuda.current_stream(out.device).synchronize()
        if rank == 0:
            self.n_gathers += 1
        self.barrier.wait()


def install(monkeypatch) -> None:
    """Route the three collectives easyrag_b200/dist.py uses through :class:`Rank` handles."""
    ws0, rk0, ag0 = tdist.get_world_size, tdist.get_rank, tdist.all_gather_into_tensor

    def get_world_size(group=None):
        return group.loop.world if isinstance(group, Rank) else ws0(group)

    def get_rank(group=None):
        return group.rank if isinstance(group, Rank) else rk0(group)

    def all_gather_into_tensor(output_tensor, input_tensor, group=None, async_op=False):
        if not isinstance(group, Rank):
            return ag0(output_tensor, input_tensor, group=group, async_op=async_op)
        assert not async_op
        group.loop.all_gather(output_tensor, input_tensor, group.rank)
        return None

    monkeypatch.setattr(tdist, "get_world_size", get_world_size)
    monkeypatch.setattr(tdist, "get_rank", get_rank)
    monkeypatch.setattr(tdist, "all_gather_into_tensor", all_gather_into_tensor)


def run_ranks(world: int, fn, timeout: float = 300.0):
    """``fn(handle)`` in one thread per rank (``handle.rank`` is the rank) -> the G return values in rank order.
    The first exception of any rank is re-raised here; the others are then aborted at the barrier."""
    loop = Loopback(world, timeout)
    out, errs = [None] * world, [None] * world

    def body(h):
        try:
            out[h.rank] = fn(h)
        except BaseException as e:          # noqa: BLE001 -- handed to the test thread below
            errs[h.rank] = e
            loop.barrier.abort()

    threads = [threading.Thread(target=body, args=(h,), name=f"loopback-rank{h.rank}") for h in loop.handles()]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    first = [e for e in errs if e is not None and not isinstance(e, threading.BrokenBarrierError)]
    first = first or [e for e in errs if e is not None]
    if first:
        raise first[0]
    return out
