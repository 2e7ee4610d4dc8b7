"""CPU: the host side of pair-split reranking -- token-balanced runs of whole pairs, and (2 ranks, gloo) the score
exchange and the cross-rank input check.  The GPU path is covered by tests/test_gpu_rerank_dist.py."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from easyrag_b200 import dist as ezdist


def _cu(lens):
    return np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)


def _check_runs(cu, world):
    runs = ezdist.token_balanced_ranges(cu, world)
    n, t = cu.size - 1, int(cu[-1])
    assert len(runs) == world
    assert runs[0][0] == 0 and runs[-1][1] == n
    assert all(lo <= hi for lo, hi in runs)
    assert all(a[1] == b[0] for a, b in zip(runs, runs[1:]))              # every pair once, in order
    for r, (lo, hi) in enumerate(runs):
        if hi > lo:
            # the run starts at the first pair starting at or after r T / world ...
            assert cu[lo] * world >= r * t and (lo == 0 or cu[lo - 1] * world < r * t)
            # ... so it holds less than T / world tokens plus its last pair
            assert (cu[hi] - cu[lo]) * world < t + world * (cu[hi] - cu[hi - 1])
    return runs


@pytest.mark.parametrize("world", [1, 2, 3, 4, 7, 8])
def test_token_balanced_ranges_cover_every_pair_once(world):
    rng = np.random.default_rng(world)
    for lens in (rng.integers(10, 513, 3072),              # Q = 16 x 192 pairs of a real workload
                 rng.integers(3, 20, 50),
                 np.r_[rng.integers(5, 10, 40), 5000, rng.integers(5, 10, 40)],   # one pair longer than a share
                 np.full(64, 37)):
        runs = _check_runs(_cu(lens), world)
        tok = [int(_cu(lens)[hi] - _cu(lens)[lo]) for lo, hi in runs]
        assert sum(tok) == int(lens.sum())


def test_token_balanced_ranges_balance_equal_pairs_exactly():
    assert ezdist.token_balanced_ranges(_cu([10] * 12), 4) == [(0, 3), (3, 6), (6, 9), (9, 12)]
    assert ezdist.token_balanced_ranges(_cu([10] * 12), 1) == [(0, 12)]


@pytest.mark.parametrize("n_pairs,world", [(0, 1), (0, 3), (1, 2), (2, 4), (3, 8)])
def test_token_balanced_ranges_leave_ranks_empty_when_pairs_are_few(n_pairs, world):
    cu = _cu(np.full(n_pairs, 50))
    runs = _check_runs(cu, world)
    assert sum(1 for lo, hi in runs if hi > lo) == n_pairs
    with pytest.raises(ValueError):
        ezdist.token_balanced_ranges(cu, 0)


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _scores(n):
    """What the head writes: sigmoids in [+0.0, 1.0], saturated ends, the smallest subnormal and values a ulp apart."""
    rng = np.random.default_rng(9)
    s = (1.0 / (1.0 + np.exp(-rng.normal(0, 6, n)))).astype(np.float32)
    s[::7] = 1.0
    s[3::11] = 0.0
    s[5::13] = np.float32(2.0 ** -149)
    s[1::17] = np.nextafter(np.float32(1.0), np.float32(0.0))
    return torch.from_numpy(s)


def _worker(rank, world, port, ret):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        fails = []
        # the exchange: each rank writes its run of the [P] vector into a zeroed buffer; one all-reduce completes it
        # uneven runs; P < world; P = world with a pair longer than a share, so the last rank gets nothing
        for lens in ([30] * 1000 + [400] * 5, [12], [5, 900]):
            cu = _cu(lens)
            full = _scores(len(lens))
            lo, hi = ezdist.token_balanced_ranges(cu, world)[rank]
            sig = torch.zeros(len(lens), dtype=torch.float32)
            sig[lo:hi] = full[lo:hi]
            ezdist.exchange_pair_scores(sig)
            if sig.numpy().tobytes() != full.numpy().tobytes():
                fails.append(f"exchange {len(lens)} pairs")
            if len(lens) <= 2 and ezdist.token_balanced_ranges(cu, world)[-1] != (len(lens), len(lens)):
                fails.append("no empty rank in a few-pairs case")
        # the input check passes equal inputs and refuses unequal ones on every rank
        ezdist.check_replicated((16, 192, 3072, 900_000), "shapes")
        try:
            ezdist.check_replicated((16, 192 if rank == 0 else 191), "shapes")
            fails.append("unequal inputs accepted")
        except ValueError as e:
            if "differ across ranks" not in str(e):
                fails.append(str(e))
        ret[rank] = fails
    finally:
        dist.destroy_process_group()


def test_two_rank_score_exchange_is_bit_exact():
    world = 2
    mgr = mp.get_context("spawn").Manager()
    ret = mgr.dict()
    mp.spawn(_worker, args=(world, _free_port(), ret), nprocs=world, join=True)
    assert dict(ret) == {r: [] for r in range(world)}
