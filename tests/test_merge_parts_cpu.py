"""CPU: the merge-by-rank that ``ezr_merge_sorted_parts`` (csrc/merge.cu) runs, restated in numpy, against a lexsort of
the union; and the per-route depths of ``RecordLayout`` (easyrag_b200/dist.py).

Merge by rank: every part is in canonical order (score desc, id desc) up to its first id < 0 and ids are distinct
across parts, so an element's output rank is its index in its own list plus, for every other part, the number of that
part's elements that are better than it.  Ranks < k are the output slots."""
import numpy as np
import pytest

from easyrag_b200 import dist as ezdist


def _better(sa, ia, sb, ib):
    return (sa > sb) | ((sa == sb) & (ia > ib))


def merge_by_rank(s, ids, k):
    """s, ids: [G, n] parts of one row (canonical prefix, then ids < 0) -> (ids [k] -1 padded, scores [k], count)."""
    G, n = ids.shape
    cnt = [int(np.argmax(ids[p] < 0)) if (ids[p] < 0).any() else n for p in range(G)]
    out_i, out_s = np.full(k, -1, np.int32), np.full(k, -np.inf, s.dtype)
    for p in range(G):
        for j in range(min(cnt[p], k)):
            rank = j
            for q in range(G):
                if q != p:
                    # the elements of q better than (s, id) form a prefix of q's list: a binary search
                    b = _better(s[q, :cnt[q]], ids[q, :cnt[q]], s[p, j], ids[p, j])
                    lo = int(np.searchsorted(~b, True))
                    assert not b[lo:].any() and b[:lo].all()
                    rank += lo
            if rank < k:
                assert out_i[rank] == -1, "two elements with one rank"
                out_i[rank], out_s[rank] = ids[p, j], s[p, j]
    count = min(sum(cnt), k)
    assert (out_i[:count] >= 0).all() and (out_i[count:] == -1).all()
    return out_i, out_s, count


def _parts(rng, G, n, values, counts):
    span = 2 * n + 3
    s = rng.choice(values, (G, n))
    ids = np.stack([rng.permutation(span)[:n] + p * span for p in range(G)]).astype(np.int32)
    order = np.lexsort((-ids, -s), axis=-1)
    s, ids = np.take_along_axis(s, order, -1), np.take_along_axis(ids, order, -1)
    past = np.arange(n)[None, :] >= np.asarray(counts)[:, None]
    return np.where(past, np.inf, s), np.where(past, -1, ids).astype(np.int32)


def _lexsort_ref(s, ids, k):
    v = ids.reshape(-1) >= 0
    sv, iv = s.reshape(-1)[v], ids.reshape(-1)[v]
    o = np.lexsort((-iv, -sv))[:k]
    return iv[o], sv[o], min(int(v.sum()), k)


@pytest.mark.parametrize("values", ["random", "tied", "signed_zeros"])
def test_merge_by_rank_against_lexsort(values):
    rng = np.random.default_rng(7)
    vals = dict(random=rng.standard_normal(1000), tied=np.array([1.0, 2.0, 3.0]),
                signed_zeros=np.array([-0.0, 0.0, 0.5]))[values]
    cases = 0
    for G in (1, 2, 3, 8):
        for n in (1, 5, 33):
            for k in (1, 4, 33, 70):
                for counts in ([n] * G, [0] * G, list(rng.integers(0, n + 1, G)), [0] * (G - 1) + [n]):
                    s, ids = _parts(rng, G, n, vals, counts)
                    gi, gs, gc = merge_by_rank(s, ids, k)
                    ri, rs, rc = _lexsort_ref(s, ids, k)
                    assert gc == rc and np.array_equal(gi[:gc], ri)
                    assert gs[:gc].tobytes() == rs.tobytes(), "score bytes (the sign of a zero included)"
                    cases += 1
    assert cases == 4 * 3 * 4 * 4


def test_record_layout_equal_k_is_todays_formula():
    """An equal-k layout (k_sparse None or == k) has exactly the offsets and size of the one-depth record."""
    for q, k, sb in ((1, 1, 8), (7, 10, 8), (10_000, 10, 4), (3, 33, 8), (5, 288, 4)):
        n = q * k
        want, o = [], 0
        for s in (n * 4, n * 4, n * sb, n * 4):
            want.append(o)
            o += (s + 15) // 16 * 16
        for lay in (ezdist.RecordLayout(q, k, sb), ezdist.RecordLayout(q, k, sb, k_sparse=k)):
            assert lay.offsets == (want, o) and lay.nbytes == o
            assert lay.sizes == (n * 4, n * 4, n * sb, n * 4)


def test_record_layout_per_route_depth():
    import torch
    for q, kd, ks, sb in ((1, 1, 1024, 8), (7, 288, 192, 8), (9, 288, 192, 4), (3, 6, 193, 4), (10, 1024, 33, 8)):
        lay = ezdist.RecordLayout(q, kd, sb, k_sparse=ks)
        offs, total = lay.offsets
        assert all(o % 16 == 0 for o in offs) and total % 16 == 0 and total == lay.nbytes
        assert lay.sizes == (q * kd * 4, q * kd * 4, q * ks * sb, q * ks * 4)
        assert all(offs[i] + lay.sizes[i] <= offs[i + 1] for i in range(3)) and offs[3] + lay.sizes[3] <= total
        buf = torch.zeros(2 * total, dtype=torch.uint8)
        views = ezdist.record_views(lay, buf[total:])
        assert [tuple(v.shape) for v in views] == [(q, kd), (q, kd), (q, ks), (q, ks)]
        assert [v.dtype for v in views] == [torch.float32, torch.int32,
                                           torch.float64 if sb == 8 else torch.float32, torch.int32]
        for j, v in enumerate(views):
            v.fill_(j + 1)
        raw = buf[total:]
        for j, v in enumerate(views):
            assert v.data_ptr() == raw.data_ptr() + offs[j]
        assert not buf[:total].any()
