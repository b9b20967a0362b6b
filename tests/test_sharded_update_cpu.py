"""The sharded delete and append of tests/sharded_update.py: for random partitions of random indexes, every rank's
local patch equals its slice of the global patch, and the new bounds tile the remaining documents."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import sharded_update as su  # noqa: E402


def _index(rng, D, K):
    """a random inverted file: each doc in a few centroids' lists, lists in ascending id order"""
    lists = [[] for _ in range(K)]
    codes, dl = [], []
    for d in range(D):
        n = int(rng.integers(1, 6))
        c = rng.integers(0, K, n)
        codes.extend(c.tolist())
        dl.append(n)
        for x in sorted(set(c.tolist())):
            lists[x].append(d)
    ivf = np.array([d for l in lists for d in l], np.int64)
    return ivf, np.array([len(l) for l in lists], np.int32), np.array(codes, np.int64), np.array(dl, np.int64)


def _bounds(rng, D, W, empty_rank=None):
    cut = np.sort(rng.integers(0, D + 1, W - 1))
    b = np.concatenate([[0], cut, [D]]).astype(np.int64)
    if W == 1:
        return b
    if empty_rank == W - 1:                       # rank empty_rank holds nothing
        b[W - 1] = D
    elif empty_rank is not None:
        b[empty_rank + 1] = b[empty_rank]
        b = np.maximum.accumulate(b)
    return b


def _patterns(rng, D, bounds):
    yield "scattered_invalid_repeated", np.concatenate([rng.choice(D, D // 7, replace=False), [-1, -5, D, D + 3],
                                                        rng.choice(D, 5)])
    yield "oldest", np.arange(0, int(bounds[1]) + 2)
    yield "newest", np.arange(D - D // 5, D)
    yield "across_a_boundary", np.arange(max(int(bounds[1]) - 3, 0), min(int(bounds[1]) + 3, D))
    yield "every_other", np.arange(0, D, 2)
    yield "all", np.arange(D)
    yield "none", np.array([-1, D], np.int64)


@pytest.mark.parametrize("W", [1, 2, 3, 8])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_rank_delete_equals_slice_of_global_delete(W, seed):
    rng = np.random.default_rng(seed * 10 + W)
    D, K = int(rng.integers(40, 120)), 16
    ivf, lens, _, _ = _index(rng, D, K)
    for bounds in (_bounds(rng, D, W), _bounds(rng, D, W, empty_rank=W // 2)):
        for name, ids in _patterns(rng, D, bounds):
            nb = su.delete_bounds(bounds, ids)
            removed = len(su.deleted_set(ids, D))
            assert nb[0] == 0 and nb[-1] == D - removed and np.all(np.diff(nb) >= 0), name
            for r in range(W):                    # each rank's new size is its old one minus its own deletions
                mine = su.deleted_set(ids, D)
                own = int(((mine >= bounds[r]) & (mine < bounds[r + 1])).sum())
                assert nb[r + 1] - nb[r] == bounds[r + 1] - bounds[r] - own, (name, r)
            want = su.global_delete_slices(ivf, lens, bounds, ids)
            for r in range(W):
                got = su.rank_delete(ivf, lens, bounds, r, ids)
                assert np.array_equal(got[0], want[r][0]) and np.array_equal(got[1], want[r][1]), (name, r)


@pytest.mark.parametrize("W", [1, 2, 3, 8])
@pytest.mark.parametrize("seed", [0, 1])
def test_last_rank_append_equals_slice_of_global_merge(W, seed):
    rng = np.random.default_rng(100 + seed * 10 + W)
    D, K = int(rng.integers(40, 120)), 16
    ivf, lens, _, _ = _index(rng, D, K)
    for bounds in (_bounds(rng, D, W), _bounds(rng, D, W, empty_rank=W - 1)):
        for n in (0, 1, 13):
            dl = rng.integers(0, 5, n)
            codes = rng.integers(0, K, int(dl.sum()))
            got = su.rank_append(ivf, lens, bounds, codes, dl, K)
            want = su.global_append_slice(ivf, lens, bounds, codes, dl, K)
            assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]), n
            for r in range(W - 1):                # the other ranks' slices do not move
                from ivf_merge import merge_ivf
                from ivf_slice import ivf_slice
                g = merge_ivf(ivf, lens, codes, dl, D, K)
                mine = ivf_slice(g[0], g[1], int(bounds[r]), int(bounds[r + 1]))
                orig = ivf_slice(ivf, lens, int(bounds[r]), int(bounds[r + 1]))
                assert np.array_equal(mine[0], orig[0]) and np.array_equal(mine[1], orig[1])


def test_append_then_delete_cycle_keeps_ranks_equal_to_global():
    rng = np.random.default_rng(7)
    D, K, W = 90, 12, 3
    ivf, lens, _, _ = _index(rng, D, K)
    bounds = _bounds(rng, D, W)
    ranks = [su.ivf_slice(ivf, lens, int(bounds[r]), int(bounds[r + 1])) for r in range(W)]
    for step in range(4):
        dl = rng.integers(1, 4, 10)
        codes = rng.integers(0, K, int(dl.sum()))
        from ivf_merge import merge_ivf
        ranks[-1] = merge_ivf(ranks[-1][0], ranks[-1][1], codes, dl, int(bounds[-1] - bounds[-2]), K)
        ivf, lens = merge_ivf(ivf, lens, codes, dl, int(bounds[-1]), K)
        bounds = bounds.copy()
        bounds[-1] += len(dl)
        ids = rng.choice(int(bounds[-1]), 15, replace=False)
        from ivf_delete import delete_ivf
        for r in range(W):
            b, e = int(bounds[r]), int(bounds[r + 1])
            mine = su.deleted_set(ids, int(bounds[-1]))
            ranks[r] = delete_ivf(ranks[r][0], ranks[r][1], mine[(mine >= b) & (mine < e)] - b, e - b)
        want = su.global_delete_slices(ivf, lens, bounds, ids)
        ivf, lens = delete_ivf(ivf, lens, su.deleted_set(ids, int(bounds[-1])), int(bounds[-1]))
        bounds = su.delete_bounds(bounds, ids)
        for r in range(W):
            assert np.array_equal(ranks[r][0], want[r][0]) and np.array_equal(ranks[r][1], want[r][1]), (step, r)
