"""The numpy restatement of pb_index_rebalance_sharded (tests/sharded_rebalance.py) against the definitions it must
meet: the distributed balanced bounds equal pb_index_dir_shard_bounds' rule over all doc lengths, and each rank's new
inverted file is the slice of the deployment's global lists at its new range -- ivf_slice of the global inverted file
when the lists are sorted, the slice of the rank-order concatenation when they are not."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import sharded_rebalance as sr  # noqa: E402
from ivf_slice import ivf_slice, shard_bounds  # noqa: E402


def _partition(rng, D, W, empty_ok=True):
    cuts = np.sort(rng.integers(0, D + 1, W - 1))
    if not empty_ok:
        cuts = np.sort(rng.choice(np.arange(1, D), W - 1, replace=False))
    return np.concatenate([[0], cuts, [D]]).astype(np.int64)


def _ragged(rng, D):
    dl = rng.integers(0, 60, D)
    dl[rng.random(D) < 0.1] = 0                       # empty docs
    dl[rng.random(D) < 0.02] = 400                    # a few long ones
    return dl.astype(np.int64)


def _sorted_ivf(rng, D, K):
    lists = [np.sort(rng.choice(D, rng.integers(0, D // 3 + 1), replace=False)) for _ in range(K)]
    return np.concatenate(lists).astype(np.int64), np.array([len(x) for x in lists], np.int32)


@pytest.mark.parametrize("seed", range(12))
def test_balanced_bounds_equal_shard_bounds(seed):
    rng = np.random.default_rng(seed)
    D = int(rng.integers(1, 400))
    W = int(rng.integers(1, 9))
    dl = _ragged(rng, D)
    if seed == 0:
        dl[:] = 0                                      # no tokens at all
    old = _partition(rng, D, W)
    by_rank = [dl[old[r]:old[r + 1]] for r in range(W)]
    assert np.array_equal(sr.balanced_bounds(by_rank), shard_bounds(dl, W))


def test_balanced_bounds_one_long_doc():
    for W in (2, 3, 5):
        dl = np.array([1000], np.int64)
        assert np.array_equal(sr.balanced_bounds([dl[:0]] * (W - 1) + [dl]), shard_bounds(dl, W))
        assert np.array_equal(sr.balanced_bounds([dl] + [dl[:0]] * (W - 1)), shard_bounds(dl, W))


@pytest.mark.parametrize("seed", range(10))
def test_plan_tiles_old_and_new_ranges(seed):
    rng = np.random.default_rng(100 + seed)
    D, W = int(rng.integers(0, 300)), int(rng.integers(1, 8))
    old, new = _partition(rng, D, W), _partition(rng, D, W)
    p = sr.plan(old, new)
    for r in range(W):
        got = sorted(v for (s, t), v in p.items() if t == r)
        assert sum(hi - lo for lo, hi in got) == new[r + 1] - new[r]
        assert all(a[1] == b[0] for a, b in zip(got, got[1:]))
        got = sorted(v for (s, t), v in p.items() if s == r)
        assert sum(hi - lo for lo, hi in got) == old[r + 1] - old[r]


@pytest.mark.parametrize("seed", range(10))
def test_sorted_lists_give_the_global_slice(seed):
    rng = np.random.default_rng(200 + seed)
    D, W, K = int(rng.integers(1, 300)), int(rng.integers(1, 7)), int(rng.integers(1, 12))
    giv, gln = _sorted_ivf(rng, D, K)
    old = _partition(rng, D, W)
    new = _partition(rng, D, W) if seed % 2 else sr.balanced_bounds([_ragged(rng, 0)] * (W - 1) + [_ragged(rng, D)])
    ranks = [ivf_slice(giv, gln, int(old[s]), int(old[s + 1])) for s in range(W)]
    for r in range(W):
        iv, ln = sr.rank_ivf(ranks, old, new, r, K)
        want = ivf_slice(giv, gln, int(new[r]), int(new[r + 1]))
        assert np.array_equal(iv, want[0]) and np.array_equal(ln, want[1]), r


@pytest.mark.parametrize("seed", range(10))
def test_unsorted_lists_give_the_slice_of_the_rank_order_concatenation(seed):
    rng = np.random.default_rng(300 + seed)
    D, W, K = int(rng.integers(1, 300)), int(rng.integers(2, 7)), int(rng.integers(1, 12))
    giv, gln = _sorted_ivf(rng, D, K)
    old = _partition(rng, D, W)
    ranks = []
    for s in range(W):
        iv, ln = ivf_slice(giv, gln, int(old[s]), int(old[s + 1]))
        off = np.concatenate([[0], np.cumsum(ln)]).astype(np.int64)
        iv = np.concatenate([rng.permutation(iv[off[c]:off[c + 1]]) for c in range(K)]).astype(np.int64)
        ranks.append((iv, ln))
    cat = sr.global_lists(ranks, old, K)
    new = _partition(rng, D, W)
    for r in range(W):
        iv, ln = sr.rank_ivf(ranks, old, new, r, K)
        want = ivf_slice(cat[0], cat[1], int(new[r]), int(new[r + 1]))
        assert np.array_equal(iv, want[0]) and np.array_equal(ln, want[1]), r
