"""CPU checks of the device row cache (DESIGN.md 4s): the numpy selection rule the GPU tests compare fills against, and
the entry points' argument refusals, which come before any device use."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import row_cache  # noqa: E402

PB_ERR_INVALID = 1


@pytest.mark.parametrize("seed", range(6))
def test_fill_by_counts_orders_skips_and_fits(seed):
    rng = np.random.default_rng(seed)
    D = int(rng.integers(1, 400))
    counts = rng.integers(0, 6, D) * (rng.random(D) < 0.6)
    lengths = rng.integers(0, 90, D)
    packed = int(rng.choice([6, 12, 32, 64]))
    budget = int(rng.integers(0, int(lengths.sum()) * packed + 2))
    order = row_cache.order_by_counts(counts)
    assert all(counts[d] > 0 for d in order) and len(order) == int((counts > 0).sum())
    for a, b in zip(order[:-1], order[1:]):
        assert counts[a] > counts[b] or (counts[a] == counts[b] and a < b)
    taken, used = row_cache.fit_or_skip(order, lengths, packed, budget)
    assert used == int(lengths[taken].sum()) * packed <= budget
    # taken keeps the order, and every doc left out did not fit after the docs taken before it
    pos = {int(d): i for i, d in enumerate(order)}
    assert [pos[int(d)] for d in taken] == sorted(pos[int(d)] for d in taken)
    run = 0
    for d in order:
        if d in set(taken.tolist()):
            run += int(lengths[d]) * packed
        else:
            assert run + int(lengths[d]) * packed > budget


def test_fill_with_ids_ignores_outside_and_repeats():
    order = row_cache.order_of_ids([5, -1, 3, 5, 10, 12, 3, 0], 11, base=0)
    assert order.tolist() == [5, 3, 10, 0]
    assert row_cache.order_of_ids([100, 104, 99, 110], 10, base=100).tolist() == [0, 4]
    lengths = np.array([4, 1, 1, 10, 1, 2, 1, 1, 1, 1, 3])
    taken, used = row_cache.fit_or_skip(order, lengths, 2, 18)
    assert taken.tolist() == [5, 10, 0] and used == 18       # doc 3 (20 bytes) skipped, later ones still taken
    assert row_cache.fit_or_skip(order, lengths, 2, 1)[0].tolist() == []  # a budget smaller than one doc


def test_keep_counts_of_kept_lists():
    c = row_cache.keep_counts([[3, 1], [1], [], [4, 3, 1]], 5)
    assert c.tolist() == [0, 3, 0, 2, 1]
    assert row_cache.order_by_counts(c).tolist() == [1, 3, 4]


@pytest.fixture(scope="module")
def lib():
    import next_plaid_b200 as m
    m.build_library()
    return m.load_library()


def test_argument_refusals_come_first(lib):
    n = C.c_int64(7)
    assert lib.pb_index_set_row_cache(None, -1) == PB_ERR_INVALID
    assert b"< 0" in lib.pb_last_error()
    assert lib.pb_index_set_row_cache(None, 1 << 20) == PB_ERR_INVALID
    assert lib.pb_index_fill_row_cache(None, None, 0, None, 0, C.byref(n)) == PB_ERR_INVALID
    assert n.value == 7
    ids = np.arange(3, dtype=np.int64)
    assert lib.pb_index_fill_row_cache(None, ids.ctypes.data_as(C.c_void_p), 3, None, 0, None) == PB_ERR_INVALID
    assert lib.pb_index_row_cache_stats(None, None, 0) == PB_ERR_INVALID
