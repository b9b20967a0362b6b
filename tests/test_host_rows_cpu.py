"""The segmented pinned row store of host-tier handles (tests/host_rows.py restates it): how byte ranges split into
segment pieces, how the store opens and grows, and that a delete's windows and pieces give np.delete of the rows."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import host_rows as hr  # noqa: E402


@pytest.mark.parametrize("shift", [8, 9, 12])
def test_pieces_cover_the_range_in_order(shift):
    rng = np.random.default_rng(shift)
    S = 1 << shift
    for _ in range(300):
        b, n = int(rng.integers(0, 5 * S)), int(rng.integers(0, 4 * S))
        ps = hr.pieces(b, n, shift)
        assert sum(m for *_, m in ps) == n
        done = 0
        for k, o, r, m in ps:
            assert r == done and 0 < m <= S - o and k * S + o == b + done
            done += m
        assert len(ps) == (0 if n == 0 else ((b + n - 1) >> shift) - (b >> shift) + 1)


@pytest.mark.parametrize("packed", [6, 8, 16, 32, 64, 128])
def test_rows_straddle_segments_but_load_units_do_not(packed):
    # dim 48 at 1 bit: 6-byte rows, 2-byte units; 4-byte units when packed % 4 == 0, 16-byte ones when packed % 16 == 0
    shift = 8
    unit = 16 if packed % 16 == 0 else 2 if packed % 4 else 4
    straddle = 0
    for t in range(1000):
        ps = hr.pieces(t * packed, packed, shift)
        straddle += len(ps) > 1
        for u in range(0, packed, unit):
            assert len(hr.pieces(t * packed + u, unit, shift)) == 1
    assert straddle == 0 if (1 << shift) % packed == 0 else straddle > 0


def test_open_and_grow():
    shift = 8
    assert hr.open_sizes(0, shift) == []
    assert hr.open_sizes(256, shift) == [256]
    assert hr.open_sizes(600, shift) == [256, 256, 88]
    assert hr.grow_sizes([256, 256, 88], 500, shift) == [256, 256, 88]      # enough capacity: nothing changes
    assert hr.grow_sizes([256, 256, 88], 601, shift) == [256, 256, 256]     # the short segment becomes a full one
    assert hr.grow_sizes([256, 256, 88], 1025, shift) == [256] * 5
    assert hr.grow_sizes([], 1, shift) == [256]


def test_write_read_round_trip_through_a_grown_store():
    rng = np.random.default_rng(3)
    shift, packed = 8, 6
    rows = rng.integers(0, 256, (150, packed), dtype=np.uint8)
    segs = hr.store(rows, shift)
    assert [len(s) for s in segs] == hr.open_sizes(rows.size, shift)
    new = rng.integers(0, 256, (77, packed), dtype=np.uint8)
    sizes = hr.grow_sizes([len(s) for s in segs], rows.size + new.size, shift)
    grown = [np.zeros(m, np.uint8) for m in sizes]
    for k, s in enumerate(segs):
        grown[k][:len(s)] = s
    hr.write(grown, rows.size, new.reshape(-1), shift)
    assert np.array_equal(hr.read(grown, 0, rows.size + new.size, shift), np.concatenate([rows, new]).reshape(-1))


@pytest.mark.parametrize("shift", [8, 12, 20])
@pytest.mark.parametrize("packed", [6, 16, 64])
def test_delete_equals_np_delete(shift, packed):
    rng = np.random.default_rng(shift * 100 + packed)
    for trial in range(40):
        D = int(rng.integers(1, 120))
        dl = rng.integers(0, 30, D)
        rows = rng.integers(0, 256, (int(dl.sum()), packed), dtype=np.uint8)
        pattern = trial % 5
        if pattern == 0:
            gone = rng.choice(D, int(rng.integers(0, D + 1)), replace=False)      # scattered
        elif pattern == 1:
            gone = np.arange(int(rng.integers(0, D + 1)))                          # oldest
        elif pattern == 2:
            gone = np.arange(int(rng.integers(0, D + 1)), D)                       # newest
        elif pattern == 3:
            gone = np.arange(D)                                                    # all
        else:
            gone = np.zeros(0, np.int64)                                           # none
        window = int(rng.choice([1, 7, 40, 1 << 22]))
        kept, old_off, new_off, wins = hr.delete_plan(dl, gone, window)
        assert np.all(new_off[:-1] <= old_off[kept])                               # survivors only move down
        for j0, j1 in wins:                                                        # windows fit, or hold one long doc
            assert j1 - j0 == 1 or new_off[j1] - new_off[j0] <= window
        segs, n_tok = hr.compact(hr.store(rows, shift), dl, gone, window, packed, shift)
        old_off_rows = np.repeat(np.arange(D), dl)
        want = rows[~np.isin(old_off_rows, gone)]
        assert n_tok == len(want)
        assert np.array_equal(hr.read(segs, 0, n_tok * packed, shift), want.reshape(-1)), (trial, window)
