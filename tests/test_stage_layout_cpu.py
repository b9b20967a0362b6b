"""The slot layout of the host-tier exact stage (tests/stage_layout.py) on random kept lists: empty queries, queries
that keep Mcap docs, zero-length docs.  Reading a doc's rows through the staged offsets of its slot gives the rows the
resident handle reads through doc_off, and the map back turns any list of slots into the docs they stand for."""
import numpy as np
import pytest

import stage_layout as sl


def _case(seed, B, Mcap, D):
    rng = np.random.default_rng(seed)
    lengths = rng.integers(0, 40, D)
    lengths[rng.random(D) < 0.2] = 0                           # zero-length docs
    doc_off = np.concatenate([[0], np.cumsum(lengths)])
    nkept = rng.integers(0, Mcap + 1, B)
    nkept[0] = 0                                                # an empty query
    nkept[-1] = Mcap                                            # a full one
    kept = np.zeros(B * Mcap, np.uint32)
    tokp = np.zeros((B, Mcap + 1), np.int64)
    for b in range(B):
        docs = rng.choice(D, nkept[b], replace=False)           # one query's kept docs are distinct
        kept[b * Mcap:b * Mcap + nkept[b]] = docs
        tokp[b, 1:nkept[b] + 1] = np.cumsum(lengths[docs])
        tokp[b, nkept[b] + 1:] = rng.integers(0, 1000, Mcap - nkept[b])  # past nkept: whatever the cut left there
    return doc_off, kept, nkept, tokp


@pytest.mark.parametrize("seed,B,Mcap,D", [(0, 1, 1, 3), (1, 4, 8, 50), (2, 7, 16, 20), (3, 32, 33, 400), (4, 3, 64, 64)])
def test_slot_layout(seed, B, Mcap, D):
    doc_off, kept, nkept, tokp = _case(seed, B, Mcap, D)
    soff, kept_s = sl.layout(nkept, tokp, Mcap)
    assert np.array_equal(kept_s, np.arange(B * Mcap))
    assert np.all(np.diff(soff) >= 0)
    assert soff[0] == 0 and soff[-1] == sum(tokp[b, nkept[b]] for b in range(B))
    for b in range(B):
        for j in range(Mcap):
            s = b * Mcap + j
            want = doc_off[kept[s] + 1] - doc_off[kept[s]] if j < nkept[b] else 0
            assert soff[s + 1] - soff[s] == want, (b, j)
            if j <= nkept[b]:                                  # the kernels' token prefix is unchanged
                assert soff[s] - soff[b * Mcap] == tokp[b, j]


@pytest.mark.parametrize("seed", range(4))
def test_staged_rows_equal_resident_rows(seed):
    doc_off, kept, nkept, tokp = _case(seed, 5, 12, 90)
    Mcap = 12
    rng = np.random.default_rng(seed + 100)
    N = int(doc_off[-1])
    res = rng.integers(0, 256, (N, 16), dtype=np.uint8)
    codes = rng.integers(0, 1000, N).astype(np.uint32)
    soff, kept_s = sl.layout(nkept, tokp, Mcap)
    s_res = sl.stage(res, doc_off, kept, nkept, soff, Mcap)
    s_codes = sl.stage(codes, doc_off, kept, nkept, soff, Mcap)
    for b in range(len(nkept)):
        for j in range(nkept[b]):
            d, s = kept[b * Mcap + j], kept_s[b * Mcap + j]
            assert np.array_equal(s_res[soff[s]:soff[s + 1]], res[doc_off[d]:doc_off[d + 1]])
            assert np.array_equal(s_codes[soff[s]:soff[s + 1]], codes[doc_off[d]:doc_off[d + 1]])


@pytest.mark.parametrize("seed", range(4))
def test_map_back(seed):
    doc_off, kept, nkept, tokp = _case(seed, 6, 10, 70)
    Mcap = 10
    _, kept_s = sl.layout(nkept, tokp, Mcap)
    # the kept list itself
    assert np.array_equal(sl.unstage(kept_s, nkept, Mcap, kept)[_valid(nkept, Mcap)], kept[_valid(nkept, Mcap)])
    # a survivor list: an ordered subset of each query's slots, as the filter leaves it
    rng = np.random.default_rng(seed)
    surv = np.zeros(len(nkept) * Mcap, np.uint32)
    nsurv = np.zeros(len(nkept), np.int64)
    for b in range(len(nkept)):
        pick = np.sort(rng.choice(nkept[b], rng.integers(0, nkept[b] + 1), replace=False)) if nkept[b] else []
        nsurv[b] = len(pick)
        surv[b * Mcap:b * Mcap + len(pick)] = b * Mcap + np.asarray(pick, np.int64)
    got = sl.unstage(surv, nsurv, Mcap, kept)
    for b in range(len(nkept)):
        idx = surv[b * Mcap:b * Mcap + nsurv[b]]
        assert np.array_equal(got[b * Mcap:b * Mcap + nsurv[b]], kept[idx])


def _valid(nkept, Mcap):
    return np.concatenate([np.arange(Mcap) < n for n in nkept])
