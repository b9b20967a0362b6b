"""The pruned first pass of a5 keeps the dense band doc for doc (tests/a5_prune.py restates both), on random and
adversarial inputs: ties at theta1 and at tau, all-equal bounds, fewer candidates than M, floors of 0 and 65535."""
import numpy as np
import pytest

import a5_prune as P


def _case(seed, K=300, nq=8, D=400, lo=0, hi=65536, doclen=(1, 12)):
    rng = np.random.default_rng(seed)
    T = rng.integers(lo, hi, (K, nq)).astype(np.int64)
    docs = [rng.choice(K, int(rng.integers(*doclen)), replace=False) for _ in range(D)]
    return T, docs


def _check(T, docs, f, M, M1, W):
    L = P.first_pass(T, docs)
    U, _ = P.bound(T, docs, f)
    assert (U >= L).all()
    band, n_dense = P.pruned_band(L, U, M, M1, W)
    assert band == P.dense_band(L, M, W)
    assert n_dense <= len(docs)
    return n_dense


@pytest.mark.parametrize("seed", range(12))
def test_random_floors(seed):
    T, docs = _case(seed)
    rng = np.random.default_rng(100 + seed)
    for f in (np.zeros(T.shape[1]), np.full(T.shape[1], 65535), np.full(T.shape[1], 65536),
              rng.integers(0, 65536, T.shape[1]), np.quantile(T, 0.97, axis=0).astype(np.int64)):
        for M, M1 in ((16, 16), (16, 40), (64, 128), (500, 600)):
            _check(T, docs, f, M, M1, W=4 * T.shape[1] + 8)


def test_floor_zero_is_the_dense_pass():
    T, docs = _case(1)
    U, live_rows = P.bound(T, docs, np.zeros(T.shape[1]))
    assert (U == P.first_pass(T, docs)).all() and live_rows == sum(len(d) for d in docs)


def test_floor_above_every_code_keeps_every_doc():
    T, docs = _case(2)
    L = P.first_pass(T, docs)
    U, live_rows = P.bound(T, docs, np.full(T.shape[1], 65536))
    assert live_rows == 0 and len(set(U.tolist())) == 1
    assert P.pruned_band(L, U, 16, 32, 40)[1] == len(docs)


def test_ties_at_theta1_and_tau():
    # a narrow code range makes many equal sums: ties at theta1 (U) and at tau (L)
    T, docs = _case(3, lo=100, hi=104, doclen=(1, 3))
    f = np.full(T.shape[1], 103)
    L = P.first_pass(T, docs)
    U, _ = P.bound(T, docs, f)
    theta1 = P.select(U, 32, 0)
    assert (U == theta1).sum() > 1 and (L == P.select(L, 16, 0)).sum() > 1
    for W in (0, 1, 40):
        _check(T, docs, f, 16, 32, W)


def test_all_equal_bounds_and_few_candidates():
    T, docs = _case(4, D=10)
    for f in (np.zeros(T.shape[1]), np.full(T.shape[1], 65536), np.full(T.shape[1], 30000)):
        _check(T, docs, f, 16, 32, 40)   # fewer candidates than M: everything is kept
        _check(T, docs, f, 4, 32, 0)     # fewer than M1 but more than M


def test_round_two_is_needed_when_m1_is_m():
    # with a high floor and M1 = M, round 1 alone misses part of the band: the result still equals the dense one
    for seed in range(20):
        T, docs = _case(seed, D=600)
        f = np.quantile(T, 0.995, axis=0).astype(np.int64)
        L = P.first_pass(T, docs)
        U, _ = P.bound(T, docs, f)
        theta1 = P.select(U, 16, 0)
        r1 = np.flatnonzero(U >= theta1)
        if not P.dense_band(L, 16, 40) <= set(r1.tolist()):
            assert _check(T, docs, f, 16, 16, 40) > len(r1)
            return
    pytest.fail("no case where round 1 alone misses the band")
