"""CPU checks for changing a deployment's number of ranks (pb_index_add_devices / pb_index_remove_ranks, DESIGN.md 4t):
the argument checks that come before any device is touched, also in a process that sees no device, and a numpy
restatement of the balanced bounds of a removal -- each rank offers, per boundary of the surviving world, the least doc
of its closed range that qualifies; the least offer wins; a leaving rank gets the empty range where the next surviving
rank starts -- which must give pb_index_dir_shard_bounds of the new world whatever the current layout."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PB_ERR_INVALID = 1


@pytest.fixture(scope="module")
def npb():
    import next_plaid_b200 as m
    m.build_library()
    return m


def _null_calls(L):
    """(name, status) of each call with a null argument"""
    dv = np.zeros(2, np.int32)
    b = np.zeros(4, np.int64)
    p = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    return [("add: null handle", L.pb_index_add_devices(None, p(dv), 1, None, None)),
            ("add: null handle and bounds", L.pb_index_add_devices(None, p(dv), 2, p(b), p(b))),
            ("add: null devices", L.pb_index_add_devices(None, None, 1, None, None)),
            ("remove: null handle", L.pb_index_remove_ranks(None, p(dv), 1, None, None)),
            ("remove: null ranks", L.pb_index_remove_ranks(None, None, 1, p(b), None))]


def test_null_arguments_are_invalid(npb):
    L = npb.load_library()
    for name, st in _null_calls(L):
        assert st == PB_ERR_INVALID, name
        assert "null argument" in L.pb_last_error().decode(), name


def test_null_arguments_without_a_device():
    code = (
        "import sys\n"
        f"sys.path.insert(0, {ROOT!r}); sys.path.insert(0, {os.path.dirname(os.path.abspath(__file__))!r})\n"
        "import next_plaid_b200 as m\n"
        "from test_deployment_resize_cpu import _null_calls\n"
        "L = m.load_library()\n"
        "assert m.device_count() == 0\n"
        "assert all(st == 1 for _, st in _null_calls(L)), _null_calls(L)\n"
        "print('ok')\n")
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and r.stdout.strip() == "ok", r.stdout + r.stderr


def _layout_dir(path, doclens):
    """A directory with only what the bounds read: metadata.json and one doclens file"""
    os.makedirs(path, exist_ok=True)
    with open(os.path.join(path, "doclens.0.json"), "w") as f:
        json.dump([int(x) for x in doclens], f)
    with open(os.path.join(path, "metadata.json"), "w") as f:
        json.dump({"num_chunks": 1, "nbits": 4, "num_embeddings": int(np.sum(doclens))}, f)
    return path


def removal_bounds(doclens, old, stays):
    """The bounds over the old world after a removal: the balanced split over the S surviving ranks, computed from the
    offers of every rank (leaving ones included: they still hold documents), expanded with empty ranges"""
    off = np.concatenate([[0], np.cumsum(doclens)]).astype(np.int64)
    D, N, W = len(doclens), int(off[-1]), len(old) - 1
    S = int(np.sum(stays))
    offers = np.full((W, S + 1), D, np.int64)
    for s in range(W):
        for j in range(1, S):
            ok = [d for d in range(old[s], old[s + 1] + 1) if off[d] * S >= N * j]
            if ok:
                offers[s, j] = ok[0]
    c = offers.min(axis=0)
    c[0], c[S] = 0, D
    b, j = [], 0
    for r in range(W):
        b.append(int(c[j]))
        j += int(stays[r])
    return b + [D]


def test_removal_bounds_are_the_new_worlds_split(npb, tmp_path):
    rng = np.random.default_rng(23)
    cases = [rng.integers(1, 60, 80), rng.integers(0, 4, 30), np.array([1, 1, 500, 1, 1, 1]), rng.integers(1, 9, 7)]
    for ci, doclens in enumerate(cases):
        path = _layout_dir(str(tmp_path / f"c{ci}"), doclens)
        D = len(doclens)
        for _ in range(25):
            W = int(rng.integers(2, 10))
            old = [0] + sorted(rng.integers(0, D + 1, W - 1).tolist()) + [D]   # any partition, empty ranks included
            n = int(rng.integers(1, W))
            stays = np.ones(W, bool)
            stays[rng.choice(W, n, replace=False)] = False
            b = removal_bounds(doclens, old, stays)
            assert b[0] == 0 and b[-1] == D and all(x <= y for x, y in zip(b, b[1:]))
            assert all(b[r] == b[r + 1] for r in range(W) if not stays[r]), (old, stays, b)
            kept = [b[r] for r in range(W) if stays[r]] + [D]
            assert kept == npb.shard_bounds(path, W - n).tolist(), (old, stays, b)
            # no rank leaving: the rebalance's own balanced split over the old world
            assert removal_bounds(doclens, old, np.ones(W, bool)) == npb.shard_bounds(path, W).tolist()
