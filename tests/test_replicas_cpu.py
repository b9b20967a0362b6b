"""CPU checks for a replica set behind one handle (pb_index_load_replicas): the argument checks come before any device is
touched, in their stated order, and without a usable device the load fails with PB_ERR_CUDA (there is no CPU path).
The no-device case runs in a child process that sees no device, so it holds on a GPU machine as well."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PB_ERR_INVALID, PB_ERR_CUDA = 1, 2


@pytest.fixture(scope="module")
def npb():
    import next_plaid_b200 as m
    m.build_library()
    return m


@pytest.fixture(scope="module")
def index_dir(oracle, tmp_path_factory):
    docs = oracle.synthetic_corpus(60, 10, dim=32, seed=8, ragged=True)
    ix = oracle.create_index(docs, nbits=4, seed=1, num_partitions=16)
    d = str(tmp_path_factory.mktemp("ix"))
    oracle.write_index(ix, d, chunk_docs=25)
    return d


def _load(npb, path, devices, n=None, shards=1, out=True):
    """raw pb_index_load_replicas: (status, message, handle)"""
    L = npb.load_library()
    dv = None if devices is None else np.ascontiguousarray(devices, np.int32)
    h = C.c_void_p()
    st = L.pb_index_load_replicas(None if path is None else os.fsencode(path),
                                  None if dv is None else dv.ctypes.data_as(C.c_void_p),
                                  len(dv) if n is None else n, shards, 0, C.byref(h) if out else None)
    return st, L.pb_last_error().decode(), h


def test_argument_checks_come_first(npb, index_dir):
    # each row breaks one rule, and every later one too: the first rule decides the message
    cases = [((None, [0], None, 1), "null argument"),
             ((index_dir, None, 1, 1), "null argument"),
             ((index_dir, [0], None, 1, False), "null argument"),
             ((index_dir, [0] * 65, None, 0), "n_shards 0 < 1"),
             ((index_dir, [0] * 65, None, -2), "n_shards -2 < 1"),
             ((index_dir, [0] * 3, None, 2), "not a positive multiple of n_shards 2"),
             ((index_dir, [0], 0, 1), "not a positive multiple"),
             ((index_dir, [0], -4, 1), "not a positive multiple"),
             ((index_dir, [0] * 66, None, 2), "above 64 members"),
             (("/nonexistent/dir", [-1] * 65, None, 1), "above 64 members")]
    for args, text in cases:
        st, msg, h = _load(npb, *args)
        assert st == PB_ERR_INVALID and not h.value and text in msg, (args[1:], msg)


def test_device_ids_are_checked_after_the_device_count(npb, index_dir):
    have = npb.device_count()
    for devices, shards in (([-1], 1), ([0, have], 1), ([0, 0, 0, have + 1000], 2)):
        st, msg, h = _load(npb, index_dir, devices, shards=shards)
        assert st == (PB_ERR_INVALID if have else PB_ERR_CUDA) and not h.value, (devices, msg)


def test_layout_and_stats_of_a_null_handle_are_invalid(npb):
    L = npb.load_library()
    r, s = C.c_int32(), C.c_int32()
    assert L.pb_index_replica_layout(None, C.byref(r), C.byref(s), None) == PB_ERR_INVALID
    assert L.pb_index_replica_stats(None, None, None, 0) == PB_ERR_INVALID


def test_without_a_device_the_load_fails_with_cuda(index_dir):
    code = (
        "import ctypes as C, os, sys, numpy as np\n"
        f"sys.path.insert(0, {ROOT!r})\n"
        "import next_plaid_b200 as m\n"
        "L = m.load_library()\n"
        "assert m.device_count() == 0\n"
        "h = C.c_void_p()\n"
        "for dirname, n, shards in ((sys.argv[1], 2, 1), ('/nonexistent/dir', 4, 2)):\n"
        "    dv = np.zeros(n, np.int32)\n"
        "    st = L.pb_index_load_replicas(os.fsencode(dirname), dv.ctypes.data_as(C.c_void_p), n, shards, 0,\n"
        "                                  C.byref(h))\n"
        "    assert st == 2 and not h.value, (st, L.pb_last_error())\n"
        "    assert b'no CPU fallback' in L.pb_last_error()\n"
        "try:\n"
        "    m.MmapIndex.load_replicas(sys.argv[1], [0, 0])\n"
        "except m.PlaidError as e:\n"
        "    assert e.status == 2\n"
        "else:\n"
        "    raise AssertionError('loaded without a device')\n"
        "print('ok')\n")
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([sys.executable, "-c", code, index_dir], env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and r.stdout.strip() == "ok", r.stdout + r.stderr
