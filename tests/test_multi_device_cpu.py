"""CPU checks for a deployment behind one handle (pb_index_load_devices): the argument checks come before any device is
touched, in their stated order, and without a usable device the load fails with PB_ERR_CUDA (there is no CPU path).
The no-device case runs in a child process that sees no device, so it holds on a GPU machine as well."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PB_ERR_INVALID, PB_ERR_CUDA, PB_ERR_IO = 1, 2, 3


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


def _load(npb, path, devices, n=None):
    """raw pb_index_load_devices: (status, message, handle)"""
    L = npb.load_library()
    dv = None if devices is None else np.ascontiguousarray(devices, np.int32)
    h = C.c_void_p()
    st = L.pb_index_load_devices(None if path is None else os.fsencode(path),
                                 None if dv is None else dv.ctypes.data_as(C.c_void_p),
                                 len(dv) if n is None else n, 0, C.byref(h))
    return st, L.pb_last_error().decode(), h


def test_argument_checks_come_first(npb, index_dir):
    L = npb.load_library()
    for path, devices, n in ((None, [0], None), (index_dir, None, 1), (index_dir, [0], 0), (index_dir, [0] * 65, None),
                             (index_dir, [0], -3), ("/nonexistent/dir", [0] * 65, None)):
        st, msg, h = _load(npb, path, devices, n)
        assert st == PB_ERR_INVALID and not h.value, (path, n, msg)
    st = L.pb_index_load_devices(os.fsencode(index_dir), np.zeros(1, np.int32).ctypes.data_as(C.c_void_p), 1, 0, None)
    assert st == PB_ERR_INVALID                                       # out == NULL


def test_device_ids_are_checked_after_the_device_count(npb, index_dir):
    have = npb.device_count()
    for devices in ([-1], [0, have], [have + 1000]):
        st, msg, h = _load(npb, index_dir, devices)
        assert st == (PB_ERR_INVALID if have else PB_ERR_CUDA) and not h.value, (devices, msg)


def test_layout_of_a_null_handle_is_invalid(npb):
    w = C.c_int32()
    assert npb.load_library().pb_index_shard_layout(None, C.byref(w), None, None) == PB_ERR_INVALID


def test_without_a_device_the_load_fails_with_cuda(index_dir):
    code = (
        "import ctypes as C, os, sys, numpy as np\n"
        f"sys.path.insert(0, {ROOT!r})\n"
        "import next_plaid_b200 as m\n"
        "L = m.load_library()\n"
        "assert m.device_count() == 0\n"
        "h = C.c_void_p()\n"
        "for dirname in (sys.argv[1], '/nonexistent/dir'):\n"
        "    dv = np.zeros(2, np.int32)\n"
        "    st = L.pb_index_load_devices(os.fsencode(dirname), dv.ctypes.data_as(C.c_void_p), 2, 0, C.byref(h))\n"
        "    assert st == 2 and not h.value, (st, L.pb_last_error())\n"
        "    assert b'no CPU fallback' in L.pb_last_error()\n"
        "try:\n"
        "    m.MmapIndex.load_devices(sys.argv[1], [0])\n"
        "except m.PlaidError as e:\n"
        "    assert e.status == 2\n"
        "else:\n"
        "    raise AssertionError('loaded without a device')\n"
        "print('ok')\n")
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([sys.executable, "-c", code, index_dir], env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and r.stdout.strip() == "ok", r.stdout + r.stderr
