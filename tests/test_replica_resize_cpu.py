"""CPU checks for changing a replica set's number of replicas (pb_index_add_replicas / pb_index_remove_replicas,
DESIGN.md 4u): the null checks come before every other check -- before the handle's kind and before the counts and
device ids, which need a set -- also in a process that sees no device.  The checks that need a live set run on the GPU
(test_gpu_replica_resize.py)."""
import ctypes as C
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
    """(name, status) of each call with a null argument, the other arguments both valid and invalid"""
    dv = np.zeros(4, np.int32)
    bad = np.array([-1, 99], np.int32)
    p = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    return [("add: null handle", L.pb_index_add_replicas(None, p(dv), 1)),
            ("add: null handle, no devices", L.pb_index_add_replicas(None, p(dv), 0)),
            ("add: null handle, bad devices", L.pb_index_add_replicas(None, p(bad), 2)),
            ("add: null handle, above 64", L.pb_index_add_replicas(None, p(dv), 65)),
            ("add: null devices", L.pb_index_add_replicas(None, None, 1)),
            ("remove: null handle", L.pb_index_remove_replicas(None, p(dv), 1)),
            ("remove: null handle, none listed", L.pb_index_remove_replicas(None, p(dv), 0)),
            ("remove: null handle, repeated", L.pb_index_remove_replicas(None, p(dv), 2)),
            ("remove: null handle, out of range", L.pb_index_remove_replicas(None, p(bad), 2)),
            ("remove: null replicas", L.pb_index_remove_replicas(None, None, 1))]


def test_null_arguments_are_invalid(npb):
    L = npb.load_library()
    for name, st in _null_calls(L):
        assert st == PB_ERR_INVALID, name
        assert "null argument" in L.pb_last_error().decode(), name


def test_bindings_declare_both_calls(npb):
    L = npb.load_library()
    assert len(L.pb_index_add_replicas.argtypes) == 3 and len(L.pb_index_remove_replicas.argtypes) == 3
    assert callable(npb.MmapIndex.add_replicas) and callable(npb.MmapIndex.remove_replicas)


def test_null_arguments_without_a_device():
    code = (
        "import sys\n"
        f"sys.path.insert(0, {ROOT!r}); sys.path.insert(0, {os.path.dirname(os.path.abspath(__file__))!r})\n"
        "import next_plaid_b200 as m\n"
        "from test_replica_resize_cpu import _null_calls\n"
        "L = m.load_library()\n"
        "assert m.device_count() == 0\n"
        "got = _null_calls(L)\n"
        "assert all(st == 1 for _, st in got), got\n"
        "print('ok')\n")
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and r.stdout.strip() == "ok", r.stdout + r.stderr
