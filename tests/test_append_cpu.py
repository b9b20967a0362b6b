"""CPU checks for the incremental append: the numpy restatement of update_index's inverted-file merge, and the C-ABI
header with the append section compiles as plain C."""
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from ivf_merge import merge_ivf  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_merge_ivf_hand_built():
    # 3 old docs, K = 4: doc 0 -> {0, 2}, doc 1 -> {2}, doc 2 -> {} (empty)
    old_ivf, old_len = np.array([0, 0, 1]), np.array([1, 0, 2, 0])
    # new docs 3 (codes 2, 2, 3), 4 (empty), 5 (codes 0, 3)
    ivf, lens = merge_ivf(old_ivf, old_len, [2, 2, 3, 0, 3], [3, 0, 2], 3, 4)
    assert lens.tolist() == [2, 0, 3, 2]
    assert ivf.tolist() == [0, 5, 0, 1, 3, 3, 5]
    assert ivf.dtype == np.int64 and lens.dtype == np.int32
    # nothing appended: unchanged
    ivf2, lens2 = merge_ivf(old_ivf, old_len, [], [], 3, 4)
    assert ivf2.tolist() == old_ivf.tolist() and lens2.tolist() == old_len.tolist()


def test_merge_ivf_equals_build_ivf_of_the_concatenation(oracle):
    rng = np.random.default_rng(3)
    for K, D0, D1 in ((16, 40, 25), (300, 200, 1), (64, 0, 30), (8, 50, 0)):
        dl0 = rng.integers(0, 12, D0)
        dl1 = rng.integers(0, 12, D1)
        c0 = rng.integers(0, K, int(dl0.sum()))
        c1 = rng.integers(0, K, int(dl1.sum()))
        ivf0, len0 = oracle.build_ivf(c0, dl0, K)
        got = merge_ivf(ivf0, len0, c1, dl1, D0, K)
        want = oracle.build_ivf(np.concatenate([c0, c1]), np.concatenate([dl0, dl1]), K)
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]), (K, D0, D1)


def test_header_compiles_as_plain_c(tmp_path):
    src = tmp_path / "h.c"
    src.write_text('#include "plaid_b200.h"\n'
                   'pb_status (*f0)(pb_index *, pb_codec *, const float *, const int64_t *, int64_t, int32_t, const char *,'
                   ' int64_t, int64_t *) = pb_index_append;\n'
                   'pb_status (*f1)(pb_index *, const int64_t *, const uint8_t *, const int64_t *, int64_t, int32_t,'
                   ' int64_t *) = pb_index_append_encoded;\n'
                   'pb_status (*f2)(pb_index *, int64_t, int64_t) = pb_index_reserve;\n')
    for std in ("c99", "c11"):
        r = subprocess.run(["cc", f"-std={std}", "-pedantic-errors", "-Wall", "-Werror", "-c", str(src), "-I",
                            os.path.join(ROOT, "include"), "-o", str(tmp_path / "h.o")], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
