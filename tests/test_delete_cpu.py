"""CPU checks for the incremental delete: the numpy restatement of delete_from_index's inverted-file patch against
build_ivf of the filtered index, and the C-ABI header with the delete section compiles as plain C."""
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from ivf_delete import delete_ivf, keep_mask  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_delete_ivf_hand_built():
    # 5 docs, K = 4: doc 0 -> {0, 2}, doc 1 -> {2}, doc 2 -> {}, doc 3 -> {1, 2}, doc 4 -> {0, 3}
    ivf, lens = np.array([0, 4, 3, 0, 1, 3, 4]), np.array([2, 1, 3, 1])
    got, gl = delete_ivf(ivf, lens, [1, 3], 5)
    # docs 0, 2, 4 stay as 0, 1, 2
    assert gl.tolist() == [2, 0, 1, 1]
    assert got.tolist() == [0, 2, 0, 2]
    assert got.dtype == np.int64 and gl.dtype == np.int32
    # ids outside the index, negative and repeated ids change nothing more
    got2, gl2 = delete_ivf(ivf, lens, [3, -1, 1, 3, 9], 5)
    assert got2.tolist() == got.tolist() and gl2.tolist() == gl.tolist()
    # nothing deleted: unchanged; everything deleted: every list empty
    got3, gl3 = delete_ivf(ivf, lens, [], 5)
    assert got3.tolist() == ivf.tolist() and gl3.tolist() == lens.tolist()
    got4, gl4 = delete_ivf(ivf, lens, range(5), 5)
    assert got4.tolist() == [] and gl4.tolist() == [0, 0, 0, 0]


def test_delete_ivf_equals_build_ivf_of_the_filtered_index(oracle):
    rng = np.random.default_rng(5)
    for K, D in ((16, 60), (300, 200), (8, 1), (64, 0)):
        dl = rng.integers(0, 12, D)
        codes = rng.integers(0, K, int(dl.sum()))
        ivf, lens = oracle.build_ivf(codes, dl, K)
        cases = {"none": [], "all": list(range(D)), "prefix": list(range(D // 3)),
                 "suffix": list(range(D - D // 4, D)), "every_other": list(range(0, D, 2)),
                 "scattered": rng.choice(max(D, 1), min(D, 7), replace=False).tolist() if D else [],
                 "outside": [D, D + 3, -1, -(1 << 40), 1 << 62],
                 "duplicates": ([D - 1] * 3 + [0, 0]) if D else []}
        for name, ids in cases.items():
            docs, toks = keep_mask(dl, ids)
            want = oracle.build_ivf(codes[toks], dl[docs], K)
            got = delete_ivf(ivf, lens, ids, D)
            assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]), (K, D, name)


def test_header_compiles_as_plain_c(tmp_path):
    src = tmp_path / "h.c"
    src.write_text('#include "plaid_b200.h"\n'
                   'pb_status (*f0)(pb_index *, const int64_t *, int64_t, const char *, int64_t *) = pb_index_delete;\n'
                   'pb_status (*f1)(pb_index *, float *) = pb_last_delete_ms;\n')
    for std in ("c99", "c11"):
        r = subprocess.run(["cc", f"-std={std}", "-pedantic-errors", "-Wall", "-Werror", "-c", str(src), "-I",
                            os.path.join(ROOT, "include"), "-o", str(tmp_path / "h.o")], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
