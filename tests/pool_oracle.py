"""ctypes face of pool_oracle.c, the CPU restatement of next-plaid-onnx's token pooling (test infrastructure).

The library is compiled on first use into a temporary directory keyed by the source's hash, with the flags of the
search oracle (-ffp-contract=off: every multiply and add rounds separately, as in the reference)."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile
from typing import List, Sequence

import numpy as np

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "pool_oracle.c")
CFLAGS = ["-O3", "-std=c11", "-fPIC", "-fopenmp", "-ffp-contract=off", "-fno-fast-math", "-mavx2", "-mfma", "-shared"]
_lib = None


def lib():
    global _lib
    if _lib is None:
        src = open(_SRC, "rb").read()
        tag = hashlib.sha256(src + " ".join(CFLAGS).encode()).hexdigest()[:16]
        d = os.path.join(tempfile.gettempdir(), f"plaid_pool_oracle_{os.getuid()}_{tag}")
        so = os.path.join(d, "libpool_oracle.so")
        if not os.path.exists(so):
            os.makedirs(d, exist_ok=True)
            tmp = so + f".{os.getpid()}"
            subprocess.run(["gcc", *CFLAGS, "-o", tmp, _SRC, "-lm"], check=True)
            os.replace(tmp, so)
        L = C.CDLL(so)
        L.po_pdist_cosine.argtypes = [C.c_void_p, C.c_int64, C.c_int32, C.c_void_p]
        L.po_pdist_cosine.restype = None
        L.po_ward_linkage.argtypes = [C.c_void_p, C.c_int64, C.c_int64, C.c_void_p]
        L.po_pooled_doc_length.argtypes = [C.c_int64, C.c_int64]
        L.po_pooled_doc_length.restype = C.c_int64
        L.po_pool_embeddings.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_int64, C.c_void_p,
                                         C.c_void_p]
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def pdist_cosine(x: np.ndarray) -> np.ndarray:
    """hierarchy::pdist_cosine: condensed f64 cosine distances of the rows of x."""
    x = np.ascontiguousarray(x, np.float32)
    n = x.shape[0]
    out = np.zeros(max(n * (n - 1) // 2, 1), np.float64)
    lib().po_pdist_cosine(_p(x), n, x.shape[1], _p(out))
    return out[:n * (n - 1) // 2]


def ward_linkage(dist: np.ndarray, n: int, max_merges: int = -1) -> np.ndarray:
    """hierarchy::linkage(.., Ward): rows [min id, max id, distance, size] in the order the chain merges, the first
    max_merges of them (all n - 1 by default)."""
    m = n - 1 if max_merges < 0 else min(max_merges, n - 1)
    d = np.ascontiguousarray(dist, np.float64)
    out = np.zeros((max(m, 1), 4), np.float64)
    rc = lib().po_ward_linkage(_p(d), n, m, _p(out))
    if rc:
        raise RuntimeError("the nearest-neighbour chain does not terminate")
    return out[:m]


def pooled_doc_length(n: int, pool_factor: int) -> int:
    return int(lib().po_pooled_doc_length(n, pool_factor))


def pool_embeddings(docs: Sequence[np.ndarray], pool_factor: int) -> List[np.ndarray]:
    """pool_document_embeddings(docs, Some(pool_factor)): one f32 array per document."""
    if not len(docs):
        return []
    dim = docs[0].shape[1]
    lens = np.array([d.shape[0] for d in docs], np.int64)
    flat = np.ascontiguousarray(np.concatenate([np.asarray(d, np.float32).reshape(-1, dim) for d in docs], 0))
    olens = np.array([pooled_doc_length(int(n), pool_factor) for n in lens], np.int64)
    out = np.zeros((max(int(olens.sum()), 1), dim), np.float32)
    got = np.zeros(len(docs), np.int64)
    rc = lib().po_pool_embeddings(_p(flat), _p(lens), len(docs), dim, pool_factor, _p(out), _p(got))
    if rc:
        raise RuntimeError("the nearest-neighbour chain does not terminate")
    assert np.array_equal(got, olens)
    offs = np.concatenate([[0], np.cumsum(olens)])
    return [out[offs[i]:offs[i + 1]].copy() for i in range(len(docs))]
