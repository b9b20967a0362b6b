"""Token pooling on the CPU side: the C restatement (pool_oracle.c) against the reference's known answers and against an
independent Python restatement of pool_embeddings_hierarchical (lib.rs:2249-2317, hierarchy.rs:128-653); the length
rule of pb_pooled_doc_length; and the C-ABI's argument refusals, which come before any device is touched."""
import ctypes as C
import json
import math
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import pool_oracle  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "pool_kats.json")


def _f32(bits, shape):
    return np.array(bits, np.uint32).reshape(shape).view(np.float32)


# ---- an independent restatement, in Python floats (IEEE f64, no contraction) and numpy f32 -----------------------

def _py_pdist(x):
    t = len(x)
    norms = [math.sqrt(sum_seq(float(v) * float(v) for v in row)) for row in x]
    out = []
    for i in range(t):
        for j in range(i + 1, t):
            dot = sum_seq(float(a) * float(b) for a, b in zip(x[i], x[j]))
            cs = dot / (norms[i] * norms[j]) if norms[i] > 0.0 and norms[j] > 0.0 else 0.0
            out.append(min(max(1.0 - cs, 0.0), 2.0))
    return out


def sum_seq(vals):
    s = 0.0
    for v in vals:
        s += v
    return s


def _py_ward(dist, n):
    """linkage_ward, rows (a, b) in chain order with the reference's cluster ids"""
    T = 2 * n - 1
    inf = float("inf")
    dsq = [[inf] * T for _ in range(T)]
    c = 0
    for i in range(n):
        for j in range(i + 1, n):
            dsq[i][j] = dsq[j][i] = dist[c] * dist[c]
            c += 1
    sizes = [1] * T
    active = list(range(n))

    def nn_of(i):
        best, bn = inf, None
        for j in active:
            if j != i and dsq[i][j] < best:
                best, bn = dsq[i][j], j
        return bn, best

    cache = [None] * T
    for i in range(n):
        cache[i] = nn_of(i)
    chain, rows, nxt = [], [], n
    for _ in range(n - 1):
        if not chain:
            chain.append(active[0])
        while True:
            cur = chain[-1]
            if cache[cur] is None or cache[cur][0] is None:
                cache[cur] = nn_of(cur)
            nn, d = cache[cur]
            if len(chain) >= 2 and chain[-2] == nn:
                a, b = chain.pop(), chain.pop()
                rows.append((min(a, b), max(a, b), math.sqrt(d), sizes[a] + sizes[b]))
                active = [x for x in active if x != a and x != b]
                sizes[nxt] = sizes[a] + sizes[b]
                for k in active:
                    nk = sizes[k]
                    v = ((sizes[a] + nk) * dsq[a][k] + (sizes[b] + nk) * dsq[b][k] - nk * d) / (sizes[a] + sizes[b] + nk)
                    dsq[nxt][k] = dsq[k][nxt] = v
                    if cache[k] is not None and cache[k][0] in (a, b):
                        cache[k] = None
                active.append(nxt)
                cache[nxt] = nn_of(nxt)
                nxt += 1
                break
            assert len(chain) < len(active), "chain revisits a cluster"
            chain.append(nn)
    return rows


def _py_pool(x, pf):
    x = np.asarray(x, np.float32)
    n = x.shape[0]
    if pf <= 1 or n <= 2:
        return x.copy()
    t = n - 1
    k = max(t // pf, 1)
    if k >= t:
        return x.copy()
    tp = x[1:]
    rows = _py_ward(_py_pdist(tp.tolist()), t)
    members = {i: [i] for i in range(t)}
    for r, (a, b, _, _) in enumerate(rows):
        members[t + r] = members[a] + members[b]
    comp = list(range(t))
    for a, b, _, _ in rows[:t - k]:
        ra, rb = comp[members[a][0]], comp[members[b][0]]
        comp = [ra if c == rb else c for c in comp]
    labels, order = [], {}
    for i in range(t):
        labels.append(order.setdefault(comp[i], len(order)))
    out = [x[0]]
    for c in range(k):
        s = np.zeros(x.shape[1], np.float32)
        cnt = 0
        for i in range(t):
            if labels[i] == c:
                s = (s + tp[i]).astype(np.float32)
                cnt += 1
        out.append((s / np.float32(cnt)).astype(np.float32))
    return np.array(out, np.float32)


# ---- known answers --------------------------------------------------------------------------------------------

def _kats():
    with open(GOLDEN) as f:
        return json.load(f)


@pytest.mark.parametrize("case", _kats()["pool"], ids=lambda c: c["name"])
def test_oracle_matches_known_answers(case):
    x = _f32(case["input"], case["shape"])
    want = _f32(case["expected"], case["expected_shape"])
    for impl in (pool_oracle.pool_embeddings, lambda docs, pf: [_py_pool(d, pf) for d in docs]):
        got = impl([x], case["pool_factor"])[0]
        assert got.shape == want.shape
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), got


def test_chain_order_case_linkage():
    case = next(c for c in _kats()["pool"] if "linkage_ids" in c)
    x = _f32(case["input"], case["shape"])[1:]
    L = pool_oracle.ward_linkage(pool_oracle.pdist_cosine(x), x.shape[0])
    assert L[:, :2].astype(int).tolist() == case["linkage_ids"]
    assert L[:, 3].astype(int).tolist() == case["linkage_sizes"]
    assert any(L[i, 2] > L[i + 1, 2] for i in range(len(L) - 1)), "the case must merge out of height order"


def test_pdist_cosine_known_answer():
    pd = _kats()["pdist"]
    got = pool_oracle.pdist_cosine(np.array(pd["input"], np.float32))
    assert got.tolist() == pd["expected"]


# ---- the oracle against the Python restatement --------------------------------------------------------------

def _small_docs(seed):
    rng = np.random.default_rng(seed)
    docs = []
    for n in (3, 4, 5, 6, 7, 9, 12, 17, 24, 33):
        docs.append(rng.standard_normal((n, 8)).astype(np.float32))
        # exact ties: tokens drawn from a few integer vectors, duplicated
        base = rng.integers(-2, 3, size=(4, 8)).astype(np.float32)
        base[np.abs(base).sum(1) == 0, 0] = 1
        docs.append(base[rng.integers(0, 4, size=n)])
    docs.append(np.ones((11, 8), np.float32))                          # every distance 0
    z = rng.standard_normal((10, 8)).astype(np.float32)
    z[3:6] = 0                                                         # zero vectors: distance 1
    docs.append(z)
    o = rng.standard_normal((10, 8)).astype(np.float32)
    o[5:] = -o[:5]                                                     # opposite pairs: clamped at 2
    docs.append(o)
    return docs


@pytest.mark.parametrize("seed", [1, 2, 3])
@pytest.mark.parametrize("pf", [1, 2, 3, 4, 1000])
def test_oracle_matches_python_restatement(seed, pf):
    docs = _small_docs(seed)
    got = pool_oracle.pool_embeddings(docs, pf)
    for d, g in zip(docs, got):
        want = _py_pool(d, pf)
        assert g.shape == want.shape
        assert np.array_equal(g.view(np.uint32), want.view(np.uint32))


def test_oracle_linkage_matches_python_restatement():
    for d in _small_docs(4):
        t = d.shape[0] - 1
        dist = pool_oracle.pdist_cosine(d[1:])
        assert dist.tolist() == _py_pdist(d[1:].tolist())
        L = pool_oracle.ward_linkage(dist, t)
        want = _py_ward(dist.tolist(), t)
        assert [(int(a), int(b), h, int(s)) for a, b, h, s in L] == [(a, b, h, s) for a, b, h, s in want]


# ---- the C-ABI --------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def npb():
    import next_plaid_b200 as m
    m.build_library()
    return m


def _rule(n, pf):
    if pf <= 1 or n <= 2:
        return n
    k = max((n - 1) // pf, 1)
    return n if k >= n - 1 else 1 + k


def test_pooled_doc_length_rule(npb):
    L = npb.load_library()
    for pf in range(0, 9):
        for n in range(0, 601):
            assert L.pb_pooled_doc_length(n, pf) == _rule(n, pf) == pool_oracle.pooled_doc_length(n, pf), (n, pf)
            assert npb.pooled_doc_length(n, pf) == _rule(n, pf)
    assert L.pb_pooled_doc_length(-1, 2) == -1 and L.pb_pooled_doc_length(5, -1) == -1


def _call(L, emb, lens, dim=128, pf=2, space=0, out=True, n_docs=None, device=0):
    lens = np.asarray(lens, np.int64)
    x = None if emb is None else np.ascontiguousarray(emb, np.float32)
    y = np.zeros((max(int(sum(max(_rule(int(n), max(pf, 0)), 0) for n in lens)), 1), dim), np.float32)
    olens = np.full(len(lens), 77, np.int64)
    st = L.pb_pool_embeddings(device, None if x is None else x.ctypes.data_as(C.c_void_p),
                              lens.ctypes.data_as(C.c_void_p), len(lens) if n_docs is None else n_docs, dim, pf, space,
                              y.ctypes.data_as(C.c_void_p) if out else None, olens.ctypes.data_as(C.c_void_p))
    return st, olens


def test_argument_refusals_before_the_device(npb):
    L = npb.load_library()
    x = np.zeros((10, 128), np.float32)
    assert _call(L, x, [4, 6], pf=-1)[0] == npb.index.PB_ERR_INVALID
    assert _call(L, x, [4, 6], n_docs=-1)[0] == npb.index.PB_ERR_INVALID
    assert _call(L, x, [-4, 14])[0] == npb.index.PB_ERR_INVALID
    assert _call(L, x, [4, 6], space=2)[0] == npb.index.PB_ERR_INVALID
    assert _call(L, None, [4, 6])[0] == npb.index.PB_ERR_INVALID
    assert _call(L, x, [4, 6], out=False)[0] == npb.index.PB_ERR_INVALID
    assert _call(L, np.zeros((10, 100), np.float32), [4, 6], dim=100)[0] == npb.index.PB_ERR_UNSUPPORTED
    big = np.zeros((8194, 128), np.float32)
    assert _call(L, big, [8194])[0] == npb.index.PB_ERR_UNSUPPORTED
    st, olens = _call(L, x, [4, 6], pf=1, device=-1)            # valid arguments: only now the device is asked for
    assert st in (npb.index.PB_ERR_INVALID, npb.index.PB_ERR_CUDA)
    assert (olens == 77).all(), "a refused call writes no lengths"
