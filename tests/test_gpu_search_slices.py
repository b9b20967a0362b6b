"""Batch searches cut into slices (DESIGN.md 4c', 4q): the lanes of a plain handle, the slices of a replica set, and
lanes inside a replica's slice, with per-query parameters of mixed top_k, per-query subsets and a shared subset.

Every call goes through the C-ABI into outputs filled with a sentinel and is compared with one plain handle at one
lane: the counts, entries [0, count) of each row, and the per-query work counters.  A row is written only up to its
query's own top_k, so every entry past it must still hold the sentinel, also in a slice whose largest top_k is below
the call's.  Then the refusals a deployment and a set of deployments keep, each leaving the handle usable.

Everything runs on device 0, repeated where a layout needs several devices."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
PB_ERR_INVALID, PB_ERR_UNSUPPORTED = 1, 4
NBITS, K, DIM, CHUNK = 4, 256, 128, 200
SENT_ID, SENT_SCORE = -7, np.float32(-7.5)
SIZES = (15, 16, 17, 33, 69)
# query 0 alone has the call's largest top_k, so every later slice's rows are wider than its own largest top_k
FIRST = dict(top_k=60, n_ivf_probe=16, n_full_scores=512)
MIXED = [dict(top_k=10, n_ivf_probe=8, n_full_scores=256),
         dict(top_k=3, n_ivf_probe=4, n_full_scores=64, centroid_batch_size=100),
         dict(top_k=0, n_ivf_probe=8, n_full_scores=256),
         dict(top_k=25, n_ivf_probe=8, n_full_scores=256, centroid_score_threshold=None)]
SHARED = dict(top_k=10, n_ivf_probe=8, n_full_scores=256)
# per-query counters: they add up over slices to the uncut call's
WORK_KEYS = ("n_queries", "n_query_tokens", "n_candidates", "n_exact_docs")


@pytest.fixture(scope="module")
def npb():
    import next_plaid_b200 as m
    m.build_library()
    if m.device_count() < 1:
        pytest.fail("GPU tests need an H100; the library has no CPU fallback")
    return m


@pytest.fixture(scope="module")
def corpus(oracle, tmp_path_factory):
    docs = oracle.synthetic_corpus(1000, 40, dim=DIM, seed=23, ragged=True)
    ix = oracle.create_index(docs[:900], nbits=NBITS, seed=5, num_partitions=K)
    qs, _ = oracle.synthetic_queries(docs[:900], max(SIZES), nq=32, seed=29)
    qs = [q[:4 + (7 * i) % 29] for i, q in enumerate(qs)]  # ragged: 4 .. 32 tokens
    path = str(tmp_path_factory.mktemp("ix"))
    oracle.write_index(ix, path, chunk_docs=CHUNK)
    return dict(qs=qs, path=path, D=ix.num_documents)


@pytest.fixture(scope="module")
def handles(npb, corpus):
    path = corpus["path"]
    hs = dict(plain=npb.MmapIndex.load(path), dep=npb.MmapIndex.load_devices(path, [0, 0]),
              rep21=npb.MmapIndex.load_replicas(path, [0, 0], shards=1),
              rep22=npb.MmapIndex.load_replicas(path, [0, 0, 0, 0], shards=2))
    yield hs
    for h in hs.values():
        h.close()


def _ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _queries(qs, n):
    offs = np.zeros(n + 1, np.int64)
    offs[1:] = np.cumsum([q.shape[0] for q in qs[:n]])
    return np.ascontiguousarray(np.concatenate(qs[:n]), np.float32), offs


def _outputs(n, width):
    return (np.full((n, max(width, 1)), SENT_ID, np.int64), np.full((n, max(width, 1)), SENT_SCORE, np.float32),
            np.full(n, -1, np.int32))


def _params_call(npb, L, h, qs, n, D):
    """pb_search_batch_params: mixed top_k, a subset for most queries (some empty); (top_k per query, outputs)"""
    rng = np.random.default_rng(n)
    params = [npb.SearchParameters(**(FIRST if i == 0 else MIXED[i % len(MIXED)])) for i in range(n)]
    subsets = [None if i % 3 == 0 else [] if i % 5 == 1 else rng.choice(D, int(rng.integers(30, 120)), replace=False)
               for i in range(n)]
    has = np.array([s is not None for s in subsets], np.uint8)
    so = np.zeros(n + 1, np.int64)
    so[1:] = np.cumsum([0 if s is None else len(s) for s in subsets])
    si = np.concatenate([np.asarray(s, np.int64) for s in subsets if s is not None] + [np.zeros(1, np.int64)])
    c = [p._c() for p in params]
    arr = (type(c[0]) * n)(*c)
    flat, offs = _queries(qs, n)
    top_k = [p.top_k for p in params]
    ids, sc, cn = _outputs(n, max(top_k))
    st = L.pb_search_batch_params(h._h, _ptr(flat), _ptr(offs), n, C.cast(arr, C.POINTER(type(c[0]))), _ptr(so),
                                  _ptr(si), _ptr(has), _ptr(ids), _ptr(sc), _ptr(cn), None)
    assert st == 0, L.pb_last_error()
    return top_k, (ids, sc, cn)


def _shared_call(npb, L, h, qs, n, D):
    """pb_search_batch with one subset for every query"""
    p = npb.SearchParameters(**SHARED)
    sub = np.arange(0, D, 3, dtype=np.int64)
    flat, offs = _queries(qs, n)
    ids, sc, cn = _outputs(n, p.top_k)
    st = L.pb_search_batch(h._h, _ptr(flat), _ptr(offs), n, C.byref(p._c()), _ptr(sub), len(sub), _ptr(ids), _ptr(sc),
                           _ptr(cn))
    assert st == 0, L.pb_last_error()
    return [p.top_k] * n, (ids, sc, cn)


def _rows(top_k, out):
    """each row's count and entries [0, count); asserts that nothing past the query's own top_k was written"""
    ids, sc, cn = out
    rows = []
    for b, k in enumerate(top_k):
        assert 0 <= cn[b] <= k, (b, cn[b], k)
        assert (ids[b, k:] == SENT_ID).all() and (sc[b, k:] == SENT_SCORE).all(), (b, k)
        rows.append((int(cn[b]), ids[b, :cn[b]].tolist(), sc[b, :cn[b]].tobytes()))
    return rows


def _work(h):
    w = h.last_work_counters()
    return {k: w[k] for k in WORK_KEYS}


@pytest.mark.parametrize("call", [_params_call, _shared_call], ids=["params_subsets", "shared_subset"])
def test_slices_equal_one_uncut_call(npb, corpus, handles, call):
    L = npb.load_library()
    qs, D = corpus["qs"], corpus["D"]
    try:
        for n in SIZES:
            top_k, out = call(npb, L, handles["plain"], qs, n, D)
            want = _rows(top_k, out)
            assert any(r[0] for r in want), n  # the searches find something
            work = {1: _work(handles["plain"])}
            top_k, out = call(npb, L, handles["dep"], qs, n, D)
            assert _rows(top_k, out) == want, ("dep", n)
            work[2] = _work(handles["dep"])  # a rank's counters: the reference of the sets of deployments
            for name, S in (("plain", 1), ("rep21", 1), ("rep22", 2)):
                for lanes in (1, 3):
                    handles[name].set_lanes(lanes)
                    top_k, out = call(npb, L, handles[name], qs, n, D)
                    assert _rows(top_k, out) == want, (name, lanes, n)
                    assert _work(handles[name]) == work[S], (name, lanes, n)
                handles[name].set_lanes(1)
    finally:
        for h in handles.values():
            h.set_lanes(1)


def test_refusals_leave_deployments_usable(npb, corpus, handles):
    L = npb.load_library()
    qs, n = corpus["qs"], 40
    p = npb.SearchParameters(**SHARED)
    want = [(r.passage_ids.tolist(), r.scores.tobytes()) for r in handles["plain"].search_batch(qs[:n], p)]
    flat, offs = _queries(qs, n)
    sub = np.arange(10, dtype=np.int64)
    so = np.arange(n + 1, dtype=np.int64) + 1  # subset_offsets[0] != 0
    trace = npb.index._Trace()  # refused before it is read
    for name in ("dep", "rep22"):
        h = handles[name]
        ids, sc, cn = _outputs(n, p.top_k)
        refusals = {
            "a traced call with n_subset < 0": (PB_ERR_UNSUPPORTED, lambda: L.pb_search_batch_traced(
                h._h, _ptr(flat), _ptr(offs), n, C.byref(p._c()), _ptr(sub), -1, _ptr(ids), _ptr(sc), _ptr(cn),
                C.byref(trace))),
            "subset_offsets[0] != 0": (PB_ERR_INVALID, lambda: L.pb_search_batch_subsets(
                h._h, _ptr(flat), _ptr(offs), n, C.byref(p._c()), _ptr(so), _ptr(sub), None, _ptr(ids), _ptr(sc),
                _ptr(cn), None)),
        }
        for what, (status, call) in refusals.items():
            assert call() == status, (name, what, L.pb_last_error())
            got = [(r.passage_ids.tolist(), r.scores.tobytes()) for r in h.search_batch(qs[:n], p)]
            assert got == want, (name, what)
