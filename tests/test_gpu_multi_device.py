"""A deployment behind one handle (pb_index_load_devices, DESIGN.md 4o): an index directory doc-sharded over a list of
devices, used through the ordinary entry points.  Every check compares it with pb_index_load of the same directory on
one device: searches of every batch entry point and pb_search bit for bit (and the CPU oracle on a sample), coalesced
searches from many threads, the accessors and readers, appends and deletes that keep the directory in sync, the
rebalance, the calls it refuses, and that no thread outlives the handle.

The ranks run on device 0 repeated (worlds 1, 2, 3, 8, and 8 ranks over a directory of 5 documents, which leaves
ranks empty); with two or more GPUs also on devices 0, 1, ..."""
import filecmp
import os
import shutil
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
PB_ERR_INVALID, PB_ERR_IO, PB_ERR_UNSUPPORTED = 1, 3, 4
NBITS, K, DIM, CHUNK = 4, 256, 128, 200
WAIT_US = 10_000


@pytest.fixture(scope="module")
def npb():
    import next_plaid_b200 as m
    m.build_library()
    if m.device_count() < 1:
        pytest.fail("GPU tests need an H100; the library has no CPU fallback")
    return m


def _layouts(npb):
    out = [("w1", [0]), ("w2", [0, 0]), ("w3", [0, 0, 0]), ("w8", [0] * 8)]
    n = npb.device_count()
    if n >= 2:
        out.append((f"gpus{n}", list(range(n))))
    return out


@pytest.fixture(scope="module")
def corpus(oracle, tmp_path_factory):
    docs = oracle.synthetic_corpus(1000, 40, dim=DIM, seed=91, ragged=True)
    ix = oracle.create_index(docs[:900], nbits=NBITS, seed=4, num_partitions=K)
    qs, _ = oracle.synthetic_queries(docs[:900], 8, nq=32, seed=19)
    path = str(tmp_path_factory.mktemp("ix"))
    oracle.write_index(ix, path, chunk_docs=CHUNK)
    tiny = oracle.create_index(docs[900:905], nbits=NBITS, seed=4, num_partitions=16)
    tiny_path = str(tmp_path_factory.mktemp("tiny"))
    oracle.write_index(tiny, tiny_path, chunk_docs=CHUNK)
    return dict(docs=docs, ix=ix, qs=qs, path=path, tiny=tiny, tiny_path=tiny_path)


def _res(rs):
    return [(r.passage_ids.tolist(), r.scores.tobytes()) for r in rs]


PARAMS = [dict(top_k=10, n_ivf_probe=8, n_full_scores=256),
          dict(top_k=5, n_ivf_probe=4, n_full_scores=64, centroid_batch_size=100),
          dict(top_k=10, n_ivf_probe=8, n_full_scores=256, centroid_score_threshold=None),
          dict(top_k=100, n_ivf_probe=32, n_full_scores=1024)]


def _searches(npb, h, qs, D):
    """Everything the search entry points return, for mixed parameters and subsets (some that miss ranks)"""
    rng = np.random.default_rng(3)
    subsets = [None, [], list(range(0, min(D, 60))), list(range(D - 30, D)), sorted(rng.choice(D, min(D, 40), replace=False).tolist()),
               [D + 3, -1, 0, 0], list(range(0, D, 7)), None]
    out = []
    for kw in PARAMS:
        p = npb.SearchParameters(**kw)
        out.append(_res(h.search_batch(qs, p)))
        out.append(_res(h.search_batch(qs, p, subset=subsets[2])))
        out.append(_res(h.search_batch_subsets(qs, p, subsets)))
        out.append([_res([h.search(q, p, subset=s)]) for q, s in zip(qs, subsets)])
    mixed = [npb.SearchParameters(**PARAMS[i % len(PARAMS)]) for i in range(len(qs))]
    out.append(_res(h.search_batch_params(qs, mixed)))
    out.append(_res(h.search_batch_params(qs, mixed, subsets)))
    return out


def _threads(n, body):
    out, err, gate = [None] * n, [None] * n, threading.Barrier(n)

    def run(t):
        try:
            gate.wait()
            out[t] = body(t)
        except Exception as e:  # noqa: BLE001 - re-raised below
            err[t] = e
    ths = [threading.Thread(target=run, args=(t,)) for t in range(n)]
    [t.start() for t in ths]
    [t.join() for t in ths]
    for e in err:
        if e is not None:
            raise e
    return out


def test_search_parity(npb, oracle, corpus):
    path, qs, D = corpus["path"], corpus["qs"], corpus["ix"].num_documents
    for host in (False, True):
        full = npb.MmapIndex.load(path, host_residuals=host)
        try:
            want = _searches(npb, full, qs, D)
            for name, devices in _layouts(npb):
                dep = npb.MmapIndex.load_devices(path, devices, host_residuals=host)
                try:
                    assert _searches(npb, dep, qs, D) == want, (name, host)
                finally:
                    dep.close()
        finally:
            full.close()
    # and the CPU oracle on a sample
    dep = npb.MmapIndex.load_devices(path, [0, 0, 0])
    try:
        for kw in PARAMS[:2]:
            got = dep.search_batch(qs[:4], npb.SearchParameters(**kw))
            for q, g in zip(qs[:4], got):
                w = oracle.search_one(corpus["ix"], q, oracle.SearchParameters(**kw))
                assert g.passage_ids.tolist() == w.passage_ids.tolist() and np.array_equal(g.scores, w.scores)
    finally:
        dep.close()


def test_empty_ranks(npb, corpus):
    path, qs, D = corpus["tiny_path"], corpus["qs"], corpus["tiny"].num_documents
    full = npb.MmapIndex.load(path)
    dep = npb.MmapIndex.load_devices(path, [0] * 8)
    try:
        b, _ = dep.shard_layout()
        assert (np.diff(b) == 0).any() and b.tolist() == npb.shard_bounds(path, 8).tolist()
        assert _searches(npb, dep, qs, D) == _searches(npb, full, qs, D)
        ids = [4, 0, 2, 9, -1, 4]
        e1, l1 = dep.decompress_documents(ids)
        e2, l2 = full.decompress_documents(ids)
        assert l1.tolist() == l2.tolist() and np.array_equal(e1, e2)
        assert np.array_equal(dep.exhaustive_scores(qs[:3]), full.exhaustive_scores(qs[:3]))
    finally:
        dep.close()
        full.close()


def _requests(oracle, corpus):
    docs, D = corpus["docs"][:900], corpus["ix"].num_documents
    rng = np.random.default_rng(5)
    subs = [None, [], sorted(rng.choice(D, 40, replace=False).tolist()), list(range(0, D, 2)), list(range(D - 50, D)),
            [D, D + 5, -1], list(range(0, 100))]
    out = []
    for i in range(14):
        q = oracle.synthetic_queries(docs, 1, nq=[32, 1, 64, 20][i % 4], seed=300 + i)[0][0]
        kw = dict(PARAMS[i % len(PARAMS)])
        kw.setdefault("centroid_batch_size", 100_000)
        out.append((q, kw, subs[i % len(subs)]))
    return out


def _coalesced(npb, dep, reqs, alone, T=16, rounds=6):
    dep.set_coalescing(32, max_wait_us=WAIT_US)
    dep.coalesce_stats(reset=True)

    def body(t):
        for i in range(rounds):
            j = (t * 5 + i) % len(reqs)
            q, k, s = reqs[j]
            assert _res([dep.search(q, npb.SearchParameters(**k), subset=s)]) == alone[j], (t, j)
    try:
        _threads(T, body)
    finally:
        dep.set_coalescing(1)
    st = dep.coalesce_stats()
    assert st["n_requests"] == T * rounds and st["n_refused"] == 0 and st["n_rerun_alone"] == 0, st
    assert st["max_batch"] > 1, st


BAD = [(dict(n_ivf_probe=0), PB_ERR_INVALID, "n_ivf_probe must be >= 1"),
       (dict(top_k=10, n_full_scores=80000), PB_ERR_UNSUPPORTED, "exceeds 16384"),
       (dict(n_ivf_probe=193, centroid_batch_size=64), PB_ERR_UNSUPPORTED, "batched variant"),
       (dict(top_k=-1), PB_ERR_INVALID, "must be >= 0"),
       (dict(n_ivf_probe=64), PB_ERR_UNSUPPORTED, "exceeds 8192")]    # with a 130-token query: 192 x 64 rows


def _refusals(npb, h, q_long):
    """(status, message) of each bad request on h, from concurrent threads with coalescing on"""
    h.set_coalescing(32, max_wait_us=WAIT_US)
    h.coalesce_stats(reset=True)

    def body(t):
        d, _, _ = BAD[t % len(BAD)]
        kw = dict(dict(top_k=10, n_full_scores=256, n_ivf_probe=8, centroid_batch_size=100_000), **d)
        with pytest.raises(npb.PlaidError) as e:
            h.search(q_long, npb.SearchParameters(**kw))
        return e.value.status, str(e.value)
    try:
        got = _threads(2 * len(BAD), body)
    finally:
        h.set_coalescing(1)
    assert h.coalesce_stats()["n_refused"] == 2 * len(BAD)
    return got


def test_coalescing(npb, oracle, corpus):
    path = corpus["path"]
    reqs = _requests(oracle, corpus)
    q_long = np.ascontiguousarray(np.concatenate([reqs[2][0]] * 3, 0)[:130])
    full = npb.MmapIndex.load(path)
    try:
        alone = [_res(full.search_batch_params([q], [npb.SearchParameters(**k)], [s])) for q, k, s in reqs]
        want_bad = _refusals(npb, full, q_long)
        for (d, status, text), (st, msg) in zip(BAD, want_bad):
            assert st == status and text in msg, (d, msg)
        for name, devices in _layouts(npb):
            dep = npb.MmapIndex.load_devices(path, devices)
            try:
                _coalesced(npb, dep, reqs, alone)
                assert _refusals(npb, dep, q_long) == want_bad, name
                if len(devices) > 1:                               # rank 0 left empty: the deployment's D decides
                    D = dep.num_documents()
                    dep.rebalance_sharded([0, 0] + [D] * (len(devices) - 1))
                    assert dep.shard_layout()[0][:2].tolist() == [0, 0]
                    _coalesced(npb, dep, reqs, alone)
                    assert _refusals(npb, dep, q_long) == want_bad, name
            finally:
                dep.close()
    finally:
        full.close()


def test_accessors_and_readers(npb, corpus):
    path, qs, D = corpus["path"], corpus["qs"], corpus["ix"].num_documents
    full = npb.MmapIndex.load(path)
    try:
        acc = lambda h: [h.num_documents(), h.num_embeddings(), h.num_partitions(), h.avg_doclen(),  # noqa: E731
                         h.embedding_dim(), h.nbits()]
        ids = [899, 0, 450, 450, 200, 199, 5, -1, 900, 10 ** 9, 3]
        e_full, l_full = full.decompress_documents(ids)
        ex_full = full.exhaustive_scores(qs)
        cs_full = full.centroid_scores(qs[0])
        assert full.shard_layout()[0].tolist() == [0, D]
        for name, devices in _layouts(npb):
            dep = npb.MmapIndex.load_devices(path, devices)
            try:
                assert acc(dep) == acc(full), name
                b, dv = dep.shard_layout()
                assert b.tolist() == npb.shard_bounds(path, len(devices)).tolist() and dv.tolist() == devices
                mem = {"device_bytes": 0, "host_bytes": 0}
                for r in range(len(devices)):
                    s = npb.MmapIndex.load_range(path, int(b[r]), int(b[r + 1]), device=devices[r])
                    for k, v in s.memory_usage().items():
                        mem[k] += v
                    s.close()
                assert dep.memory_usage() == mem, name
                e, lens = dep.decompress_documents(ids)
                assert lens.tolist() == l_full.tolist() and np.array_equal(e, e_full), name
                assert np.array_equal(dep.exhaustive_scores(qs), ex_full), name
                assert np.array_equal(dep.centroid_scores(qs[0]), cs_full), name
            finally:
                dep.close()
    finally:
        full.close()


@pytest.mark.parametrize("W", [2, 3])
def test_updates_keep_the_directory(npb, oracle, tmp_path, W):
    docs = oracle.synthetic_corpus(1400, 40, dim=DIM, seed=92, ragged=True)
    a, b = str(tmp_path / "a"), str(tmp_path / "b")
    npb.create_index(docs[:1100], a, nbits=NBITS, num_partitions=K, batch_size=400, seed=7).close()
    shutil.copytree(a, b)
    base = oracle.load_index(a)
    codec = npb.ResidualCodec(NBITS, base.centroids, base.bucket_cutoffs)
    qs, _ = oracle.synthetic_queries(docs, 5, nq=32, seed=15)
    dep = npb.MmapIndex.load_devices(a, [0] * W)
    single = npb.MmapIndex.load(b)
    p = npb.SearchParameters(top_k=10, n_ivf_probe=8, n_full_scores=256)

    def same_files():
        fa, fb = sorted(os.listdir(a)), sorted(os.listdir(b))
        assert fa == fb
        for f in fa:
            assert filecmp.cmp(os.path.join(a, f), os.path.join(b, f), shallow=False), f

    try:
        rng = np.random.default_rng(4)
        gone = rng.choice(1100, 200, replace=False)
        assert dep.delete(gone, a) == single.delete(gone, b) == 200
        assert dep.append(docs[1100:1400], codec, a, batch_size=150) == single.append(docs[1100:1400], codec, b,
                                                                                       batch_size=150)
        same_files()
        fresh = npb.MmapIndex.load(a)
        try:
            want = _res(fresh.search_batch(qs, p))
        finally:
            fresh.close()
        assert _res(dep.search_batch(qs, p)) == want == _res(single.search_batch(qs, p))
        assert dep.rebalance_sharded(None).tolist() == npb.shard_bounds(a, W).tolist()
        assert dep.shard_layout()[0].tolist() == npb.shard_bounds(a, W).tolist()
        assert _res(dep.search_batch(qs, p)) == want
        # documents already encoded go to the last rank only; the other ranks get null codes and residuals
        extra = docs[1300:1400]
        codes, packed = codec.encode_chunk(np.concatenate(extra, 0))
        dl = [e.shape[0] for e in extra]
        assert dep.append_encoded(codes, packed, dl) == single.append_encoded(codes, packed, dl)
        assert [dep.num_documents(), dep.num_embeddings()] == [single.num_documents(), single.num_embeddings()]
        assert _res(dep.search_batch(qs, p)) == _res(single.search_batch(qs, p))
        # a codec the last rank refuses: the caller gets that rank's own message, and nothing changes
        other = np.random.default_rng(0).standard_normal((K, DIM)).astype(np.float32)
        bad = npb.ResidualCodec(NBITS, other, base.bucket_cutoffs)
        try:
            before = (dep.num_documents(), _res(dep.search_batch(qs, p)))
            with pytest.raises(npb.PlaidError) as e:
                dep.append(docs[1100:1105], bad)
            assert e.value.status == PB_ERR_INVALID
            assert f"rank {W - 1}: " in str(e.value) and "of the group failed" not in str(e.value), str(e.value)
            assert (dep.num_documents(), _res(dep.search_batch(qs, p))) == before
        finally:
            bad.close()
        if npb.device_count() >= 2:   # a codec on another device than the last rank's: refused, nothing changes
            other = npb.MmapIndex.load_devices(a, [1] * W)
            try:
                before = (other.num_documents(), _res(other.search_batch(qs, p)))
                with pytest.raises(npb.PlaidError) as e:
                    other.append(docs[1100:1110], codec)
                assert e.value.status == PB_ERR_INVALID
                assert (other.num_documents(), _res(other.search_batch(qs, p))) == before
            finally:
                other.close()
    finally:
        codec.close()
        dep.close()
        single.close()


def test_refused_calls_leave_it_usable(npb, corpus):
    import ctypes as C
    path, qs = corpus["path"], corpus["qs"]
    L = npb.load_library()
    p = npb.SearchParameters(**PARAMS[0])
    full = npb.MmapIndex.load(path)
    dep = npb.MmapIndex.load_devices(path, [0, 0, 0])
    try:
        want = _res(full.search_batch(qs, p))
        h = dep._h
        z = np.zeros(16, np.int64)
        zp = z.ctypes.data_as(C.c_void_p)
        grp = C.c_void_p()
        assert L.pb_shard_group_create(1, C.byref(grp)) == 0
        uid = np.zeros(128, np.uint8)
        calls = {
            "pb_index_comm_init": lambda: L.pb_index_comm_init(h, uid.ctypes.data_as(C.c_void_p), 0, 1),
            "pb_index_group_join": lambda: L.pb_index_group_join(h, grp, 0),
            "pb_index_delete_sharded": lambda: L.pb_index_delete_sharded(h, zp, 1, None, None),
            "pb_index_append_sharded": lambda: L.pb_index_append_sharded(h, None, None, zp, 0, 0, None, 1, None),
            "pb_index_append_encoded_sharded": lambda: L.pb_index_append_encoded_sharded(h, None, None, zp, 0, 0, None),
            "pb_index_reserve": lambda: L.pb_index_reserve(h, 10 ** 4, 10 ** 6),
            "pb_index_export_ivf": lambda: L.pb_index_export_ivf(h, None, None, zp),
            "pb_last_delete_ms": lambda: L.pb_last_delete_ms(h, zp),
            "pb_search_batch_device": lambda: L.pb_search_batch_device(h, zp, zp, 0, C.byref(p._c()), zp, zp, zp),
        }
        for name, call in calls.items():
            assert call() == PB_ERR_UNSUPPORTED, name
            assert name in L.pb_last_error().decode(), name
            assert _res(dep.search_batch(qs, p)) == want, name
        with pytest.raises(npb.PlaidError) as e:
            dep.search_batch(qs, p, trace=True)
        assert e.value.status == PB_ERR_UNSUPPORTED
        assert _res(dep.search_batch(qs, p)) == want
        L.pb_shard_group_destroy(grp)
    finally:
        dep.close()
        full.close()


def _threads_now():
    return len(os.listdir("/proc/self/task"))


def test_no_thread_outlives_the_handle(npb, corpus, tmp_path):
    path = corpus["path"]
    warm = npb.MmapIndex.load_devices(path, [0] * 8)   # threads the CUDA runtime keeps for the process start here
    warm.search_batch(corpus["qs"], npb.SearchParameters(**PARAMS[0]))
    warm.close()
    before = _threads_now()
    dep = npb.MmapIndex.load_devices(path, [0] * 8)
    assert _threads_now() >= before + 7
    dep.search_batch(corpus["qs"], npb.SearchParameters(**PARAMS[0]))
    dep.close()
    assert _threads_now() == before
    with pytest.raises(npb.PlaidError) as e:
        npb.MmapIndex.load_devices(str(tmp_path / "missing"), [0, 0, 0])
    assert e.value.status == PB_ERR_IO
    assert _threads_now() == before
    # a corrupt chunk on the last rank's range: the load fails, and nothing is left behind
    bad = str(tmp_path / "bad")
    shutil.copytree(path, bad)
    with open(os.path.join(bad, "4.residuals.npy"), "r+b") as f:
        f.truncate(os.path.getsize(os.path.join(bad, "4.residuals.npy")) - 64)
    with pytest.raises(npb.PlaidError) as e:
        npb.MmapIndex.load_devices(bad, [0, 0, 0])
    assert e.value.status == PB_ERR_IO
    assert _threads_now() == before
