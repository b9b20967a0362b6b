"""A replica set behind one handle (pb_index_load_replicas, DESIGN.md 4q): R copies of an index directory, each a plain
handle (S = 1) or a deployment over S devices, used through the ordinary entry points.  Every check compares it with
pb_index_load (S = 1) or pb_index_load_devices (S > 1) of the same directory: searches of every batch entry point cut
into slices, the routing, coalesced searches from many threads, the readers, the host tier, appends, deletes, reserve
and rebalance that keep every replica and the directory in step, what a search sees while a delete runs, and the calls
the set refuses.

The replicas run on device 0 repeated ((R, S) = (1, 1), (2, 1), (3, 1), (2, 2)); with two or more GPUs also one replica
per GPU."""
import filecmp
import os
import shutil
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
PB_ERR_INVALID, PB_ERR_UNSUPPORTED = 1, 4
NBITS, K, DIM, CHUNK = 4, 256, 128, 200


@pytest.fixture(scope="module")
def npb():
    import next_plaid_b200 as m
    m.build_library()
    if m.device_count() < 1:
        pytest.fail("GPU tests need an H100; the library has no CPU fallback")
    return m


def _layouts(npb):
    out = [(1, 1, [0]), (2, 1, [0, 0]), (3, 1, [0, 0, 0]), (2, 2, [0, 0, 0, 0])]
    n = npb.device_count()
    if n >= 2:
        out.append((n, 1, list(range(n))))
    return out


def _plain(npb, path, S, host=False):
    return npb.MmapIndex.load(path, host_residuals=host) if S == 1 else \
        npb.MmapIndex.load_devices(path, [0] * S, host_residuals=host)


@pytest.fixture(scope="module")
def corpus(oracle, tmp_path_factory):
    docs = oracle.synthetic_corpus(1000, 40, dim=DIM, seed=91, ragged=True)
    ix = oracle.create_index(docs[:900], nbits=NBITS, seed=4, num_partitions=K)
    qs, _ = oracle.synthetic_queries(docs[:900], 3 * 32 + 5, nq=32, seed=19)
    path = str(tmp_path_factory.mktemp("ix"))
    oracle.write_index(ix, path, chunk_docs=CHUNK)
    return dict(docs=docs, ix=ix, qs=qs, path=path)


def _res(rs):
    return [(r.passage_ids.tolist(), r.scores.tobytes()) for r in rs]


PARAMS = [dict(top_k=10, n_ivf_probe=8, n_full_scores=256),
          dict(top_k=5, n_ivf_probe=4, n_full_scores=64, centroid_batch_size=100),
          dict(top_k=10, n_ivf_probe=8, n_full_scores=256, centroid_score_threshold=None),
          dict(top_k=100, n_ivf_probe=32, n_full_scores=1024)]
SIZE_KEYS = ("n_queries", "n_query_tokens", "n_cells", "n_candidates", "n_exact_docs", "n_exact_tokens")


def _searches(npb, h, qs, D, R):
    """results and work counters of the search entry points at the sizes where the cut changes (a refusal as its
    status and message)"""
    rng = np.random.default_rng(3)
    out = []

    def _res(rs):
        try:
            return globals()["_res"](rs())
        except npb.PlaidError as e:
            return e.status, str(e)
    for n in (0, 1, 31, 32, 33, R * 32 + 5):
        q = qs[:n]
        subsets = [[int(x) for x in rng.choice(D, 40, replace=False)] if i % 3 else None for i in range(n)]
        mixed = [npb.SearchParameters(**PARAMS[i % len(PARAMS)]) for i in range(n)]
        for kw in PARAMS[:2]:
            p = npb.SearchParameters(**kw)
            out.append(_res(lambda: h.search_batch(q, p)))
            w = h.last_work_counters()
            # one slice: every counter is the plain handle's; several: the per-query ones add up to it
            out.append(w if n <= 32 else {k: w[k] for k in SIZE_KEYS})
            out.append(_res(lambda: h.search_batch(q, p, subset=list(range(0, D, 3)))))
        out.append(_res(lambda: h.search_batch_subsets(q, npb.SearchParameters(**PARAMS[0]), subsets)))
        out.append(_res(lambda: h.search_batch_params(q, mixed)))
        out.append(_res(lambda: h.search_batch_params(q, mixed, subsets)))
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


def test_search_routing_and_readers(npb, corpus):
    path, qs, D = corpus["path"], corpus["qs"], corpus["ix"].num_documents
    ids = [899, 0, 450, 450, 200, 199, 5, -1, 900, 10 ** 9, 3]
    for R, S, devices in _layouts(npb):
        plain = _plain(npb, path, S)
        rep = npb.MmapIndex.load_replicas(path, devices, shards=S)
        try:
            r, s, dv = rep.replica_layout()
            assert (r, s, dv.tolist()) == (R, S, np.reshape(devices, (R, S)).tolist())
            # an idle set's call of R * 32 queries reaches every replica, with 32 queries each; this also checks every
            # replica against the plain handle, since each answered a slice of the same call
            rep.replica_stats(reset=True)
            p = npb.SearchParameters(**PARAMS[0])
            assert _res(rep.search_batch(qs[:R * 32], p)) == _res(plain.search_batch(qs[:R * 32], p)), (R, S)
            calls, queries = rep.replica_stats()
            assert calls.tolist() == [1] * R and queries.tolist() == [32] * R, (R, S, calls, queries)
            assert _searches(npb, rep, qs, D, R) == _searches(npb, plain, qs, D, R), (R, S)
            acc = lambda h: [h.num_documents(), h.num_embeddings(), h.num_partitions(), h.avg_doclen(),  # noqa: E731
                             h.embedding_dim(), h.nbits(), h.shard_layout()[0].tolist(),
                             npb.load_library().pb_index_device(h._h)]
            assert acc(rep) == acc(plain)
            e1, l1 = rep.decompress_documents(ids)
            e2, l2 = plain.decompress_documents(ids)
            assert l1.tolist() == l2.tolist() and np.array_equal(e1, e2)
            assert np.array_equal(rep.exhaustive_scores(qs[:5]), plain.exhaustive_scores(qs[:5]))
            assert np.array_equal(rep.centroid_scores(qs[0]), plain.centroid_scores(qs[0]))
            if S == 1:
                a, b = rep.export_ivf(), plain.export_ivf()
                assert all(np.array_equal(x, y) for x, y in zip(a, b))
                assert rep.last_delete_ms() == plain.last_delete_ms()
            m1, m0 = rep.memory_usage(), plain.memory_usage()
            assert m1 == {"device_bytes": R * m0["device_bytes"], "host_bytes": 0}, (m1, m0)
        finally:
            rep.close()
            plain.close()


def test_coalesced_searches_equal_serial_ones(npb, corpus):
    path, qs = corpus["path"], corpus["qs"]
    p = npb.SearchParameters(**PARAMS[0])
    for R, S, devices in _layouts(npb)[1:4]:
        rep = npb.MmapIndex.load_replicas(path, devices, shards=S)
        try:
            alone = [_res(rep.search_batch([q], p)) for q in qs[:40]]
            rep.set_coalescing(16, max_wait_us=2000, max_inflight=1)
            rep.coalesce_stats(reset=True)

            def body(t):
                for i in range(20):
                    j = (t * 7 + i) % 40
                    assert _res([rep.search(qs[j], p)]) == alone[j], (t, j)
            _threads(8, body)
            st = rep.coalesce_stats()
            assert st["n_requests"] == 160 and st["n_refused"] == 0 and st["n_rerun_alone"] == 0, st
        finally:
            rep.set_coalescing(1)
            rep.close()


def test_host_tier(npb, corpus):
    path, qs = corpus["path"], corpus["qs"]
    p = npb.SearchParameters(**PARAMS[0])
    for R, S, devices in _layouts(npb)[1:4]:
        resident = npb.MmapIndex.load_replicas(path, devices, shards=S)
        host = npb.MmapIndex.load_replicas(path, devices, shards=S, host_residuals=True)
        one = _plain(npb, path, S, host=True)
        try:
            assert host.memory_usage()["host_bytes"] == one.memory_usage()["host_bytes"] > 0
            n = R * 32 + 5
            assert _res(host.search_batch(qs[:n], p)) == _res(resident.search_batch(qs[:n], p)), (R, S)
        finally:
            one.close()
            host.close()
            resident.close()


def _same_files(a, b):
    fa, fb = sorted(os.listdir(a)), sorted(os.listdir(b))
    assert fa == fb
    for f in fa:
        assert filecmp.cmp(os.path.join(a, f), os.path.join(b, f), shallow=False), f


@pytest.mark.parametrize("RS", [(2, 1), (3, 1), (2, 2)])
def test_mutations_keep_every_replica_and_the_directory(npb, oracle, tmp_path, RS):
    R, S = RS
    docs = oracle.synthetic_corpus(1400, 40, dim=DIM, seed=92, ragged=True)
    a, b = str(tmp_path / "a"), str(tmp_path / "b")
    npb.create_index(docs[:1100], a, nbits=NBITS, num_partitions=K, batch_size=400, seed=7).close()
    shutil.copytree(a, b)
    base = oracle.load_index(a)
    codec = npb.ResidualCodec(NBITS, base.centroids, base.bucket_cutoffs)
    qs, _ = oracle.synthetic_queries(docs, R * 32, nq=32, seed=15)
    rep = npb.MmapIndex.load_replicas(a, [0] * (R * S), shards=S)
    single = _plain(npb, b, S)
    p = npb.SearchParameters(top_k=10, n_ivf_probe=8, n_full_scores=256)

    def every_replica_equals(h):   # R * 32 queries: each replica answers a slice
        rep.replica_stats(reset=True)
        got = _res(rep.search_batch(qs, p))
        assert rep.replica_stats()[1].tolist() == [32] * R
        assert got == _res(h.search_batch(qs, p))
        assert [rep.num_documents(), rep.num_embeddings()] == [h.num_documents(), h.num_embeddings()]

    def fresh_equals():
        fresh = _plain(npb, a, S)
        try:
            every_replica_equals(fresh)
        finally:
            fresh.close()

    try:
        rng = np.random.default_rng(4)
        gone = rng.choice(1100, 200, replace=False)
        assert rep.delete(gone, a) == single.delete(gone, b) == 200
        _same_files(a, b)
        fresh_equals()
        assert rep.append(docs[1100:1300], codec, a, batch_size=150) == single.append(docs[1100:1300], codec, b,
                                                                                      batch_size=150)
        # the stat of the codec's last encode: the call's tokens (it is overwritten per encode, so it cannot tell one
        # encode from R; that only replica 0 encodes follows from the code path)
        assert codec.last_assign_stats()["tokens"] == sum(d.shape[0] for d in docs[1100:1300])
        _same_files(a, b)
        fresh_equals()
        extra = docs[1300:1400]
        codes, packed = codec.encode_chunk(np.concatenate(extra, 0))
        dl = [e.shape[0] for e in extra]
        assert rep.append_encoded(codes, packed, dl) == single.append_encoded(codes, packed, dl)
        every_replica_equals(single)
        if S == 1:
            rep.reserve(rep.num_documents() + 500, rep.num_embeddings() + 20000)
            single.reserve(single.num_documents() + 500, single.num_embeddings() + 20000)
            assert rep.memory_usage()["device_bytes"] == R * single.memory_usage()["device_bytes"]
            every_replica_equals(single)
        else:
            D = rep.num_documents()
            assert rep.rebalance_sharded([0, D // 3, D]).tolist() == single.rebalance_sharded([0, D // 3, D]).tolist()
            assert rep.shard_layout()[0].tolist() == [0, D // 3, D]
            every_replica_equals(single)
        # refused mutations change no replica and no file
        before = (rep.num_documents(), _res(rep.search_batch(qs, p)))
        other = np.random.default_rng(0).standard_normal((K, DIM)).astype(np.float32)
        bad = npb.ResidualCodec(NBITS, other, base.bucket_cutoffs)
        try:
            with pytest.raises(npb.PlaidError) as e:
                rep.append(docs[1100:1105], bad, a, batch_size=150)
            assert e.value.status == PB_ERR_INVALID
        finally:
            bad.close()
        if npb.device_count() >= 2:
            far = npb.ResidualCodec(NBITS, base.centroids, base.bucket_cutoffs, device=1)
            try:
                with pytest.raises(npb.PlaidError) as e:
                    rep.append(docs[1100:1105], far, a, batch_size=150)
                assert e.value.status == PB_ERR_INVALID
            finally:
                far.close()
        if S > 1:
            # a directory the write refuses (no metadata.json): the failure comes after every replica prepared, on
            # replica 0's last rank alone, and no replica commits
            empty = str(tmp_path / "empty")
            os.makedirs(empty)
            with pytest.raises(npb.PlaidError):
                rep.delete([1, 2, 3], empty)
            # and an append whose encode replica 0 refuses: the replicas waiting for its rows append nothing
            bad = npb.ResidualCodec(NBITS, other, base.bucket_cutoffs)
            try:
                with pytest.raises(npb.PlaidError):
                    rep.append(docs[1100:1105], bad)
            finally:
                bad.close()
        assert (rep.num_documents(), _res(rep.search_batch(qs, p))) == before
        _same_files(a, b)
        every_replica_equals(single)
    finally:
        codec.close()
        rep.close()
        single.close()


def test_searches_see_a_delete_whole(npb, oracle, tmp_path):
    docs = oracle.synthetic_corpus(1000, 40, dim=DIM, seed=93, ragged=True)
    a = str(tmp_path / "a")
    npb.create_index(docs, a, nbits=NBITS, num_partitions=K, batch_size=400, seed=7).close()
    qs, _ = oracle.synthetic_queries(docs, 3 * 32, nq=32, seed=16)
    p = npb.SearchParameters(top_k=10, n_ivf_probe=8, n_full_scores=256)
    gone = np.random.default_rng(5).choice(1000, 300, replace=False)
    plain = npb.MmapIndex.load(a)
    pre = _res(plain.search_batch(qs, p))
    plain.delete(gone)
    post = _res(plain.search_batch(qs, p))
    plain.close()
    assert pre != post
    rep = npb.MmapIndex.load_replicas(a, [0, 0, 0])
    try:
        started, stop = threading.Event(), threading.Event()

        def body(t):
            if t == 0:
                started.wait()
                assert rep.delete(gone) == 300
                stop.set()
                return 0
            n = 0
            while not stop.is_set():
                got = _res(rep.search_batch(qs, p))
                assert got in (pre, post), t
                started.set()
                n += 1
            assert _res(rep.search_batch(qs, p)) == post
            return n
        _threads(5, body)
        for _ in range(3):
            assert _res(rep.search_batch(qs, p)) == post
    finally:
        rep.close()


def test_refused_calls_leave_it_usable(npb, corpus):
    import ctypes as C
    path, qs = corpus["path"], corpus["qs"]
    L = npb.load_library()
    p = npb.SearchParameters(**PARAMS[0])
    for S in (1, 2):
        plain = _plain(npb, path, S)
        rep = npb.MmapIndex.load_replicas(path, [0] * (2 * S), shards=S)
        try:
            want = _res(plain.search_batch(qs, p))
            h = rep._h
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
                "pb_index_append_encoded_sharded": lambda: L.pb_index_append_encoded_sharded(h, None, None, zp, 0, 0,
                                                                                             None),
                "pb_search_batch_device": lambda: L.pb_search_batch_device(h, zp, zp, 0, C.byref(p._c()), zp, zp, zp),
            }
            if S == 2:   # what a deployment refuses, the set of deployments refuses with its message
                calls.update({
                    "pb_index_reserve": lambda: L.pb_index_reserve(h, 10 ** 4, 10 ** 6),
                    "pb_index_export_ivf": lambda: L.pb_index_export_ivf(h, None, None, zp),
                    "pb_last_delete_ms": lambda: L.pb_last_delete_ms(h, zp)})
            for name, call in calls.items():
                assert call() == PB_ERR_UNSUPPORTED, name
                assert name in L.pb_last_error().decode(), name
                assert _res(rep.search_batch(qs, p)) == want, name
            # a trace follows one call: it runs whole on one replica (S = 1), and a deployment refuses it (S = 2)
            if S == 1:
                assert _res(rep.search_batch_params(qs[:40], [p] * 40, trace=True)[0]) == want[:40]
            else:
                with pytest.raises(npb.PlaidError) as e:
                    rep.search_batch_params(qs, [p] * len(qs), trace=True)
                assert e.value.status == PB_ERR_UNSUPPORTED
            # a refusal of a cut call is the plain handle's own.  (Not with S = 2: a deployment refused by its own
            # argument checks, before the plan exchange, leaves its group broken, DESIGN §4q.)
            if S == 1:
                bad = [npb.SearchParameters(**PARAMS[0]) for _ in range(80)]
                bad[70] = npb.SearchParameters(top_k=-1)
                msgs = []
                for hd in (plain, rep):
                    with pytest.raises(npb.PlaidError) as e:
                        hd.search_batch_params(qs[:80], bad)
                    msgs.append((e.value.status, str(e.value)))
                assert msgs[0] == msgs[1]
                assert _res(rep.search_batch(qs, p)) == want
            L.pb_shard_group_destroy(grp)
        finally:
            rep.close()
            plain.close()
