"""Adding replicas to and removing replicas from a live replica set (pb_index_add_replicas / pb_index_remove_replicas,
DESIGN.md 4u).  After every resize the set must equal pb_index_load (S = 1) or pb_index_load_devices (S > 1) of the same
directory on every entry point, and a fresh pb_index_load_replicas on the new devices in its layout, accessors and
memory; kept replicas keep their routing counts and new ones serve slices.  Also: host-tier sets whose replica 0 leaves
while the set keeps appending and deleting, row caches that a copy takes with it, switches that hold on new replicas,
searches and mutations racing resizes, and every refusal.

The replicas run on device 0 repeated; with two or more GPUs new replicas also go one per GPU."""
import os
import shutil

import numpy as np
import pytest

from test_gpu_replicas import PARAMS, _plain, _res, _same_files, _searches, _threads

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


@pytest.fixture(scope="module")
def corpus(oracle, tmp_path_factory):
    docs = oracle.synthetic_corpus(1000, 40, dim=DIM, seed=93, ragged=True)
    ix = oracle.create_index(docs[:900], nbits=NBITS, seed=5, num_partitions=K)
    qs, _ = oracle.synthetic_queries(docs[:900], 4 * 32 + 5, nq=32, seed=21)
    path = str(tmp_path_factory.mktemp("ix"))
    oracle.write_index(ix, path, chunk_docs=CHUNK)
    return dict(docs=docs, ix=ix, qs=qs, path=path)


def _device(npb, h):
    return npb.load_library().pb_index_device(h._h)


def _accessors(npb, h):
    return [h.num_documents(), h.num_embeddings(), h.num_partitions(), h.avg_doclen(), h.embedding_dim(), h.nbits(),
            h.shard_layout()[0].tolist(), _device(npb, h)]


def _coalesced(rep, qs, p, alone):
    rep.set_coalescing(16, max_wait_us=2000, max_inflight=1)
    rep.coalesce_stats(reset=True)
    try:
        def body(t):
            for i in range(12):
                j = (t * 7 + i) % len(alone)
                assert _res([rep.search(qs[j], p)]) == alone[j], (t, j)
        _threads(8, body)
        st = rep.coalesce_stats()
        assert st["n_requests"] == 96 and st["n_refused"] == 0 and st["n_rerun_alone"] == 0, st
    finally:
        rep.set_coalescing(1)


def _check_set(npb, rep, plain, path, devices, S, qs, D, before):
    """rep after a resize to `devices` against the plain handle and a fresh load_replicas; `before` are the counts each
    replica had before the resize (None for a new replica)"""
    R = len(devices) // S
    r, s, dv = rep.replica_layout()
    assert (r, s, dv.tolist()) == (R, S, np.reshape(devices, (R, S)).tolist())
    calls, queries = rep.replica_stats()
    assert calls.tolist() == [c if c is not None else 0 for c, _ in before]
    assert queries.tolist() == [q if q is not None else 0 for _, q in before]
    p = npb.SearchParameters(**PARAMS[0])
    assert _res(rep.search_batch(qs[:R * 32], p)) == _res(plain.search_batch(qs[:R * 32], p)), R
    c2, q2 = rep.replica_stats()
    assert (c2 - calls).tolist() == [1] * R and (q2 - queries).tolist() == [32] * R, (c2, q2)
    assert _searches(npb, rep, qs, D, R) == _searches(npb, plain, qs, D, R), R
    alone = [_res(plain.search_batch([q], p)) for q in qs[:24]]
    _coalesced(rep, qs, p, alone)
    fresh = npb.MmapIndex.load_replicas(path, devices, shards=S)
    try:
        assert _accessors(npb, rep) == _accessors(npb, fresh) == _accessors(npb, plain)
        assert rep.memory_usage() == fresh.memory_usage()
        assert fresh.replica_layout()[2].tolist() == dv.tolist()
    finally:
        fresh.close()
    e1, l1 = rep.decompress_documents([899, 0, 450, 7])
    e2, l2 = plain.decompress_documents([899, 0, 450, 7])
    assert l1.tolist() == l2.tolist() and np.array_equal(e1, e2)
    assert np.array_equal(rep.exhaustive_scores(qs[:3]), plain.exhaustive_scores(qs[:3]))
    return [tuple(int(x) for x in cq) for cq in zip(*rep.replica_stats())]


def _new_devices(npb, k):
    """devices for k new replicas: device 0, or one per GPU when there are several"""
    n = npb.device_count()
    return [i % n for i in range(1, k + 1)] if n >= 2 else [0] * k


def test_walk_one_to_four_and_back(npb, corpus):
    path, qs, D = corpus["path"], corpus["qs"], corpus["ix"].num_documents
    plain = _plain(npb, path, 1)
    rep = npb.MmapIndex.load_replicas(path, [0])
    try:
        devices = [0]
        counts = _check_set(npb, rep, plain, path, devices, 1, qs, D, [(0, 0)])
        for step in ("add 1", "add 2", "remove middle", "remove 0", "remove last"):
            if step.startswith("add"):
                new = _new_devices(npb, int(step[-1]))
                rep.add_replicas(new)
                devices = devices + new
                before = counts + [(None, None)] * len(new)
            else:
                R = len(devices)
                g = {"remove middle": 1, "remove 0": 0, "remove last": R - 1}[step]
                rep.remove_replicas([g])
                devices = devices[:g] + devices[g + 1:]
                before = counts[:g] + counts[g + 1:]
            counts = _check_set(npb, rep, plain, path, devices, 1, qs, D, before)
        assert len(devices) == 1
    finally:
        rep.close()
        plain.close()


def test_sets_of_deployments(npb, corpus):
    path, qs, D = corpus["path"], corpus["qs"], corpus["ix"].num_documents
    plain = _plain(npb, path, 2)
    rep = npb.MmapIndex.load_replicas(path, [0, 0], shards=2)
    try:
        counts = [tuple(int(x) for x in cq) for cq in zip(*rep.replica_stats())]
        rep.add_replicas([0, 0])
        counts = _check_set(npb, rep, plain, path, [0, 0, 0, 0], 2, qs, D, counts + [(None, None)])
        rep.remove_replicas([0])
        _check_set(npb, rep, plain, path, [0, 0], 2, qs, D, counts[1:])
    finally:
        rep.close()
        plain.close()


def test_host_tier_set_loses_replica_0_and_keeps_writing(npb, oracle, tmp_path):
    docs = oracle.synthetic_corpus(1300, 40, dim=DIM, seed=94, ragged=True)
    a, b, c = str(tmp_path / "a"), str(tmp_path / "b"), str(tmp_path / "c")
    npb.create_index(docs[:1000], a, nbits=NBITS, num_partitions=K, batch_size=400, seed=7).close()
    shutil.copytree(a, b)
    shutil.copytree(a, c)
    base = oracle.load_index(a)
    codec = npb.ResidualCodec(NBITS, base.centroids, base.bucket_cutoffs)
    qs, _ = oracle.synthetic_queries(docs, 2 * 32, nq=32, seed=16)
    p = npb.SearchParameters(top_k=10, n_ivf_probe=8, n_full_scores=256)
    rep = npb.MmapIndex.load_replicas(a, [0], host_residuals=True, mutable=True)
    single = npb.MmapIndex.load(b)                                      # resident
    host = npb.MmapIndex.load(c, host_residuals=True, mutable=True)    # the store rep's replica 0 grows alike
    rng = np.random.default_rng(8)

    def same(R):
        rep.replica_stats(reset=True)
        assert _res(rep.search_batch(qs[:R * 32], p)) == _res(single.search_batch(qs[:R * 32], p))
        assert rep.replica_stats()[1].tolist() == [32] * R
        assert rep.memory_usage()["host_bytes"] == host.memory_usage()["host_bytes"] > 0
        assert [rep.num_documents(), rep.num_embeddings()] == [single.num_documents(), single.num_embeddings()]
        _same_files(a, b)

    def mutate(lo, hi):
        assert rep.append(docs[lo:hi], codec, a, batch_size=150) == single.append(docs[lo:hi], codec, b, batch_size=150)
        host.append(docs[lo:hi], codec, c, batch_size=150)
        gone = rng.choice(rep.num_documents(), 60, replace=False)
        assert rep.delete(gone, a) == single.delete(gone, b) == host.delete(gone, c) == 60

    try:
        rep.add_replicas([0])
        same(2)
        mutate(1000, 1150)
        same(2)
        rep.remove_replicas([0])           # the copy becomes replica 0: it writes the directory and the shared store
        assert _device(npb, rep) == 0
        same(1)
        mutate(1150, 1300)
        same(1)
        rep.add_replicas([0])
        same(2)
    finally:
        rep.close()
        single.close()
        host.close()


def test_row_cache_goes_with_the_copy(npb, corpus):
    path, qs = corpus["path"], corpus["qs"]
    p = npb.SearchParameters(**PARAMS[0])
    resident = npb.MmapIndex.load(path)
    rep = npb.MmapIndex.load_replicas(path, [0], host_residuals=True)
    try:
        want = _res(resident.search_batch(qs[:64], p))
        rep.set_row_cache(400_000)
        rep.search_batch(qs[:64], p)
        assert len(rep.fill_row_cache()) > 0
        one = rep.row_cache_stats()
        assert one["cached_docs"] > 0
        rep.add_replicas([0])
        two = rep.row_cache_stats()
        for k in ("budget_bytes", "cached_docs", "cached_bytes"):
            assert two[k] == 2 * one[k], (k, one, two)
        # the copy alone: its cache serves hits, with the same results
        rep.remove_replicas([0])
        rep.row_cache_stats(reset=True)
        assert _res(rep.search_batch(qs[:64], p)) == want
        st = rep.row_cache_stats()
        assert st["cached_docs"] == one["cached_docs"] and st["hit_docs"] > 0, st
        # a later fill covers every replica, the new ones included
        rep.add_replicas([0, 0])
        ids = list(range(0, 900, 15))
        got = rep.fill_row_cache(ids)
        assert len(got) == 3 * len(ids) and rep.row_cache_stats()["cached_docs"] == 3 * len(ids)
        rep.replica_stats(reset=True)
        assert _res(rep.search_batch(qs[:96], p)) == _res(resident.search_batch(qs[:96], p))
        assert rep.replica_stats()[1].tolist() == [32] * 3
    finally:
        rep.close()
        resident.close()


def test_switches_hold_on_new_replicas(npb, corpus):
    path, qs = corpus["path"], corpus["qs"]
    p = npb.SearchParameters(**PARAMS[0])
    rep = npb.MmapIndex.load_replicas(path, [0])
    try:
        rep.set_fast_exact(False)
        rep.add_replicas([0, 0])
        rep.replica_stats(reset=True)
        rep.search_batch(qs[:96], p)       # a slice on each replica; the counters are the slices' sums
        assert rep.replica_stats()[0].tolist() == [1, 1, 1]
        assert rep.last_work_counters()["n_filter_docs"] == 0
        rep.set_fast_exact(True)
        rep.search_batch(qs[:96], p)
        assert rep.last_work_counters()["n_filter_docs"] > 0
        # coalesced searches after a removal
        rep.remove_replicas([1])
        alone = [_res(rep.search_batch([q], p)) for q in qs[:16]]
        _coalesced(rep, qs, p, alone)
    finally:
        rep.close()


def test_searches_and_mutations_race_resizes(npb, corpus, oracle, tmp_path):
    path, qs = corpus["path"], corpus["qs"]
    p = npb.SearchParameters(**PARAMS[0])
    rep = npb.MmapIndex.load_replicas(path, [0])
    plain = npb.MmapIndex.load(path)
    try:
        batch = _res(plain.search_batch(qs[:70], p))
        alone = [_res(plain.search_batch([q], p)) for q in qs[:20]]
        rep.set_coalescing(8, max_wait_us=500, max_inflight=1)
        stop = []

        def body(t):
            if t == 7:
                try:
                    for i in range(3):
                        rep.add_replicas(_new_devices(npb, 2))
                        rep.remove_replicas([0] if i % 2 else [1])
                        rep.remove_replicas([rep.replica_layout()[0] - 1])
                finally:
                    stop.append(1)
                return
            i = 0
            while not stop or i < 3:
                if t < 3:
                    assert _res(rep.search_batch(qs[:70], p)) == batch, t
                else:
                    j = (t * 5 + i) % 20
                    assert _res([rep.search(qs[j], p)]) == alone[j], (t, j)
                i += 1
        _threads(8, body)
        assert rep.replica_layout()[0] == 1
    finally:
        rep.set_coalescing(1)
        rep.close()
        plain.close()

    # an append races an add: the set ends with both, equal to a single handle with the append
    docs = oracle.synthetic_corpus(1100, 40, dim=DIM, seed=95, ragged=True)
    a = str(tmp_path / "a")
    npb.create_index(docs[:1000], a, nbits=NBITS, num_partitions=K, batch_size=400, seed=7).close()
    base = oracle.load_index(a)
    codec = npb.ResidualCodec(NBITS, base.centroids, base.bucket_cutoffs)
    codes, packed = codec.encode_chunk(np.concatenate(docs[1000:], 0))
    dl = [d.shape[0] for d in docs[1000:]]
    rep = npb.MmapIndex.load_replicas(a, [0])
    single = npb.MmapIndex.load(a)
    try:
        single.append_encoded(codes, packed, dl)
        _threads(2, lambda t: rep.append_encoded(codes, packed, dl) if t == 0 else rep.add_replicas([0]))
        rep.replica_stats(reset=True)
        q2, _ = oracle.synthetic_queries(docs, 64, nq=32, seed=17)
        assert _res(rep.search_batch(q2, p)) == _res(single.search_batch(q2, p))
        assert rep.replica_stats()[1].tolist() == [32, 32]
        assert rep.num_documents() == single.num_documents() == 1100
    finally:
        rep.close()
        single.close()


def _threads_now():
    return len(os.listdir("/proc/self/task"))


def test_refusals_leave_the_set_usable(npb, corpus):
    path, qs = corpus["path"], corpus["qs"]
    p = npb.SearchParameters(**PARAMS[0])
    plain = npb.MmapIndex.load(path)
    want = _res(plain.search_batch(qs[:40], p))
    rep = npb.MmapIndex.load_replicas(path, [0, 0, 0])
    deps = npb.MmapIndex.load_replicas(path, [0, 0], shards=2)
    dep = npb.MmapIndex.load_devices(path, [0, 0])
    n = npb.device_count()
    try:
        cases = [(rep, "add", [], PB_ERR_INVALID), (rep, "add", [0] * 62, PB_ERR_INVALID),
                 (rep, "add", [n], PB_ERR_INVALID), (rep, "add", [0, -1], PB_ERR_INVALID),
                 (deps, "add", [0], PB_ERR_INVALID), (deps, "add", [0] * 64, PB_ERR_INVALID),
                 (rep, "remove", [], PB_ERR_INVALID), (rep, "remove", [0, 1, 2], PB_ERR_INVALID),
                 (rep, "remove", [3], PB_ERR_INVALID), (rep, "remove", [-1], PB_ERR_INVALID),
                 (rep, "remove", [1, 1], PB_ERR_INVALID), (deps, "remove", [0], PB_ERR_INVALID),
                 (plain, "add", [0], PB_ERR_UNSUPPORTED), (plain, "remove", [0], PB_ERR_UNSUPPORTED),
                 (dep, "add", [0], PB_ERR_UNSUPPORTED), (dep, "remove", [0], PB_ERR_UNSUPPORTED)]
        for h, op, arg, status in cases:
            before = (h.replica_layout()[0], h.replica_layout()[2].tolist(), h.memory_usage())
            with pytest.raises(npb.PlaidError) as e:
                (h.add_replicas if op == "add" else h.remove_replicas)(arg)
            assert e.value.status == status, (op, arg, str(e.value))
            assert (h.replica_layout()[0], h.replica_layout()[2].tolist(), h.memory_usage()) == before
            assert _res(h.search_batch(qs[:40], p)) == want, (op, arg)
    finally:
        for h in (rep, deps, plain, dep):
            h.close()
    # no library thread outlives a set that was resized
    warm = npb.MmapIndex.load_replicas(path, [0, 0])
    warm.search_batch(qs[:70], p)
    warm.close()
    t0 = _threads_now()
    rep = npb.MmapIndex.load_replicas(path, [0])
    rep.add_replicas([0, 0])
    rep.search_batch(qs[:100], p)
    rep.remove_replicas([1])
    rep.search_batch(qs[:70], p)
    rep.close()
    assert _threads_now() <= t0
