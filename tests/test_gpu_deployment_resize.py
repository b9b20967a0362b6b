"""Changing a live deployment's number of ranks (pb_index_add_devices / pb_index_remove_ranks, DESIGN.md 4t).  After
every step the handle must give what pb_index_load of the directory gives, and what a fresh pb_index_load_devices on
the new devices gives, bit for bit: every search entry point, decompression and exhaustive scores, the accessors and
the layout; the directory stays byte for byte as it was.  Also: explicit (skewed) bounds, appends and deletes across
resizes, resizes while other threads search, the refusals, threads and memory.

The ranks run on device 0 repeated; with two or more GPUs the new ranks go to distinct devices."""
import filecmp
import hashlib
import os
import shutil
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
PB_ERR_INVALID, PB_ERR_UNSUPPORTED = 1, 4
NBITS, K, DIM, CHUNK = 4, 256, 128, 200
WAIT_US = 10_000


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
    ix = oracle.create_index(docs[:900], nbits=NBITS, seed=4, num_partitions=K)
    qs, _ = oracle.synthetic_queries(docs[:900], 8, nq=32, seed=21)
    path = str(tmp_path_factory.mktemp("ix"))
    oracle.write_index(ix, path, chunk_docs=CHUNK)
    return dict(docs=docs, ix=ix, qs=qs, path=path)


def _devs(npb, n, start):
    """n devices for new ranks: device 0 repeated, or distinct devices in turn when there are several"""
    c = npb.device_count()
    return [0] * n if c < 2 else [(start + i) % c for i in range(n)]


def _res(rs):
    return [(r.passage_ids.tolist(), r.scores.tobytes()) for r in rs]


PARAMS = [dict(top_k=10, n_ivf_probe=8, n_full_scores=256),
          dict(top_k=100, n_ivf_probe=32, n_full_scores=1024, centroid_batch_size=100)]


def _searches(npb, h, qs, D):
    rng = np.random.default_rng(3)
    subsets = [None, [], list(range(0, 60)), list(range(D - 30, D)), sorted(rng.choice(D, 40, replace=False).tolist()),
               [D + 3, -1, 0, 0], list(range(0, D, 7)), None]
    out = []
    for kw in PARAMS:
        p = npb.SearchParameters(**kw)
        out.append(_res(h.search_batch(qs, p)))
        out.append(_res(h.search_batch_subsets(qs, p, subsets)))
        out.append([_res([h.search(q, p, subset=s)]) for q, s in zip(qs[:8], subsets)])
    mixed = [npb.SearchParameters(**PARAMS[i % len(PARAMS)]) for i in range(len(qs))]
    out.append(_res(h.search_batch_params(qs, mixed, subsets)))
    return out


IDS = [899, 0, 450, 450, 200, 199, 5, -1, 900, 10 ** 9, 3, 120, 777]


def _readers(h, qs):
    e, lens = h.decompress_documents(IDS)
    return [lens.tolist(), e.tobytes(), h.exhaustive_scores(qs[:5]).tobytes(), h.num_documents(), h.num_embeddings(),
            h.num_partitions(), h.avg_doclen(), h.embedding_dim(), h.nbits()]


def _digest(path):
    h = hashlib.sha256()
    for f in sorted(os.listdir(path)):
        h.update(f.encode())
        with open(os.path.join(path, f), "rb") as fh:
            h.update(fh.read())
    return h.hexdigest()


def _device_of(npb, h):
    return int(npb.load_library().pb_index_device(h._h))


def test_parity_through_adds_and_removes(npb, corpus):
    path, qs, D = corpus["path"], corpus["qs"], corpus["ix"].num_documents
    digest = _digest(path)
    full = npb.MmapIndex.load(path)
    want, want_rd = _searches(npb, full, qs, D), _readers(full, qs)
    full.close()
    devices = _devs(npb, 2, 0)
    dep = npb.MmapIndex.load_devices(path, devices)

    def check(step):
        b, dv = dep.shard_layout()
        W = len(devices)
        assert b.tolist() == npb.shard_bounds(path, W).tolist() and dv.tolist() == devices, step
        assert _device_of(npb, dep) == devices[0], step
        assert _searches(npb, dep, qs, D) == want, step
        assert _readers(dep, qs) == want_rd, step
        fresh = npb.MmapIndex.load_devices(path, devices)
        try:
            assert _searches(npb, fresh, qs, D) == want, step
        finally:
            fresh.close()
        assert _digest(path) == digest, step

    steps = [("add", 1), ("add", 2), ("remove", [2]), ("remove", [0]), ("remove", "last"),   # 2 -> 3 -> 5 -> 2
             ("remove", [0]), ("add", 7), ("remove", list(range(1, 8)))]                    # 1 -> 8 -> 1
    try:
        check("load")
        for i, (op, arg) in enumerate(steps):
            if op == "add":
                new = _devs(npb, arg, len(devices))
                got = dep.add_devices(new)
                devices = devices + new
            else:
                rk = [len(devices) - 1] if arg == "last" else arg
                got = dep.remove_ranks(rk)
                devices = [d for r, d in enumerate(devices) if r not in rk]
            assert got.tolist() == npb.shard_bounds(path, len(devices)).tolist(), (i, op, arg)
            check((i, op, arg))
    finally:
        dep.close()


def test_explicit_bounds(npb, corpus):
    path, qs, D = corpus["path"], corpus["qs"], corpus["ix"].num_documents
    full = npb.MmapIndex.load(path)
    want = _res(full.search_batch(qs, npb.SearchParameters(**PARAMS[1])))
    want_rd = _readers(full, qs)
    full.close()
    dep = npb.MmapIndex.load_devices(path, [0, 0])
    p = npb.SearchParameters(**PARAMS[1])
    try:
        for op, arg, bounds in (("add", [0, 0], [0, 0, 17, 850, 900]),          # rank 0 left empty
                                ("add", [0], [0, 0, 17, 850, 900, 900]),         # and the new last rank too
                                ("remove", [1], [0, 0, 880, 900, 900]),
                                ("remove", [0, 3], [0, 900, 900]),               # the last rank empty
                                ("add", [0, 0], [0, 1, 2, 3, 900])):
            got = dep.add_devices(arg, bounds) if op == "add" else dep.remove_ranks(arg, bounds)
            assert got.tolist() == bounds and dep.shard_layout()[0].tolist() == bounds, (op, arg)
            assert _res(dep.search_batch(qs, p)) == want, (op, arg)
            assert _readers(dep, qs) == want_rd, (op, arg)
        W = len(dep.shard_layout()[1])
        assert dep.rebalance_sharded(None).tolist() == npb.shard_bounds(path, W).tolist()
        assert _res(dep.search_batch(qs, p)) == want
    finally:
        dep.close()
    assert D == 900


def test_mutations_across_resizes(npb, oracle, tmp_path):
    docs = oracle.synthetic_corpus(1500, 40, dim=DIM, seed=94, ragged=True)
    a, b = str(tmp_path / "a"), str(tmp_path / "b")
    npb.create_index(docs[:1100], a, nbits=NBITS, num_partitions=K, batch_size=400, seed=7).close()
    shutil.copytree(a, b)
    base = oracle.load_index(a)
    codec = npb.ResidualCodec(NBITS, base.centroids, base.bucket_cutoffs)
    qs, _ = oracle.synthetic_queries(docs, 5, nq=32, seed=16)
    p = npb.SearchParameters(top_k=10, n_ivf_probe=8, n_full_scores=256)
    dep = npb.MmapIndex.load_devices(a, [0, 0])
    single = npb.MmapIndex.load(b)

    def same():
        fa, fb = sorted(os.listdir(a)), sorted(os.listdir(b))
        assert fa == fb
        for f in fa:
            assert filecmp.cmp(os.path.join(a, f), os.path.join(b, f), shallow=False), f
        fresh = npb.MmapIndex.load(a)
        try:
            w = _res(fresh.search_batch(qs, p))
        finally:
            fresh.close()
        assert _res(dep.search_batch(qs, p)) == w == _res(single.search_batch(qs, p))
        assert [dep.num_documents(), dep.num_embeddings()] == [single.num_documents(), single.num_embeddings()]

    try:
        dep.add_devices([0])                                    # the codec's device: the last rank encodes
        before = dep.shard_layout()[0]
        ids = dep.append(docs[1100:1250], codec, a, batch_size=150)
        assert ids == single.append(docs[1100:1250], codec, b, batch_size=150) and ids[0] == 1100
        after = dep.shard_layout()[0]
        assert after[:-1].tolist() == before[:-1].tolist() and after[-1] == 1250   # on the new last rank only
        same()
        rng = np.random.default_rng(6)
        gone = rng.choice(1250, 150, replace=False)                                  # across every rank
        assert dep.delete(gone, a) == single.delete(gone, b) == 150
        same()
        dep.remove_ranks([1])
        assert dep.shard_layout()[0].tolist() == npb.shard_bounds(a, 2).tolist()
        same()
        ids = dep.append(docs[1250:1500], codec, a, batch_size=150)
        assert ids == single.append(docs[1250:1500], codec, b, batch_size=150) and ids[0] == 1100
        assert dep.shard_layout()[0][-2] <= ids[0]
        same()
    finally:
        codec.close()
        dep.close()
        single.close()


def _threads(n, body):
    out, err = [None] * n, [None] * n

    def run(t):
        try:
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


def test_searches_during_resizes(npb, corpus):
    path, qs = corpus["path"], corpus["qs"]
    p = npb.SearchParameters(**PARAMS[0])
    full = npb.MmapIndex.load(path)
    batch = _res(full.search_batch(qs[:8], p))
    alone = [_res([full.search(q, p)]) for q in qs]
    full.close()
    dep = npb.MmapIndex.load_devices(path, [0, 0])
    dep.set_coalescing(32, max_wait_us=WAIT_US)
    done = threading.Event()
    counts = [0] * 8

    def body(t):
        if t == 0:                      # the resizer
            try:
                for k in range(3):                                   # 2 -> 3 + k -> 2 + k -> 4 + k -> 2
                    dep.add_devices(_devs(npb, 1 + k, k))
                    dep.remove_ranks([0])
                    dep.add_devices(_devs(npb, 2, k + 1), None)
                    dep.remove_ranks(list(range(1, 3 + k)))
            finally:
                done.set()
            return
        while not done.is_set():
            if t % 2:
                assert _res(dep.search_batch(qs[:8], p)) == batch, t
            else:
                i = (t + counts[t]) % len(qs)
                assert _res([dep.search(qs[i], p)]) == alone[i], (t, i)
            counts[t] += 1
    try:
        _threads(8, body)
        assert all(c > 0 for c in counts[1:]), counts
        assert dep.coalesce_stats()["n_refused"] == 0
        assert _res(dep.search_batch(qs[:8], p)) == batch
    finally:
        dep.close()


def test_refusals_leave_the_handle_as_it_was(npb, corpus):
    import ctypes as C
    path, qs = corpus["path"], corpus["qs"]
    L = npb.load_library()
    p = npb.SearchParameters(**PARAMS[0])
    n = npb.device_count()
    dep = npb.MmapIndex.load_devices(path, [0, 0, 0])
    want = _res(dep.search_batch(qs, p))
    layout = [x.tolist() for x in dep.shard_layout()]

    def raw(call, arr, n_items, bounds=None):
        a = np.ascontiguousarray(arr, np.int32)
        bb = None if bounds is None else np.ascontiguousarray(bounds, np.int64)
        out = np.zeros(70, np.int64)
        return call(dep._h, a.ctypes.data_as(C.c_void_p), n_items,
                    None if bb is None else bb.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p))

    add, rem = L.pb_index_add_devices, L.pb_index_remove_ranks
    cases = {
        "device -1": lambda: raw(add, [-1], 1),
        "device out of range": lambda: raw(add, [n], 1),
        "no device": lambda: raw(add, [0], 0),
        "world 65": lambda: raw(add, [0] * 62, 62),
        "add: bounds short of D": lambda: raw(add, [0], 1, [0, 100, 200, 300, 899]),
        "add: bounds decreasing": lambda: raw(add, [0], 1, [0, 300, 200, 400, 900]),
        "rank -1": lambda: raw(rem, [-1], 1),
        "rank 3": lambda: raw(rem, [3], 1),
        "rank twice": lambda: raw(rem, [1, 1], 2),
        "every rank": lambda: raw(rem, [0, 1, 2], 3),
        "no rank": lambda: raw(rem, [0], 0),
        "remove: bounds not from 0": lambda: raw(rem, [1], 1, [1, 500, 900]),
    }
    try:
        for name, call in cases.items():
            assert call() == PB_ERR_INVALID, (name, L.pb_last_error())
            assert [x.tolist() for x in dep.shard_layout()] == layout, name
            assert _res(dep.search_batch(qs, p)) == want, name
        with pytest.raises(npb.PlaidError) as e:        # the binding checks the bounds' length
            dep.add_devices([0], [0, 900])
        assert e.value.status == PB_ERR_INVALID
    finally:
        dep.close()

    def unsupported(h):
        for call in (lambda: h.add_devices([0]), lambda: h.remove_ranks([0])):
            with pytest.raises(npb.PlaidError) as e:
                call()
            assert e.value.status == PB_ERR_UNSUPPORTED, str(e.value)
        assert _res(h.search_batch(qs, p)) == want
    plain = npb.MmapIndex.load(path)
    reps = npb.MmapIndex.load_replicas(path, [0, 0])
    host = npb.MmapIndex.load_devices(path, [0, 0], host_residuals=True)
    try:
        unsupported(plain)
        unsupported(reps)
        unsupported(host)
        assert host.shard_layout()[0].tolist() == npb.shard_bounds(path, 2).tolist()
    finally:
        plain.close()
        reps.close()
        host.close()
    # a rank of an in-process group (as an NCCL-joined handle): not a deployment
    shard = npb.MmapIndex.load(path)
    grp = C.c_void_p()
    assert L.pb_shard_group_create(1, C.byref(grp)) == 0
    try:
        assert L.pb_index_group_join(shard._h, grp, 0) == 0
        unsupported(shard)
    finally:
        shard.close()
        L.pb_shard_group_destroy(grp)


def _threads_now():
    return len(os.listdir("/proc/self/task"))


def test_threads_and_memory(npb, corpus):
    path, qs, D = corpus["path"], corpus["qs"], corpus["ix"].num_documents
    p = npb.SearchParameters(**PARAMS[0])
    warm = npb.MmapIndex.load_devices(path, [0] * 8)
    warm.search_batch(qs, p)
    warm.close()
    before = _threads_now()
    dep = npb.MmapIndex.load_devices(path, [0, 0])
    two = _threads_now()
    try:
        dep.add_devices([0] * 6)
        assert _threads_now() >= two + 6
        dep.search_batch(qs, p)

        def fresh_memory(devices):
            f = npb.MmapIndex.load_devices(path, devices)
            try:
                return f.memory_usage()
            finally:
                f.close()
        # a resized rank holds arrays sized to their contents; a loaded one has the allocator's slack (1/8 + 256 bytes
        # per array), and the last rank keeps the little spare its empty arrays had
        for W in (8, 3):
            if W == 3:
                dep.remove_ranks([0, 2, 4, 6, 7])
            got, fresh = dep.memory_usage(), fresh_memory([0] * W)
            assert got["host_bytes"] == fresh["host_bytes"] == 0
            assert fresh["device_bytes"] * 8 // 9 - 4096 * W <= got["device_bytes"] <= fresh["device_bytes"] + 4096, W
        dep.remove_ranks([1])
        assert _threads_now() == two
    finally:
        dep.close()
    assert _threads_now() == before
    # an empty rank opened from rank 0 equals load_range of an empty range: a deployment of one rank grown by one
    # empty rank (nothing moves) holds exactly what the two loads hold
    dep = npb.MmapIndex.load_devices(path, [0])
    try:
        assert dep.add_devices([0], [0, D, D]).tolist() == [0, D, D]
        mem = {"device_bytes": 0, "host_bytes": 0}
        for b, e in ((0, D), (D, D)):
            s = npb.MmapIndex.load_range(path, b, e, device=0)
            assert s.num_documents() == e - b and s.shard_layout()[0].tolist() == [b, e]
            for k, v in s.memory_usage().items():
                mem[k] += v
            s.close()
        assert dep.memory_usage() == mem
        full = npb.MmapIndex.load(path)
        try:
            assert _res(dep.search_batch(qs, p)) == _res(full.search_batch(qs, p))
        finally:
            full.close()
    finally:
        dep.close()
    assert _threads_now() == before
