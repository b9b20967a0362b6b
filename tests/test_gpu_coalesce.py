"""pb_search and the request coalescer (DESIGN.md 4m): single-query calls from many host threads, merged into shared
pb_search_batch_params calls.  With coalescing off pb_search is the batch of one; with it on every request must get,
bit for bit, what the CPU oracle computes for it and what it gets alone, whatever batch it rode in: mixed parameters,
subsets of every probe kind, both variants, refusals, failed merged calls, appends and deletes under way, host-tier
handles, lanes, shard groups, and the thread-local stats of a follower.

Batches are made to form by releasing the threads from a barrier with max_wait_us at its largest, never by timing an
assertion: the checks on batch sizes are all `>=`."""
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
PB_ERR_INVALID, PB_ERR_UNSUPPORTED = 1, 4
WAIT_US = 10_000


@pytest.fixture(scope="module")
def npb():
    import next_plaid_b200 as m
    m.build_library()
    if m.device_count() < 1:
        pytest.fail("GPU tests need an H100; the library has no CPU fallback")
    return m


def _open(npb, ix, **kw):
    return npb.MmapIndex.from_arrays(ix.centroids, ix.bucket_weights, ix.codes, ix.residuals,
                                     ix.doc_lengths, ix.ivf, ix.ivf_lengths, ix.nbits, **kw)


def _same(a, b):
    return a.passage_ids.tolist() == b.passage_ids.tolist() and np.array_equal(a.scores, b.scores)


# the mix of test_gpu_search_params.py: (query tokens, parameters)
MIX = [
    (32, dict(top_k=10, n_full_scores=256, n_ivf_probe=8)),
    (1, dict(top_k=1, n_full_scores=4, n_ivf_probe=1, centroid_score_threshold=None)),
    (64, dict(top_k=100, n_full_scores=1024, n_ivf_probe=64)),
    (33, dict(top_k=0, n_full_scores=256, n_ivf_probe=8)),
    (65, dict(top_k=300, n_full_scores=64, n_ivf_probe=65, centroid_score_threshold=None)),
    (32, dict(top_k=10, n_full_scores=4096, n_ivf_probe=192, centroid_batch_size=128)),
    (32, dict(top_k=10, n_full_scores=0, n_ivf_probe=8)),
    (20, dict(top_k=100, n_full_scores=1024, n_ivf_probe=8, centroid_score_threshold=1e9)),
    (33, dict(top_k=10, n_full_scores=64, n_ivf_probe=32, centroid_batch_size=64)),
    (32, dict(top_k=100, n_full_scores=4096, n_ivf_probe=8, centroid_batch_size=128, centroid_score_threshold=None)),
    (1, dict(top_k=10, n_full_scores=256, n_ivf_probe=16)),
    (64, dict(top_k=10, n_full_scores=1024, n_ivf_probe=8, centroid_batch_size=64, centroid_score_threshold=None)),
]


def _kw(d):
    k = dict(centroid_batch_size=100_000, centroid_score_threshold=0.4)
    k.update(d)
    return k


def _requests(oracle, docs, D, seed):
    """(query, parameter kwargs, subset): the mix without subsets, then with a subset of every probe kind"""
    qs = [oracle.synthetic_queries(docs, 1, nq=n, seed=seed + i)[0][0] for i, (n, _) in enumerate(MIX)]
    kws = [_kw(d) for _, d in MIX]
    rng = np.random.default_rng(4)
    subs = [None, [], [5, 5, 17, 10 ** 7, -3, 17], sorted(rng.choice(D, 40, replace=False).tolist()),
            list(range(0, D, 2)), list(range(1, D, 20)), list(range(D)), [D, D + 5, -1], None,
            list(range(0, D, 3)), list(range(1, D, 20)), None]
    return [(q, k, None) for q, k in zip(qs, kws)] + [(q, k, s) for q, k, s in zip(qs, kws, subs)]


def _alone(npb, gpu, reqs):
    return [gpu.search_batch_params([q], [npb.SearchParameters(**k)], [s])[0] for q, k, s in reqs]


def _threads(n, body):
    """body(t) on n threads released together; the per-thread return values, or the first exception"""
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


def _bucket(n):
    b = 0
    while b < 7 and (1 << b) < n:
        b += 1
    return b


@pytest.fixture(scope="module", params=[(128, 4), (48, 2)], ids=["d128n4", "d48n2"])
def corpus(request, oracle, npb):
    dim, nbits = request.param
    docs = oracle.synthetic_corpus(3000, 40, dim=dim, seed=dim + nbits + 5, ragged=True)
    ix = oracle.create_index(docs, nbits=nbits, seed=3, num_partitions=512)
    gpu = _open(npb, ix)
    reqs = _requests(oracle, docs, ix.num_documents, 100)
    want = [oracle.search_one(ix, q, oracle.SearchParameters(**k), subset=s) for q, k, s in reqs]
    alone = _alone(npb, gpu, reqs)
    yield ix, gpu, reqs, want, alone
    gpu.close()


def test_off_is_the_batch_of_one(npb, corpus):
    ix, gpu, reqs, want, alone = corpus
    gpu.coalesce_stats(reset=True)
    for (q, k, s), w in zip(reqs, want):
        p = npb.SearchParameters(**k)
        one = gpu.search_batch_params([q], [p], [s])[0]
        wc, wl = gpu.last_work_counters(), gpu.last_stage_stats()[1]
        r = gpu.search(q, p, subset=s)
        assert _same(r, one) and _same(r, w) and r.query_id == 0
        assert gpu.last_work_counters() == wc and gpu.last_stage_stats()[1] == wl
    st = gpu.coalesce_stats()
    assert st["n_bypassed"] == len(reqs) and st["n_requests"] == 0 and st["n_batches"] == 0


@pytest.mark.parametrize("T,rounds", [(16, 24), (64, 6)])
def test_threads_share_batches_and_get_their_own_results(npb, corpus, T, rounds):
    ix, gpu, reqs, want, alone = corpus
    gpu.set_coalescing(32, max_wait_us=WAIT_US, max_inflight=2)
    gpu.coalesce_stats(reset=True)

    def body(t):
        seen = []
        for i in range(rounds):
            j = (t * 5 + i) % len(reqs)                  # each thread its own rotation
            q, k, s = reqs[j]
            r = gpu.search(q, npb.SearchParameters(**k), subset=s)
            assert _same(r, want[j]) and _same(r, alone[j]), (t, j)
            seen.append(gpu.last_work_counters()["n_queries"])   # the batch this thread's request rode in
        return seen
    try:
        seen = _threads(T, body)
    finally:
        gpu.set_coalescing(1)
    st = gpu.coalesce_stats()
    assert st["n_requests"] == T * rounds and st["n_refused"] == 0 and st["n_rerun_alone"] == 0
    assert 2 <= st["max_batch"] <= 32 and st["n_batches"] < st["n_requests"]
    assert sum(st["batch_hist"]) == st["n_batches"] and sum(st["batch_hist"][6:]) == 0
    # every thread of a batch reports the batch's counters (n_queries: its queries that ran a pass, so the ones with
    # top_k = 0, n_full_scores = 0 or nothing eligible are not in it): were it only the leaders, at most one report per
    # merged batch could exceed 1
    sizes = [n for per in seen for n in per]
    assert all(0 <= n <= st["max_batch"] for n in sizes)
    assert sum(n >= 2 for n in sizes) > sum(st["batch_hist"][1:])


def test_wait_zero_and_one_thread_runs_alone(npb, corpus):
    ix, gpu, reqs, want, alone = corpus
    gpu.set_coalescing(32, max_wait_us=0)
    gpu.coalesce_stats(reset=True)
    try:
        for j, (q, k, s) in enumerate(reqs):
            assert _same(gpu.search(q, npb.SearchParameters(**k), subset=s), want[j])
    finally:
        gpu.set_coalescing(1)
    st = gpu.coalesce_stats()
    assert st["n_requests"] == len(reqs) and st["batch_hist"] == [len(reqs)] + [0] * 7


def test_refused_request_leaves_its_neighbours_alone(npb, corpus):
    ix, gpu, reqs, want, alone = corpus
    q0 = reqs[0][0]
    bad = {3: (dict(n_ivf_probe=0), PB_ERR_INVALID, "n_ivf_probe must be >= 1"),
           7: (dict(top_k=10, n_full_scores=80000), PB_ERR_UNSUPPORTED, "exceeds 16384"),
           11: (dict(n_ivf_probe=193, centroid_batch_size=64), PB_ERR_UNSUPPORTED, "batched variant"),
           13: (dict(top_k=-1), PB_ERR_INVALID, "must be >= 0")}
    gpu.set_coalescing(32, max_wait_us=WAIT_US)
    gpu.coalesce_stats(reset=True)

    def body(t):
        for i in range(4):
            if t in bad:
                d, status, text = bad[t]
                p = npb.SearchParameters(**_kw(dict(dict(top_k=10, n_full_scores=256, n_ivf_probe=8), **d)))
                with pytest.raises(npb.PlaidError) as e:
                    gpu.search(q0, p)
                assert e.value.status == status and text in str(e.value), (t, str(e.value))
            else:
                j = (t + i) % len(reqs)
                q, k, s = reqs[j]
                assert _same(gpu.search(q, npb.SearchParameters(**k), subset=s), want[j]), (t, j)
    try:
        _threads(16, body)
    finally:
        gpu.set_coalescing(1)
    st = gpu.coalesce_stats()
    assert st["n_refused"] == 16 and st["n_requests"] == 12 * 4 and st["n_rerun_alone"] == 0


def test_failed_merged_call_reruns_its_members_alone(oracle, npb, corpus):
    """A dense-variant query with a subset gets its probe width from its eligible centroids, counted on the device, so
    its limit (query tokens x width <= 8192) cannot be checked before it is queued: the merged call is refused, every
    member runs again alone, the offender gets its own status and the others their results."""
    ix, gpu, reqs, want, alone = corpus
    D = ix.num_documents
    wide = np.ascontiguousarray(np.concatenate([reqs[2][0]] * 3, 0)[:130])   # 130 tokens: rows of 192
    p_wide = npb.SearchParameters(**_kw(dict(top_k=10, n_full_scores=256, n_ivf_probe=16)))
    sub = list(range(0, D, 3))                                               # 16 x 3 = 48 cells: 192 x 48 > 8192
    with pytest.raises(npb.PlaidError) as e:
        gpu.search(wide, p_wide, subset=sub)
    assert e.value.status == PB_ERR_UNSUPPORTED and "exceeds 8192" in str(e.value)
    gpu.set_coalescing(32, max_wait_us=WAIT_US)
    gpu.coalesce_stats(reset=True)

    def body(t):
        for i in range(4):
            if t == 5:
                with pytest.raises(npb.PlaidError) as e:
                    gpu.search(wide, p_wide, subset=sub)
                assert e.value.status == PB_ERR_UNSUPPORTED and "exceeds 8192" in str(e.value)
            else:
                j = (t + i) % len(reqs)
                q, k, s = reqs[j]
                assert _same(gpu.search(q, npb.SearchParameters(**k), subset=s), want[j]), (t, j)
    try:
        _threads(16, body)
    finally:
        gpu.set_coalescing(1)
    st = gpu.coalesce_stats()
    assert st["n_refused"] == 0 and st["n_requests"] == 64 and st["n_rerun_alone"] >= 2


def test_appends_and_deletes_under_way(oracle, npb):
    docs = oracle.synthetic_corpus(2500, 36, dim=128, seed=78, ragged=True)
    ix = oracle.create_index(docs, nbits=4, seed=9, num_partitions=256)
    D0 = 1800
    t0 = int(ix.doc_offsets[D0])
    ivf, ivf_lengths = oracle.build_ivf(ix.codes[:t0], ix.doc_lengths[:D0], ix.num_centroids)
    head = oracle.Index(ix.centroids, ix.bucket_weights, ix.bucket_cutoffs, ix.codes[:t0], ix.residuals[:t0],
                        ix.doc_lengths[:D0], ivf, ivf_lengths, ix.nbits)
    reqs = _requests(oracle, docs, D0, 300)
    gone = list(range(0, ix.num_documents, 7))

    def mutate(h, between):
        between(0)
        h.append_encoded(ix.codes[t0:], ix.residuals[t0:], ix.doc_lengths[D0:])
        between(1)
        assert h.delete(gone) > 0
        between(2)

    # the three states of the index, on a handle searched serially
    ref, states = _open(npb, head), []
    try:
        mutate(ref, lambda _: states.append(_alone(npb, ref, reqs)))
    finally:
        ref.close()
    for j, (q, k, s) in enumerate(reqs):                 # the oracle pins the states it can rebuild
        assert _same(states[0][j], oracle.search_one(head, q, oracle.SearchParameters(**k), subset=s))
        assert _same(states[1][j], oracle.search_one(ix, q, oracle.SearchParameters(**k), subset=s))

    gpu = _open(npb, head)
    gpu.set_coalescing(32, max_wait_us=200)
    stop = threading.Event()

    def body(t):
        if t == 16:                                      # the writer
            try:
                mutate(gpu, lambda _: [gpu.search(*_req(reqs[0], npb)) for _ in range(20)])
            finally:
                stop.set()
            return 0
        n = 0
        while not stop.is_set() or n < 8:
            j = (t * 3 + n) % len(reqs)
            r = gpu.search(*_req(reqs[j], npb))
            assert any(_same(r, st[j]) for st in states), (t, j)   # one state whole, never a mixture
            n += 1
        return n
    try:
        _threads(17, body)
        final = [gpu.search(*_req(r, npb)) for r in reqs]
        assert all(_same(a, b) for a, b in zip(final, states[2]))
        assert gpu.coalesce_stats()["n_requests"] > 0
    finally:
        gpu.close()


def _req(r, npb):
    q, k, s = r
    return q, npb.SearchParameters(**k), s


def test_host_tier_and_lanes(npb, corpus):
    ix, gpu, reqs, want, alone = corpus
    host = _open(npb, ix, host_residuals=True)
    host.set_lanes(2)
    host.set_coalescing(32, max_wait_us=WAIT_US, max_inflight=1)

    def body(t):
        for i in range(4):
            j = (t * 7 + i) % len(reqs)
            assert _same(host.search(*_req(reqs[j], npb)), want[j]), (t, j)
    try:
        _threads(32, body)
        st = host.coalesce_stats()
        assert st["n_requests"] == 128 and st["max_batch"] >= 2
    finally:
        host.close()


def test_environment_default(npb, corpus, monkeypatch):
    ix, gpu, reqs, want, alone = corpus
    monkeypatch.setenv("PB_COALESCE", "8")
    monkeypatch.setenv("PB_COALESCE_WAIT_US", "50")
    h = _open(npb, ix)
    monkeypatch.delenv("PB_COALESCE")
    try:
        assert _same(h.search(*_req(reqs[0], npb)), want[0])
        assert h.coalesce_stats()["n_requests"] == 1
        h.set_coalescing(1)
        assert _same(h.search(*_req(reqs[0], npb)), want[0])
        assert h.coalesce_stats()["n_bypassed"] == 1
        for bad in ((0, 0, 2), (8, -1, 2), (8, 0, 0)):
            with pytest.raises(npb.PlaidError) as e:
                h.set_coalescing(*bad)
            assert e.value.status == PB_ERR_INVALID
    finally:
        h.close()


def test_shard_group_refuses_coalescing_and_search_stays_a_collective(oracle, npb, corpus):
    ix, gpu, reqs, want, alone = corpus
    D = ix.num_documents
    bounds = [0, D // 2, D]
    shards = []
    for r in range(2):
        d0, d1 = bounds[r], bounds[r + 1]
        a, b = int(ix.doc_offsets[d0]), int(ix.doc_offsets[d1])
        ivf, ivf_lengths = oracle.build_ivf(ix.codes[a:b], ix.doc_lengths[d0:d1], ix.num_centroids)
        part = oracle.Index(ix.centroids, ix.bucket_weights, ix.bucket_cutoffs, ix.codes[a:b], ix.residuals[a:b],
                            ix.doc_lengths[d0:d1], ivf, ivf_lengths, ix.nbits)
        shards.append(_open(npb, part, device=0, doc_id_base=d0))
    shards[0].set_coalescing(32)                         # joining turns it off
    grp = npb.ShardGroup(shards)
    try:
        for s in shards:
            with pytest.raises(npb.PlaidError) as e:
                s.set_coalescing(32)
            assert e.value.status == PB_ERR_UNSUPPORTED
            s.set_coalescing(1)                          # off is always accepted
        for j in (0, 2, 8, 16, 21):
            res = grp._collective(lambda r, s: s.search(*_req(reqs[j], npb)))
            assert all(_same(x, want[j]) for x in res), j
        assert shards[0].coalesce_stats()["n_requests"] == 0 and shards[0].coalesce_stats()["n_bypassed"] == 5
    finally:
        grp.close()
