"""pb_search_batch_subsets: a subset per query (None, [] or an id list) in one call.  Every query's result must be
bit-identical to the CPU oracle searching it alone with its subset, and to pb_search_batch of that query alone; a
call whose queries share one subset is pb_search_batch with it, work counters included.  Covers both variants, the
probe kinds a subset can lead to (streaming over the eligible centroids, radix select past 64, every eligible
centroid, nothing eligible), lanes, small workspace budgets, concurrent callers, host-tier handles, appends and
deletes, traces, in-process shard groups and argument errors."""
import ctypes as C
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
PB_ERR_INVALID = 1


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


def _queries(oracle, docs, lengths, seed):
    return [oracle.synthetic_queries(docs, 1, nq=n, seed=seed + i)[0][0] for i, n in enumerate(lengths)]


def _mix(D, seed):
    """one of each kind a subset leads to (n_ivf_probe = 8): None, Some([]), out-of-range / negative / duplicated ids,
    a tiny list (every eligible centroid), half the docs (scaled probe 16, streaming), 5 % (scaled 160: radix select),
    the full id range, and a list of nothing in range (no eligible centroid)"""
    rng = np.random.default_rng(seed)
    return [None, [], [5, 5, 17, 10 ** 7, -3, 17], sorted(rng.choice(D, 40, replace=False).tolist()),
            list(range(0, D, 2)), list(range(1, D, 20)), list(range(D)), [D, D + 5, -1]]


@pytest.fixture(scope="module", params=[(128, 4), (64, 2), (48, 4)], ids=["d128n4", "d64n2", "d48n4"])
def corpus(request, oracle, npb):
    dim, nbits = request.param
    docs = oracle.synthetic_corpus(3000, 40, dim=dim, seed=dim + nbits, ragged=True)
    ix = oracle.create_index(docs, nbits=nbits, seed=3, num_partitions=512)
    gpu = _open(npb, ix)
    yield docs, ix, gpu
    gpu.close()


LENGTHS = (1, 32, 33, 64, 65, 32, 33, 1)


@pytest.mark.parametrize("cbs", [100_000, 128])
@pytest.mark.parametrize("thr", [0.4, None])
def test_each_query_equals_the_oracle_with_its_subset(oracle, npb, corpus, cbs, thr):
    docs, ix, gpu = corpus
    D = ix.num_documents
    subs = _mix(D, 1)
    qs = _queries(oracle, docs, LENGTHS, 100)
    kw = dict(top_k=10, n_ivf_probe=8, n_full_scores=256, centroid_batch_size=cbs, centroid_score_threshold=thr)
    res = gpu.search_batch_subsets(qs, npb.SearchParameters(**kw), subs)
    po = oracle.SearchParameters(**kw)
    for i, (q, s, r) in enumerate(zip(qs, subs, res)):
        w = oracle.search_one(ix, q, po, subset=s)
        assert _same(r, w), (i, cbs, thr)
        assert r.query_id == i
        if s is not None:
            assert set(r.passage_ids.tolist()) <= set(s)
    assert len(res[1].passage_ids) == 0 and len(res[7].passage_ids) == 0     # Some([]), nothing eligible
    assert len(res[0].passage_ids) > 0 and len(res[6].passage_ids) > 0       # their neighbours still find docs


def test_shared_subset_and_none_equal_search_batch(oracle, npb, corpus):
    docs, ix, gpu = corpus
    D = ix.num_documents
    qs = _queries(oracle, docs, (32, 1, 65, 33, 64, 32), 200)
    for cbs in (100_000, 128):
        pg = npb.SearchParameters(top_k=10, n_ivf_probe=8, n_full_scores=256, centroid_batch_size=cbs)
        for s in _mix(D, 2):
            want = gpu.search_batch(qs, pg, subset=s)
            wc = gpu.last_work_counters()
            got = gpu.search_batch_subsets(qs, pg, [s] * len(qs))
            assert gpu.last_work_counters() == wc, (cbs, s is None)
            for a, b in zip(got, want):
                assert _same(a, b), (cbs, s is None)


@pytest.mark.parametrize("knob", [None, "scores_tc", "fast_exact", "fast_approx"])
def test_distinct_subsets_equal_batch_of_one(oracle, npb, corpus, knob):
    docs, ix, gpu = corpus
    D = ix.num_documents
    subs = _mix(D, 3)
    qs = _queries(oracle, docs, LENGTHS, 300)
    if knob:
        getattr(gpu, "set_" + knob)(0)
    try:
        for cbs in (100_000, 128):
            pg = npb.SearchParameters(top_k=10, n_ivf_probe=8, n_full_scores=256, centroid_batch_size=cbs)
            got = gpu.search_batch_subsets(qs, pg, subs)
            for q, s, r in zip(qs, subs, got):
                assert _same(r, gpu.search_batch([q], pg, subset=s)[0]), (knob, cbs)
    finally:
        if knob:
            getattr(gpu, "set_" + knob)(1)


def test_unfiltered_queries_keep_the_tensor_core_path(oracle, npb, corpus):
    docs, ix, gpu = corpus
    D = ix.num_documents
    qs = _queries(oracle, docs, (32,) * 8, 400)
    pg = npb.SearchParameters(top_k=10, n_ivf_probe=8, n_full_scores=256)
    plain = [0, 2, 4, 6]
    gpu.search_batch([qs[i] for i in plain], pg)
    alone = gpu.last_work_counters()
    subs = [None, list(range(0, D, 2)), None, list(range(0, D, 3)), None, list(range(1, D, 20)), None, [3, 4]]
    res = gpu.search_batch_subsets(qs, pg, subs)
    mixed = gpu.last_work_counters()
    assert mixed["n_k1_tc"] >= alone["n_k1_tc"] and mixed["n_probe_threshold"] >= alone["n_probe_threshold"]
    assert alone["n_k1_tc"] + alone["n_probe_threshold"] > 0
    po = oracle.SearchParameters(top_k=10, n_ivf_probe=8, n_full_scores=256)
    for q, s, r in zip(qs, subs, res):
        assert _same(r, oracle.search_one(ix, q, po, subset=s))


def test_trace_per_query(oracle, npb, corpus):
    docs, ix, gpu = corpus
    subs = _mix(ix.num_documents, 4)
    qs = _queries(oracle, docs, LENGTHS, 500)
    for cbs in (100_000, 128):
        kw = dict(top_k=10, n_ivf_probe=8, n_full_scores=256, centroid_batch_size=cbs)
        res, tr = gpu.search_batch_subsets(qs, npb.SearchParameters(**kw), subs, trace=True)
        for i, (q, s) in enumerate(zip(qs, subs)):
            want, wt = oracle.search_one(ix, q, oracle.SearchParameters(**kw), subset=s, trace=True)
            assert _same(res[i], want), (i, cbs)
            assert tr.cells[i].tolist() == wt.cells.tolist(), (i, cbs)
            assert tr.candidates[i].tolist() == wt.candidates.tolist(), (i, cbs)
            assert np.array_equal(tr.approx[i], wt.approx), (i, cbs)
            assert tr.kept[i].tolist() == wt.kept.tolist(), (i, cbs)
            assert np.array_equal(tr.kept_exact[i], wt.kept_exact), (i, cbs)


@pytest.fixture(scope="module")
def small(oracle):
    docs = oracle.synthetic_corpus(2500, 36, dim=128, seed=77, ragged=True)
    ix = oracle.create_index(docs, nbits=4, seed=9, num_partitions=256)
    subs = (_mix(2500, 5) * 3)[:24]
    qs = _queries(oracle, docs, [(1, 32, 33, 64, 65, 20)[i % 6] for i in range(24)], 600)
    return docs, ix, qs, subs


def _want(oracle, ix, qs, subs, kw):
    po = oracle.SearchParameters(**kw)
    return [oracle.search_one(ix, q, po, subset=s) for q, s in zip(qs, subs)]


def test_lanes_budget_threads_and_host_tier(oracle, npb, small, monkeypatch):
    docs, ix, qs, subs = small
    for cbs in (100_000, 64):
        kw = dict(top_k=10, n_ivf_probe=8, n_full_scores=256, centroid_batch_size=cbs)
        pg = npb.SearchParameters(**kw)
        want = _want(oracle, ix, qs, subs, kw)
        gpu = _open(npb, ix)
        try:
            for lanes in (2, 4):
                gpu.set_lanes(lanes)
                assert all(_same(a, b) for a, b in zip(gpu.search_batch_subsets(qs, pg, subs), want)), (cbs, lanes)
            gpu.set_lanes(1)
            # 4 host threads at once, each with its own rotation of the subsets
            out, err = [None] * 4, [None] * 4

            def run(t):
                try:
                    rot = subs[t:] + subs[:t]
                    out[t] = (rot, gpu.search_batch_subsets(qs, pg, rot))
                except Exception as e:  # noqa: BLE001 - re-raised below
                    err[t] = e
            ths = [threading.Thread(target=run, args=(t,)) for t in range(4)]
            [t.start() for t in ths]
            [t.join() for t in ths]
            assert err == [None] * 4, err
            for rot, res in out:
                for q, s, r in zip(qs, rot, res):
                    assert _same(r, gpu.search_batch([q], pg, subset=s)[0]), cbs
        finally:
            gpu.close()
        monkeypatch.setenv("PB_WS_BUDGET_MB", "1")       # many sub-batches
        tiny = _open(npb, ix)
        monkeypatch.delenv("PB_WS_BUDGET_MB")
        host = _open(npb, ix, host_residuals=True)
        try:
            assert all(_same(a, b) for a, b in zip(tiny.search_batch_subsets(qs, pg, subs), want)), cbs
            assert all(_same(a, b) for a, b in zip(host.search_batch_subsets(qs, pg, subs), want)), cbs
        finally:
            tiny.close()
            host.close()


def test_after_append_and_delete(oracle, npb, small):
    docs, ix, qs, subs = small
    D0 = 1800
    t0 = int(ix.doc_offsets[D0])
    ivf, ivf_lengths = oracle.build_ivf(ix.codes[:t0], ix.doc_lengths[:D0], ix.num_centroids)
    head = oracle.Index(ix.centroids, ix.bucket_weights, ix.bucket_cutoffs, ix.codes[:t0], ix.residuals[:t0],
                        ix.doc_lengths[:D0], ivf, ivf_lengths, ix.nbits)
    gpu = _open(npb, head)
    try:
        new = gpu.append_encoded(ix.codes[t0:], ix.residuals[t0:], ix.doc_lengths[D0:])
        assert new == list(range(D0, ix.num_documents))
        named = [None, list(range(D0, ix.num_documents, 3)), list(range(D0 - 50, D0 + 50)), [D0 + 1, 2, D0 + 7]]
        sub2 = (named * 6)[:len(qs)]
        for cbs in (100_000, 64):
            kw = dict(top_k=10, n_ivf_probe=8, n_full_scores=256, centroid_batch_size=cbs)
            got = gpu.search_batch_subsets(qs, npb.SearchParameters(**kw), sub2)
            assert all(_same(a, b) for a, b in zip(got, _want(oracle, ix, qs, sub2, kw))), cbs
        gone = list(range(0, ix.num_documents, 7)) + [D0 + 1, D0 + 7]
        assert gpu.delete(gone) == len(set(gone))
        for cbs in (100_000, 64):
            pg = npb.SearchParameters(top_k=10, n_ivf_probe=8, n_full_scores=256, centroid_batch_size=cbs)
            got = gpu.search_batch_subsets(qs, pg, sub2)
            for q, s, r in zip(qs, sub2, got):
                assert _same(r, gpu.search_batch([q], pg, subset=s)[0]), cbs
    finally:
        gpu.close()


# -- in-process shard groups ---------------------------------------------------------------------------------------

def _shard(oracle, ix, d0, d1):
    t0, t1 = int(ix.doc_offsets[d0]), int(ix.doc_offsets[d1])
    codes, res, dl = ix.codes[t0:t1], ix.residuals[t0:t1], ix.doc_lengths[d0:d1]
    ivf, ivf_lengths = oracle.build_ivf(codes, dl, ix.num_centroids)
    return oracle.Index(ix.centroids, ix.bucket_weights, ix.bucket_cutoffs, codes, res, dl, ivf, ivf_lengths, ix.nbits)


def _group(npb, oracle, ix, bounds, host=(), budget_mb=None, monkeypatch=None):
    shards = []
    for r in range(len(bounds) - 1):
        if budget_mb and budget_mb[r]:
            monkeypatch.setenv("PB_WS_BUDGET_MB", str(budget_mb[r]))
        sh = _shard(oracle, ix, bounds[r], bounds[r + 1])
        shards.append(_open(npb, sh, device=0, doc_id_base=bounds[r], host_residuals=r in host))
        if budget_mb and budget_mb[r]:
            monkeypatch.delenv("PB_WS_BUDGET_MB")
    return npb.ShardGroup(shards)


def _check_group(grp, res, want):
    for per_rank in grp.all_results:                      # every rank holds the same global answer
        assert all(_same(a, b) for a, b in zip(per_rank, res))
    assert all(_same(a, b) for a, b in zip(res, want))


@pytest.mark.parametrize("G", [2, 3, 8])
def test_group_per_query_and_single_subsets_dense(oracle, npb, small, G):
    docs, ix, qs, subs = small
    D = ix.num_documents
    bounds = [g * D // G for g in range(G + 1)]
    if G == 3:
        bounds = [0, 1000, 1000, D]                       # an empty shard
    grp = _group(npb, oracle, ix, bounds)
    try:
        s1 = list(range(bounds[1] // 2, bounds[1]))       # one shard only
        s2 = list(range(0, bounds[1])) + list(range(bounds[-2], D, 2))   # the middle shards hold no subset doc
        per_q = ([s1, s2] + subs)[:len(qs)]
        for cbs in (100_000, 64):
            kw = dict(top_k=10, n_ivf_probe=8, n_full_scores=256, centroid_batch_size=cbs)
            pg = npb.SearchParameters(**kw)
            res = grp.search_batch_subsets(qs, pg, per_q)
            _check_group(grp, res, _want(oracle, ix, qs, per_q, kw))
            for s in (s1, s2, list(range(1, D, 20))):     # pb_search_batch with one subset, now also dense
                res = grp.search_batch(qs, pg, subset=s)
                _check_group(grp, res, _want(oracle, ix, qs, [s] * len(qs), kw))
    finally:
        grp.close()


def test_group_mixed_tiers_and_budgets(oracle, npb, small, monkeypatch):
    """ranks with different sub-batch bounds (a host-tier rank, a small budget) agree on the smallest"""
    docs, ix, qs, subs = small
    D = ix.num_documents
    grp = _group(npb, oracle, ix, [0, 800, 1700, D], host=(1,), budget_mb=[1, 0, 2], monkeypatch=monkeypatch)
    try:
        for cbs in (100_000, 64):
            kw = dict(top_k=10, n_ivf_probe=8, n_full_scores=256, centroid_batch_size=cbs)
            pg = npb.SearchParameters(**kw)
            _check_group(grp, grp.search_batch_subsets(qs, pg, subs), _want(oracle, ix, qs, subs, kw))
            _check_group(grp, grp.search_batch(qs, pg), _want(oracle, ix, qs, [None] * len(qs), kw))
    finally:
        grp.close()


def test_group_ranks_with_different_subsets_refuse_together(oracle, npb, small):
    docs, ix, qs, subs = small
    D = ix.num_documents
    grp = _group(npb, oracle, ix, [0, D // 2, D])
    try:
        kw = dict(top_k=10, n_ivf_probe=8, n_full_scores=256)
        pg = npb.SearchParameters(**kw)

        def call(r, s):
            mine = [list(range(r, D, 3))] + subs[1:]
            try:
                s.search_batch_subsets(qs, pg, mine)
                return None
            except npb.PlaidError as e:
                return e.status
        assert grp._collective(call) == [PB_ERR_INVALID] * 2
        _check_group(grp, grp.search_batch_subsets(qs, pg, subs), _want(oracle, ix, qs, subs, kw))
    finally:
        grp.close()


# -- argument errors ---------------------------------------------------------------------------------------------

def test_malformed_arguments_change_nothing(oracle, npb, small):
    docs, ix, qs, subs = small
    gpu = _open(npb, ix)
    L = npb.load_library()
    try:
        q = np.ascontiguousarray(np.concatenate(qs[:3], 0), np.float32)
        qo = np.array([0, len(qs[0]), len(qs[0]) + len(qs[1]), len(q)], np.int64)
        p = npb.SearchParameters(top_k=5, n_ivf_probe=8, n_full_scores=64)._c()
        ids = np.full((3, 5), 77, np.int64)
        sc = np.full((3, 5), 7.5, np.float32)
        cn = np.full(3, 9, np.int32)
        sid = np.arange(30, dtype=np.int64)
        P = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)  # noqa: E731
        cases = [(3, np.array([1, 10, 20, 30], np.int64), sid),          # does not start at 0
                 (3, np.array([0, 20, 10, 30], np.int64), sid),          # not monotone
                 (-1, np.array([0, 10, 20, 30], np.int64), sid),         # n_queries < 0
                 (3, np.array([0, 10, 20, 30], np.int64), None)]         # ids missing
        for n, so, si in cases:
            st = L.pb_search_batch_subsets(gpu._h, P(q), P(qo), n, C.byref(p), P(so), P(si), None,
                                           P(ids), P(sc), P(cn), None)
            assert st == PB_ERR_INVALID, (n, so, si is None)
            assert (ids == 77).all() and (sc == 7.5).all() and (cn == 9).all()
    finally:
        gpu.close()
