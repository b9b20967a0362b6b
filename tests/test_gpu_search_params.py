"""pb_search_batch_params: search parameters per query (top_k, n_full_scores, n_ivf_probe, threshold, variant) in one
call.  Every query's result must be bit-identical to the CPU oracle searching it alone with its parameters, and to
pb_search_batch of that query alone; a call whose queries share one struct is pb_search_batch (and with subsets
pb_search_batch_subsets), work counters, stage launches and traces included.  Covers the switches of the pipeline,
traces, per-query subsets, lanes, small workspace budgets, concurrent callers, host-tier handles, appends and deletes,
the tensor-core probe next to queries that cannot take it, flagged queries, in-process shard groups and argument
errors."""
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


# (query tokens, parameters): top_k 1 / 10 / 100 / above M, n_full_scores 4 / 64 / 1024 / 4096, n_ivf_probe 1 / 8 / 64 /
# 65 (radix select) / 192, thresholds None / 0.4 / above every score, the dense variant (K = 512 <= 100000) and the
# batched one with two slab widths, and queries with top_k = 0 and n_full_scores = 0 in the middle
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


def _params(npb, kws):
    return [npb.SearchParameters(**k) for k in kws]


def _want(oracle, ix, qs, kws, subs=None):
    subs = subs or [None] * len(qs)
    return [oracle.search_one(ix, q, oracle.SearchParameters(**k), subset=s) for q, k, s in zip(qs, kws, subs)]


@pytest.fixture(scope="module", params=[(128, 4), (64, 2), (48, 4)], ids=["d128n4", "d64n2", "d48n4"])
def corpus(request, oracle, npb):
    dim, nbits = request.param
    docs = oracle.synthetic_corpus(3000, 40, dim=dim, seed=dim + nbits + 1, ragged=True)
    ix = oracle.create_index(docs, nbits=nbits, seed=3, num_partitions=512)
    gpu = _open(npb, ix)
    qs = _queries(oracle, docs, [n for n, _ in MIX], 100)
    kws = [_kw(d) for _, d in MIX]
    yield docs, ix, gpu, qs, kws, _want(oracle, ix, qs, kws)
    gpu.close()


@pytest.mark.parametrize("knob", [None, "scores_tc", "fast_exact", "fast_approx"])
def test_each_query_equals_the_oracle_and_batch_of_one(npb, corpus, knob):
    docs, ix, gpu, qs, kws, want = corpus
    ps = _params(npb, kws)
    if knob:
        getattr(gpu, "set_" + knob)(0)
    try:
        res = gpu.search_batch_params(qs, ps)
        for i, (q, p, r, w) in enumerate(zip(qs, ps, res, want)):
            assert _same(r, w), (i, knob)
            assert _same(r, gpu.search_batch([q], p)[0]), (i, knob)
            assert r.query_id == i
            assert len(r.passage_ids) <= p.top_k
    finally:
        if knob:
            getattr(gpu, "set_" + knob)(1)
    assert len(res[3].passage_ids) == 0 and len(res[6].passage_ids) == 0    # top_k = 0, n_full_scores = 0
    assert len(res[7].passage_ids) == 0                                     # a threshold above every score
    assert len(res[2].passage_ids) == 100 and len(res[4].passage_ids) == 64  # top_k 100; top_k above M = 64


def test_uniform_params_are_the_old_calls(oracle, npb, corpus):
    docs, ix, gpu, qs, kws, _ = corpus
    D = ix.num_documents
    subs = [None, [], list(range(0, D, 2)), list(range(1, D, 20)), [5, 5, 17], None, list(range(D)), [D + 1]] * 2
    subs = subs[:len(qs)]
    for d in ({}, dict(centroid_batch_size=128), dict(top_k=100, n_full_scores=1024, centroid_score_threshold=None)):
        p = npb.SearchParameters(**_kw({**dict(top_k=10, n_full_scores=256, n_ivf_probe=8), **d}))
        want = gpu.search_batch(qs, p)
        wc, wl = gpu.last_work_counters(), gpu.last_stage_stats()[1]
        got = gpu.search_batch_params(qs, [p] * len(qs))
        assert gpu.last_work_counters() == wc and gpu.last_stage_stats()[1] == wl, d
        assert all(_same(a, b) for a, b in zip(got, want)), d
        want = gpu.search_batch_subsets(qs, p, subs)
        wc, wl = gpu.last_work_counters(), gpu.last_stage_stats()[1]
        got = gpu.search_batch_params(qs, [p] * len(qs), subs)
        assert gpu.last_work_counters() == wc and gpu.last_stage_stats()[1] == wl, d
        assert all(_same(a, b) for a, b in zip(got, want)), d
        want, wt = gpu.search_batch_subsets(qs, p, subs, trace=True)
        got, gt = gpu.search_batch_params(qs, [p] * len(qs), subs, trace=True)
        assert all(_same(a, b) for a, b in zip(got, want)), d
        for f in ("cells", "candidates", "approx", "kept", "kept_exact"):
            assert all(np.array_equal(a, b) for a, b in zip(getattr(gt, f), getattr(wt, f))), (d, f)


def test_trace_per_query(npb, corpus):
    docs, ix, gpu, qs, kws, want = corpus
    ps = _params(npb, kws)
    res, tr = gpu.search_batch_params(qs, ps, trace=True)
    for i, (q, p) in enumerate(zip(qs, ps)):
        one, ot = gpu.search_batch([q], p, trace=True)
        assert _same(res[i], one[0]) and _same(res[i], want[i]), i
        for f in ("cells", "candidates", "approx", "kept", "kept_exact"):
            assert np.array_equal(getattr(tr, f)[i], getattr(ot, f)[0]), (i, f)


def test_subsets_of_every_probe_kind(oracle, npb, corpus):
    docs, ix, gpu, qs, kws, _ = corpus
    D = ix.num_documents
    rng = np.random.default_rng(4)
    subs = [None, [], [5, 5, 17, 10 ** 7, -3, 17], sorted(rng.choice(D, 40, replace=False).tolist()),
            list(range(0, D, 2)), list(range(1, D, 20)), list(range(D)), [D, D + 5, -1], None,
            list(range(0, D, 3)), list(range(1, D, 20)), None]
    res = gpu.search_batch_params(qs, _params(npb, kws), subs)
    for i, (r, w) in enumerate(zip(res, _want(oracle, ix, qs, kws, subs))):
        assert _same(r, w), i


@pytest.fixture(scope="module")
def small(oracle):
    docs = oracle.synthetic_corpus(2500, 36, dim=128, seed=78, ragged=True)
    ix = oracle.create_index(docs, nbits=4, seed=9, num_partitions=256)
    mix = (MIX * 2)[:24]
    qs = _queries(oracle, docs, [n for n, _ in mix], 600)
    kws = [_kw(d) for _, d in mix]
    return docs, ix, qs, kws


def test_lanes_budget_threads_and_host_tier(oracle, npb, small, monkeypatch):
    docs, ix, qs, kws = small
    ps = _params(npb, kws)
    want = _want(oracle, ix, qs, kws)
    gpu = _open(npb, ix)
    try:
        gpu.set_lanes(2)
        assert all(_same(a, b) for a, b in zip(gpu.search_batch_params(qs, ps), want))
        gpu.set_lanes(1)
        out, err = [None] * 8, [None] * 8

        def run(t):                                       # 8 host threads, each with its own rotation of the batch
            try:
                out[t] = (t, gpu.search_batch_params(qs[t:] + qs[:t], ps[t:] + ps[:t]))
            except Exception as e:  # noqa: BLE001 - re-raised below
                err[t] = e
        ths = [threading.Thread(target=run, args=(t,)) for t in range(8)]
        [t.start() for t in ths]
        [t.join() for t in ths]
        assert err == [None] * 8, err
        for t, res in out:
            for q, p, r in zip(qs[t:] + qs[:t], ps[t:] + ps[:t], res):
                assert _same(r, gpu.search_batch([q], p)[0]), t
    finally:
        gpu.close()
    monkeypatch.setenv("PB_WS_BUDGET_MB", "1")           # many sub-batches
    tiny = _open(npb, ix)
    monkeypatch.delenv("PB_WS_BUDGET_MB")
    host = _open(npb, ix, host_residuals=True)
    try:
        assert all(_same(a, b) for a, b in zip(tiny.search_batch_params(qs, ps), want))
        assert all(_same(a, b) for a, b in zip(host.search_batch_params(qs, ps), want))
        assert host.last_staging_stats()["docs"] > 0
    finally:
        tiny.close()
        host.close()


def test_after_append_and_delete(oracle, npb, small):
    docs, ix, qs, kws = small
    ps = _params(npb, kws)
    D0 = 1800
    t0 = int(ix.doc_offsets[D0])
    ivf, ivf_lengths = oracle.build_ivf(ix.codes[:t0], ix.doc_lengths[:D0], ix.num_centroids)
    head = oracle.Index(ix.centroids, ix.bucket_weights, ix.bucket_cutoffs, ix.codes[:t0], ix.residuals[:t0],
                        ix.doc_lengths[:D0], ivf, ivf_lengths, ix.nbits)
    gpu = _open(npb, head)
    try:
        gpu.append_encoded(ix.codes[t0:], ix.residuals[t0:], ix.doc_lengths[D0:])
        assert all(_same(a, b) for a, b in zip(gpu.search_batch_params(qs, ps), _want(oracle, ix, qs, kws)))
        assert gpu.delete(list(range(0, ix.num_documents, 7))) > 0
        for q, p, r in zip(qs, ps, gpu.search_batch_params(qs, ps)):
            assert _same(r, gpu.search_batch([q], p)[0])
    finally:
        gpu.close()


ADDITIVE = ("n_cells", "n_candidates", "n_candidate_tokens", "n_exact_docs", "n_exact_tokens", "n_filter_docs",
            "n_filter_tokens", "n_recheck_docs", "n_exact_pairs", "n_a5_live_rows", "n_a5_dense_docs")


def test_tensor_core_probe_kept_next_to_wide_n(oracle, npb, small):
    """n = 8 queries share a call with n = 32 ones (more than the 8 threshold-first chunks at K = 256): they still run on
    the threshold-first table, and the per-query work adds up to that of the single-query calls"""
    docs, ix, qs, _ = small
    qs = qs[:8]
    kws = [_kw(dict(top_k=10, n_full_scores=256, n_ivf_probe=8 if i % 2 == 0 else 32)) for i in range(8)]
    ps = _params(npb, kws)
    gpu = _open(npb, ix)
    try:
        qs = [q[:32] for q in qs]
        gpu.search_batch([qs[i] for i in range(0, 8, 2)], ps[0])
        alone = gpu.last_work_counters()
        assert alone["n_k1_tc"] + alone["n_probe_threshold"] > 0
        res = gpu.search_batch_params(qs, ps)
        mixed = gpu.last_work_counters()
        assert mixed["n_k1_tc"] >= alone["n_k1_tc"] and mixed["n_probe_threshold"] >= alone["n_probe_threshold"]
        total = dict.fromkeys(ADDITIVE, 0)
        for q, p, r in zip(qs, ps, res):
            assert _same(r, gpu.search_batch([q], p)[0])
            one = gpu.last_work_counters()
            for f in ADDITIVE:
                total[f] += one[f]
        assert {f: mixed[f] for f in ADDITIVE} == total
        assert all(_same(a, b) for a, b in zip(res, _want(oracle, ix, qs, kws)))
    finally:
        gpu.close()


def test_flagged_query_leaves_the_others_alone(npb, small):
    docs, ix, qs, kws = small
    ps = _params(npb, kws[:8])
    qs = [q.copy() for q in qs[:8]]
    qs[2][0, 0] = np.nan                                  # non-finite tokens: the exact path
    gpu = _open(npb, ix)
    try:
        res = gpu.search_batch_params(qs, ps)
        for q, p, r in zip(qs, ps, res):
            assert _same(r, gpu.search_batch([q], p)[0])
    finally:
        gpu.close()


# -- in-process shard groups ---------------------------------------------------------------------------------------

def _shard(oracle, ix, d0, d1):
    t0, t1 = int(ix.doc_offsets[d0]), int(ix.doc_offsets[d1])
    codes, res, dl = ix.codes[t0:t1], ix.residuals[t0:t1], ix.doc_lengths[d0:d1]
    ivf, ivf_lengths = oracle.build_ivf(codes, dl, ix.num_centroids)
    return oracle.Index(ix.centroids, ix.bucket_weights, ix.bucket_cutoffs, codes, res, dl, ivf, ivf_lengths, ix.nbits)


def _group(npb, oracle, ix, bounds, host=()):
    return npb.ShardGroup([_open(npb, _shard(oracle, ix, bounds[r], bounds[r + 1]), device=0, doc_id_base=bounds[r],
                                 host_residuals=r in host) for r in range(len(bounds) - 1)])


@pytest.mark.parametrize("G", [2, 3, 8])
def test_group_equals_unsharded_and_oracle(oracle, npb, small, G):
    docs, ix, qs, kws = small
    D = ix.num_documents
    bounds = [g * D // G for g in range(G + 1)]
    if G == 3:
        bounds = [0, 1000, 1000, D]                       # an empty shard
    grp = _group(npb, oracle, ix, bounds, host=(1,) if G == 2 else ())
    ps = _params(npb, kws)
    subs = ([None, list(range(0, D, 2)), None, list(range(bounds[1] // 2, bounds[1]))] * 6)[:len(qs)]
    flat = _open(npb, ix)
    try:
        for s in (None, subs):
            res = grp.search_batch_params(qs, ps, s)
            for per_rank in grp.all_results:
                assert all(_same(a, b) for a, b in zip(per_rank, res))
            assert all(_same(a, b) for a, b in zip(res, flat.search_batch_params(qs, ps, s))), G
            assert all(_same(a, b) for a, b in zip(res, _want(oracle, ix, qs, kws, s))), G
    finally:
        grp.close()
        flat.close()


def test_group_ranks_with_different_params_refuse_together(oracle, npb, small):
    docs, ix, qs, kws = small
    D = ix.num_documents
    grp = _group(npb, oracle, ix, [0, D // 2, D])
    ps = _params(npb, kws)
    try:
        def call(r, s):
            mine = [npb.SearchParameters(**_kw(dict(top_k=10, n_full_scores=256, n_ivf_probe=8 + r)))] + ps[1:]
            try:
                s.search_batch_params(qs, mine)
                return None
            except npb.PlaidError as e:
                return e.status
        assert grp._collective(call) == [PB_ERR_INVALID] * 2
        res = grp.search_batch_params(qs, ps)
        assert all(_same(a, b) for a, b in zip(res, _want(oracle, ix, qs, kws)))
    finally:
        grp.close()


# -- argument errors ---------------------------------------------------------------------------------------------

def test_refusals_match_the_query_alone(npb, small):
    docs, ix, qs, kws = small
    gpu = _open(npb, ix)
    L = npb.load_library()
    base = [npb.SearchParameters(**_kw(dict(top_k=10, n_full_scores=256, n_ivf_probe=8))) for _ in range(4)]
    qs4 = [qs[0][:32], qs[1], qs[2][:64], qs[0][:32]]
    try:
        flat = np.ascontiguousarray(np.concatenate(qs4, 0), np.float32)
        qo = np.zeros(5, np.int64)
        qo[1:] = np.cumsum([len(q) for q in qs4])
        P = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)  # noqa: E731
        ids, sc, cn = np.zeros((4, 10), np.int64), np.zeros((4, 10), np.float32), np.zeros(4, np.int32)
        assert L.pb_search_batch_params(gpu._h, P(flat), P(qo), 4, None, None, None, None, P(ids), P(sc), P(cn),
                                        None) == PB_ERR_INVALID
        bad = [dict(n_ivf_probe=0), dict(top_k=10, n_full_scores=80000), dict(n_ivf_probe=192, centroid_batch_size=64)]
        for d in bad:
            b = npb.SearchParameters(**_kw(dict(dict(top_k=10, n_full_scores=256, n_ivf_probe=8), **d)))
            ps = base[:2] + [b] + base[3:]                 # the query of 64 tokens: 64 x 192 > 8192
            alone = L.pb_search_batch(gpu._h, P(np.ascontiguousarray(qs4[2], np.float32)),
                                      P(np.array([0, len(qs4[2])], np.int64)), 1, C.byref(b._c()), None, 0,
                                      P(ids), P(sc), P(cn))
            assert alone != 0, d
            arr = (type(b._c()) * 4)(*[p._c() for p in ps])
            st = L.pb_search_batch_params(gpu._h, P(flat), P(qo), 4, arr, None, None, None, P(ids), P(sc), P(cn), None)
            assert st == alone, d
            assert len(gpu.search_batch_params(qs4, base)) == 4
    finally:
        gpu.close()
