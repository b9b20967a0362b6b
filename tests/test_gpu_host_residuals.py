"""Host-tier handles (PB_OPEN_HOST_RESIDUALS): the packed residuals live in pinned host memory and each search stages the
kept docs' rows to the device (DESIGN.md 4j).  A host-tier handle must be indistinguishable from a resident one opened on
the same arrays -- ids, scores, counts and every work counter -- on every path of the exact stage, and both must equal
the CPU oracle bit for bit.  Also: decompression and exhaustive scores, the loaders, a shard group mixing both tiers,
memory_usage(), last_staging_stats(), and the mutations that refuse such handles."""
import os
import sys
import threading

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_gpu_shape_edges import _codec_index, _queries_from  # noqa: E402

pytestmark = pytest.mark.gpu

PER_SUB_BATCH = ("n_probe_threshold", "n_probe_list", "n_k1_tc", "n_k1_tc_redo")  # counted once per sub-batch


@pytest.fixture(scope="module")
def npb():
    import next_plaid_b200 as m
    m.build_library()
    if m.device_count() < 1:
        pytest.fail("GPU tests need an H100; the library has no CPU fallback")
    return m


def _open(npb, ix, host, **kw):
    return npb.MmapIndex.from_arrays(ix.centroids, ix.bucket_weights, ix.codes, ix.residuals, ix.doc_lengths, ix.ivf,
                                     ix.ivf_lengths, ix.nbits, host_residuals=host, **kw)


def _lengths(seed, D=1200):
    """20..60 tokens, a few docs spanning several 128-token tiles, one much longer than the rest"""
    rng = np.random.default_rng(seed)
    dl = rng.integers(20, 61, D)
    dl[[7, 300, 801]] = [260, 383, 515]
    dl[500] = 1800
    return dl


def _with_repeated_doc(oracle, ix, doc):
    """doc `doc` becomes one token repeated: every token ties for every maximum, so its pair list overflows"""
    codes, res = ix.codes.copy(), ix.residuals.copy()
    t0, t1 = int(ix.doc_offsets[doc]), int(ix.doc_offsets[doc + 1])
    codes[t0:t1] = codes[t0]
    res[t0:t1] = res[t0]
    ivf, lens = oracle.build_ivf(codes, ix.doc_lengths, ix.num_centroids)
    return oracle.Index(ix.centroids, ix.bucket_weights, ix.bucket_cutoffs, codes, res, ix.doc_lengths, ivf, lens, ix.nbits)


def _query_groups(oracle, ix, seed):
    """<= 32, 33..64 and > 64 tokens, each a batch of its own (the filter needs <= 64 tokens in the sub-batch)"""
    rng = np.random.default_rng(seed)
    D = ix.num_documents
    docs = [500, 7, 300] + rng.integers(0, D, 5).tolist()
    return [_queries_from(oracle, ix, docs, nqs, seed + i)
            for i, nqs in enumerate(([32, 8, 17, 32, 1, 24, 32, 5], [33, 64, 40, 64, 50, 64, 36, 48],
                                     [65, 100, 64, 128, 70, 96, 200, 80]))]


def _run(h, qs, params, subset=None):
    res = h.search_batch(qs, params, subset=subset)
    return [(r.passage_ids.tolist(), r.scores.tobytes()) for r in res], h.last_work_counters()


def _same_tiers(npb, oracle, ix, host, res, qs, kw, subset=None, oracle_check=True, skip=()):
    got, wg = _run(host, qs, npb.SearchParameters(**kw), subset)
    want, wr = _run(res, qs, npb.SearchParameters(**kw), subset)
    assert got == want, kw
    assert {k: v for k, v in wg.items() if k not in skip} == {k: v for k, v in wr.items() if k not in skip}, kw
    if oracle_check:
        for q, (ids, sc) in zip(qs, got):
            w = oracle.search_one(ix, q, oracle.SearchParameters(**kw), subset=subset)
            assert ids == w.passage_ids.tolist() and sc == w.scores.astype(np.float32).tobytes(), kw
    return wr


CASES = [(d, nb) for d in (64, 96, 128) for nb in (1, 2, 4, 8)] + [(32, 4), (256, 4), (32, 1), (256, 8)]


@pytest.mark.parametrize("dim,nbits", CASES)
def test_search_equals_resident_and_oracle(npb, oracle, dim, nbits):
    ix = _codec_index(oracle, 512, _lengths(dim + nbits), dim=dim, nbits=nbits, seed=dim * 10 + nbits)
    groups = _query_groups(oracle, ix, dim + nbits)
    host, res = _open(npb, ix, True), _open(npb, ix, False)
    subset = sorted(set(range(0, ix.num_documents, 2)) | {500, 7, 300})
    try:
        for qs in groups:
            for kw in (dict(top_k=10, n_ivf_probe=8, n_full_scores=256),
                       dict(top_k=10, n_ivf_probe=8, n_full_scores=256, centroid_batch_size=100),
                       dict(top_k=15, n_ivf_probe=6, n_full_scores=64),          # top_k near M = 16
                       dict(top_k=16, n_ivf_probe=6, n_full_scores=64, centroid_batch_size=100)):
                _same_tiers(npb, oracle, ix, host, res, qs, kw)
            _same_tiers(npb, oracle, ix, host, res, qs, dict(top_k=10, n_ivf_probe=8, n_full_scores=256,
                                                             centroid_batch_size=100), subset=subset)
            _same_tiers(npb, oracle, ix, host, res, qs, dict(top_k=10, n_ivf_probe=8, n_full_scores=256), subset=subset)
    finally:
        host.close()
        res.close()


@pytest.fixture(scope="module")
def pcorpus(oracle):
    """dim 128, 4 bits, with the long doc 500 made of one repeated token"""
    return _with_repeated_doc(oracle, _codec_index(oracle, 512, _lengths(5), seed=77), 500)


def _pair(npb, ix, **kw):
    return _open(npb, ix, True, **kw), _open(npb, ix, False, **kw)


def test_exact_stage_switches(npb, oracle, pcorpus):
    ix = pcorpus
    qs = _query_groups(oracle, ix, 9)[0]
    kw = dict(top_k=10, n_ivf_probe=8, n_full_scores=256)
    host, res = _pair(npb, ix)
    try:
        w = _same_tiers(npb, oracle, ix, host, res, qs, kw)
        assert w["n_pair_fallback_queries"] > 0 and w["n_exact_pairs"] > 0 and w["n_filter_docs"] > 0, w
        for setter, off in (("set_fast_exact", False), ("set_fast_approx", 0), ("set_scores_tc", False)):
            for h in (host, res):
                getattr(h, setter)(off)
            w = _same_tiers(npb, oracle, ix, host, res, qs, kw)
            for h in (host, res):
                getattr(h, setter)(not off if isinstance(off, bool) else 1)
        # traced search: every stage's contents
        rh, th = host.search_batch(qs, npb.SearchParameters(**kw), trace=True)
        rr, tr = res.search_batch(qs, npb.SearchParameters(**kw), trace=True)
        assert host.last_work_counters() == res.last_work_counters()
        for a, b in zip(rh, rr):
            assert a.passage_ids.tolist() == b.passage_ids.tolist() and np.array_equal(a.scores, b.scores)
        for f in ("cells", "candidates", "approx", "kept", "kept_exact"):
            for a, b in zip(getattr(th, f), getattr(tr, f)):
                assert np.array_equal(a, b), f
        # lanes: a batch of 32 queries in 2 slices
        big = qs * 4
        for h in (host, res):
            h.set_lanes(2)
        _same_tiers(npb, oracle, ix, host, res, big, kw)
    finally:
        host.close()
        res.close()


def test_filter_diag(npb, oracle, pcorpus, monkeypatch):
    monkeypatch.setenv("PB_FILTER_DIAG", "1")
    host, res = _pair(npb, pcorpus)
    try:
        for qs in _query_groups(oracle, pcorpus, 3)[:2]:
            w = _same_tiers(npb, oracle, pcorpus, host, res, qs, dict(top_k=10, n_ivf_probe=8, n_full_scores=256))
            assert w["filter_diag_pairs"] > 0 and w["filter_err_ratio_e6"] <= 10 ** 6, w
    finally:
        host.close()
        res.close()


def test_small_workspace_budget_splits_sub_batches(npb, oracle, pcorpus, monkeypatch):
    monkeypatch.setenv("PB_WS_BUDGET_MB", "8")
    host, res = _pair(npb, pcorpus)
    try:
        qs = _query_groups(oracle, pcorpus, 4)[0] * 3
        # the staging buffer counts in the budget of a host-tier handle only, so the tiers split differently
        kw = dict(top_k=10, n_ivf_probe=8, n_full_scores=256)
        _same_tiers(npb, oracle, pcorpus, host, res, qs, kw, skip=PER_SUB_BATCH)
        _, w = _run(host, qs, npb.SearchParameters(**kw))       # the counters are the calling thread's last search's
        assert w["n_k1_tc"] + w["n_probe_threshold"] + w["n_probe_list"] > 1, w
    finally:
        host.close()
        res.close()


def test_two_threads_on_one_handle(npb, oracle, pcorpus):
    host, res = _pair(npb, pcorpus)
    groups = _query_groups(oracle, pcorpus, 6)
    p = npb.SearchParameters(top_k=10, n_ivf_probe=8, n_full_scores=256)
    try:
        want = [_run(res, qs, p) for qs in groups[:2]]
        got, err = [None, None], [None, None]

        def run(i):
            try:
                for _ in range(5):
                    r = _run(host, groups[i], p)
                    assert r == want[i], i
                got[i] = r
            except Exception as e:      # noqa: BLE001 - re-raised below
                err[i] = e
        ths = [threading.Thread(target=run, args=(i,)) for i in range(2)]
        [t.start() for t in ths]
        [t.join() for t in ths]
        assert err == [None, None], err
        assert got == want
    finally:
        host.close()
        res.close()


def test_decompress_and_exhaustive_equal_resident(npb, oracle, pcorpus):
    host, res = _pair(npb, pcorpus)
    try:
        ids = [0, 7, 500, 300, 801, 1199, 5000, -1, 500]
        eh, lh = host.decompress_documents(ids)
        er, lr = res.decompress_documents(ids)
        assert np.array_equal(lh, lr) and np.array_equal(eh, er)
        assert np.array_equal(host.decompress_documents([500])[0], oracle.get_document_embeddings(pcorpus, 500))
        qs = _query_groups(oracle, pcorpus, 8)[0][:3]
        assert np.array_equal(host.exhaustive_scores(qs), res.exhaustive_scores(qs))
    finally:
        host.close()
        res.close()


def test_memory_usage(npb, pcorpus):
    host, res = _pair(npb, pcorpus)
    try:
        mh, mr = host.memory_usage(), res.memory_usage()
        b = max(pcorpus.num_embeddings * pcorpus.residuals.shape[1], 16)
        assert mh["host_bytes"] == pcorpus.residuals.size and mr["host_bytes"] == 0
        # the resident handle's residual array: b bytes plus DevBuf's 1/8 + 256 of headroom
        assert mr["device_bytes"] - mh["device_bytes"] == b + (b >> 3) + 256, (mr, mh)
    finally:
        host.close()
        res.close()


def test_staging_stats(npb, oracle, pcorpus):
    host, res = _pair(npb, pcorpus)
    packed = pcorpus.residuals.shape[1]
    qs = _query_groups(oracle, pcorpus, 12)[0]
    p = npb.SearchParameters(top_k=10, n_ivf_probe=8, n_full_scores=256)
    try:
        host.set_profiling(True)
        for on in (True, False):
            host.set_fast_exact(on)
            host.search_batch(qs, p)
            w, s = host.last_work_counters(), host.last_staging_stats()
            docs, toks = (w["n_filter_docs"], w["n_filter_tokens"]) if on else (w["n_exact_docs"], w["n_exact_tokens"])
            assert docs > 0 and s["docs"] == docs and s["bytes"] == toks * packed and s["ms"] > 0, (on, w, s)
        res.search_batch(qs, p)
        assert res.last_staging_stats() == dict(docs=0, bytes=0, ms=0.0)
    finally:
        host.close()
        res.close()


# ---------------------------------------------------------------------------------------------------------------------
# loaders, shard groups, refusals
# ---------------------------------------------------------------------------------------------------------------------

NBITS, K, DIM, CHUNK = 4, 256, 128, 200


@pytest.fixture(scope="module")
def dcorpus(oracle, tmp_path_factory):
    docs = oracle.synthetic_corpus(960, 40, dim=DIM, seed=91, ragged=True)
    ix = oracle.create_index(docs[:900], nbits=NBITS, seed=4, num_partitions=K)
    qs, _ = oracle.synthetic_queries(docs[:900], 8, nq=32, seed=19)
    path = str(tmp_path_factory.mktemp("ix"))
    oracle.write_index(ix, path, chunk_docs=CHUNK)
    return dict(docs=docs, ix=ix, qs=qs, path=path)


def _state(npb, h, qs):
    out = [h.num_documents(), h.num_embeddings()] + [a.tolist() for a in h.export_ivf()]
    emb, lens = h.decompress_documents([h_id for h_id in range(0, 900, 97)])
    out += [lens.tolist(), emb.tobytes()]
    for kw in (dict(top_k=10, n_ivf_probe=8, n_full_scores=256),
               dict(top_k=5, n_ivf_probe=4, n_full_scores=64, centroid_batch_size=100)):
        out.append(_run(h, qs, npb.SearchParameters(**kw)))
    return out


def test_loaders_equal_resident(npb, dcorpus):
    path, qs = dcorpus["path"], dcorpus["qs"]
    pairs = [(lambda host: npb.MmapIndex.load(path, host_residuals=host)),
             (lambda host: npb.MmapIndex.load_range(path, 150, 650, host_residuals=host)),
             (lambda host: npb.MmapIndex.load_shard(path, 2, 3, host_residuals=host))]
    for make in pairs:
        a, b = make(True), make(False)
        try:
            assert a.memory_usage()["host_bytes"] == a.num_embeddings() * DIM * NBITS // 8
            assert _state(npb, a, qs) == _state(npb, b, qs)
        finally:
            a.close()
            b.close()


def test_mixed_group_equals_load(npb, oracle, dcorpus):
    path, qs = dcorpus["path"], dcorpus["qs"]
    full = npb.MmapIndex.load(path)
    grp = npb.ShardGroup([npb.MmapIndex.load_shard(path, r, 3, host_residuals=r != 1) for r in range(3)])
    try:
        for kw in (dict(top_k=10, n_ivf_probe=8, n_full_scores=256, centroid_batch_size=100_000),
                   dict(top_k=10, n_ivf_probe=8, n_full_scores=256, centroid_batch_size=128)):
            got = grp.search_batch(qs, npb.SearchParameters(**kw))
            want = full.search_batch(qs, npb.SearchParameters(**kw))
            for per_rank in grp.all_results:
                for a, b in zip(per_rank, want):
                    assert a.passage_ids.tolist() == b.passage_ids.tolist() and np.array_equal(a.scores, b.scores)
            for q, g in zip(qs, got):
                w = oracle.search_one(dcorpus["ix"], q, oracle.SearchParameters(**kw))
                assert g.passage_ids.tolist() == w.passage_ids.tolist() and np.array_equal(g.scores, w.scores)
    finally:
        grp.close()
        full.close()


def test_mutations_are_refused(npb, oracle, dcorpus):
    path, qs, ix, docs = dcorpus["path"], dcorpus["qs"], dcorpus["ix"], dcorpus["docs"]
    h = npb.MmapIndex.load(path, host_residuals=True)
    codec = npb.ResidualCodec(NBITS, ix.centroids, ix.bucket_cutoffs)
    try:
        before = _state(npb, h, qs)
        enc_codes, enc_res = codec.encode_chunk(np.concatenate(docs[900:903], 0))
        dl = [len(d) for d in docs[900:903]]
        calls = [lambda: h.append(docs[900:903], codec), lambda: h.append_encoded(enc_codes, enc_res, dl),
                 lambda: h.reserve(2000, 100_000), lambda: h.delete([1, 2, 3])]
        for call in calls:
            with pytest.raises(npb.PlaidError) as e:
                call()
            assert e.value.status == 4
        assert _state(npb, h, qs) == before
    finally:
        h.close()
    grp = npb.ShardGroup([npb.MmapIndex.load_shard(path, r, 2, host_residuals=r == 0) for r in range(2)])
    try:
        p = npb.SearchParameters(top_k=10, n_ivf_probe=8, n_full_scores=256, centroid_batch_size=128)
        before = [(r.passage_ids.tolist(), r.scores.tobytes()) for r in grp.search_batch(qs, p)]
        enc_codes, enc_res = codec.encode_chunk(np.concatenate(docs[900:903], 0))
        dl = [len(d) for d in docs[900:903]]
        for call in (lambda: grp.delete([1, 500]), lambda: grp.append(docs[900:903], codec),
                     lambda: grp.append_encoded(enc_codes, enc_res, dl), lambda: grp.rebalance([0, 300, 900])):
            with pytest.raises(npb.PlaidError) as e:
                call()
            assert e.value.status == 4
        assert [s.num_documents() for s in grp.shards] == [int(b) for b in np.diff(npb.shard_bounds(path, 2))]
        assert [(r.passage_ids.tolist(), r.scores.tobytes()) for r in grp.search_batch(qs, p)] == before
    finally:
        grp.close()
        codec.close()


def test_host_and_adopt_together_are_invalid(npb, oracle):
    torch = pytest.importorskip("torch")
    ix = _codec_index(oracle, 64, np.full(20, 10), seed=3)
    dev = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in dict(
        cen=ix.centroids, w=ix.bucket_weights, codes=ix.codes, res=ix.residuals, dl=ix.doc_lengths).items()}
    with pytest.raises(npb.PlaidError) as e:
        npb.MmapIndex.from_device_pointers(ix.dim, ix.nbits, 64, 20, 200, dev["cen"].data_ptr(), dev["w"].data_ptr(),
                                           dev["codes"].data_ptr(), dev["res"].data_ptr(), dev["dl"].data_ptr(), None,
                                           None, adopt_residuals=True, host_residuals=True)
    assert e.value.status == 1
    # device arrays with the host tier alone: copied to pinned memory
    h = npb.MmapIndex.from_device_pointers(ix.dim, ix.nbits, 64, 20, 200, dev["cen"].data_ptr(), dev["w"].data_ptr(),
                                           dev["codes"].data_ptr(), dev["res"].data_ptr(), dev["dl"].data_ptr(), None,
                                           None, host_residuals=True)
    try:
        assert h.memory_usage()["host_bytes"] == ix.residuals.size
        assert np.array_equal(h.decompress_documents([3])[0], oracle.get_document_embeddings(ix, 3))
    finally:
        h.close()
        torch.cuda.synchronize()
