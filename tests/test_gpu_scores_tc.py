"""a2 on the tensor cores (k_scores16_tc) as the default path: its certified consumers (k_collect16_tc,
k_cells_unique/k_exact_rows/k_cells_thr, k_approx_recheck) must reproduce the exact fp32 path and the CPU oracle
bit for bit -- cells, candidates, approximate scores of the kept docs, ids and scores -- and hand flagged queries and
probe-list overflows back to the exact path (search.rs:345, :171-174; k_scores_tc.cuh for the error budget)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def npb():
    import next_plaid_b200 as m
    m.build_library()
    if m.device_count() < 1:
        pytest.fail("GPU tests need an H100; the library has no CPU fallback")
    return m


def _gpu_index(npb, ix, **kw):
    return npb.MmapIndex.from_arrays(ix.centroids, ix.bucket_weights, ix.codes, ix.residuals,
                                     ix.doc_lengths, ix.ivf, ix.ivf_lengths, ix.nbits, **kw)


@pytest.fixture(scope="module")
def corpus(oracle, npb):
    docs = oracle.synthetic_corpus(3000, 48, dim=128, seed=21, ragged=True)
    ix = oracle.create_index(docs, nbits=4, seed=4, num_partitions=2048)
    qs, src = oracle.synthetic_queries(docs, 16, nq=32, seed=9)
    return docs, ix, qs, _gpu_index(npb, ix)


def _same(a, w):
    return a.passage_ids.tolist() == w.passage_ids.tolist() and np.array_equal(a.scores, w.scores, equal_nan=True)


@pytest.mark.parametrize("kw", [
    dict(top_k=10, n_ivf_probe=8, n_full_scores=256),
    dict(top_k=10, n_ivf_probe=8, n_full_scores=256, centroid_batch_size=256),
    dict(top_k=100, n_ivf_probe=4, n_full_scores=4096, centroid_batch_size=512, centroid_score_threshold=0.3),
    dict(top_k=5, n_ivf_probe=32, n_full_scores=64, centroid_score_threshold=None),
    dict(top_k=20, n_ivf_probe=1, n_full_scores=128, centroid_batch_size=100),
])
def test_tensor_core_table_equals_exact_path_and_oracle(oracle, npb, corpus, kw, monkeypatch):
    docs, ix, qs, gpu = corpus
    pg, po = npb.SearchParameters(**kw), oracle.SearchParameters(**kw)
    monkeypatch.setenv("PB_K1_TC", "0")
    plain = _gpu_index(npb, ix)
    monkeypatch.delenv("PB_K1_TC")
    try:
        a = gpu.search_batch(qs, pg)
        wa = gpu.last_work_counters()
        b = plain.search_batch(qs, pg)
        wb = plain.last_work_counters()
        assert wa["n_k1_tc"] > 0 and wa["n_k1_tc_redo"] == 0, wa            # the tensor-core pass did the work
        assert wb["n_k1_tc"] == 0 and wb["n_probe_threshold"] > 0, wb
        for k in ("n_cells", "n_candidates", "n_filter_docs"):   # same cells, candidates, kept docs (the filter's
            # survivor count may differ: its error bound includes the table's code error)
            assert wa[k] == wb[k], (k, wa, wb)
        for q, x, y in zip(qs, a, b):
            w = oracle.search_one(ix, q, po)
            assert _same(x, w) and _same(y, w), kw
    finally:
        plain.close()


def test_code_difference_against_the_exact_table_is_within_the_certificate(oracle, npb, corpus, monkeypatch):
    docs, ix, qs, gpu = corpus
    monkeypatch.setenv("PB_K1_TC_DIAG", "1")
    diag = _gpu_index(npb, ix)
    monkeypatch.delenv("PB_K1_TC_DIAG")
    try:
        odd = [qs[0] * 37.0, qs[1] * 1e-5, qs[2][:9], qs[3]]
        pg = npb.SearchParameters(top_k=10, n_ivf_probe=8, n_full_scores=256)
        diag.search_batch(qs + odd, pg)
        w = diag.last_work_counters()
        assert w["n_k1_tc"] == 0                      # the diagnostic keeps the exact table in charge
        assert 0 <= w["k1_tc_max_code_diff"] <= 1, w  # E = 1 (k1_err_codes < 1 code)
    finally:
        diag.close()


def test_scaled_queries_stay_on_the_tensor_cores_and_flagged_ones_are_redone(oracle, npb, corpus):
    docs, ix, qs, gpu = corpus
    kw = dict(top_k=10, n_ivf_probe=8, n_full_scores=256, centroid_batch_size=256)
    pg, po = npb.SearchParameters(**kw), oracle.SearchParameters(**kw)
    scaled = [qs[0] * 1e-6, qs[1] * 4096.0, qs[2] * 3e-3, qs[3]]
    res = gpu.search_batch(scaled, pg)
    w = gpu.last_work_counters()
    assert w["n_k1_tc"] > 0 and w["n_k1_tc_redo"] == 0, w
    for q, r in zip(scaled, res):
        assert _same(r, oracle.search_one(ix, q, po))
    nan_q = qs[4].copy(); nan_q[3, 5] = np.nan
    inf_q = qs[5].copy(); inf_q[0, 0] = np.inf
    zero_tok = qs[6].copy(); zero_tok[5] = 0.0          # ties all K centroids -> the probe list overflows
    for batch in ([qs[7], nan_q], [inf_q, qs[8]], [zero_tok, qs[9]]):
        res = gpu.search_batch(batch, pg)
        w = gpu.last_work_counters()
        assert w["n_k1_tc_redo"] == 1 and w["n_k1_tc"] == 0, w          # handed back to the exact path, once
        for q, r in zip(batch, res):
            assert _same(r, oracle.search_one(ix, q, po))


def test_tensor_core_path_on_small_dims_and_bit_widths(oracle, npb):
    # the threshold-first probe needs at least n_ivf_probe chunks of 1024 centroids
    for dim, nbits, K, n_probe in ((64, 2, 2100, 2), (96, 4, 1024, 1), (128, 8, 2048, 2), (128, 1, 1500, 1)):
        docs = oracle.synthetic_corpus(500, 30, dim=dim, seed=3 + dim, ragged=True)
        ix = oracle.create_index(docs, nbits=nbits, seed=2, num_partitions=K)
        qs = [oracle.synthetic_queries(docs, 1, nq=n, seed=50 + n)[0][0] for n in (1, 5, 32, 40, 64)]
        gpu = _gpu_index(npb, ix)
        try:
            for cbs in (100_000, 97):
                kw = dict(top_k=7, n_ivf_probe=n_probe, n_full_scores=200, centroid_batch_size=cbs)
                res = gpu.search_batch(qs, npb.SearchParameters(**kw))
                w = gpu.last_work_counters()
                assert w["n_k1_tc"] > 0, (dim, w)
                for q, r in zip(qs, res):
                    assert _same(r, oracle.search_one(ix, q, oracle.SearchParameters(**kw))), (dim, nbits, cbs)
        finally:
            gpu.close()


def test_trace_of_the_tensor_core_pass_matches_the_oracle_stage_by_stage(oracle, npb, corpus):
    # the traced call itself runs the exact path (it reports every candidate's exact approximate score); here the
    # untraced tensor-core pass must keep exactly the docs the oracle's cut keeps, in its order
    docs, ix, qs, gpu = corpus
    kw = dict(top_k=64, n_ivf_probe=8, n_full_scores=256, centroid_batch_size=256)
    pg, po = npb.SearchParameters(**kw), oracle.SearchParameters(**kw)
    gpu.set_fast_exact(False)                      # every kept doc is scored exactly -> top_k = M exposes the cut
    try:
        res = gpu.search_batch(qs, pg)
        assert gpu.last_work_counters()["n_k1_tc"] > 0
        for q, r in zip(qs, res):
            assert _same(r, oracle.search_one(ix, q, po))
    finally:
        gpu.set_fast_exact(True)


def _codec_domain_index(oracle, K, D, T, dim=128, nbits=4, seed=5, docs_per_topic=64, pool=64):
    """A bench-style index drawn directly in the codec domain (random unit centroids, topic pools, random residual
    bytes): K can be 2^17 without running k-means on the CPU."""
    rng = np.random.default_rng(seed)
    cent = rng.standard_normal((K, dim), dtype=np.float32)
    cent /= np.linalg.norm(cent, axis=1, keepdims=True)
    n_topics = max(D // docs_per_topic, 4)
    pools = rng.integers(0, K, (n_topics, pool))
    topic = np.repeat(rng.integers(0, n_topics, D), T)
    u = rng.random(D * T)
    from_pool = pools[topic, np.minimum((u * u * pool).astype(np.int64), pool - 1)]
    sel = rng.random(D * T)
    codes = np.where(sel < 0.75, from_pool, rng.integers(0, K, D * T)).astype(np.int64)
    res = rng.integers(0, 256, (D * T, dim * nbits // 8), dtype=np.uint8)
    nb = 1 << nbits
    w = (0.05 * np.linspace(-1.8, 1.8, nb)).astype(np.float32)
    dl = np.full(D, T, np.int64)
    ivf, ivf_lengths = oracle.build_ivf(codes, dl, K)
    return oracle.Index(cent, w, None, codes, res, dl, ivf, ivf_lengths, nbits)


def test_scale_shaped_parity_at_k_2_17_with_the_default_slab(oracle, npb):
    # K = 2^17 > centroid_batch_size = 100 000 (the reference default): the batched variant with its real slab
    # boundary (100 000 + 31 072), 128 probe chunks, 64 queries, default parameters -- on the tensor-core table and
    # on the exact one
    ix = _codec_domain_index(oracle, 1 << 17, 20_000, 64)
    rng = np.random.default_rng(11)
    qs = []
    for d in rng.integers(0, ix.num_documents, 64):
        tok = oracle.get_document_embeddings(ix, int(d))[rng.integers(0, 64, 32)]
        nz = rng.standard_normal(tok.shape).astype(np.float32)
        q = tok + 0.15 * nz / np.linalg.norm(nz, axis=1, keepdims=True)
        qs.append((q / np.linalg.norm(q, axis=1, keepdims=True)).astype(np.float32))
    gpu = _gpu_index(npb, ix)
    try:
        for kw in (dict(top_k=100), dict(top_k=10, n_ivf_probe=16, n_full_scores=1024, centroid_score_threshold=0.35)):
            pg, po = npb.SearchParameters(**kw), oracle.SearchParameters(**kw)
            want = [oracle.search_one(ix, q, po) for q in qs]
            for tc in (True, False):
                gpu.set_scores_tc(tc)
                res = gpu.search_batch(qs, pg)
                w = gpu.last_work_counters()
                assert (w["n_k1_tc"] > 0) == tc and w["n_k1_tc_redo"] == 0 and w["n_probe_list"] == 0, (tc, w)
                assert w["n_candidates"] > 64 * 100                 # the searches are not trivially empty
                assert sum(_same(r, x) for r, x in zip(res, want)) == 64, (kw, tc)
    finally:
        gpu.set_scores_tc(True)
        gpu.close()
