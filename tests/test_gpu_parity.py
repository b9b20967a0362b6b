"""GPU parity tests proper: every stage of the CUDA path, called through the C-ABI, against the CPU
oracle on the same seeded inputs.  Bar: bit-exact for ids/indices AND for fp32 values, because both
sides use the same pinned accumulation order (DESIGN.md "Numerics"); the 1e-4 tolerance of the
north star is the bound against *other* sgemm orders and is checked separately against float64."""
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
    ix = oracle.create_index(docs, nbits=4, seed=4, num_partitions=512)
    qs, src = oracle.synthetic_queries(docs, 12, nq=32, seed=9)
    return docs, ix, qs, src, _gpu_index(npb, ix)


def _params(npb, oracle, **kw):
    return npb.SearchParameters(**kw), oracle.SearchParameters(**kw)


def test_accessors(corpus):
    docs, ix, qs, src, gpu = corpus
    assert gpu.num_documents() == ix.num_documents
    assert gpu.num_embeddings() == ix.num_embeddings
    assert gpu.num_partitions() == ix.num_centroids
    assert gpu.embedding_dim() == ix.dim and gpu.nbits() == 4
    assert abs(gpu.avg_doclen() - ix.num_embeddings / ix.num_documents) < 1e-9


def test_stage1_centroid_scores_bit_exact(oracle, corpus):
    docs, ix, qs, src, gpu = corpus
    q = np.concatenate(qs[:3], 0)
    S = gpu.centroid_scores(q)
    want = oracle.centroid_scores(q, ix.centroids)
    assert np.array_equal(S, want)
    assert np.abs(S - q.astype(np.float64) @ ix.centroids.astype(np.float64).T).max() < 1e-5


def test_stage2_decompress_bit_exact(oracle, corpus):
    docs, ix, qs, src, gpu = corpus
    ids = [0, 7, 2999, 1234, 7]
    emb, lens = gpu.decompress_documents(ids)
    want = np.concatenate([oracle.get_document_embeddings(ix, d) for d in ids], 0)
    assert lens.tolist() == [int(ix.doc_lengths[d]) for d in ids]
    assert np.array_equal(emb, want)
    assert np.allclose(np.linalg.norm(emb, axis=1), 1.0, atol=1e-6)
    # unknown ids contribute length 0 (index.rs:1202-1204)
    emb2, lens2 = gpu.decompress_documents([5, 10 ** 9])
    assert lens2.tolist() == [int(ix.doc_lengths[5]), 0]
    assert np.array_equal(emb2, oracle.get_document_embeddings(ix, 5))


def test_stage3_maxsim_bit_exact(oracle, npb, corpus):
    docs, ix, qs, src, gpu = corpus
    dd = [oracle.get_document_embeddings(ix, d) for d in (1, 50, 51, 700, 2998)]
    got = npb.maxsim_scores(qs[0], dd)
    want = np.array([oracle.maxsim_score(qs[0], d) for d in dd], np.float32)
    assert np.array_equal(got, want)
    # north-star tolerance against a different accumulation order (float64 sgemm)
    ref64 = np.array([(qs[0].astype(np.float64) @ d.astype(np.float64).T).max(1).sum() for d in dd])
    assert np.abs(got - ref64).max() < 1e-4


def test_maxsim_kats_on_gpu(npb):
    # maxsim.rs:393-413 (1.7) and :498-507 (NaN row entries -> 8.0): same KATs that pin the oracle
    q = np.zeros((2, 32), np.float32); q[0, 0] = 1; q[1, 1] = 1
    d = np.zeros((3, 32), np.float32); d[0, :2] = [0.5, 0.5]; d[1, :2] = [0.8, 0.2]; d[2, 1:3] = [0.9, 0.1]
    assert abs(npb.maxsim_scores(q, [d])[0] - 1.7) < 1e-5
    q2 = np.zeros((16, 32), np.float32); q2[:, 0] = 1
    d2 = np.zeros((16, 32), np.float32); d2[:, 0] = 0.5; d2[15, 0] = np.nan
    assert abs(npb.maxsim_scores(q2, [d2])[0] - 8.0) < 1e-5


@pytest.mark.parametrize("cbs,thr", [(100_000, 0.4), (100_000, None), (128, 0.4), (128, None), (0, 0.45)])
def test_search_stages_and_results_bit_exact(oracle, npb, corpus, cbs, thr):
    docs, ix, qs, src, gpu = corpus
    pg, po = _params(npb, oracle, top_k=10, n_ivf_probe=8, n_full_scores=256,
                     centroid_batch_size=cbs, centroid_score_threshold=thr)
    res, tr = gpu.search_batch(qs, pg, trace=True)
    for i, q in enumerate(qs):
        want, wt = oracle.search_one(ix, q, po, trace=True)
        assert tr.cells[i].tolist() == wt.cells.tolist(), f"cells q{i}"
        assert tr.candidates[i].tolist() == wt.candidates.tolist(), f"candidates q{i}"
        assert np.array_equal(tr.approx[i], wt.approx), f"approx q{i}"
        assert tr.kept[i].tolist() == wt.kept.tolist(), f"kept q{i}"
        assert np.array_equal(tr.kept_exact[i], wt.kept_exact), f"exact q{i}"
        assert res[i].query_id == i
        assert res[i].passage_ids.tolist() == want.passage_ids.tolist()
        assert np.array_equal(res[i].scores, want.scores)


def test_search_single_equals_batch(oracle, npb, corpus):
    docs, ix, qs, src, gpu = corpus
    pg, po = _params(npb, oracle, top_k=5, n_full_scores=128)
    r = gpu.search(qs[3], pg)
    w = oracle.search_one(ix, qs[3], po)
    assert r.query_id == 0 and r.passage_ids.tolist() == w.passage_ids.tolist()
    assert np.array_equal(r.scores, w.scores)


def test_ragged_query_lengths_and_small_dims(oracle, npb):
    for dim, nbits in ((64, 2), (96, 4), (32, 8), (256, 4), (128, 1)):
        docs = oracle.synthetic_corpus(400, 20, dim=dim, seed=dim, ragged=True)
        ix = oracle.create_index(docs, nbits=nbits, seed=1, num_partitions=64)
        gpu = _gpu_index(npb, ix)
        qs = []
        for nq, seed in ((1, 1), (5, 2), (32, 3), (33, 4), (48, 5), (70, 6), (129, 7), (257, 8)):
            qs.append(oracle.synthetic_queries(docs, 1, nq=nq, seed=seed)[0][0])
        qs.append(np.zeros((0, dim), np.float32))       # empty query -> empty result
        pg, po = _params(npb, oracle, top_k=7, n_ivf_probe=4, n_full_scores=64, centroid_score_threshold=0.3)
        res = gpu.search_batch(qs, pg)
        for q, r in zip(qs, res):
            w = oracle.search_one(ix, q, po)
            assert r.passage_ids.tolist() == w.passage_ids.tolist(), (dim, nbits, q.shape)
            assert np.array_equal(r.scores, w.scores), (dim, nbits, q.shape)
        emb, _ = gpu.decompress_documents([0, 1, 399])
        want = np.concatenate([oracle.get_document_embeddings(ix, d) for d in (0, 1, 399)], 0)
        assert np.array_equal(emb, want), (dim, nbits)
        gpu.close()


def test_subset_prefilter(oracle, npb, corpus):
    # search.rs:350-382 (dense: eligible centroids + n_ivf_probe scaling), :434-437, :542-545
    docs, ix, qs, src, gpu = corpus
    rng = np.random.default_rng(0)
    subsets = [list(range(0, 3000, 2)),                      # 50% -> scaled probe 16
               list(range(0, 3000, 20)),                     # 5% -> scaled probe 160 (row-wise radix select)
               sorted(rng.choice(3000, 40, replace=False)),  # tiny -> every eligible centroid
               [5, 5, 17, 10 ** 7, -3],                      # duplicates and out-of-range ids
               []]
    for cbs in (100_000, 128):
        for ss in subsets:
            pg, po = _params(npb, oracle, top_k=10, n_ivf_probe=8, n_full_scores=256, centroid_batch_size=cbs)
            res = gpu.search_batch(qs[:4], pg, subset=ss)
            for q, r in zip(qs[:4], res):
                w = oracle.search_one(ix, q, po, subset=ss)
                assert r.passage_ids.tolist() == w.passage_ids.tolist(), (cbs, len(ss))
                assert np.array_equal(r.scores, w.scores)
                assert set(r.passage_ids.tolist()) <= set(ss)


def test_edge_cases(oracle, npb, corpus):
    docs, ix, qs, src, gpu = corpus
    # everything pruned by the threshold -> empty (search.rs:439-445)
    pg, po = _params(npb, oracle, top_k=10, centroid_score_threshold=2.0)
    assert all(len(r.passage_ids) == 0 for r in gpu.search_batch(qs[:2], pg))
    # top_k larger than what survives the cut: take(n_full_scores) caps first (search.rs:461-469)
    pg, po = _params(npb, oracle, top_k=500, n_full_scores=64, centroid_score_threshold=None)
    for q, r in zip(qs[:2], gpu.search_batch(qs[:2], pg)):
        w = oracle.search_one(ix, q, po)
        assert len(r.passage_ids) == len(w.passage_ids) <= 64
        assert r.passage_ids.tolist() == w.passage_ids.tolist()
    # n_ivf_probe = 1, 64 and (dense variant only) beyond the streaming lists
    for n in (1, 64, 100, 600):
        pg, po = _params(npb, oracle, top_k=10, n_ivf_probe=n, n_full_scores=128)
        for q, r in zip(qs[:3], gpu.search_batch(qs[:3], pg)):
            w = oracle.search_one(ix, q, po)
            assert r.passage_ids.tolist() == w.passage_ids.tolist()
    # zero queries
    assert gpu.search_batch([], npb.SearchParameters()) == []
    # bad arguments
    with pytest.raises(npb.PlaidError):
        gpu.search_batch(qs[:1], npb.SearchParameters(n_ivf_probe=0))
    with pytest.raises(npb.PlaidError):
        gpu.search_batch([np.zeros((4, 64), np.float32)], npb.SearchParameters())


def test_index_directory_load(oracle, npb, corpus, tmp_path):
    # the GPU loader reads the reference's on-disk format (index.rs:1026-1139) chunk by chunk
    docs, ix, qs, src, gpu = corpus
    path = str(tmp_path / "idx")
    oracle.write_index(ix, path, chunk_docs=700, merged=True)
    g2 = npb.MmapIndex.load(path)
    assert g2.num_documents() == ix.num_documents and g2.num_embeddings() == ix.num_embeddings
    pg, po = _params(npb, oracle, top_k=10, n_full_scores=256)
    for q, r in zip(qs[:4], g2.search_batch(qs[:4], pg)):
        w = oracle.search_one(ix, q, po)
        assert r.passage_ids.tolist() == w.passage_ids.tolist() and np.array_equal(r.scores, w.scores)
    g2.close()


def test_exhaustive_scores_and_recall_property(oracle, npb, corpus):
    docs, ix, qs, src, gpu = corpus
    ex = gpu.exhaustive_scores(qs[:3])
    for i in range(3):
        want = oracle.exhaustive_scores(ix, qs[i])
        assert np.array_equal(ex[i], want)
    # size-independent property: PLAID results are a subset of the corpus with exact scores equal to
    # the exhaustive score of the same doc, and the planted source doc ranks first
    pg = npb.SearchParameters(top_k=10, n_full_scores=512)
    for i, r in enumerate(gpu.search_batch(qs[:3], pg)):
        assert np.array_equal(r.scores, ex[i][r.passage_ids])
        assert r.passage_ids[0] == src[i]


def test_concurrent_searches_share_one_handle(oracle, npb, corpus):
    # state.rs:24-47: one index, many worker threads
    import threading
    docs, ix, qs, src, gpu = corpus
    pg, po = _params(npb, oracle, top_k=10, n_full_scores=256)
    want = [oracle.search_one(ix, q, po).passage_ids.tolist() for q in qs]
    errs = []

    def work(k):
        try:
            for _ in range(5):
                res = gpu.search_batch(qs[k::4], pg)
                for r, w in zip(res, want[k::4]):
                    assert r.passage_ids.tolist() == w
        except Exception as e:  # noqa
            errs.append(e)
    ts = [threading.Thread(target=work, args=(k,)) for k in range(4)]
    [t.start() for t in ts]
    [t.join() for t in ts]
    assert not errs, errs


def test_two_pass_approx_equals_single_pass_and_oracle(oracle, npb, corpus):
    # DESIGN.md "a5 two-pass": the 16-bit first pass only prunes docs that provably cannot make the cut
    docs, ix, qs, src, gpu = corpus
    for kw in (dict(top_k=10, n_full_scores=64), dict(top_k=100, n_full_scores=400),
               dict(top_k=10, n_full_scores=256, centroid_score_threshold=None, n_ivf_probe=32),
               dict(top_k=3, n_full_scores=8, centroid_batch_size=128)):
        pg, po = _params(npb, oracle, **kw)
        gpu.set_fast_approx(1)
        fast = gpu.search_batch(qs, pg)
        gpu.set_fast_approx(0)
        slow = gpu.search_batch(qs, pg)
        gpu.set_scores_tc(False)                # two-pass on the exact fp32 table (the tensor-core table's fallback)
        gpu.set_fast_approx(1)
        mid = gpu.search_batch(qs, pg)
        gpu.set_scores_tc(True)
        for q, f, s, c in zip(qs, fast, slow, mid):
            w = oracle.search_one(ix, q, po)
            assert f.passage_ids.tolist() == s.passage_ids.tolist() == c.passage_ids.tolist() == w.passage_ids.tolist(), kw
            assert np.array_equal(f.scores, w.scores) and np.array_equal(s.scores, w.scores) and np.array_equal(c.scores, w.scores)


def test_two_pass_approx_with_massive_ties_and_odd_ranges(oracle, npb):
    # many byte-identical docs -> identical approximate scores straddling the cut: the certified band
    # must keep all of them so the doc-id tie-break of the stable sort (search.rs:460) decides
    base = oracle.synthetic_corpus(40, 24, dim=64, seed=5)
    docs = [base[i % 4] if i % 3 else base[i % 40] for i in range(900)]
    ix = oracle.create_index(docs, nbits=4, seed=2, num_partitions=64)
    qs, _ = oracle.synthetic_queries(docs, 6, nq=16, seed=4)
    qs.append(qs[0] * 7.5)                      # non-unit query norms scale the 16-bit range
    qs.append(qs[1] * 1e-3)
    bad = qs[2].copy(); bad[3, 5] = np.inf      # non-finite query -> flagged, single exact pass
    qs.append(bad)
    gpu = _gpu_index(npb, ix)
    for kw in (dict(top_k=10, n_full_scores=64, centroid_score_threshold=None),
               dict(top_k=50, n_full_scores=100, centroid_score_threshold=None, n_ivf_probe=16),
               dict(top_k=5, n_full_scores=20, centroid_score_threshold=0.2)):
        pg, po = _params(npb, oracle, **kw)
        for mode in (1, 0):                     # certified paths on the tensor-core table / on the exact table
            gpu.set_scores_tc(bool(mode))
            for q, r in zip(qs, gpu.search_batch(qs, pg)):
                w = oracle.search_one(ix, q, po)
                assert r.passage_ids.tolist() == w.passage_ids.tolist(), (kw, mode)
                assert np.array_equal(r.scores, w.scores, equal_nan=True), (kw, mode)
    gpu.close()


def test_deep_cut_and_large_top_k(oracle, npb, corpus):
    # BASELINE config E shape: recall@1000 -> top_k = 1000, n_full_scores = 16384 -> 4096 docs exact-scored
    docs, ix, qs, src, gpu = corpus
    for kw in (dict(top_k=1000, n_full_scores=16384, centroid_score_threshold=None, n_ivf_probe=16),
               dict(top_k=1000, n_full_scores=2048, centroid_score_threshold=None),
               dict(top_k=64, n_full_scores=8192, n_ivf_probe=32, centroid_batch_size=128)):
        pg, po = _params(npb, oracle, **kw)
        for q, r in zip(qs[:4], gpu.search_batch(qs[:4], pg)):
            w = oracle.search_one(ix, q, po)
            assert r.passage_ids.tolist() == w.passage_ids.tolist(), kw
            assert np.array_equal(r.scores, w.scores), kw
    with pytest.raises(npb.PlaidError):      # stated limit: > 16384 docs to exact-score
        gpu.search_batch(qs[:1], npb.SearchParameters(top_k=10, n_full_scores=4 * 16385))


def test_randomized_search_parity(oracle, npb):
    """Seeded sweep over index shapes and search parameters: ids and scores bit-identical to the oracle."""
    rng = np.random.default_rng(20260923)
    checked = 0
    for case in range(24):
        dim = int(rng.choice([32, 64, 96, 128]))
        nbits = int(rng.choice([1, 2, 4, 8]))
        n_docs = int(rng.integers(150, 900))
        doclen = int(rng.integers(3, 50))
        K = int(rng.choice([32, 64, 128, 256]))
        docs = oracle.synthetic_corpus(n_docs, doclen, dim=dim, seed=1000 + case, ragged=bool(rng.integers(2)))
        ix = oracle.create_index(docs, nbits=nbits, seed=case, num_partitions=K, kmeans_niters=2)
        gpu = _gpu_index(npb, ix)
        nqs = [int(rng.integers(1, 49)) for _ in range(3)]
        qs = [oracle.synthetic_queries(docs, 1, nq=nq, seed=case * 7 + j)[0][0] for j, nq in enumerate(nqs)]
        for trial in range(2):
            kw = dict(top_k=int(rng.integers(1, 200)), n_ivf_probe=int(rng.integers(1, 33)),
                      n_full_scores=int(rng.integers(16, 2048)),
                      centroid_batch_size=int(rng.choice([0, max(ix.num_centroids // 3, 1), 100_000])),
                      centroid_score_threshold=None if rng.integers(3) == 0 else float(rng.uniform(0.2, 0.5)))
            subset = None
            if rng.integers(4) == 0:
                subset = sorted(rng.choice(n_docs, int(rng.integers(1, n_docs)), replace=False).tolist())
            pg, po = _params(npb, oracle, **kw)
            try:
                res = gpu.search_batch(qs, pg, subset=subset)
            except npb.PlaidError as e:
                assert e.status == 4, e          # only the stated limits may refuse (PB_ERR_UNSUPPORTED)
                continue
            for q, r in zip(qs, res):
                w = oracle.search_one(ix, q, po, subset=subset)
                assert r.passage_ids.tolist() == w.passage_ids.tolist(), (case, dim, nbits, kw, subset is not None)
                assert np.array_equal(r.scores, w.scores), (case, dim, nbits, kw)
                checked += 1
        gpu.close()
    assert checked >= 100


def test_tensor_core_filter_equals_full_exact_stage(oracle, npb, corpus):
    # DESIGN.md "a7' certified filter": the fp16 tensor-core estimate may only drop docs that provably cannot reach
    # the top_k, so results with the filter on / off / the oracle's are the same bits
    docs, ix, qs, src, gpu = corpus
    for kw in (dict(top_k=5, n_full_scores=2048), dict(top_k=100, n_full_scores=4096, centroid_score_threshold=None),
               dict(top_k=1, n_full_scores=512, n_ivf_probe=16), dict(top_k=30, n_full_scores=400, centroid_batch_size=128)):
        pg, po = _params(npb, oracle, **kw)
        gpu.set_fast_exact(True)
        on = gpu.search_batch(qs, pg)
        work = gpu.last_work_counters()
        gpu.set_fast_exact(False)
        off = gpu.search_batch(qs, pg)
        work_off = gpu.last_work_counters()
        gpu.set_fast_exact(True)
        assert work["n_filter_docs"] > 0 and work_off["n_filter_docs"] == 0, kw
        assert work["n_filter_docs"] == work_off["n_exact_docs"], kw
        assert 0 < work["n_exact_docs"] < work["n_filter_docs"], (kw, work)   # it did filter
        for q, a, b in zip(qs, on, off):
            w = oracle.search_one(ix, q, po)
            assert a.passage_ids.tolist() == b.passage_ids.tolist() == w.passage_ids.tolist(), kw
            assert np.array_equal(a.scores, w.scores) and np.array_equal(b.scores, w.scores), kw


def test_tensor_core_filter_with_ties_scaled_and_nonfinite_queries(oracle, npb):
    # byte-identical docs tie exactly at the top_k boundary: all of them must survive the filter so that the
    # approximate-rank tie-break (search.rs:496-515, stable sort) decides; odd query norms scale the bound
    base = oracle.synthetic_corpus(40, 40, dim=128, seed=15)
    docs = [base[i % 5] if i % 3 else base[i % 40] for i in range(700)]
    docs[17] = docs[17][:0]                      # a doc without tokens scores 0
    ix = oracle.create_index(docs, nbits=2, seed=3, num_partitions=64)
    qs, _ = oracle.synthetic_queries(docs, 5, nq=24, seed=8)
    qs.append(qs[0] * 9.0)
    qs.append(qs[1] * 1e-4)
    bad = qs[2].copy(); bad[1, 7] = np.nan
    qs.append(bad)
    gpu = _gpu_index(npb, ix)
    for kw in (dict(top_k=10, n_full_scores=1024, centroid_score_threshold=None, n_ivf_probe=16),
               dict(top_k=3, n_full_scores=2800, centroid_score_threshold=None, n_ivf_probe=64),
               dict(top_k=60, n_full_scores=600, centroid_score_threshold=0.2)):
        pg, po = _params(npb, oracle, **kw)
        for on in (True, False):
            gpu.set_fast_exact(on)
            for q, r in zip(qs, gpu.search_batch(qs, pg)):
                w = oracle.search_one(ix, q, po)
                assert r.passage_ids.tolist() == w.passage_ids.tolist(), (kw, on)
                assert np.array_equal(r.scores, w.scores, equal_nan=True), (kw, on)
    gpu.close()


def test_probe_threshold_path_and_its_fallbacks(oracle, npb, corpus, monkeypatch):
    # a3 on the 16-bit table (k_chunkmax16 / k_collect16): same cells as the per-lane list scan and the oracle, including
    # the device-side fallback (a zero query token ties every centroid -> more than `cap` entries reach the threshold)
    docs, ix, qs, src, gpu = corpus
    zero_tok = qs[1].copy(); zero_tok[5] = 0.0
    dup = qs[2].copy(); dup[7] = dup[3]
    batch = [qs[0], zero_tok, dup, qs[3] * 3.0, qs[4][:9]]
    monkeypatch.setenv("PB_PROBE16", "0")
    plain = _gpu_index(npb, ix)
    monkeypatch.delenv("PB_PROBE16")
    for kw in (dict(top_k=10, n_ivf_probe=8, n_full_scores=256), dict(top_k=10, n_ivf_probe=1, n_full_scores=64),
               dict(top_k=20, n_ivf_probe=32, n_full_scores=512, centroid_score_threshold=None),
               dict(top_k=10, n_ivf_probe=8, n_full_scores=256, centroid_batch_size=128, centroid_score_threshold=0.3)):
        pg, po = _params(npb, oracle, **kw)
        for sub in (batch, [batch[0], batch[3]]):          # with and without the query that forces the fallback
            a = gpu.search_batch(sub, pg)
            b = plain.search_batch(sub, pg)
            for q, x, y in zip(sub, a, b):
                w = oracle.search_one(ix, q, po)
                assert x.passage_ids.tolist() == y.passage_ids.tolist() == w.passage_ids.tolist(), kw
                assert np.array_equal(x.scores, w.scores) and np.array_equal(y.scores, w.scores), kw
    plain.close()



@pytest.mark.parametrize("nq", [33, 48, 64])
def test_long_queries_keep_the_fast_paths(oracle, npb, corpus, nq):
    # default_query_length() = 48 in the reference's ONNX encoder (next-plaid-onnx/src/lib.rs:628-630): the tensor-core
    # filter (N = 64 UMMA) and the threshold-first probe (QS/8 = 5, 6, 8 lanes per row) must stay engaged past 32 tokens
    docs, ix, qs, src, gpu = corpus
    ql, _ = oracle.synthetic_queries(docs, 6, nq=nq, seed=100 + nq)
    for kw in (dict(top_k=5, n_full_scores=2048), dict(top_k=20, n_full_scores=1024, centroid_batch_size=128),
               dict(top_k=10, n_full_scores=512, n_ivf_probe=16, centroid_score_threshold=None)):
        pg, po = _params(npb, oracle, **kw)
        res = gpu.search_batch(ql, pg)
        work = gpu.last_work_counters()
        assert work["n_filter_docs"] > 0 and work["n_exact_docs"] < work["n_filter_docs"], (kw, work)
        assert work["n_probe_list"] == 0 and work["n_probe_threshold"] + work["n_k1_tc"] > 0, (kw, work)
        for q, r in zip(ql, res):
            w = oracle.search_one(ix, q, po)
            assert r.passage_ids.tolist() == w.passage_ids.tolist(), (kw, nq)
            assert np.array_equal(r.scores, w.scores), (kw, nq)


@pytest.mark.parametrize("env", [{"PB_FAST_APPROX": "0"}, {"PB_K1_TC": "0"}, {"PB_PAIR_EXACT": "0"}, {},
                                 {"PB_FAST_APPROX": "0", "PB_PAIR_EXACT": "0"}])
def test_the_filter_on_the_tensor_core_table_the_exact_table_and_no_table(oracle, npb, corpus, monkeypatch, env):
    # the filter (k_maxsim_tc: centroid score from the 16-bit table + residual part on the tensor cores) on the
    # tensor-core table (default), on the exact table (PB_K1_TC=0) and without a score table (PB_FAST_APPROX=0), where
    # a2 writes the exact table's 16-bit codes for it; the exact stage on the (token, q) pairs inside the certified
    # band (default) or on every token of the survivors (PB_PAIR_EXACT=0)
    docs, ix, qs, src, _ = corpus
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    gpu = _gpu_index(npb, ix)
    for k in env:
        monkeypatch.delenv(k)
    try:
        long_q, _ = oracle.synthetic_queries(docs, 3, nq=48, seed=77)
        batch = qs[:6] + long_q + [qs[6] * 5.0, qs[7][:3]]
        for kw in (dict(top_k=5, n_full_scores=2048), dict(top_k=40, n_full_scores=400, centroid_batch_size=128)):
            pg, po = _params(npb, oracle, **kw)
            res = gpu.search_batch(batch, pg)
            w = gpu.last_work_counters()
            assert 0 < w["n_exact_docs"] < w["n_filter_docs"], (env, kw, w)
            pair_form = "PB_PAIR_EXACT" not in env
            assert (w["n_exact_pairs"] > 0) == pair_form, (env, kw, w)
            if pair_form:   # a little over one pair per (survivor, query token), never every token
                assert w["n_pair_fallback_queries"] == 0, (env, kw, w)
                assert w["n_exact_pairs"] < 0.25 * 48 * w["n_exact_tokens"], (env, kw, w)
            for q, r in zip(batch, res):
                want = oracle.search_one(ix, q, po)
                assert r.passage_ids.tolist() == want.passage_ids.tolist(), (env, kw)
                assert np.array_equal(r.scores, want.scores), (env, kw)
    finally:
        gpu.close()


def test_pair_lists_that_overflow_fall_back_to_the_token_kernel(oracle, npb):
    # docs made of one repeated token: every token of a doc holds every per-token maximum, so the (token, q) list of
    # the exact stage grows to doclen * nq per survivor and overflows -- those queries are scored by k_exact instead;
    # a second corpus mixes repeated-token docs with ordinary ones (several pairs per (doc, q), no overflow)
    rng = np.random.default_rng(5)
    base = oracle.synthetic_corpus(300, 30, dim=128, seed=23)
    rep = [np.repeat(d[:1], 200, axis=0) for d in base]
    mixed = [np.repeat(d[:6], 2, axis=0) if i % 2 else d for i, d in enumerate(base)]
    for docs, expect_overflow in ((rep, True), (mixed, False)):
        ix = oracle.create_index(docs, nbits=4, seed=2, num_partitions=64)
        qs, _ = oracle.synthetic_queries(docs, 6, nq=32, seed=9)
        gpu = _gpu_index(npb, ix)
        try:
            for kw in (dict(top_k=20, n_full_scores=256, centroid_score_threshold=None, n_ivf_probe=16),
                       dict(top_k=5, n_full_scores=1024, centroid_score_threshold=None, n_ivf_probe=32)):
                pg, po = _params(npb, oracle, **kw)
                res = gpu.search_batch(qs, pg)
                w = gpu.last_work_counters()
                if w["n_filter_docs"] > 0:
                    assert (w["n_pair_fallback_queries"] > 0) == expect_overflow, (kw, w)
                for q, r in zip(qs, res):
                    want = oracle.search_one(ix, q, po)
                    assert r.passage_ids.tolist() == want.passage_ids.tolist(), (kw, expect_overflow)
                    assert np.array_equal(r.scores, want.scores), (kw, expect_overflow)
        finally:
            gpu.close()


def test_fast_plaid_directory_serves_the_same_results(oracle, npb, corpus, tmp_path):
    # mmap.rs:1757-1811: a fast-plaid directory (f16 floats, i64 ivf_lengths) is equivalent to its f32 widening; the
    # loader reads it as it is and the searches equal the oracle's on the widened index
    docs, ix, qs, src, _ = corpus
    path = str(tmp_path / "fp")
    oracle.write_index(ix, path, chunk_docs=1000)
    import os
    for name in ("centroids.npy", "bucket_weights.npy", "bucket_cutoffs.npy"):
        p = os.path.join(path, name)
        if os.path.exists(p):
            np.save(p, np.load(p).astype(np.float16))
    np.save(os.path.join(path, "ivf_lengths.npy"), np.load(os.path.join(path, "ivf_lengths.npy")).astype(np.int64))
    wide = oracle.Index(ix.centroids.astype(np.float16).astype(np.float32),
                        ix.bucket_weights.astype(np.float16).astype(np.float32), None, ix.codes, ix.residuals,
                        ix.doc_lengths, ix.ivf, ix.ivf_lengths, ix.nbits)
    gpu = npb.MmapIndex.load(path)
    try:
        pg, po = _params(npb, oracle, top_k=10, n_ivf_probe=8, n_full_scores=256)
        for q, r in zip(qs[:6], gpu.search_batch(qs[:6], pg)):
            w = oracle.search_one(wide, q, po)
            assert r.passage_ids.tolist() == w.passage_ids.tolist() and np.array_equal(r.scores, w.scores)
    finally:
        gpu.close()


def test_batched_variant_with_more_than_64_probes(oracle, npb, corpus):
    # colgrep exposes n_ivf_probe (COLGREP_N_IVF_PROBE, colgrep/src/index/mod.rs:792-820): the batched variant's
    # streaming selection holds up to 192 entries per token; beyond that the call is refused, never silently different
    docs, ix, qs, src, gpu = corpus
    for n in (65, 100, 192):
        kw = dict(top_k=10, n_ivf_probe=n, n_full_scores=512, centroid_batch_size=128, centroid_score_threshold=0.45)
        pg, po = _params(npb, oracle, **kw)
        for q, r in zip(qs[:5], gpu.search_batch(qs[:5], pg)):
            w = oracle.search_one(ix, q, po)
            assert r.passage_ids.tolist() == w.passage_ids.tolist(), n
            assert np.array_equal(r.scores, w.scores), n
    with pytest.raises(npb.PlaidError) as e:
        gpu.search_batch(qs[:2], npb.SearchParameters(top_k=10, n_ivf_probe=193, centroid_batch_size=128))
    assert e.value.status == 4


def test_lanes_cut_a_batch_without_changing_a_bit(oracle, npb, corpus):
    # pb_set_lanes: slices of a batch run the pipeline concurrently on their own streams; ids, scores and the summed work
    # counters must not depend on the number of lanes, with host buffers, ragged queries and a subset alike
    docs, ix, qs, src, gpu = corpus
    long_q, _ = oracle.synthetic_queries(docs, 4, nq=48, seed=91)
    batch = (qs + long_q + [qs[0][:5], qs[1] * 3.0]) * 3
    assert len(batch) >= 40
    try:
        for kw, subset in ((dict(top_k=10, n_full_scores=1024), None),
                           (dict(top_k=25, n_full_scores=512, centroid_batch_size=128), None),
                           (dict(top_k=10, n_full_scores=256), list(range(0, len(docs), 2)))):
            pg, po = _params(npb, oracle, **kw)
            ref = None
            for lanes in (1, 2, 3, 5):
                gpu.set_lanes(lanes)
                res = gpu.search_batch(batch, pg, subset=subset)
                w = gpu.last_work_counters()
                got = [(r.passage_ids.tolist(), r.scores.tobytes()) for r in res]
                key = (w["n_queries"], w["n_query_tokens"], w["n_candidates"], w["n_exact_docs"])
                if ref is None:
                    ref = (got, key)
                    for q, r in zip(batch[:12], res):
                        want = oracle.search_one(ix, q, po, subset=subset)
                        assert r.passage_ids.tolist() == want.passage_ids.tolist() and np.array_equal(r.scores, want.scores)
                assert got == ref[0], (kw, lanes)
                assert key == ref[1], (kw, lanes, key, ref[1])
        # an error inside one lane is the call's error
        gpu.set_lanes(2)
        bad = _params(npb, oracle, top_k=10, n_full_scores=10 ** 6)[0]
        with pytest.raises(Exception):
            gpu.search_batch(batch, bad)
    finally:
        gpu.set_lanes(1)
