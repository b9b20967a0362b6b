"""Index-build path on the GPU (SURVEY 8 a12): nearest-centroid codes and packed residuals are
bit-identical to the CPU oracle (compress_into_codes_cpu codec.rs:297, quantize_residuals codec.rs:356);
k-means is parity-unpinned (fastkmeans-rs is not in the reference tree) and checked statistically."""
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


def test_codec_kats_on_gpu(npb):
    # maxsim.rs:444-477 -> [0,1,2,0,2]; codec.rs:637-663 -> [0,2]; codec.rs:733-752 NaN centroid -> 1;
    # last maximum wins exact ties (codec.rs:329-337)
    def pad(a, d=32):
        out = np.zeros((a.shape[0], d), np.float32); out[:, :a.shape[1]] = a; return out
    c = pad(np.eye(3, 4, dtype=np.float32))
    e = pad(np.array([[0.9, 0.1, 0, 0], [0.1, 0.9, 0, 0], [0, 0.1, 0.9, 0], [0.8, 0.2, 0, 0], [0, 0, 0.8, 0.2]], np.float32))
    assert npb.ResidualCodec(2, c).compress_into_codes(e).tolist() == [0, 1, 2, 0, 2]
    e2 = pad(np.array([[0.9, 0.1, 0, 0], [0, 0, 0.95, 0.05]], np.float32))
    assert npb.ResidualCodec(2, c).compress_into_codes(e2).tolist() == [0, 2]
    cn = pad(np.array([[np.nan, 0], [1, 0], [0, 1]], np.float32))
    assert npb.ResidualCodec(2, cn).compress_into_codes(pad(np.array([[1, 0]], np.float32))).tolist() == [1]
    ct = pad(np.array([[1, 0], [1, 0], [0, 1]], np.float32))
    assert npb.ResidualCodec(2, ct).compress_into_codes(pad(np.array([[1, 0]], np.float32))).tolist() == [1]


@pytest.mark.parametrize("dim,nbits,K", [(128, 4, 300), (128, 2, 1024), (64, 8, 77), (96, 1, 130), (32, 4, 64), (256, 4, 200)])
def test_encode_chunk_bit_exact(oracle, npb, dim, nbits, K):
    rng = np.random.default_rng(dim + nbits)
    cent = rng.standard_normal((K, dim)).astype(np.float32)
    cent /= np.linalg.norm(cent, axis=1, keepdims=True)
    cent[K // 2] = cent[3]                        # exact duplicate centroid: the LAST one must win
    emb = cent[rng.integers(0, K, 1500)] + 0.3 * rng.standard_normal((1500, dim)).astype(np.float32) / np.sqrt(dim)
    emb /= np.linalg.norm(emb, axis=1, keepdims=True)
    emb[7] = cent[3]
    want_codes = oracle.compress_into_codes(emb, cent)
    res = oracle.residuals_of(emb, cent, want_codes)
    n_opt = 1 << nbits
    cut = oracle.quantiles(res.ravel(), [i / n_opt for i in range(1, n_opt)])
    want_packed = oracle.quantize_residuals(res, cut, nbits)
    codec = npb.ResidualCodec(nbits, cent, cut)
    codes, packed = codec.encode_chunk(emb)
    st = codec.last_assign_stats()
    assert st["tokens"] == 1500
    assert st["tensor_cores"] == (dim in (64, 96, 128) and K >= 256)
    if st["tensor_cores"]:
        assert st["exact_fallback"] < 150, st     # the certified tensor-core shortlist decides >90 % of the tokens
    assert codes.tolist() == want_codes.tolist()
    assert codes[7] == max(3, K // 2)
    assert np.array_equal(packed, want_packed)
    c2, r2 = codec.compress_and_residuals(emb)
    assert c2.tolist() == want_codes.tolist() and np.array_equal(r2, res)
    assert codec.compress_into_codes(np.zeros((0, dim), np.float32)).shape == (0,)
    codec.close()


def test_codec_argument_errors(npb):
    with pytest.raises(npb.PlaidError) as e:
        npb.ResidualCodec(3, np.zeros((4, 32), np.float32))
    assert "divisor of 8" in str(e.value)                       # codec.rs:161-166
    codec = npb.ResidualCodec(4, np.eye(4, 32, dtype=np.float32))
    with pytest.raises(npb.PlaidError) as e:
        codec.encode_chunk(np.zeros((2, 32), np.float32))
    assert "bucket_cutoffs required" in str(e.value)            # codec.rs:359-362


def test_kmeans_fit_shape_norm_and_quality(oracle, npb):
    # kmeans.rs:461-534 pins shape and unit norm only; add: better than random centroids
    docs = oracle.synthetic_corpus(800, 32, dim=64, seed=3)
    x = np.concatenate(docs, 0)
    K = 256
    cent = npb.kmeans_fit(x, K, niters=4, seed=42)
    assert cent.shape == (K, 64)
    assert np.allclose(np.linalg.norm(cent, axis=1), 1.0, atol=1e-5)
    rng = np.random.default_rng(0)
    rnd = rng.standard_normal((K, 64)).astype(np.float32)
    rnd /= np.linalg.norm(rnd, axis=1, keepdims=True)
    fit = (x @ cent.T).max(1).mean()
    base = (x @ rnd.T).max(1).mean()
    ref = (x @ oracle.kmeans(x, K, 4, 42).T).max(1).mean()
    assert fit > base + 0.2 and fit > ref - 0.03


def test_gpu_built_index_serves_searches(oracle, npb):
    # create_with_kmeans (index.rs:1392) with the numeric steps on the GPU, then search it
    docs = oracle.synthetic_corpus(1200, 32, dim=128, seed=13, ragged=True)
    x = np.concatenate(docs, 0)
    cent = npb.kmeans_fit(x, 256, niters=4, seed=42)
    art = oracle.prepare_codec_artifacts(docs, cent, 4, seed=42)     # quantiles of the held-out residuals (host)
    codec = npb.ResidualCodec(4, cent, art.bucket_cutoffs)
    codes, packed = codec.encode_chunk(x)
    doclens = np.array([d.shape[0] for d in docs], np.int64)
    ivf, ivf_lengths = oracle.build_ivf(codes, doclens, 256)
    ix = oracle.Index(cent, art.bucket_weights, art.bucket_cutoffs, codes, packed, doclens, ivf, ivf_lengths, 4)
    gpu = npb.MmapIndex.from_arrays(cent, art.bucket_weights, codes, packed, doclens, ivf, ivf_lengths, 4)
    qs, src = oracle.synthetic_queries(docs, 8, nq=32, seed=1)
    pg = npb.SearchParameters(top_k=5, n_full_scores=256)
    po = oracle.SearchParameters(top_k=5, n_full_scores=256)
    hits = 0
    for q, s, r in zip(qs, src, gpu.search_batch(qs, pg)):
        w = oracle.search_one(ix, q, po)
        assert r.passage_ids.tolist() == w.passage_ids.tolist() and np.array_equal(r.scores, w.scores)
        hits += int(len(r.passage_ids) and r.passage_ids[0] == s)
    assert hits >= 7


def test_tensor_core_filter_is_exact_on_hard_inputs(oracle, npb):
    # near ties inside the fp16 error band, duplicated centroids, non-unit norms and a NaN token:
    # whatever the tensor-core shortlist cannot certify must fall back to the exact kernel
    rng = np.random.default_rng(7)
    K, dim = 2048, 128
    cent = rng.standard_normal((K, dim)).astype(np.float32)
    cent /= np.linalg.norm(cent, axis=1, keepdims=True)
    cent[1000:1016] = cent[5] + 1e-4 * rng.standard_normal((16, dim)).astype(np.float32)   # a tight cluster
    cent[1500] = cent[7]                                                                  # exact duplicate
    cent[1600:1700] *= 3.0                                                                # non-unit norms
    emb = cent[rng.integers(0, K, 4000)] + 0.2 * rng.standard_normal((4000, dim)).astype(np.float32) / np.sqrt(dim)
    emb[:300] = cent[5] + 1e-3 * rng.standard_normal((300, dim)).astype(np.float32)        # all land in the cluster
    emb[300:320] = cent[7]
    emb[320] = np.nan
    emb[321] *= 1e-6
    emb[322] *= 1e4
    want = oracle.compress_into_codes(emb, cent)
    codec = npb.ResidualCodec(4, cent)
    got = codec.compress_into_codes(emb)
    st = codec.last_assign_stats()
    assert st["tensor_cores"] and 300 <= st["exact_fallback"] < 1200, st
    assert got.tolist() == want.tolist()
    assert got[300] == 1500


@pytest.mark.parametrize("dim,K", [(128, 700), (64, 129), (256, 90), (32, 8)])
def test_find_outliers_identical_to_oracle(oracle, npb, dim, K):
    # update.rs:490-608; includes rows placed inside the 1e-5 re-check band around the threshold
    rng = np.random.default_rng(dim + K)
    cent = rng.standard_normal((K, dim)).astype(np.float32)
    cent /= np.linalg.norm(cent, axis=1, keepdims=True)
    emb = cent[rng.integers(0, K, 3000)] + rng.uniform(0.0, 1.2, (3000, 1)).astype(np.float32) * \
        rng.standard_normal((3000, dim)).astype(np.float32) / np.sqrt(dim)
    e64, c64 = emb.astype(np.float64), cent.astype(np.float64)
    d2 = ((e64 * e64).sum(1)[:, None] + (c64 * c64).sum(1)[None, :] - 2.0 * e64 @ c64.T).min(1)
    thr = float(np.median(d2))
    # nudge a few rows onto the threshold so the f64 path decides them
    for r in range(40):
        j = int(rng.integers(0, K))
        v = rng.standard_normal(dim).astype(np.float32)
        v /= np.linalg.norm(v)
        emb[r] = cent[j] + np.float32(np.sqrt(thr) * (1.0 + (r - 20) * 1e-7)) * v
    want = oracle.find_outliers(emb, cent, thr)
    got = npb.ResidualCodec(4, cent).find_outliers(emb, thr)
    assert 100 < len(want) < 2900
    assert got.tolist() == want.tolist()


def test_find_outliers_reference_kat(npb):
    # update.rs:1170-1185, padded to a built dimension
    c = np.zeros((2, 32), np.float32); c[1, :2] = 1.0
    e = np.zeros((3, 32), np.float32); e[0, :2] = 0.1; e[1, :2] = 0.9; e[2, :2] = 5.0
    assert npb.ResidualCodec(4, c).find_outliers(e, 1.0).tolist() == [2]


def test_inverted_file_is_built_on_the_device_when_none_is_given(oracle, npb):
    # index.rs:850-873: code -> sorted unique doc ids.  A handle opened without ivf builds it from the codes; the
    # export is what create_index writes to ivf.npy / ivf_lengths.npy, and searches on it equal the oracle's.
    docs = oracle.synthetic_corpus(1200, 36, dim=64, seed=77, ragged=True)
    docs[5] = docs[5][:0]                                           # a doc without tokens
    ix = oracle.create_index(docs, nbits=2, seed=9, num_partitions=300)
    gpu = npb.MmapIndex.from_arrays(ix.centroids, ix.bucket_weights, ix.codes, ix.residuals, ix.doc_lengths,
                                    None, None, ix.nbits, doc_id_base=0)
    try:
        ivf, lens = gpu.export_ivf()
        assert lens.dtype == np.int32 and ivf.dtype == np.int64
        assert np.array_equal(lens, ix.ivf_lengths) and np.array_equal(ivf, ix.ivf)
        qs, _ = oracle.synthetic_queries(docs, 6, nq=16, seed=4)
        kw = dict(top_k=10, n_ivf_probe=4, n_full_scores=128)
        for q, r in zip(qs, gpu.search_batch(qs, npb.SearchParameters(**kw))):
            w = oracle.search_one(ix, q, oracle.SearchParameters(**kw))
            assert r.passage_ids.tolist() == w.passage_ids.tolist() and np.array_equal(r.scores, w.scores)
    finally:
        gpu.close()


def test_adopted_device_residuals_are_used_in_place(oracle, npb):
    import torch
    docs = oracle.synthetic_corpus(600, 30, dim=128, seed=78)
    ix = oracle.create_index(docs, nbits=4, seed=9, num_partitions=128)
    dev = torch.device("cuda", 0)
    t = {k: torch.from_numpy(np.ascontiguousarray(v)).to(dev) for k, v in dict(
        cen=ix.centroids, w=ix.bucket_weights, codes=ix.codes.astype(np.int64), res=ix.residuals,
        dl=ix.doc_lengths.astype(np.int64)).items()}
    gpu = npb.MmapIndex.from_device_pointers(128, 4, ix.num_centroids, ix.num_documents, ix.num_embeddings,
                                             t["cen"].data_ptr(), t["w"].data_ptr(), t["codes"].data_ptr(),
                                             t["res"].data_ptr(), t["dl"].data_ptr(), None, None, device=0,
                                             adopt_residuals=True)
    try:
        qs, _ = oracle.synthetic_queries(docs, 4, nq=32, seed=5)
        kw = dict(top_k=5, n_ivf_probe=8, n_full_scores=64)
        for q, r in zip(qs, gpu.search_batch(qs, npb.SearchParameters(**kw))):
            w = oracle.search_one(ix, q, oracle.SearchParameters(**kw))
            assert r.passage_ids.tolist() == w.passage_ids.tolist() and np.array_equal(r.scores, w.scores)
    finally:
        gpu.close()


def test_data_parallel_kmeans_over_an_in_process_group(oracle, npb):
    # SURVEY 8e "Build path": sample points sharded over ranks, centroids replicated, one all-reduce of the
    # [K][dim] sums + [K] counts per iteration.  Ranks = host threads of this process on one GPU (the NCCL
    # transport runs the same kernels, tests/gpu_sharded_check.py).  k-means is parity-unpinned: the checks are
    # that every rank ends with the same unit-norm centroids, that well-separated blobs are recovered, and that the
    # clustering is as tight as the single-GPU fit's.
    rng = np.random.default_rng(3)
    dim, n_blobs = 64, 48
    centers = rng.standard_normal((n_blobs, dim)).astype(np.float32)
    centers /= np.linalg.norm(centers, axis=1, keepdims=True)
    pts = centers[rng.integers(0, n_blobs, 24_000)] + 0.05 * rng.standard_normal((24_000, dim)).astype(np.float32)
    pts /= np.linalg.norm(pts, axis=1, keepdims=True)

    def inertia(c):
        return float((1.0 - (pts @ c.T).max(1)).mean())
    single = npb.kmeans_fit(pts, n_blobs, niters=8, seed=5)
    for G in (2, 3):
        shards = np.array_split(pts, G)
        c = npb.kmeans_fit_dp(shards, n_blobs, niters=8, seed=5)        # asserts that the ranks agree bit for bit
        assert c.shape == (n_blobs, dim) and np.abs(np.linalg.norm(c, axis=1) - 1.0).max() < 1e-5
        assert inertia(c) <= 1.5 * inertia(single) + 1e-3
        found = (centers @ c.T).max(1)
        found_single = (centers @ single.T).max(1)
        assert (found > 0.98).mean() >= (found_single > 0.98).mean() - 0.2     # as many blobs recovered as by the single fit


def test_kmeans_on_the_tensor_cores_matches_the_fp32_assignment_statistically(oracle, npb, monkeypatch):
    # dims 64/96/128 with K >= 256: the Lloyd assignment step runs as the fp16 wgmma GEMM with the -|c|^2/2 bias in
    # its epilogue (k_assign_tc<., true>); PB_KMEANS_EXACT=1 keeps the fp32 kernel.  Same seed -> same start; bf16
    # rounding may move points that sit between two centroids, the clustering quality must not change.
    docs = oracle.synthetic_corpus(1500, 32, dim=128, seed=8)
    x = np.concatenate(docs, 0)
    K = 512
    tc = npb.kmeans_fit(x, K, niters=5, seed=7)
    monkeypatch.setenv("PB_KMEANS_EXACT", "1")
    ex = npb.kmeans_fit(x, K, niters=5, seed=7)
    monkeypatch.delenv("PB_KMEANS_EXACT")
    assert np.allclose(np.linalg.norm(tc, axis=1), 1.0, atol=1e-5)
    q_tc, q_ex = (x @ tc.T).max(1).mean(), (x @ ex.T).max(1).mean()
    assert abs(q_tc - q_ex) < 5e-3, (q_tc, q_ex)
    agree = ((x @ tc.T).argmax(1) == (x @ ex.T).argmax(1)).mean()
    assert agree > 0.9, agree
