"""The product builds an index by itself (SURVEY 8 a12; index.rs:551-911, kmeans.rs:261-422): pb_create_index writes the
reference's directory, the oracle loads it, and everything downstream of the (parity-unpinned) centroids and samples
is bit-identical to the CPU restatement -- codec training, codes, packed residuals, inverted file -- and searches of
the directory agree between the GPU and the oracle.  Includes BASELINE config A (10k docs x 64 tokens, K = 2^13)."""
import json
import os

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


def test_codec_training_matches_the_oracle(oracle, npb):
    rng = np.random.default_rng(5)
    docs = oracle.synthetic_corpus(400, 40, dim=128, seed=12)
    flat = np.concatenate(docs, 0)
    cent = flat[rng.choice(len(flat), 300, replace=False)].copy()
    held = flat[rng.choice(len(flat), 5000, replace=False)]
    for nbits in (1, 2, 4, 8):
        codec = npb.ResidualCodec(nbits, cent)
        cut, wts, avg, thr = codec.train(held)
        codes = oracle.compress_into_codes(held, cent)
        res = oracle.residuals_of(held, cent, codes)
        n_opt = 1 << nbits
        want_cut = oracle.quantiles(res.ravel(), [i / n_opt for i in range(1, n_opt)])
        want_wts = oracle.quantiles(res.ravel(), [(i + 0.5) / n_opt for i in range(n_opt)])
        assert np.array_equal(cut, want_cut) and np.array_equal(wts, want_wts), nbits      # utils.rs:125-149, bit for bit
        dist = np.sqrt((res.astype(np.float64) ** 2).sum(1))
        assert abs(thr - float(np.quantile(dist, 0.75))) < 1e-5                            # index.rs:249-253
        assert np.abs(avg - np.abs(res).mean(0)).max() < 1e-6                              # index.rs:255-258
        # the trained codec encodes: packed residuals equal the oracle's with these cutoffs
        c2, packed = codec.encode_chunk(held[:777])
        assert np.array_equal(c2, codes[:777])
        assert np.array_equal(packed, oracle.quantize_residuals(res[:777], want_cut, nbits))
        codec.close()


def _check_directory(oracle, npb, docs, path, gpu, nbits, queries, param_sets):
    ix = oracle.load_index(path)                                   # the reference's reader of the directory
    flat = np.concatenate(docs, 0).astype(np.float32)
    assert ix.num_documents == len(docs) and ix.num_embeddings == len(flat)
    assert np.abs(np.linalg.norm(ix.centroids, axis=1) - 1.0).max() < 1e-5           # kmeans.rs:415-419
    codes = oracle.compress_into_codes(flat, ix.centroids)
    assert np.array_equal(ix.codes, codes)                                            # codec.rs:297-343
    res = oracle.residuals_of(flat, ix.centroids, codes)
    assert np.array_equal(ix.residuals, oracle.quantize_residuals(res, ix.bucket_cutoffs, nbits))   # codec.rs:356-411
    ivf, lens = oracle.build_ivf(codes, ix.doc_lengths, ix.num_centroids)
    assert np.array_equal(ix.ivf, ivf) and np.array_equal(ix.ivf_lengths, lens)       # index.rs:850-873
    meta = json.load(open(os.path.join(path, "metadata.json")))
    assert meta["num_documents"] == len(docs) and meta["num_partitions"] == ix.num_centroids and meta["nbits"] == nbits
    assert meta["next_plaid_compatible"] is True and abs(meta["avg_doclen"] - len(flat) / len(docs)) < 1e-9
    loaded = npb.MmapIndex.load(path)                              # pb_index_load of what pb_create_index wrote
    try:
        for kw in param_sets:
            pg, po = npb.SearchParameters(**kw), oracle.SearchParameters(**kw)
            a, b = gpu.search_batch(queries, pg), loaded.search_batch(queries, pg)
            for q, x, y in zip(queries, a, b):
                w = oracle.search_one(ix, q, po)
                assert x.passage_ids.tolist() == y.passage_ids.tolist() == w.passage_ids.tolist(), kw
                assert np.array_equal(x.scores, w.scores) and np.array_equal(y.scores, w.scores), kw
    finally:
        loaded.close()
    return ix


def test_created_directory_is_the_references_and_serves_searches(oracle, npb, tmp_path):
    docs = oracle.synthetic_corpus(2500, 40, dim=128, seed=33, ragged=True)
    qs, src = oracle.synthetic_queries(docs, 12, nq=32, seed=3)
    path = str(tmp_path / "ix")
    gpu = npb.create_index(docs, path, nbits=2, num_partitions=256, batch_size=1000, seed=7)
    try:
        assert sorted(f for f in os.listdir(path) if f.endswith(".codes.npy")) == ["0.codes.npy", "1.codes.npy", "2.codes.npy"]
        _check_directory(oracle, npb, docs, path, gpu, 2, qs,
                         [dict(top_k=10, n_ivf_probe=8, n_full_scores=256), dict(top_k=5, n_ivf_probe=4, n_full_scores=64,
                                                                                 centroid_batch_size=100)])
        # the planted source doc comes back first for most queries (the index is usable, not just consistent)
        res = gpu.search_batch(qs, npb.SearchParameters(top_k=10, n_ivf_probe=8, n_full_scores=256))
        assert np.mean([int(len(r.passage_ids) and s in r.passage_ids.tolist()) for r, s in zip(res, src)]) >= 0.75
    finally:
        gpu.close()


def test_baseline_config_a(oracle, npb, tmp_path):
    # BASELINE.json configs[0]: 10k docs x 64 tok x 128-d, IndexConfig::default() -> K = 2^13 by the heuristic of
    # kmeans.rs:304-309; dense variant (K <= centroid_batch_size) and batched with centroid_batch_size = 4096
    docs = oracle.synthetic_corpus(10_000, 64, dim=128, seed=42)
    qs, src = oracle.synthetic_queries(docs, 64, nq=32, seed=7)
    path = str(tmp_path / "config_a")
    gpu = npb.create_index(docs, path)                    # nbits 4, kmeans_niters 4, seed 42, batch_size 50 000
    try:
        assert gpu.num_partitions() == 8192
        _check_directory(oracle, npb, docs, path, gpu, 4, qs,
                         [dict(top_k=10), dict(top_k=100, centroid_batch_size=4096),
                          dict(top_k=10, n_ivf_probe=16, n_full_scores=1024, centroid_score_threshold=None)])
        w = gpu.last_work_counters()
        assert w["n_queries"] == 64
    finally:
        gpu.close()
