"""Indexes of embedding dim 48 on every path.  48 is the first built width that is not a multiple of 32: the tensor-core
kernels run three wgmma K steps, the MaxSim filter's operand stage is rounded up to 128 bytes, a pinned sum of squares
spans 12 float4 groups, and 1-bit rows are 6 bytes (not whole 32-bit words: the filter stays off there and the exact
kernels score those queries).

Every search is compared bit for bit with the CPU oracle, with the tensor-core paths on and off, and the work counters
show which kernels ran: the tensor-core score table (n_k1_tc), the exact table's threshold-first probe (n_probe_threshold), the
MaxSim filter (n_filter_docs) and its pair stage (n_exact_pairs).  Then the certificates of both estimates, the build
path, mutations with an index directory, the host-residual tier, an in-process shard group with a rebalance, and the
stage entry points."""
import os
import shutil

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

DIM = 48
KW = (dict(top_k=10, n_ivf_probe=8, n_full_scores=256),                              # dense variant
      dict(top_k=10, n_ivf_probe=8, n_full_scores=256, centroid_batch_size=1000))    # batched: K > 1000
ENVS = ("PB_FILTER_DIAG", "PB_K1_TC_DIAG")


@pytest.fixture(scope="module")
def npb():
    import next_plaid_b200 as m
    m.build_library()
    if m.device_count() < 1:
        pytest.fail("GPU tests need an H100; the library has no CPU fallback")
    return m


def _codec_index(oracle, nbits, K=2048, D=3000, seed=5):
    """Codes drawn mostly from per-topic pools (so probes find dense cells), random residual bytes, unit centroids."""
    rng = np.random.default_rng(seed)
    cent = rng.standard_normal((K, DIM), dtype=np.float32)
    cent /= np.linalg.norm(cent, axis=1, keepdims=True)
    dl = rng.integers(10, 50, D).astype(np.int64)
    N = int(dl.sum())
    pools = rng.integers(0, K, (D // 64, 64))
    topic = np.repeat(rng.integers(0, len(pools), D), dl)
    u = rng.random(N)
    from_pool = pools[topic, np.minimum((u * u * 64).astype(np.int64), 63)]
    codes = np.where(rng.random(N) < 0.75, from_pool, rng.integers(0, K, N)).astype(np.int64)
    res = rng.integers(0, 256, (N, DIM * nbits // 8), dtype=np.uint8)
    w = (0.05 * np.linspace(-1.8, 1.8, 1 << nbits)).astype(np.float32)
    cut = ((w[1:] + w[:-1]) / 2).astype(np.float32)
    ivf, lens = oracle.build_ivf(codes, dl, K)
    return oracle.Index(cent, w, cut, codes, res, dl, ivf, lens, nbits)


def _queries(oracle, ix, lens, seed, noise=0.15):
    """One query per length: tokens of a random doc's decompressed embedding plus noise, renormalised."""
    rng = np.random.default_rng(seed)
    out = []
    for nq in lens:
        tok = oracle.get_document_embeddings(ix, int(rng.integers(ix.num_documents)))
        tok = tok[rng.integers(0, len(tok), nq)]
        nz = rng.standard_normal(tok.shape).astype(np.float32)
        q = tok + noise * nz / np.linalg.norm(nz, axis=1, keepdims=True)
        out.append((q / np.linalg.norm(q, axis=1, keepdims=True)).astype(np.float32))
    return out


def _open(npb, ix, monkeypatch=None, env=None, **kw):
    for k in ENVS:
        if monkeypatch:
            monkeypatch.delenv(k, raising=False)
    for k, v in (env or {}).items():
        monkeypatch.setenv(k, v)
    try:
        return npb.MmapIndex.from_arrays(ix.centroids, ix.bucket_weights, ix.codes, ix.residuals, ix.doc_lengths,
                                         ix.ivf, ix.ivf_lengths, ix.nbits, **kw)
    finally:
        for k in env or {}:
            monkeypatch.delenv(k)


def _same(r, w):
    return r.passage_ids.tolist() == w.passage_ids.tolist() and np.array_equal(r.scores, w.scores)


@pytest.fixture(scope="module")
def corpora(oracle):
    return {nb: _codec_index(oracle, nb, seed=40 + nb) for nb in (1, 2, 4, 8)}


LENS = [1, 31, 32, 33, 48, 64, 65]


# ---------------------------------------------------------------------------------------------------------------------
# search parity and the paths that ran
# ---------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("nbits", [1, 2, 4, 8])
@pytest.mark.parametrize("nq", LENS)
def test_search_parity_and_paths(oracle, npb, corpora, nbits, nq):
    ix = corpora[nbits]
    qs = _queries(oracle, ix, [nq] * 3, seed=nq * 10 + nbits)
    subset = sorted(np.random.default_rng(nq).choice(ix.num_documents, 1500, replace=False).tolist())
    gpu = _open(npb, ix)
    try:
        assert gpu.embedding_dim() == DIM and gpu.nbits() == nbits
        for kw in KW:
            batched = "centroid_batch_size" in kw
            for sub in (None, subset):
                pg, po = npb.SearchParameters(**kw), oracle.SearchParameters(**kw)
                want = [oracle.search_one(ix, q, po, subset=sub) for q in qs]
                assert any(len(w.passage_ids) for w in want)
                res = gpu.search_batch(qs, pg, subset=sub)
                w = gpu.last_work_counters()
                mode = (kw, sub is not None, w)
                for r, x in zip(res, want):
                    assert _same(r, x), mode
                # the tensor-core table, unless a dense-variant subset keeps the sub-batch on the exact kernels
                tc_pass = sub is None or batched
                if tc_pass:
                    assert w["n_k1_tc"] > 0, mode
                filt = nbits != 1 and nq <= 64
                assert (w["n_filter_docs"] > 0) == filt, mode
                if filt:
                    assert w["n_exact_pairs"] > 0, mode
                # the same ids and scores with each fast path off
                for off in ("set_scores_tc", "set_fast_exact", "set_fast_approx"):
                    getattr(gpu, off)(False)
                    try:
                        res = gpu.search_batch(qs, pg, subset=sub)
                    finally:
                        getattr(gpu, off)(True)
                    wo = gpu.last_work_counters()
                    if off != "set_fast_exact":
                        assert wo["n_k1_tc"] == 0, (off, mode)
                        if off == "set_scores_tc" and tc_pass:   # threshold-first probe on the exact table
                            assert wo["n_probe_threshold"] > 0, (off, mode)
                    else:
                        assert wo["n_filter_docs"] == 0, (off, mode)
                    for r, x in zip(res, want):
                        assert _same(r, x), (off, mode)
    finally:
        gpu.close()


# ---------------------------------------------------------------------------------------------------------------------
# certificates
# ---------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("nbits", [2, 4, 8])
def test_score_table_certificate(oracle, npb, corpora, monkeypatch, nbits):
    ix = corpora[nbits]
    qs = _queries(oracle, ix, LENS, seed=nbits)
    gpu = _open(npb, ix, monkeypatch, {"PB_K1_TC_DIAG": "1"})
    try:
        for kw in KW:
            res = gpu.search_batch(qs, npb.SearchParameters(**kw))
            w = gpu.last_work_counters()
            assert 0 <= w["k1_tc_max_code_diff"] <= 1 and w["k1_rows_mismatch"] == 0, (kw, w)
            assert w["n_k1_tc"] == 0, (kw, w)               # the diagnostic keeps the exact table in charge
            for q, r in zip(qs, res):
                assert _same(r, oracle.search_one(ix, q, oracle.SearchParameters(**kw))), kw
    finally:
        gpu.close()


@pytest.mark.parametrize("nbits", [2, 4, 8])
@pytest.mark.parametrize("scores_tc", [True, False])
def test_filter_certificate(oracle, npb, corpora, monkeypatch, nbits, scores_tc):
    ix = corpora[nbits]
    rng = np.random.default_rng(nbits)
    base = [q / np.linalg.norm(q, axis=1, keepdims=True) for q in
            (rng.standard_normal((n, DIM)).astype(np.float32) for n in (1, 32, 33, 64))]
    kw = dict(top_k=10, n_ivf_probe=8, n_full_scores=256, centroid_score_threshold=None)
    gpu = _open(npb, ix, monkeypatch, {"PB_FILTER_DIAG": "1"})
    gpu.set_scores_tc(scores_tc)
    try:
        for lo, hi in ((0, 2), (2, 4)):                  # N = 32 and N = 64 operands of k_maxsim_tc
            batch = []
            for i, q in enumerate(base[lo:hi]):
                batch += [(q * np.float32(s)).astype(np.float32) for s in (1e-8, 1e-6, 1e-4, 1.0, 4096.0, 1e6)]
                big = q.astype(np.float32).copy()
                big[0, i % DIM] = 1e5
                batch.append(big)
            gpu.search_batch(batch, npb.SearchParameters(**kw))
            w = gpu.last_work_counters()
            assert w["n_filter_docs"] > 0 and w["filter_diag_pairs"] > 0, (lo, w)
            assert 0 < w["filter_err_ratio_e6"] <= 1_000_000, (lo, w["filter_err_ratio_e6"])
    finally:
        gpu.close()


# ---------------------------------------------------------------------------------------------------------------------
# build path
# ---------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("nbits,K", [(1, 300), (2, 1024), (4, 256), (8, 300), (4, 200)])
def test_encode_chunk_bit_exact(oracle, npb, nbits, K):
    rng = np.random.default_rng(nbits + K)
    cent = rng.standard_normal((K, DIM)).astype(np.float32)
    cent /= np.linalg.norm(cent, axis=1, keepdims=True)
    cent[K // 2] = cent[3]                                      # duplicate centroid: the last one wins
    emb = cent[rng.integers(0, K, 3000)] + 0.3 * rng.standard_normal((3000, DIM)).astype(np.float32) / np.sqrt(DIM)
    emb /= np.linalg.norm(emb, axis=1, keepdims=True)
    emb[7] = cent[3]
    want_codes = oracle.compress_into_codes(emb, cent)
    res = oracle.residuals_of(emb, cent, want_codes)
    n_opt = 1 << nbits
    cut = oracle.quantiles(res.ravel(), [i / n_opt for i in range(1, n_opt)])
    codec = npb.ResidualCodec(nbits, cent, cut)
    try:
        codes, packed = codec.encode_chunk(emb)
        st = codec.last_assign_stats()
        assert st["tokens"] == 3000
        assert st["tensor_cores"] == (K >= 256), st
        if st["tensor_cores"]:
            assert st["exact_fallback"] < 300, st               # < 10 %: the shortlist decides most tokens
        assert codes.tolist() == want_codes.tolist() and codes[7] == max(3, K // 2)
        assert np.array_equal(packed, oracle.quantize_residuals(res, cut, nbits))
        c2, r2 = codec.compress_and_residuals(emb)
        assert c2.tolist() == want_codes.tolist() and np.array_equal(r2, res)
    finally:
        codec.close()


def test_kmeans_on_the_tensor_cores(oracle, npb):
    docs = oracle.synthetic_corpus(800, 32, dim=DIM, seed=3)
    x = np.concatenate(docs, 0)
    cent = npb.kmeans_fit(x, 256, niters=4, seed=42)
    assert cent.shape == (256, DIM) and np.allclose(np.linalg.norm(cent, axis=1), 1.0, atol=1e-5)
    ref = (x @ oracle.kmeans(x, 256, 4, 42).T).max(1).mean()
    assert (x @ cent.T).max(1).mean() > ref - 0.03


@pytest.fixture(scope="module")
def built(oracle, npb, tmp_path_factory):
    """A directory written by create_index at dim 48 (K = 256: the tensor-core assignment) and its documents."""
    docs = oracle.synthetic_corpus(2600, 40, dim=DIM, seed=33, ragged=True)
    path = str(tmp_path_factory.mktemp("dim48") / "ix")
    npb.create_index(docs[:2400], path, nbits=4, num_partitions=256, batch_size=1000, seed=7).close()
    return path, docs


def test_created_directory_searches_as_the_oracle(oracle, npb, built):
    path, docs = built
    ix = oracle.load_index(path)
    assert ix.dim == DIM and ix.num_documents == 2400
    qs, _ = oracle.synthetic_queries(docs[:2400], 8, nq=32, seed=3)
    gpu = npb.MmapIndex.load(path)
    try:
        for kw in KW:
            res = gpu.search_batch(qs, npb.SearchParameters(**kw))
            w = gpu.last_work_counters()
            assert w["n_k1_tc"] > 0 and w["n_filter_docs"] > 0, (kw, w)
            for q, r in zip(qs, res):
                assert _same(r, oracle.search_one(ix, q, oracle.SearchParameters(**kw))), kw
    finally:
        gpu.close()


# ---------------------------------------------------------------------------------------------------------------------
# mutations, tiers, shards
# ---------------------------------------------------------------------------------------------------------------------

def _dir_files(path):
    return {f: open(os.path.join(path, f), "rb").read() for f in sorted(os.listdir(path))}


def _check_handle(oracle, npb, gpu, path, qs):
    ix = oracle.load_index(path)
    fresh = npb.MmapIndex.load(path)
    try:
        for kw in KW:
            a = gpu.search_batch(qs, npb.SearchParameters(**kw))
            b = fresh.search_batch(qs, npb.SearchParameters(**kw))
            for q, x, y in zip(qs, a, b):
                w = oracle.search_one(ix, q, oracle.SearchParameters(**kw))
                assert _same(x, w) and _same(y, w), kw
    finally:
        fresh.close()


def test_append_and_delete_with_the_directory(oracle, npb, built, tmp_path):
    src, docs = built
    single, sharded = str(tmp_path / "single"), str(tmp_path / "sharded")
    shutil.copytree(src, single)
    shutil.copytree(src, sharded)
    base = oracle.load_index(src)
    qs, _ = oracle.synthetic_queries(docs, 6, nq=32, seed=4)
    codec = npb.ResidualCodec(4, base.centroids, base.bucket_cutoffs)
    live = npb.MmapIndex.load(single)
    grp = npb.ShardGroup([npb.MmapIndex.load_shard(sharded, r, 3) for r in range(3)])
    try:
        assert live.append(docs[2400:2600], codec, index_dir=single, batch_size=1000) == list(range(2400, 2600))
        assert grp.append(docs[2400:2600], codec, index_dir=sharded, batch_size=1000) == list(range(2400, 2600))
        _check_handle(oracle, npb, live, single, qs)
        ids = [0, 5, 999, 1000, 2399, 2400, 2599]
        assert live.delete(ids, index_dir=single) == len(ids)
        assert grp.delete(ids, index_dir=sharded) == len(ids)
        _check_handle(oracle, npb, live, single, qs)
        assert _dir_files(single) == _dir_files(sharded)
        ix = oracle.load_index(single)
        for kw in KW:
            for q, r in zip(qs, grp.search_batch(qs, npb.SearchParameters(**kw))):
                assert _same(r, oracle.search_one(ix, q, oracle.SearchParameters(**kw))), kw
    finally:
        codec.close()
        live.close()
        grp.close()


@pytest.mark.parametrize("nbits", [1, 4])
def test_host_residuals_equal_resident(oracle, npb, corpora, nbits):
    ix = corpora[nbits]
    qs = _queries(oracle, ix, [1, 32, 48, 64, 65], seed=70 + nbits)
    dev, host = _open(npb, ix), _open(npb, ix, host_residuals=True)
    try:
        for kw in KW:
            a = dev.search_batch(qs, npb.SearchParameters(**kw))
            b = host.search_batch(qs, npb.SearchParameters(**kw))
            assert host.last_staging_stats()["docs"] > 0
            for q, x, y in zip(qs, a, b):
                assert _same(x, y) and _same(x, oracle.search_one(ix, q, oracle.SearchParameters(**kw))), kw
        ids = [0, 17, 2999]
        ea, la = dev.decompress_documents(ids)
        eb, lb = host.decompress_documents(ids)
        assert np.array_equal(ea, eb) and np.array_equal(la, lb)
        assert np.array_equal(dev.exhaustive_scores(qs[:2]), host.exhaustive_scores(qs[:2]))
    finally:
        dev.close()
        host.close()


@pytest.mark.parametrize("nbits", [1, 4])
def test_shard_group_and_rebalance(oracle, npb, corpora, tmp_path, nbits):
    ix = corpora[nbits]
    path = str(tmp_path / "ix")
    oracle.write_index(ix, path, chunk_docs=700)
    qs = _queries(oracle, ix, [1, 32, 33, 64], seed=90 + nbits)
    single = npb.MmapIndex.load(path)
    grp = npb.ShardGroup([npb.MmapIndex.load_range(path, b0, b1) for b0, b1 in ((0, 0), (0, 2000), (2000, 3000))])
    try:
        for bounds in (None, [0, 1000, 1001, 3000]):
            for kw in KW:
                want = single.search_batch(qs, npb.SearchParameters(**kw))
                got = grp.search_batch(qs, npb.SearchParameters(**kw))
                for q, x, y in zip(qs, want, got):
                    assert _same(x, y) and _same(x, oracle.search_one(ix, q, oracle.SearchParameters(**kw))), kw
            grp.rebalance(bounds)
        for kw in KW:
            for x, y in zip(single.search_batch(qs, npb.SearchParameters(**kw)),
                            grp.search_batch(qs, npb.SearchParameters(**kw))):
                assert _same(x, y), kw
    finally:
        single.close()
        grp.close()


# ---------------------------------------------------------------------------------------------------------------------
# stage entry points
# ---------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("nbits", [1, 2, 4, 8])
def test_decompress_and_exhaustive(oracle, npb, corpora, nbits):
    ix = corpora[nbits]
    ids = [0, 1, 1500, 2999, 10 ** 9]
    gpu = _open(npb, ix)
    try:
        emb, lens = gpu.decompress_documents(ids)
        assert lens.tolist() == [int(ix.doc_lengths[d]) for d in ids[:-1]] + [0]
        assert np.array_equal(emb, np.concatenate([oracle.get_document_embeddings(ix, d) for d in ids[:-1]], 0))
        qs = _queries(oracle, ix, [1, 33, 65, 48], seed=nbits)
        ex = gpu.exhaustive_scores(qs)
        for i, q in enumerate(qs):
            assert np.array_equal(ex[i], oracle.exhaustive_scores(ix, q)), i
    finally:
        gpu.close()


@pytest.mark.parametrize("nq", [1, 31, 32, 33, 64, 65, 300])
def test_maxsim_scores(oracle, npb, nq):
    rng = np.random.default_rng(nq)
    unit = lambda n: (lambda x: (x / np.maximum(np.linalg.norm(x, axis=1, keepdims=True), 1e-30)).astype(np.float32))(  # noqa: E731
        rng.standard_normal((n, DIM)).astype(np.float32))
    docs = [unit(n) for n in (0, 1, 127, 128, 129, 1000)]
    q = unit(nq)
    q[0] = docs[5][17]
    got = npb.maxsim_scores(q, docs)
    assert np.array_equal(got, np.array([oracle.maxsim_score(q, d) for d in docs], np.float32))
    assert got[0] == 0.0


def test_unbuilt_dims_are_refused(npb):
    for dim in (16, 80):
        with pytest.raises(npb.PlaidError) as e:
            npb.ResidualCodec(4, np.eye(8, dim, dtype=np.float32))
        assert e.value.status == 4 and "48" in str(e.value)
