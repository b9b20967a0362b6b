"""Search and scoring at the shapes where the engine switches kernels, tile loops and block sizes: query lengths past
the 64-token column block of k_approx16, past the QS <= 256 limit of the tensor-core table and the pair form, up to the
QS x n_ivf_probe <= 8192 limit; documents that span several 128-token tiles; exhaustive scores over more than one
block of 65536 documents and 32 queries; the device-resident search call; maxsim_scores at odd query and doc lengths.

Every comparison with the CPU oracle is bit-exact (ids, scores, counts).  The float64 checks bound the difference by
the pinned summation order (see _fp32_bound), not by a fixed tolerance: a sum of 1000 terms near 1 is already off by
more than 1e-4 in fp32.  Each case also asserts the work counters that name the path it ran on."""
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


def _params(npb, oracle, **kw):
    return npb.SearchParameters(**kw), oracle.SearchParameters(**kw)


def _codec_index(oracle, K, doc_lengths, dim=128, nbits=4, seed=5, docs_per_topic=64, pool=64):
    """An index drawn directly in the codec domain with the given per-doc lengths: random unit centroids, codes mostly
    from a per-topic pool, random residual bytes (so the tokens of a doc are distinct even where codes repeat)."""
    rng = np.random.default_rng(seed)
    cent = rng.standard_normal((K, dim), dtype=np.float32)
    cent /= np.linalg.norm(cent, axis=1, keepdims=True)
    dl = np.asarray(doc_lengths, np.int64)
    D, N = len(dl), int(dl.sum())
    n_topics = max(D // docs_per_topic, 4)
    pools = rng.integers(0, K, (n_topics, pool))
    topic = np.repeat(rng.integers(0, n_topics, D), dl)
    u = rng.random(N)
    from_pool = pools[topic, np.minimum((u * u * pool).astype(np.int64), pool - 1)]
    codes = np.where(rng.random(N) < 0.75, from_pool, rng.integers(0, K, N)).astype(np.int64)
    res = rng.integers(0, 256, (N, dim * nbits // 8), dtype=np.uint8)
    w = (0.05 * np.linspace(-1.8, 1.8, 1 << nbits)).astype(np.float32)
    cut = ((w[1:] + w[:-1]) / 2).astype(np.float32)
    ivf, ivf_lengths = oracle.build_ivf(codes, dl, K)
    return oracle.Index(cent, w, cut, codes, res, dl, ivf, ivf_lengths, nbits)


def _queries_from(oracle, ix, doc_ids, nqs, seed, noise=0.15):
    """One query per (doc, length): tokens of the doc's decompressed embedding plus noise, renormalised."""
    rng = np.random.default_rng(seed)
    out = []
    for d, nq in zip(doc_ids, nqs):
        if nq == 0:
            out.append(np.zeros((0, ix.dim), np.float32))
            continue
        tok = oracle.get_document_embeddings(ix, int(d))
        tok = tok[rng.integers(0, len(tok), nq)]
        nz = rng.standard_normal(tok.shape).astype(np.float32)
        q = tok + noise * nz / np.linalg.norm(nz, axis=1, keepdims=True)
        out.append((q / np.linalg.norm(q, axis=1, keepdims=True)).astype(np.float32))
    return out


def _same(r, w):
    return r.passage_ids.tolist() == w.passage_ids.tolist() and np.array_equal(r.scores, w.scores)


def _maxsim64(q, d):
    """MaxSim in float64; a query token with no doc token adds nothing (an empty doc scores 0)."""
    if len(q) == 0 or len(d) == 0:
        return 0.0
    return float((q.astype(np.float64) @ d.astype(np.float64).T).max(1).sum())


def _fp32_bound(q, d):
    """Largest |fp32 MaxSim - exact| for the pinned order: each similarity is a chain of `dim` fp32 FMAs, so it is off by
    at most g(dim) |q_i| |d_t| (Cauchy-Schwarz on sum |q_ij d_tj|) and so is its maximum over t; the nq maxima are then
    added one by one in fp32, which adds at most g(nq - 1) sum_i |m_i| with |m_i| <= (1 + g(dim)) |q_i| max_t |d_t|.
    g(n) = n u / (1 - n u), u = 2^-24.  The float64 reference's own error (~1e-13) is covered by the 1e-9 slack."""
    if len(q) == 0 or len(d) == 0:
        return 1e-9
    u = 2.0 ** -24
    g = lambda n: n * u / (1.0 - n * u)  # noqa: E731
    s = float((np.linalg.norm(q.astype(np.float64), axis=1) * np.linalg.norm(d.astype(np.float64), axis=1).max()).sum())
    return s * (g(q.shape[1]) + g(max(len(q) - 1, 0)) * (1.0 + g(q.shape[1]))) + 1e-9


def _check_float64(scores, qs, docs):
    for i, q in enumerate(qs):
        for j, d in enumerate(docs):
            err = abs(float(scores[i, j]) - _maxsim64(q, d))
            assert err <= _fp32_bound(q, d), (i, j, len(q), len(d), err, _fp32_bound(q, d))


# ---------------------------------------------------------------------------------------------------------------------
# 1. long and mixed-length queries
# ---------------------------------------------------------------------------------------------------------------------

def _query_row_tokens(nq):
    return max(8, (nq + 7) & ~7) if nq <= 32 else (nq + 63) & ~63


@pytest.fixture(scope="module")
def qcorpus(oracle):
    """4000 docs of 20..60 tokens over K = 4096: the tensor-core score table and the threshold-first probe engage."""
    rng = np.random.default_rng(3)
    ix = _codec_index(oracle, 4096, rng.integers(20, 61, 4000), seed=31)
    return ix


@pytest.mark.parametrize("nq", [32, 64, 65, 127, 128, 129, 192, 193, 255, 256, 257, 320, 511, 1000])
def test_long_queries_on_every_path(oracle, npb, qcorpus, nq):
    ix = qcorpus
    QS = _query_row_tokens(nq)
    n = min(16, 8192 // QS)                                       # QS x n_ivf_probe <= 8192
    qs = _queries_from(oracle, ix, [11, 1234, 3999], [nq] * 3, seed=nq)
    gpu = _gpu_index(npb, ix)
    try:
        # top_k = n_full_scores / 4 returns every doc the cut keeps, so a wrong approximate score shows in the ids
        for kw in (dict(top_k=10, n_ivf_probe=n, n_full_scores=256),
                   dict(top_k=10, n_ivf_probe=n, n_full_scores=256, centroid_batch_size=1000),   # batched: K > 1000
                   dict(top_k=64, n_ivf_probe=n, n_full_scores=256, centroid_score_threshold=None)):
            pg, po = _params(npb, oracle, **kw)
            want = [oracle.search_one(ix, q, po) for q in qs]
            assert all(len(w.passage_ids) == kw["top_k"] for w in want)
            for tc in (True, False):
                for approx in (1, 0):
                    for exact in (True, False):
                        gpu.set_scores_tc(tc)
                        gpu.set_fast_approx(approx)
                        gpu.set_fast_exact(exact)
                        res = gpu.search_batch(qs, pg)
                        w = gpu.last_work_counters()
                        mode = (kw, tc, approx, exact, w)
                        # the MaxSim filter runs up to 64 query tokens, when the cut keeps more than top_k docs
                        filt = exact and nq <= 64 and kw["top_k"] < kw["n_full_scores"] // 4
                        assert (w["n_filter_docs"] > 0) == filt, mode
                        if QS <= 256:      # the tensor-core table: QS <= 256 and the two-pass approximate stage
                            assert (w["n_k1_tc"] > 0) == (tc and approx == 1), mode
                        else:              # past 256 tokens: the exact table and the per-lane list probe
                            assert w["n_k1_tc"] == 0 and w["n_probe_list"] > 0, mode
                        for r, x in zip(res, want):
                            assert _same(r, x), mode
    finally:
        gpu.close()


def test_mixed_length_batch_takes_the_longest_query_row(oracle, npb, qcorpus):
    # 257 tokens set QS = 320 for the whole batch: the 0-, 1- and 33-token queries run on 320-token rows too
    ix = qcorpus
    lens = [257, 1, 0, 33, 64, 256] * 3
    qs = _queries_from(oracle, ix, np.random.default_rng(7).integers(0, ix.num_documents, len(lens)), lens, seed=8)
    gpu = _gpu_index(npb, ix)
    try:
        for kw in (dict(top_k=10, n_ivf_probe=16, n_full_scores=256),
                   dict(top_k=20, n_ivf_probe=8, n_full_scores=512, centroid_batch_size=1000)):
            pg, po = _params(npb, oracle, **kw)
            want = [oracle.search_one(ix, q, po) for q in qs]
            for lanes in (1, 3):
                gpu.set_lanes(lanes)
                res = gpu.search_batch(qs, pg)
                w = gpu.last_work_counters()
                assert w["n_k1_tc"] == 0 and w["n_probe_list"] > 0 and w["n_filter_docs"] == 0, (kw, lanes, w)
                assert w["n_query_tokens"] == sum(lens), (kw, lanes, w)
                for i, (r, x) in enumerate(zip(res, want)):
                    assert _same(r, x), (kw, lanes, i, lens[i])
                assert len(res[2].passage_ids) == 0
    finally:
        gpu.set_lanes(1)
        gpu.close()


def test_query_tokens_times_probes_limit(oracle, npb, qcorpus):
    # 1000 tokens -> QS = 1024: n_ivf_probe = 8 is the largest accepted (8192), 9 is refused, never silently different
    ix = qcorpus
    q = _queries_from(oracle, ix, [5], [1000], seed=1)
    gpu = _gpu_index(npb, ix)
    try:
        pg, po = _params(npb, oracle, top_k=10, n_ivf_probe=8, n_full_scores=256)
        assert _same(gpu.search_batch(q, pg)[0], oracle.search_one(ix, q[0], po))
        for cbs in (100_000, 1000):
            with pytest.raises(npb.PlaidError) as e:
                gpu.search_batch(q, npb.SearchParameters(top_k=10, n_ivf_probe=9, n_full_scores=256,
                                                         centroid_batch_size=cbs))
            assert e.value.status == 4
    finally:
        gpu.close()


# ---------------------------------------------------------------------------------------------------------------------
# 2. long documents
# ---------------------------------------------------------------------------------------------------------------------

LONG_LENGTHS = [0, 1, 127, 128, 129, 255, 256, 257, 300, 1000, 4097]


@pytest.fixture(scope="module")
def dcorpus(oracle):
    """600 docs of 8..48 tokens with the lengths of LONG_LENGTHS spread among them; returns (index, their ids)."""
    rng = np.random.default_rng(17)
    dl = rng.integers(8, 49, 600)
    where = np.sort(rng.choice(600, len(LONG_LENGTHS), replace=False))
    dl[where] = LONG_LENGTHS
    return _codec_index(oracle, 1024, dl, seed=41), where


def test_long_documents_search(oracle, npb, dcorpus, monkeypatch):
    ix, where = dcorpus
    long_ids = [int(d) for d, n in zip(where, LONG_LENGTHS) if n >= 129]
    qs = _queries_from(oracle, ix, long_ids, [32] * len(long_ids), seed=3)
    monkeypatch.setenv("PB_PAIR_EXACT", "0")
    tokens = _gpu_index(npb, ix)
    monkeypatch.delenv("PB_PAIR_EXACT")
    gpu = _gpu_index(npb, ix)
    try:
        for kw in (dict(top_k=10, n_ivf_probe=8, n_full_scores=256),
                   dict(top_k=5, n_ivf_probe=16, n_full_scores=1024, centroid_score_threshold=None)):
            pg, po = _params(npb, oracle, **kw)
            want = [oracle.search_one(ix, q, po) for q in qs]
            for d, x in zip(long_ids, want):
                assert d in x.passage_ids.tolist(), (d, kw)      # the long docs reach the cut and the top_k
            for name, h, exact in (("pairs", gpu, True), ("tokens", tokens, True), ("no filter", gpu, False)):
                h.set_fast_exact(exact)
                res = h.search_batch(qs, pg)
                w = h.last_work_counters()
                h.set_fast_exact(True)
                assert (w["n_filter_docs"] > 0) == exact, (name, kw, w)
                assert (w["n_exact_pairs"] > 0) == (name == "pairs"), (name, kw, w)
                for r, x in zip(res, want):
                    assert _same(r, x), (name, kw)
    finally:
        tokens.close()
        gpu.close()


def test_long_documents_decompress_and_exhaustive(oracle, npb, dcorpus):
    ix, where = dcorpus
    ids = [int(d) for d in where] + [int(where[-1]), 0, 10 ** 9]
    gpu = _gpu_index(npb, ix)
    try:
        emb, lens = gpu.decompress_documents(ids)
        assert lens.tolist() == LONG_LENGTHS + [4097, int(ix.doc_lengths[0]), 0]
        want = np.concatenate([oracle.get_document_embeddings(ix, d) for d in ids[:-1]], 0)
        assert np.array_equal(emb, want)
        long_ids = [int(d) for d, n in zip(where, LONG_LENGTHS) if n >= 129]
        qs = _queries_from(oracle, ix, long_ids[:3] + [0], [32, 65, 1, 0], seed=5)
        ex = gpu.exhaustive_scores(qs)
        for i, q in enumerate(qs):
            assert np.array_equal(ex[i], oracle.exhaustive_scores(ix, q)), i
        docs = [oracle.get_document_embeddings(ix, int(d)) for d in where]
        _check_float64(ex[:, where], qs, docs)
    finally:
        gpu.close()


def test_append_one_very_long_document_then_delete_it(oracle, npb):
    # max_doclen grows from 40 to 3000 on the open handle: the exact stage's token grid must follow it
    rng = np.random.default_rng(23)
    K, D = 512, 800
    oix = _codec_index(oracle, K, np.concatenate([rng.integers(5, 41, D), [3000]]), seed=29)
    T = int(oix.doc_offsets[D])
    ivf, lens = oracle.build_ivf(oix.codes[:T], oix.doc_lengths[:D], K)
    base = oracle.Index(oix.centroids, oix.bucket_weights, oix.bucket_cutoffs, oix.codes[:T], oix.residuals[:T],
                        oix.doc_lengths[:D], ivf, lens, oix.nbits)
    new_codes, new_res = oix.codes[T:], oix.residuals[T:]
    gpu = _gpu_index(npb, base)
    try:
        assert gpu.append_encoded(new_codes, new_res, [3000]) == [D]
        qs = _queries_from(oracle, oix, [D, D, D, 7], [32, 48, 8, 32], seed=2)
        kws = (dict(top_k=10, n_ivf_probe=8, n_full_scores=256),
               dict(top_k=20, n_ivf_probe=4, n_full_scores=512, centroid_batch_size=100))
        for kw in kws:
            pg, po = _params(npb, oracle, **kw)
            res_ = gpu.search_batch(qs, pg)
            w = gpu.last_work_counters()
            assert w["n_filter_docs"] > 0, (kw, w)
            for i, (q, r) in enumerate(zip(qs, res_)):
                assert _same(r, oracle.search_one(oix, q, po)), (kw, i)
                if i < 3:
                    assert r.passage_ids[0] == D, (kw, i)
        assert gpu.delete([D]) == 1 and gpu.num_documents() == D
        for kw in kws:
            pg, po = _params(npb, oracle, **kw)
            for i, (q, r) in enumerate(zip(qs, gpu.search_batch(qs, pg))):
                assert _same(r, oracle.search_one(base, q, po)), (kw, i)
                assert D not in r.passage_ids.tolist()
    finally:
        gpu.close()


# ---------------------------------------------------------------------------------------------------------------------
# 3. exhaustive scores across blocks of 65536 documents and 32 queries
# ---------------------------------------------------------------------------------------------------------------------

def test_exhaustive_scores_across_doc_and_query_blocks(oracle, npb, tmp_path):
    # 65536 + 3000 docs (two doc blocks), 70 queries (two full query blocks and a partial one of 6); each block holds
    # one 300-token query, so every block runs with QS = 304 (maxkey 32 x 65536 x 304 x 4 bytes = 2.5 GB)
    D = (1 << 16) + 3000
    rng = np.random.default_rng(61)
    dl = rng.integers(0, 4, D)
    dl[65530:65542] = [0, 1, 130, 2, 3, 1, 129, 0, 1, 257, 2, 1]      # long docs on both sides of d = 65536
    ix = _codec_index(oracle, 512, dl, dim=32, nbits=4, seed=62, docs_per_topic=1024)
    blk = ([0, 1, 64, 65] * 8)[:31]
    lens = blk[:15] + [300] + blk[15:] + blk[::-1][:3] + [300] + blk[::-1][3:] + [65, 0, 300, 1, 64, 65]
    assert len(lens) == 70
    src = rng.integers(0, D, len(lens))
    src = [int(s) if dl[s] else 65532 for s in src]
    qs = _queries_from(oracle, ix, src, lens, seed=63)
    gpu = _gpu_index(npb, ix)
    try:
        ex = gpu.exhaustive_scores(qs)
        for i, q in enumerate(qs):
            assert np.array_equal(ex[i], oracle.exhaustive_scores(ix, q)), (i, len(q))
        cols = list(range(0, 4)) + list(range(65528, 65544)) + [D - 1]
        _check_float64(ex[:, cols], qs, [oracle.get_document_embeddings(ix, d) for d in cols])
        # a document-range shard (as bench.py scores each rank's docs): the same columns of the whole matrix, here
        # with a range that itself spans two doc blocks
        path = str(tmp_path / "idx")
        oracle.write_index(ix, path, chunk_docs=20_000)
        shard = npb.MmapIndex.load_range(path, 1000, D)
        try:
            assert np.array_equal(shard.exhaustive_scores(qs), ex[:, 1000:])
        finally:
            shard.close()
    finally:
        gpu.close()


@pytest.mark.parametrize("dim", [32, 64, 96, 256])
@pytest.mark.parametrize("nbits", [1, 2, 8])
def test_exhaustive_scores_small_dims_and_bit_widths(oracle, npb, dim, nbits):
    rng = np.random.default_rng(dim * 10 + nbits)
    dl = np.concatenate([rng.integers(0, 30, 200), [0, 1, 127, 128, 129, 300]])
    ix = _codec_index(oracle, 128, dl, dim=dim, nbits=nbits, seed=dim + nbits)
    qs = _queries_from(oracle, ix, [201, 203, 205, 204, 5], [1, 33, 65, 8, 0], seed=nbits)
    gpu = _gpu_index(npb, ix)
    try:
        ex = gpu.exhaustive_scores(qs)
        for i, q in enumerate(qs):
            assert np.array_equal(ex[i], oracle.exhaustive_scores(ix, q)), (dim, nbits, i)
        cols = list(range(200, 206))
        _check_float64(ex[:, cols], qs, [oracle.get_document_embeddings(ix, d) for d in cols])
    finally:
        gpu.close()


# ---------------------------------------------------------------------------------------------------------------------
# 4. the device-resident search call
# ---------------------------------------------------------------------------------------------------------------------

def _search_device(gpu, qs, pg, torch):
    """search_batch_device on torch tensors; the outputs start as garbage so that untouched entries show"""
    dim = gpu.embedding_dim()
    flat = np.concatenate([q.reshape(-1, dim) for q in qs], 0).astype(np.float32)
    offs = np.zeros(len(qs) + 1, np.int64)
    offs[1:] = np.cumsum([len(q) for q in qs])
    d_q = torch.from_numpy(flat).cuda()
    d_ids = torch.full((len(qs), pg.top_k), -7, dtype=torch.int64, device="cuda")
    d_sc = torch.full((len(qs), pg.top_k), -7.0, dtype=torch.float32, device="cuda")
    d_cn = torch.full((len(qs),), -7, dtype=torch.int32, device="cuda")
    gpu.search_batch_device(d_q.data_ptr(), offs, pg, d_ids.data_ptr(), d_sc.data_ptr(), d_cn.data_ptr())
    torch.cuda.synchronize()
    return d_ids.cpu().numpy(), d_sc.cpu().numpy(), d_cn.cpu().numpy()


def test_device_resident_search_equals_host_search(oracle, npb, qcorpus):
    import torch
    ix = qcorpus
    lens = [32, 0, 5, 48, 64, 1, 100, 32, 17, 65, 32, 9, 0, 40, 33, 2, 32, 31]
    qs = _queries_from(oracle, ix, np.random.default_rng(9).integers(0, ix.num_documents, len(lens)), lens, seed=10)
    b0 = 1500                                            # a doc range opened on its own, ids offset by b0
    t0, t1 = int(ix.doc_offsets[b0]), int(ix.doc_offsets[3500])
    part_dl = ix.doc_lengths[b0:3500]
    handles = [("whole", _gpu_index(npb, ix)),
               ("range", npb.MmapIndex.from_arrays(ix.centroids, ix.bucket_weights, ix.codes[t0:t1],
                                                   ix.residuals[t0:t1], part_dl, None, None, ix.nbits,
                                                   doc_id_base=b0))]
    try:
        for name, gpu in handles:
            for kw in (dict(top_k=10, n_ivf_probe=8, n_full_scores=256),
                       dict(top_k=25, n_ivf_probe=16, n_full_scores=512, centroid_batch_size=1000)):
                pg = npb.SearchParameters(**kw)
                for lanes in (1, 3):
                    gpu.set_lanes(lanes)
                    host = gpu.search_batch(qs, pg)
                    wh = gpu.last_work_counters()
                    ids, sc, cn = _search_device(gpu, qs, pg, torch)
                    wd = gpu.last_work_counters()
                    assert wd["n_candidates"] == wh["n_candidates"] > 0 and wd["n_k1_tc"] == wh["n_k1_tc"] > 0, (wh, wd)
                    for i, r in enumerate(host):
                        assert cn[i] == len(r.passage_ids), (name, kw, lanes, i)
                        assert ids[i, :cn[i]].tolist() == r.passage_ids.tolist(), (name, kw, lanes, i)
                        assert np.array_equal(sc[i, :cn[i]], r.scores), (name, kw, lanes, i)
                    assert cn[1] == 0 and cn[12] == 0
                    if name == "range":
                        assert all(b0 <= v < 3500 for i in range(len(qs)) for v in ids[i, :cn[i]])
            # everything pruned by the threshold: the counts are cleared on the device
            pg = npb.SearchParameters(top_k=10, centroid_score_threshold=2.0)
            for lanes in (1, 3):
                gpu.set_lanes(lanes)
                ids, sc, cn = _search_device(gpu, qs, pg, torch)
                assert cn.tolist() == [0] * len(qs), (name, lanes)
        # the host search of the whole index is the oracle's (the device one equals it above)
        gpu = handles[0][1]
        gpu.set_lanes(1)
        pg, po = _params(npb, oracle, top_k=10, n_ivf_probe=8, n_full_scores=256)
        for q, r in zip(qs[:6], gpu.search_batch(qs[:6], pg)):
            assert _same(r, oracle.search_one(ix, q, po))
    finally:
        for _, h in handles:
            h.set_lanes(1)
            h.close()


# ---------------------------------------------------------------------------------------------------------------------
# 5. maxsim_scores
# ---------------------------------------------------------------------------------------------------------------------

def _unit(rng, n, dim):
    x = rng.standard_normal((n, dim)).astype(np.float32)
    return (x / np.maximum(np.linalg.norm(x, axis=1, keepdims=True), 1e-30)).astype(np.float32)


@pytest.mark.parametrize("dim", [32, 64, 96, 128, 256])
@pytest.mark.parametrize("nq", [1, 31, 32, 33, 64, 65, 300])
def test_maxsim_scores_at_odd_lengths(oracle, npb, dim, nq):
    rng = np.random.default_rng(dim * 1000 + nq)
    docs = [_unit(rng, n, dim) for n in (0, 1, 127, 128, 129, 1000, 5, 0, 3)]
    q = _unit(rng, nq, dim)
    q[0] = docs[5][17]                                   # an exact match in the 1000-token doc
    got = npb.maxsim_scores(q, docs)
    want = np.array([oracle.maxsim_score(q, d) for d in docs], np.float32)
    assert np.array_equal(got, want), (dim, nq)
    assert got[0] == 0.0 and got[7] == 0.0
    _check_float64(got[None, :], [q], docs)


def test_maxsim_scores_over_more_than_one_grid_wave(oracle, npb):
    # the kernel's grid is at most 16 CTAs per SM over 128-token tiles (270 336 tokens on 132 SMs): 560 000 tokens make
    # every CTA loop, and documents of 127..1000 tokens span tiles at every offset
    rng = np.random.default_rng(77)
    lens = rng.integers(0, 29, 50_000)
    lens[::997] = rng.choice([127, 128, 129, 1000], len(lens[::997]))
    dim = 32
    flat = _unit(rng, int(lens.sum()), dim)
    off = np.concatenate([[0], np.cumsum(lens)])
    assert off[-1] > 2 * 132 * 16 * 128
    docs = [flat[off[i]:off[i + 1]] for i in range(len(lens))]
    q = _unit(rng, 33, dim)
    got = npb.maxsim_scores(q, docs)
    want = np.array([oracle.maxsim_score(q, d) for d in docs], np.float32)
    assert np.array_equal(got, want)
    pick = list(range(0, len(docs), 211)) + [len(docs) - 1]
    _check_float64(got[None, pick], [q], [docs[i] for i in pick])
