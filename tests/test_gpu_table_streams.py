"""One stream of the tensor-core score table for a3 and a5: the probe's chunk maxima come from k_scores16_tc's epilogue
(16-row slab maxima, k_chunkmax_slabs) and the live-row bitmap of the pruned first approximate pass from
k_collect16_tc's loads.  PB_TABLE_DIAG=1 reruns the standalone k_chunkmax16 and k_a5_live on the same table and counts
the words that differ (table_diag_mismatch); it must stay 0 while the results equal the CPU oracle.

Covered: dims 48 / 64 / 96 / 128; every query-row width of the path, each length searched as its own batch (QS = 8, 16,
24, 32, 64: 1, 2, 3, 4 and 8 lanes per table row, QS = 24 leaving two lanes of a warp idle); chunks of 32, 64, 128, 256
and 1024 centroids; K not a multiple of 128; K = 2^20 (the bitmap read from global memory by k_a5_bound) with the batch
cut into 3 lanes; per-query n_ivf_probe; the PB_A5_LIVE extremes; and a batch with a non-finite query (redone on the
exact path).  Each check also confirms that the diagnostic ran: its 4 launches per tensor-core pass show in the probe
stage's launch count against a handle without it."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ENVS = ("PB_TABLE_DIAG", "PB_A5_LIVE", "PB_A5_PRUNE", "PB_K1_TC")
LENS = [1, 8, 12, 20, 31, 32, 33, 48, 64]   # QS 8, 8, 16, 24, 32, 32, 64, 64, 64


@pytest.fixture(scope="module")
def npb():
    import next_plaid_b200 as m
    m.build_library()
    if m.device_count() < 1:
        pytest.fail("GPU tests need an H100; the library has no CPU fallback")
    return m


def _codec_index(oracle, dim, K, D=3000, nbits=4, seed=5):
    """Codes drawn mostly from per-topic pools (so probes find dense cells), random residual bytes, unit centroids."""
    rng = np.random.default_rng(seed)
    cent = rng.standard_normal((K, dim), dtype=np.float32)
    cent /= np.linalg.norm(cent, axis=1, keepdims=True)
    dl = rng.integers(10, 50, D).astype(np.int64)
    N = int(dl.sum())
    pools = rng.integers(0, K, (D // 64, 64))
    topic = np.repeat(rng.integers(0, len(pools), D), dl)
    u = rng.random(N)
    from_pool = pools[topic, np.minimum((u * u * 64).astype(np.int64), 63)]
    codes = np.where(rng.random(N) < 0.75, from_pool, rng.integers(0, K, N)).astype(np.int64)
    res = rng.integers(0, 256, (N, dim * nbits // 8), dtype=np.uint8)
    w = (0.05 * np.linspace(-1.8, 1.8, 1 << nbits)).astype(np.float32)
    cut = ((w[1:] + w[:-1]) / 2).astype(np.float32)
    ivf, lens = oracle.build_ivf(codes, dl, K)
    return oracle.Index(cent, w, cut, codes, res, dl, ivf, lens, nbits)


def _queries(oracle, ix, lens, seed, noise=0.15):
    rng = np.random.default_rng(seed)
    out = []
    for nq in lens:
        tok = oracle.get_document_embeddings(ix, int(rng.integers(ix.num_documents)))
        tok = tok[rng.integers(0, len(tok), nq)]
        nz = rng.standard_normal(tok.shape).astype(np.float32)
        q = tok + noise * nz / np.linalg.norm(nz, axis=1, keepdims=True)
        out.append((q / np.linalg.norm(q, axis=1, keepdims=True)).astype(np.float32))
    return out


def _open(npb, ix, monkeypatch, env, diag=True):
    for k in ENVS:
        monkeypatch.delenv(k, raising=False)
    env = dict(env, PB_TABLE_DIAG="1") if diag else dict(env)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    try:
        return npb.MmapIndex.from_arrays(ix.centroids, ix.bucket_weights, ix.codes, ix.residuals, ix.doc_lengths,
                                         ix.ivf, ix.ivf_lengths, ix.nbits)
    finally:
        for k in env:
            monkeypatch.delenv(k)


def _same(r, w):
    return r.passage_ids.tolist() == w.passage_ids.tolist() and np.array_equal(r.scores, w.scores)


def _probe_launches(h):
    return h.last_stage_stats()[1]["probe"]


def _check(npb, h, plain, qs, kws, want, lanes=1):
    """search qs (one parameter set per query) on the diagnostic handle: fused = standalone, results = the oracle's
    (want), and the diagnostic's k_chunkmax16 / k_a5_live / two compares ran once per tensor-core pass (QS <= 64: the
    pass prunes, so both compares run) -- counted against the same search on `plain`, a handle without it"""
    ps = [npb.SearchParameters(**kw) for kw in kws]
    for x in (h, plain):
        x.set_lanes(lanes)
    plain.search_batch_params(qs, ps)
    base = _probe_launches(plain)
    got = h.search_batch_params(qs, ps)
    w = h.last_work_counters()
    assert w["table_diag_mismatch"] == 0, (kws[0], len(qs[0]), w)
    assert w["n_k1_tc"] > 0 and w["n_k1_tc_redo"] == 0, w
    assert _probe_launches(h) - base == 4 * w["n_k1_tc"], (_probe_launches(h), base, w)
    for i, (r, x) in enumerate(zip(got, want)):
        assert _same(r, x), (i, len(qs[i]), kws[i])
    return w


# (K, n_ivf_probe) -> chunk_rows: 1024 centroids unless fewer than 2 n chunks would exist
@pytest.mark.parametrize("dim,K,n,chunk_rows", [
    (48, 1000, 16, 32), (64, 1024, 8, 64), (96, 2048, 8, 128), (128, 5000, 2, 1024), (128, 2048, 4, 256),
])
def test_fused_chunk_maxima_and_live_bits_equal_the_standalone_kernels(oracle, npb, dim, K, n, chunk_rows, monkeypatch):
    ix = _codec_index(oracle, dim, K, seed=dim + K)
    plain = _open(npb, ix, monkeypatch, {}, diag=False)
    handles = {name: _open(npb, ix, monkeypatch, env) for name, env in
               (("default", {}), ("all_live", {"PB_A5_LIVE": str(1 << 40)}), ("none_live", {"PB_A5_LIVE": "0"}))}
    try:
        for nq in LENS:   # one batch per length: the pass's QS is that of its longest query
            qs = _queries(oracle, ix, [nq] * 3, seed=dim + n + nq)
            for kws in ([dict(top_k=10, n_ivf_probe=n, n_full_scores=64)] * len(qs),
                        [dict(top_k=10, n_ivf_probe=max(1, n >> i), n_full_scores=64,
                              centroid_batch_size=(None if i % 2 else 300)) for i in range(len(qs))]):
                kws = [{k: v for k, v in kw.items() if v is not None} for kw in kws]
                want = [oracle.search_one(ix, q, oracle.SearchParameters(**kw)) for q, kw in zip(qs, kws)]
                for name, h in handles.items():
                    w = _check(npb, h, plain, qs, kws, want)
                    if name == "none_live":
                        assert w["n_a5_live_rows"] == 0, w
                    if name == "all_live":
                        assert w["n_a5_live_rows"] == w["n_candidate_tokens"], w
    finally:
        plain.close()
        for h in handles.values():
            h.close()


def test_k_2_20_with_lanes(oracle, npb, monkeypatch):
    # K = 2^20: the live bitmap (128 KiB per query) stays in global memory for k_a5_bound.  24 queries: 3 lanes of 8
    # (a batch is laned from 16 queries on, at most one lane per 8), each one tensor-core pass
    ix = _codec_index(oracle, 48, 1 << 20, D=2000, seed=20)
    plain = _open(npb, ix, monkeypatch, {}, diag=False)
    h = _open(npb, ix, monkeypatch, {})
    try:
        kw = dict(top_k=10, n_ivf_probe=8, n_full_scores=64)
        for nq in (20, 32):
            qs = _queries(oracle, ix, [nq] * 24, seed=21 + nq)
            want = [oracle.search_one(ix, q, oracle.SearchParameters(**kw)) for q in qs]
            for lanes in (1, 3):
                w = _check(npb, h, plain, qs, [kw] * len(qs), want, lanes=lanes)
                assert w["n_k1_tc"] == lanes, (lanes, w)   # the batch really was cut into `lanes` slices
                assert w["n_a5_live_rows"] > 0, w
    finally:
        plain.close()
        h.close()


def test_non_finite_query_is_redone_on_the_exact_path(oracle, npb, monkeypatch):
    ix = _codec_index(oracle, 128, 2048, seed=9)
    qs = _queries(oracle, ix, [32, 32, 17], seed=10)
    bad = qs[1].copy()
    bad[2, 3] = np.nan
    batch = [qs[0], bad, qs[2]]
    h = _open(npb, ix, monkeypatch, {})
    try:
        kw = dict(top_k=10, n_ivf_probe=8, n_full_scores=64)
        got = h.search_batch(batch, npb.SearchParameters(**kw))
        w = h.last_work_counters()
        assert w["n_k1_tc_redo"] > 0 and w["table_diag_mismatch"] == 0, w
        po = oracle.SearchParameters(**kw)
        for i in (0, 2):
            assert _same(got[i], oracle.search_one(ix, batch[i], po)), i
    finally:
        h.close()
