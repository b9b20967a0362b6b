"""The boundaries of k_scores16_tc's pipeline.  Each consumer warpgroup keeps two accumulators and issues the MMAs of
query group g + 1 before it runs the epilogue of group g, so the first group, the steady state, an odd last group and a
partial last group each take their own branch of the kernel.  None of them may change a code of the table.

Covered: 1, 2, 3 and 8 query groups of 128 rows (B QS = 128, 256, 384, 1024), a partial last group (7 queries of 20
tokens, QS = 24: 168 rows), QS = 64, K = 5000 (a partial centroid tile) and K = 2^20, dims 48 / 64 / 96 / 128, a
24-query batch in 3 lanes, and a batch with a NaN query.  Every case checks the results against the CPU oracle bit for
bit, the estimate codes against the exact table (PB_K1_TC_DIAG: at most 1 code apart), the epilogue's slab maxima
against the standalone kernels (PB_TABLE_DIAG: no word differs) and the redo counter (0, or 1 for the NaN batch)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ENVS = ("PB_TABLE_DIAG", "PB_K1_TC_DIAG", "PB_A5_LIVE", "PB_A5_PRUNE", "PB_K1_TC")


@pytest.fixture(scope="module")
def npb():
    import next_plaid_b200 as m
    m.build_library()
    if m.device_count() < 1:
        pytest.fail("GPU tests need an H100; the library has no CPU fallback")
    return m


def _codec_index(oracle, dim, K, D=2000, nbits=4, seed=5):
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


def _open(npb, ix, monkeypatch, env):
    for k in ENVS:
        monkeypatch.delenv(k, raising=False)
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


def _run(oracle, npb, monkeypatch, ix, qs, lanes, nan_at=None):
    """search qs on a handle with the table diagnostic (the tensor-core pass in charge) and on one with the code
    diagnostic (the exact table in charge, the tensor-core table computed beside it); both against the oracle"""
    kw = dict(top_k=10, n_ivf_probe=min(8, ix.centroids.shape[0] // 1024), n_full_scores=64)
    po, pg = oracle.SearchParameters(**kw), npb.SearchParameters(**kw)
    want = [None if i == nan_at else oracle.search_one(ix, q, po) for i, q in enumerate(qs)]
    table = _open(npb, ix, monkeypatch, {"PB_TABLE_DIAG": "1"})
    codes = _open(npb, ix, monkeypatch, {"PB_K1_TC_DIAG": "1"})
    try:
        table.set_lanes(lanes)
        got = table.search_batch(qs, pg)
        w = table.last_work_counters()
        assert w["table_diag_mismatch"] == 0, w
        if nan_at is None:
            assert w["n_k1_tc"] == lanes and w["n_k1_tc_redo"] == 0, (lanes, w)
        else:   # the flagged batch is handed back to the exact path, once
            assert w["n_k1_tc"] == 0 and w["n_k1_tc_redo"] == 1, w
        for i, (r, x) in enumerate(zip(got, want)):
            if x is not None:
                assert _same(r, x), (i, len(qs[i]))
        if nan_at is None:   # the code diagnostic compares every real token's codes; a NaN token has none to compare
            codes.set_lanes(lanes)
            got = codes.search_batch(qs, pg)
            w = codes.last_work_counters()
            assert w["n_k1_tc"] == 0 and 0 <= w["k1_tc_max_code_diff"] <= 1, w
            for i, (r, x) in enumerate(zip(got, want)):
                assert _same(r, x), (i, len(qs[i]))
    finally:
        table.close()
        codes.close()


# (dim, K, query lengths of the batch): B QS rows = 128 n_groups
@pytest.mark.parametrize("dim,K,lens", [
    (128, 2048, [32] * 4),             # 1 group
    (64, 2048, [32] * 8),              # 2 groups
    (96, 5000, [32] * 12),             # 3 groups (odd), a partial centroid tile
    (128, 4096, [32] * 32),            # 8 groups (config B's batch)
    (48, 5000, [20] * 7),              # QS = 24: 168 rows, the second group partial
    (128, 2048, [64, 40, 33, 64, 50]), # QS = 64: 320 rows, 3 groups
    (64, 3000, [1, 8, 5]),             # QS = 8: 24 rows, one partial group
])
def test_pipeline_boundaries(oracle, npb, monkeypatch, dim, K, lens):
    ix = _codec_index(oracle, dim, K, seed=dim + K + len(lens))
    _run(oracle, npb, monkeypatch, ix, _queries(oracle, ix, lens, seed=dim + len(lens)), lanes=1)


def test_k_2_20_and_a_batch_in_three_lanes(oracle, npb, monkeypatch):
    # 24 queries of 32 tokens: one pass of 6 groups, or 3 lanes of 8 queries (2 groups each)
    ix = _codec_index(oracle, 48, 1 << 20, seed=20)
    qs = _queries(oracle, ix, [32] * 24, seed=21)
    for lanes in (1, 3):
        _run(oracle, npb, monkeypatch, ix, qs, lanes=lanes)


def test_nan_query_is_flagged_and_redone(oracle, npb, monkeypatch):
    ix = _codec_index(oracle, 128, 2048, seed=9)
    qs = _queries(oracle, ix, [32, 32, 17], seed=10)
    qs[1] = qs[1].copy()
    qs[1][2, 3] = np.nan
    _run(oracle, npb, monkeypatch, ix, qs, lanes=1, nan_at=1)
