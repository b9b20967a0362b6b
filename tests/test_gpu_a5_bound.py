"""k_a5_bound's staging (next-plaid_b200/csrc/k_approx16.cuh): the shapes its ring of bulk copies and its bitmap
placement switch on.  Every result and counter of the pruned first pass equals the dense first pass (PB_A5_PRUNE=0).

Covered: K = 2^20 (the live bitmap does not fit shared memory and is tested from global memory), doc lists that span
several ring slots (more than 256 distinct codes, more slots than a consumer warp owns, and a doc above PB_UCODE_MAX
tokens that keeps its raw code list), and one batch whose queries' candidate counts differ by orders of magnitude.
Both row-group widths run: queries of up to 32 tokens (LPR = 4) and of 33 to 64 (LPR = 8)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

KW = dict(top_k=10, n_ivf_probe=8, n_full_scores=64)
COUNTERS = ("n_candidates", "n_candidate_tokens", "n_recheck_docs", "n_exact_docs", "n_exact_pairs", "n_filter_docs")
ENVS = ("PB_A5_PRUNE", "PB_A5_LIVE", "PB_A5_M1", "PB_A5_WAVES")
PRUNED = {"default": {}, "all_live": {"PB_A5_LIVE": str(1 << 40)}, "one_wave": {"PB_A5_WAVES": "1"}}


@pytest.fixture(scope="module")
def npb():
    import next_plaid_b200 as m
    m.build_library()
    if m.device_count() < 1:
        pytest.fail("GPU tests need an H100; the library has no CPU fallback")
    return m


def _index(oracle, dim, K, doc_lengths, seed, pool_frac=0.75):
    """Codes drawn mostly from per-topic pools of 64 centroids (so probes find shared cells), the rest uniformly over
    all K; random residual bytes, unit centroids, 4-bit."""
    rng = np.random.default_rng(seed)
    cent = rng.standard_normal((K, dim), dtype=np.float32)
    cent /= np.linalg.norm(cent, axis=1, keepdims=True)
    dl = np.asarray(doc_lengths, np.int64)
    D, N = len(dl), int(dl.sum())
    pools = rng.integers(0, K, (max(D // 32, 2), 64))
    topic = np.repeat(rng.integers(0, len(pools), D), dl)
    u = rng.random(N)
    from_pool = pools[topic, np.minimum((u * u * 64).astype(np.int64), 63)]
    codes = np.where(rng.random(N) < pool_frac, from_pool, rng.integers(0, K, N)).astype(np.int64)
    res = rng.integers(0, 256, (N, dim // 2), dtype=np.uint8)
    w = (0.05 * np.linspace(-1.8, 1.8, 16)).astype(np.float32)
    cut = ((w[1:] + w[:-1]) / 2).astype(np.float32)
    ivf, lens = oracle.build_ivf(codes, dl, K)
    return oracle.Index(cent, w, cut, codes, res, dl, ivf, lens, 4)


def _queries(oracle, ix, lens, seed, docs=None):
    rng = np.random.default_rng(seed)
    out = []
    for k, nq in enumerate(lens):
        d = int(docs[k]) if docs is not None else int(rng.integers(ix.num_documents))
        tok = oracle.get_document_embeddings(ix, d)
        tok = tok[rng.integers(0, len(tok), nq)]
        nz = rng.standard_normal(tok.shape).astype(np.float32)
        q = tok + 0.15 * nz / np.linalg.norm(nz, axis=1, keepdims=True)
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


def _flat(res):
    return [(r.passage_ids.tolist(), r.scores.tobytes()) for r in res]


def _compare(npb, ix, monkeypatch, batches, search=None):
    """every batch on the dense first pass and on each pruned variant: results and counters identical.  Returns the
    dense pass's (results, counters) per batch."""
    search = search or (lambda h, qs, pg: h.search_batch(qs, pg))
    pg = npb.SearchParameters(**KW)
    dense = _open(npb, ix, monkeypatch, {"PB_A5_PRUNE": "0"})
    pruned = {name: _open(npb, ix, monkeypatch, env) for name, env in PRUNED.items()}
    seen = []
    try:
        for qs in batches:
            want = search(dense, qs, pg)
            wd = dense.last_work_counters()
            assert wd["n_a5_live_rows"] == 0 and wd["n_a5_dense_docs"] == 0, wd
            for name, h in pruned.items():
                got = search(h, qs, pg)
                w = h.last_work_counters()
                mode = (name, [len(q) for q in qs], w, wd)
                assert _flat(got) == _flat(want), mode
                for k in COUNTERS:
                    assert w[k] == wd[k], (k, mode)
                assert 0 < w["n_a5_dense_docs"] <= w["n_candidates"], mode
                if name == "all_live":
                    assert w["n_a5_live_rows"] == w["n_candidate_tokens"], mode
            seen.append((want, wd))
    finally:
        dense.close()
        for h in pruned.values():
            h.close()
    return seen


def test_bitmap_beyond_shared_memory(oracle, npb, monkeypatch):
    """K = 2^20: 128 KiB of live bits per query, tested from global memory"""
    rng = np.random.default_rng(20)
    ix = _index(oracle, 48, 1 << 20, rng.integers(20, 120, 600), seed=20, pool_frac=0.9)
    batches = [_queries(oracle, ix, [32] * 4, seed=1), _queries(oracle, ix, [40, 64, 1], seed=2)]
    seen = _compare(npb, ix, monkeypatch, batches)
    assert all(w["n_candidates"] > 0 for _, w in seen), seen


def test_lists_spanning_ring_slots(oracle, npb, monkeypatch):
    """docs with 300 to ~1900 distinct codes (2 to 8 slots of 256; a consumer warp owns 4) and one of 6000 tokens,
    above PB_UCODE_MAX = 4096, whose raw list fills 24 slots"""
    rng = np.random.default_rng(7)
    dl = rng.integers(20, 80, 1500)
    long_docs = [3, 4, 5, 100, 101, 700, 1499]
    dl[long_docs] = [600, 1200, 2500, 900, 400, 3000, 1800]
    dl[1000] = 6000
    ix = _index(oracle, 64, 8192, dl, seed=8, pool_frac=0.3)
    # queries taken from the long docs, so that they are candidates (and score near the cut)
    src = long_docs + [1000]
    batches = [_queries(oracle, ix, [32] * len(src), seed=3, docs=src),
               _queries(oracle, ix, [48] * len(src), seed=4, docs=src)]
    seen = _compare(npb, ix, monkeypatch, batches)
    # the long lists were bounded: every long doc is a candidate of (and returned for) the query drawn from it
    for res, _ in seen:
        for d, r in zip(src, res):
            assert d in r.passage_ids.tolist(), (d, r.passage_ids)


def test_candidate_counts_far_apart(oracle, npb, monkeypatch):
    """one batch whose queries hold from a handful to thousands of candidates: subsets of 4 docs, 64 docs and none,
    at 1 and 32 query tokens"""
    rng = np.random.default_rng(11)
    ix = _index(oracle, 128, 4096, rng.integers(20, 60, 8000), seed=12)
    qs = _queries(oracle, ix, [32, 32, 1, 32, 32, 1], seed=5)
    subsets = [None, sorted(rng.choice(8000, 4, replace=False).tolist()), None,
               sorted(rng.choice(8000, 64, replace=False).tolist()), None, [0, 1, 2, 3]]
    pg = npb.SearchParameters(**KW)
    counts = []
    probe = _open(npb, ix, monkeypatch, {})
    try:
        for q, s in zip(qs, subsets):
            probe.search_batch_subsets([q], pg, [s])
            counts.append(probe.last_work_counters()["n_candidates"])
    finally:
        probe.close()
    assert max(counts) >= 100 * max(1, min(counts)), counts
    _compare(npb, ix, monkeypatch, [qs], search=lambda h, b, p: h.search_batch_subsets(b, p, subsets))
