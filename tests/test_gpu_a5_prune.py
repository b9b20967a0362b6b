"""The pruned first pass of a5 (k_a5_bound and its two k_approx16 rounds, next-plaid_b200/csrc/k_approx16.cuh): every
result and every downstream counter equals the dense first pass (PB_A5_PRUNE=0) bit for bit, and the CPU oracle.

Covered: dims 48 / 64 / 96 / 128, nbits 1 / 2 / 4 / 8, query lengths on both sides of the QS <= 64 gate, the dense and
batched variants and subsets, lanes 1 and 3, forced floors (0: every row live; above every code: none; high ones with
M1 = M, so that round 2 runs), a host-tier handle, a 2-shard group, and an index after appends and deletes."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

KW = (dict(top_k=10, n_ivf_probe=8, n_full_scores=64),
      dict(top_k=10, n_ivf_probe=8, n_full_scores=64, centroid_batch_size=1000))
LENS = [1, 31, 32, 33, 64, 65]
COUNTERS = ("n_candidates", "n_candidate_tokens", "n_recheck_docs", "n_exact_docs", "n_exact_pairs", "n_filter_docs")
ENVS = ("PB_A5_PRUNE", "PB_A5_LIVE", "PB_A5_M1")


@pytest.fixture(scope="module")
def npb():
    import next_plaid_b200 as m
    m.build_library()
    if m.device_count() < 1:
        pytest.fail("GPU tests need an H100; the library has no CPU fallback")
    return m


def _codec_index(oracle, dim, nbits, K=2048, D=4000, seed=5):
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


def _open(npb, ix, monkeypatch, env, **kw):
    for k in ENVS:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    try:
        return npb.MmapIndex.from_arrays(ix.centroids, ix.bucket_weights, ix.codes, ix.residuals, ix.doc_lengths,
                                         ix.ivf, ix.ivf_lengths, ix.nbits, **kw)
    finally:
        for k in env:
            monkeypatch.delenv(k)


def _flat(res):
    return [(r.passage_ids.tolist(), r.scores.tobytes()) for r in res]


def _same(r, w):
    return r.passage_ids.tolist() == w.passage_ids.tolist() and np.array_equal(r.scores, w.scores)


FLOORS = {"default": {}, "all_live": {"PB_A5_LIVE": str(1 << 40)}, "none_live": {"PB_A5_LIVE": "0"},
          **{f"high{n}": {"PB_A5_LIVE": str(n), "PB_A5_M1": "1"} for n in (1, 4, 16)}}   # high floors with M1 = M


def _cut(kw):
    """M, the docs of the cut: min(n_full_scores, max(n_full_scores / 4, top_k))"""
    return min(kw["n_full_scores"], max(kw["n_full_scores"] // 4, kw["top_k"]))


@pytest.mark.parametrize("dim,nbits", [(48, 4), (64, 4), (96, 4), (128, 1), (128, 2), (128, 4), (128, 8)])
def test_pruned_first_pass_equals_dense_and_oracle(oracle, npb, dim, nbits, monkeypatch):
    ix = _codec_index(oracle, dim, nbits, seed=dim + nbits)
    subset = sorted(np.random.default_rng(dim).choice(ix.num_documents, 2500, replace=False).tolist())
    dense = _open(npb, ix, monkeypatch, {"PB_A5_PRUNE": "0"})
    pruned = {name: _open(npb, ix, monkeypatch, env) for name, env in FLOORS.items()}
    try:
        pruned_any = round2 = False
        for nq in LENS:
            qs = _queries(oracle, ix, [nq] * 3, seed=nq * 10 + dim + nbits)
            for kw in KW:
                pg, po = npb.SearchParameters(**kw), oracle.SearchParameters(**kw)
                for sub in (None, subset):
                    want = dense.search_batch(qs, pg, subset=sub)
                    wd = dense.last_work_counters()
                    assert wd["n_a5_dense_docs"] == 0 and wd["n_a5_live_rows"] == 0, wd
                    if nq in (1, 33, 65):
                        for q, r in zip(qs, want):
                            assert _same(r, oracle.search_one(ix, q, po, subset=sub)), (nq, kw)
                    for name, h in pruned.items():
                        got = h.search_batch(qs, pg, subset=sub)
                        w = h.last_work_counters()
                        mode = (nq, kw, sub is not None, name, w, wd)
                        assert _flat(got) == _flat(want), mode
                        for k in COUNTERS:
                            assert w[k] == wd[k], (k, mode)
                        if nq > 64:   # QS > 64: the dense first pass
                            assert w["n_a5_dense_docs"] == 0, mode
                            continue
                        assert 0 < w["n_a5_dense_docs"] <= w["n_candidates"], mode
                        if name == "default":
                            pruned_any |= w["n_a5_dense_docs"] < w["n_candidates"]
                        if name == "none_live":
                            assert w["n_a5_live_rows"] == 0, mode
                        if name == "all_live":
                            assert w["n_a5_live_rows"] == w["n_candidate_tokens"], mode
                        if name.startswith("high"):   # |R1| = M per query (no ties at theta1): more is round 2
                            round2 |= w["n_a5_dense_docs"] > len(qs) * _cut(kw) and \
                                w["n_a5_dense_docs"] < w["n_candidates"]
        assert pruned_any, "the default floor never pruned a candidate"
        assert round2, "round 2 of the pruned pass never ran"
    finally:
        dense.close()
        for h in pruned.values():
            h.close()


def test_lanes_and_host_tier(oracle, npb, monkeypatch):
    ix = _codec_index(oracle, 128, 4, seed=77)
    qs = _queries(oracle, ix, [32] * 7, seed=3)
    dense = _open(npb, ix, monkeypatch, {"PB_A5_PRUNE": "0"})
    hosts = [_open(npb, ix, monkeypatch, {}, host_residuals=hr) for hr in (False, True)]
    try:
        for kw in KW:
            pg = npb.SearchParameters(**kw)
            want = dense.search_batch(qs, pg)
            wd = dense.last_work_counters()
            for h in hosts:
                for lanes in (1, 3):
                    h.set_lanes(lanes)
                    got = h.search_batch(qs, pg)
                    w = h.last_work_counters()
                    assert _flat(got) == _flat(want), (kw, lanes, w)
                    for k in COUNTERS:
                        assert w[k] == wd[k], (k, kw, lanes, w, wd)
                    assert 0 < w["n_a5_dense_docs"] < w["n_candidates"], (kw, lanes, w)
    finally:
        dense.close()
        for h in hosts:
            h.close()


def test_shard_group_after_appends_and_deletes(oracle, npb, tmp_path, monkeypatch):
    docs = oracle.synthetic_corpus(3200, 40, dim=128, seed=33, ragged=True)
    path = str(tmp_path / "ix")
    npb.create_index(docs[:3000], path, nbits=4, num_partitions=256, batch_size=1000, seed=7).close()
    base = oracle.load_index(path)
    qs, _ = oracle.synthetic_queries(docs, 6, nq=32, seed=4)
    codec = npb.ResidualCodec(4, base.centroids, base.bucket_cutoffs)
    for k in ENVS:
        monkeypatch.delenv(k, raising=False)
    grp = npb.ShardGroup([npb.MmapIndex.load_shard(path, r, 2) for r in range(2)])
    live = npb.MmapIndex.load(path)
    monkeypatch.setenv("PB_A5_PRUNE", "0")
    dense = npb.MmapIndex.load(path)
    monkeypatch.delenv("PB_A5_PRUNE")
    try:
        for step in ("as built", "appended", "deleted"):
            if step == "appended":
                for h in (live, dense):
                    assert h.append_encoded(*_encode(codec, docs[3000:3200])) == list(range(3000, 3200))
                grp.append_encoded(*_encode(codec, docs[3000:3200]))
            if step == "deleted":
                ids = [0, 5, 999, 1000, 2999, 3000, 3199]
                for h in (live, dense):
                    assert h.delete(ids) == len(ids)
                grp.delete(ids)
            for kw in KW:
                pg = npb.SearchParameters(**kw)
                want = dense.search_batch(qs, pg)
                wd = dense.last_work_counters()
                got = live.search_batch(qs, pg)
                w = live.last_work_counters()
                assert _flat(got) == _flat(want), (step, kw)
                for k in COUNTERS:
                    assert w[k] == wd[k], (k, step, kw, w, wd)
                assert w["n_a5_dense_docs"] > 0, (step, kw, w)
                assert _flat(grp.search_batch(qs, pg)) == _flat(want), (step, kw)
                if step == "as built":
                    po = oracle.SearchParameters(**kw)
                    for q, r in zip(qs, want):
                        assert _same(r, oracle.search_one(base, q, po)), kw
    finally:
        codec.close()
        live.close()
        dense.close()
        grp.close()


def _encode(codec, docs):
    codes, packed = codec.encode_chunk(np.concatenate(docs, 0))
    return codes, packed, [len(d) for d in docs]
