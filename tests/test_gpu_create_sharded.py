"""pb_create_index_sharded on one H100: G build ranks of an in-process group (one host thread each, all on device 0)
build one index directory together.  With the same centroids it is pb_create_index's directory byte for byte; with
k-means at 0 iterations too (sample membership, K, the fit subsample and the seeds are pinned); each rank's returned
shard is pb_index_load_range of its range, and a ShardGroup of them searches as the unsharded index does."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_gpu_create_index import _check_directory  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def npb():
    import next_plaid_b200 as m
    m.build_library()
    if m.device_count() < 1:
        pytest.fail("GPU tests need an H100; the library has no CPU fallback")
    return m


def _files(path):
    return {f: open(os.path.join(path, f), "rb").read() for f in sorted(os.listdir(path))}


def _assert_same_dir(a, b):
    fa, fb = _files(a), _files(b)
    assert sorted(fa) == sorted(fb)
    for f in fa:
        assert fa[f] == fb[f], f


def _split(docs, sizes):
    assert sum(sizes) == len(docs)
    out, o = [], 0
    for n in sizes:
        out.append(docs[o:o + n])
        o += n
    return out


def _close(handles):
    for h in handles:
        h.close()


# 700 docs in chunks of 100: even splits, a boundary on a chunk edge, and an empty rank with chunk 1 (docs 100-199)
# spread over ranks 0, 2, 3 and 4
SPLITS = {1: [[700]], 2: [[350, 350]], 3: [[234, 233, 233], [200, 300, 200]],
          5: [[140] * 5, [120, 0, 30, 40, 510]]}


@pytest.mark.parametrize("dim,nbits", [(128, 4), (128, 2), (48, 4)])
def test_given_centroids_same_bytes(npb, oracle, tmp_path, dim, nbits):
    docs = oracle.synthetic_corpus(700, 30, dim=dim, seed=dim + nbits, ragged=True)
    a = str(tmp_path / "a")
    npb.create_index(docs, a, nbits=nbits, num_partitions=256, batch_size=100, seed=3).close()
    cen = np.load(os.path.join(a, "centroids.npy"))
    for G, splits in SPLITS.items():
        for sizes in splits:
            b = str(tmp_path / f"b{G}_{'_'.join(map(str, sizes))}")
            hs = npb.create_index_sharded(_split(docs, sizes), b, centroids=cen, nbits=nbits, num_partitions=256,
                                          batch_size=100, seed=3)
            _close(hs)
            _assert_same_dir(a, b)


@pytest.fixture(scope="module")
def big(oracle):
    # D > 30 720 short docs: the k-means and codec samples are strict subsets, and K * 256 < sampled tokens
    return oracle.synthetic_corpus(32_000, 6, dim=128, seed=21, ragged=True), None


def test_big_corpus_given_centroids(npb, tmp_path, big):
    docs, _ = big
    a = str(tmp_path / "a")
    npb.create_index(docs, a, num_partitions=256, batch_size=5000, kmeans_niters=1).close()
    cen = np.load(os.path.join(a, "centroids.npy"))
    b = str(tmp_path / "b")
    _close(npb.create_index_sharded(_split(docs, [9000, 0, 13000, 10000]), b, centroids=cen, num_partitions=256,
                                    batch_size=5000, kmeans_niters=1))
    _assert_same_dir(a, b)


@pytest.mark.parametrize("G", [1, 3])
def test_kmeans_pinned_at_zero_iterations(npb, oracle, tmp_path, big, G):
    docs, _ = big
    a = str(tmp_path / "a")
    npb.create_index(docs, a, num_partitions=256, batch_size=5000, kmeans_niters=0).close()
    b = str(tmp_path / "b")
    sizes = [len(docs)] if G == 1 else [5001, 20000, len(docs) - 25001]
    _close(npb.create_index_sharded(_split(docs, sizes), b, num_partitions=256, batch_size=5000, kmeans_niters=0))
    _assert_same_dir(a, b)
    # the K heuristic of kmeans.rs:304-309 as well
    small = oracle.synthetic_corpus(900, 20, dim=64, seed=4, ragged=True)
    c, d = str(tmp_path / "c"), str(tmp_path / "d")
    npb.create_index(small, c, kmeans_niters=0, batch_size=200).close()
    _close(npb.create_index_sharded(_split(small, [300, 0, 600][:G] if G == 3 else [900]), d, kmeans_niters=0,
                                    batch_size=200))
    _assert_same_dir(c, d)


def test_kmeans_running(npb, oracle, tmp_path):
    docs = oracle.synthetic_corpus(2500, 40, dim=128, seed=33, ragged=True)
    qs, _ = oracle.synthetic_queries(docs, 12, nq=32, seed=3)
    a = str(tmp_path / "a")
    ref = npb.create_index(docs, a, nbits=2, batch_size=1000, seed=7)
    K = ref.num_partitions()
    ref.close()
    b = str(tmp_path / "b")
    hs = npb.create_index_sharded(_split(docs, [800, 1, 1699]), b, nbits=2, batch_size=1000, seed=7)
    try:
        assert [h.num_partitions() for h in hs] == [K] * 3
        probe = np.concatenate(qs[:2], 0)
        sc = [h.centroid_scores(probe) for h in hs]                 # every rank holds the same centroids
        assert all(np.array_equal(s, sc[0]) for s in sc)
        loaded = npb.MmapIndex.load(b)
        try:
            got = _check_directory(oracle, npb, docs, b, loaded, 2, qs, [dict(top_k=10, n_ivf_probe=8, n_full_scores=256)])
            assert got.num_centroids == K
        finally:
            loaded.close()
    finally:
        _close(hs)


def _state(h, ids):
    emb, lens = h.decompress_documents(ids)
    return ([h.num_documents(), h.num_embeddings(), h.num_partitions(), h.embedding_dim(), h.nbits()],
            [a.tolist() for a in h.export_ivf()], emb.tobytes(), lens.tolist(), h.memory_usage())


def test_shards_equal_load_range_and_search_as_one(npb, oracle, tmp_path):
    docs = oracle.synthetic_corpus(1500, 40, dim=128, seed=8, ragged=True)
    qs, _ = oracle.synthetic_queries(docs, 10, nq=32, seed=2)
    b = str(tmp_path / "b")
    sizes = [400, 0, 350, 750]
    hs = npb.create_index_sharded(_split(docs, sizes), b, num_partitions=512, batch_size=300, seed=11)
    full = npb.MmapIndex.load(b)
    oix = oracle.load_index(b)
    try:
        base = np.concatenate([[0], np.cumsum(sizes)])
        for r, h in enumerate(hs):
            assert h.first_doc_id == base[r]
            want = npb.MmapIndex.load_range(b, int(base[r]), int(base[r + 1]))
            try:
                ids = list(range(int(base[r]), int(base[r + 1])))
                assert _state(h, ids) == _state(want, ids), r
            finally:
                want.close()
        grp = npb.ShardGroup(hs)
        try:
            subset = list(range(0, 1500, 3))
            for kw, sub in [(dict(top_k=10, n_ivf_probe=8, n_full_scores=256), None),
                            (dict(top_k=20, n_ivf_probe=4, n_full_scores=64, centroid_batch_size=100), None),
                            (dict(top_k=10, n_ivf_probe=8, n_full_scores=256), subset)]:
                pg, po = npb.SearchParameters(**kw), oracle.SearchParameters(**kw)
                got = grp.search_batch(qs, pg, subset=sub)
                one = full.search_batch(qs, pg, subset=sub)
                for q, x, y in zip(qs, got, one):
                    w = oracle.search_one(oix, q, po, subset=sub)
                    assert x.passage_ids.tolist() == y.passage_ids.tolist() == w.passage_ids.tolist(), kw
                    assert np.array_equal(x.scores, y.scores) and np.array_equal(x.scores, w.scores), kw
        finally:
            grp.close()
    finally:
        full.close()
        _close(hs)


def test_device_input_same_directory(npb, oracle, tmp_path):
    import torch
    docs = oracle.synthetic_corpus(600, 30, dim=128, seed=14, ragged=True)
    a, b = str(tmp_path / "a"), str(tmp_path / "b")
    sizes = [250, 0, 350]
    _close(npb.create_index_sharded(_split(docs, sizes), a, num_partitions=256, batch_size=100, kmeans_niters=0))
    dev = [[torch.from_numpy(np.ascontiguousarray(d, np.float32)).cuda() for d in part] for part in _split(docs, sizes)]
    _close(npb.create_index_sharded(dev, b, num_partitions=256, batch_size=100, kmeans_niters=0, dim=128))
    _assert_same_dir(a, b)


def _refused(npb, G, call):
    """call(r) on every rank of an in-process build group; every rank must fail with the same status"""
    import ctypes as C
    from next_plaid_b200.index import _per_rank
    L = npb.load_library()
    g = C.c_void_p()
    assert L.pb_shard_group_create(G, C.byref(g)) == 0
    out = [None] * G

    def run(r):
        h = C.c_void_p()
        assert L.pb_build_comm_group(g, r, 0, C.byref(h)) == 0
        try:
            out[r] = call(r, h)
        finally:
            L.pb_build_comm_destroy(h)
    try:
        _per_rank(G, run)
    finally:
        L.pb_shard_group_destroy(g)
    return out


def test_refusals(npb, oracle, tmp_path):
    import ctypes as C
    from next_plaid_b200.index import _CreateParams, _ptr
    L = npb.load_library()
    docs = oracle.synthetic_corpus(90, 10, dim=128, seed=2, ragged=True)
    parts = _split(docs, [30, 30, 30])
    flat = [np.ascontiguousarray(np.concatenate(p, 0), np.float32) for p in parts]
    lens = [np.array([len(d) for d in p], np.int64) for p in parts]
    cen = np.ascontiguousarray(flat[0][:64], np.float32)
    tmp = str(tmp_path)

    def case(path_of=lambda r: os.path.join(tmp, "x"), params_of=lambda r: {}, cen_of=lambda r: None,
             n_of=lambda r: len(lens[r]), lens_of=lambda r: lens[r], dim=128):
        def call(r, h):
            kw = dict(nbits=4, kmeans_niters=1, max_points_per_centroid=256, device=0, num_partitions=16,
                      batch_size=20, seed=1)
            kw.update(params_of(r))
            p = _CreateParams(**kw)
            c = cen_of(r)
            ix, first = C.c_void_p(), C.c_int64(-1)
            st = L.pb_create_index_sharded(h, _ptr(flat[r]), _ptr(lens_of(r)), n_of(r), dim, 0, _ptr(c),
                                           0 if c is None else c.shape[0], C.byref(p), os.fsencode(path_of(r)),
                                           C.byref(ix), C.byref(first))
            return st, ix.value
        res = _refused(npb, 3, call)
        assert len({s for s, _ in res}) == 1 and res[0][0] != 0, res
        assert all(h is None for _, h in res), res
        return res[0][0]

    INVALID, IO, UNSUPPORTED = 1, 3, 4
    assert case(params_of=lambda r: dict(seed=2) if r == 1 else {}) == INVALID
    assert case(params_of=lambda r: dict(batch_size=21) if r == 2 else {}) == INVALID
    assert case(cen_of=lambda r: cen if r != 1 else cen * 2) == INVALID
    assert case(path_of=lambda r: os.path.join(tmp, "y" if r == 2 else "x")) == INVALID
    assert case(n_of=lambda r: 0) == INVALID                                       # no documents at all
    assert case(lens_of=lambda r: np.array([-1] + [1] * 29, np.int64) if r == 1 else lens[r]) == INVALID
    assert case(dim=100) == UNSUPPORTED
    open(os.path.join(tmp, "file"), "w").close()
    assert case(path_of=lambda r: os.path.join(tmp, "file", "ix")) == IO
    for d in ("x", "y"):                                                          # nothing but the directory
        p = os.path.join(tmp, d)
        assert not os.path.exists(p) or os.listdir(p) == [], d
    # centroids of the wrong dim are refused before any rank starts
    with pytest.raises(npb.PlaidError) as e:
        npb.create_index_sharded(parts, os.path.join(tmp, "z"), centroids=cen[:, :64])
    assert e.value.status == INVALID
