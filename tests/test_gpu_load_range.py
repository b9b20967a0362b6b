"""A document range of an index directory as one shard (pb_index_load_range, pb_index_dir_shard_bounds): each range
handle equals pb_index_open of the numpy-sliced arrays with the slice of ivf.npy (tests/ivf_slice.py) -- accessors,
inverted file, decompression, searches bit for bit with their work counters -- [0, D) equals pb_index_load, and an
in-process shard group of load_shard handles returns what load and the CPU oracle on the directory return."""
import json
import os
import sys
import threading

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from ivf_slice import ivf_slice, shard_arrays, shard_bounds  # noqa: E402
from test_gpu_append import PARAMS, _search, _set_paths  # noqa: E402

pytestmark = pytest.mark.gpu

NBITS, K, DIM, CHUNK = 4, 256, 128, 200


@pytest.fixture(scope="module")
def npb():
    import next_plaid_b200 as m
    m.build_library()
    if m.device_count() < 1:
        pytest.fail("GPU tests need an H100; the library has no CPU fallback")
    return m


@pytest.fixture(scope="module")
def corpus(oracle):
    docs = oracle.synthetic_corpus(1000, 40, dim=DIM, seed=91, ragged=True)
    ix = oracle.create_index(docs[:900], nbits=NBITS, seed=4, num_partitions=K)
    qs, _ = oracle.synthetic_queries(docs[:900], 8, nq=32, seed=19)
    return dict(docs=docs, ix=ix, qs=qs)


@pytest.fixture(scope="module")
def written(oracle, corpus, tmp_path_factory):
    path = str(tmp_path_factory.mktemp("ix"))
    oracle.write_index(corpus["ix"], path, chunk_docs=CHUNK)      # chunks of 200 docs, the last of 100
    return path


def _state(npb, h, qs, ids):
    """Everything a handle shows: accessors, inverted file (global ids), decompression, searches with counters."""
    out = [h.num_documents(), h.num_embeddings(), h.num_partitions(), h.avg_doclen(), h.embedding_dim(), h.nbits()]
    out += [a.tolist() for a in h.export_ivf()]
    emb, lens = h.decompress_documents(ids)
    out += [lens.tolist(), emb.tobytes()]
    for on in (True, False):
        _set_paths(h, on)
        for kw in PARAMS:
            out.append(_search(h, npb, qs, kw))
    _set_paths(h, True)
    return out


def _probe_ids(b, e):
    return sorted({b, (b + e) // 2, e - 1}) if e > b else []


def _from_slice(npb, ix, b, e):
    codes, res, dl, ivf, lens = shard_arrays(ix, b, e)
    return npb.MmapIndex.from_arrays(ix.centroids, ix.bucket_weights, codes, res, dl, ivf, lens, ix.nbits,
                                     doc_id_base=b)


def _check_range(npb, oracle, path, ix, qs, b, e):
    """load_range(b, e) of the directory holding `ix` == pb_index_open of the sliced arrays"""
    got = npb.MmapIndex.load_range(path, b, e)
    want = _from_slice(npb, ix, b, e)
    try:
        sl, sll = ivf_slice(ix.ivf, ix.ivf_lengths, b, e)
        gi, gl = got.export_ivf()
        assert np.array_equal(gi, sl + b) and np.array_equal(gl, sll), (b, e)
        ids = _probe_ids(b, e)
        assert _state(npb, got, qs, ids) == _state(npb, want, qs, ids), (b, e)
        for d in ids:                                          # decompression takes global ids
            assert np.array_equal(got.decompress_documents([d])[0], oracle.get_document_embeddings(ix, d)), d
    finally:
        got.close()
        want.close()


def test_whole_range_equals_load(npb, corpus, written):
    D, qs = corpus["ix"].num_documents, corpus["qs"]
    full, rng = npb.MmapIndex.load(written), npb.MmapIndex.load_range(written, 0, D)
    try:
        ids = [0, 199, 200, 450, D - 1]
        assert _state(npb, rng, qs, ids) == _state(npb, full, qs, ids)
        assert [a.tolist() for a in full.export_ivf()] == [corpus["ix"].ivf.tolist(), corpus["ix"].ivf_lengths.tolist()]
    finally:
        full.close()
        rng.close()


def _ranges(npb, path, D):
    out = set()
    for W in (1, 2, 3, 8):                                     # token-balanced
        b = npb.shard_bounds(path, W)
        assert b.tolist() == shard_bounds(np.concatenate([json.load(open(os.path.join(path, f"doclens.{i}.json")))
                                                          for i in range((D + CHUNK - 1) // CHUNK)]), W).tolist()
        out |={(int(b[r]), int(b[r + 1])) for r in range(W)}
    out |= {(r * D // 4, (r + 1) * D // 4) for r in range(4)}   # equal-doc
    for c in (200, 400):                                       # at a chunk boundary and one doc either side
        for x in (c - 1, c, c + 1):
            out |= {(x, 600), (100, x)}
    out |= {(437, 438), (0, 1), (D - 1, D), (300, 300), (0, 0), (D, D), (800, D)}   # one doc, empty, last chunk
    return sorted(out)


def test_each_range_equals_an_open_of_the_sliced_arrays(npb, oracle, corpus, written):
    ix = corpus["ix"]
    for b, e in _ranges(npb, written, ix.num_documents):
        _check_range(npb, oracle, written, ix, corpus["qs"], b, e)


@pytest.mark.parametrize("slab", ["1", "31", "1000"])
def test_lists_straddling_staging_slabs(npb, oracle, corpus, written, monkeypatch, slab):
    """ivf.npy streamed in slabs of a few entries: lists straddle slabs, count and write passes re-read the file"""
    monkeypatch.setenv("PB_LOAD_IVF_SLAB", slab)
    ix = corpus["ix"]
    for b, e in ((0, ix.num_documents), (199, 601), (437, 438)):
        _check_range(npb, oracle, written, ix, corpus["qs"][:4], b, e)


def _group_check(npb, oracle, path, oix, qs, W):
    """load_shard group == load == the oracle on the directory, on every rank"""
    full = npb.MmapIndex.load(path)
    grp = npb.ShardGroup([npb.MmapIndex.load_shard(path, r, W) for r in range(W)])
    D = oix.num_documents
    try:
        cases = [(dict(top_k=10, n_ivf_probe=8, n_full_scores=256, centroid_batch_size=cbs), None)
                 for cbs in (100_000, 128)]
        # top_k > n_full_scores / 4; subset with the batched variant (the dense one is not built for doc shards)
        cases += [(dict(top_k=50, n_ivf_probe=4, n_full_scores=64, centroid_batch_size=128), None),
                  (dict(top_k=10, n_ivf_probe=8, n_full_scores=256, centroid_batch_size=128), list(range(0, D, 3)))]
        for kw, sub in cases:
            res = grp.search_batch(qs, npb.SearchParameters(**kw), subset=sub)
            ref = full.search_batch(qs, npb.SearchParameters(**kw), subset=sub)
            for per_rank in grp.all_results:
                for a, b in zip(per_rank, res):
                    assert a.passage_ids.tolist() == b.passage_ids.tolist() and np.array_equal(a.scores, b.scores)
            for q, g, f in zip(qs, res, ref):
                w = oracle.search_one(oix, q, oracle.SearchParameters(**kw), subset=sub)
                assert g.passage_ids.tolist() == f.passage_ids.tolist() == w.passage_ids.tolist(), (W, kw)
                assert np.array_equal(g.scores, f.scores) and np.array_equal(g.scores, w.scores), (W, kw)
    finally:
        grp.close()
        full.close()


@pytest.mark.parametrize("W", [2, 3])
def test_group_of_load_shard_equals_load_and_oracle(npb, oracle, corpus, written, W):
    _group_check(npb, oracle, written, oracle.load_index(written), corpus["qs"], W)


def test_ivf_that_is_not_the_rebuild(npb, oracle, corpus, written, tmp_path):
    """Lists with extra valid doc ids: a shard must hold the slice of ivf.npy, which a per-shard rebuild is not."""
    import shutil
    path = str(tmp_path / "ix")
    shutil.copytree(written, path)
    ix = corpus["ix"]
    rng = np.random.default_rng(23)
    off = ix.ivf_offsets
    lists = []
    for c in range(K):
        lst = set(ix.ivf[off[c]:off[c + 1]].tolist())
        if c % 3 == 0:
            lst |= set(rng.integers(0, ix.num_documents, 12).tolist())
        lists.append(sorted(lst))
    np.save(os.path.join(path, "ivf.npy"), np.array([x for lst in lists for x in lst], np.int64))
    np.save(os.path.join(path, "ivf_lengths.npy"), np.array([len(lst) for lst in lists], np.int32))
    oix = oracle.load_index(path)
    assert len(oix.ivf) > len(ix.ivf)
    b = npb.shard_bounds(path, 3)
    for r in range(3):
        sh = npb.MmapIndex.load_shard(path, r, 3)
        try:
            s, e = int(b[r]), int(b[r + 1])
            sl, sll = ivf_slice(oix.ivf, oix.ivf_lengths, s, e)
            t0, t1 = int(oix.doc_offsets[s]), int(oix.doc_offsets[e])
            rebuilt = oracle.build_ivf(oix.codes[t0:t1], oix.doc_lengths[s:e], K)
            assert not np.array_equal(sl, rebuilt[0])
            gi, gl = sh.export_ivf()
            assert np.array_equal(gi, sl + s) and np.array_equal(gl, sll)
        finally:
            sh.close()
    _check_range(npb, oracle, path, oix, corpus["qs"], 150, 650)
    _group_check(npb, oracle, path, oix, corpus["qs"], 3)


def test_fast_plaid_directory(npb, oracle, corpus, written, tmp_path):
    import shutil
    path = str(tmp_path / "ix")
    shutil.copytree(written, path)
    for name in ("centroids.npy", "bucket_weights.npy", "bucket_cutoffs.npy", "avg_residual.npy"):
        p = os.path.join(path, name)
        np.save(p, np.load(p).astype(np.float16))
    p = os.path.join(path, "ivf_lengths.npy")
    np.save(p, np.load(p).astype(np.int64))
    oix = oracle.load_index(path)                             # widened: the values the loader uses
    for b, e in ((0, oix.num_documents), (150, 650), (800, 900)):
        _check_range(npb, oracle, path, oix, corpus["qs"], b, e)


def test_directory_after_append_and_delete(npb, oracle, corpus, tmp_path):
    docs, qs = corpus["docs"], corpus["qs"]
    path = str(tmp_path / "ix")
    npb.create_index(docs[:900], path, nbits=NBITS, num_partitions=K, batch_size=CHUNK, seed=7).close()
    live = npb.MmapIndex.load(path)
    try:
        assert live.delete(list(range(200, 400)) + [5, 650], index_dir=path) == 202     # chunk 1 emptied
        base = oracle.load_index(path)
        codec = npb.ResidualCodec(NBITS, base.centroids, base.bucket_cutoffs)
        try:
            live.append(docs[900:950], codec, index_dir=path, batch_size=CHUNK)
        finally:
            codec.close()
    finally:
        live.close()
    assert json.load(open(os.path.join(path, "doclens.1.json"))) == []
    oix = oracle.load_index(path)
    D = oix.num_documents
    assert D == 748
    # doc 199 is the first after chunk 0, which is also where the emptied chunk 1 sits
    for b, e in ((150, 250), (199, 300), (100, 199), (199, 199), (198, 200), (0, D), (600, D)):
        _check_range(npb, oracle, path, oix, qs, b, e)
    _group_check(npb, oracle, path, oix, qs, 3)


def test_concurrent_loads_equal_sequential(npb, corpus, written):
    W, qs = 4, corpus["qs"][:4]
    b = npb.shard_bounds(written, W)
    seq = []
    for r in range(W):
        h = npb.MmapIndex.load_shard(written, r, W)
        seq.append(_state(npb, h, qs, _probe_ids(int(b[r]), int(b[r + 1]))))
        h.close()
    hs, err = [None] * W, [None] * W

    def run(r):
        try:
            hs[r] = npb.MmapIndex.load_shard(written, r, W)
        except Exception as e:      # noqa: BLE001 - re-raised below
            err[r] = e
    ths = [threading.Thread(target=run, args=(r,)) for r in range(W)]
    [t.start() for t in ths]
    [t.join() for t in ths]
    try:
        assert err == [None] * W, err
        for r in range(W):
            assert _state(npb, hs[r], qs, _probe_ids(int(b[r]), int(b[r + 1]))) == seq[r], r
    finally:
        for h in hs:
            if h is not None:
                h.close()


def test_out_of_range_ivf_entry_is_refused_by_every_rank(npb, corpus, written, tmp_path):
    import shutil
    path = str(tmp_path / "ix")
    shutil.copytree(written, path)
    ix = corpus["ix"]
    D = ix.num_documents
    W = 3
    b = npb.shard_bounds(path, W)
    ivf = ix.ivf.copy()
    # a list entry in the last shard's range becomes D: only that shard's range would have read it
    j = int(np.flatnonzero(ivf >= b[W - 1])[0])
    ivf[j] = D
    np.save(os.path.join(path, "ivf.npy"), ivf)
    for r in range(W):
        with pytest.raises(npb.PlaidError) as e:
            npb.MmapIndex.load_shard(path, r, W)
        assert e.value.status == 1 and "ivf" in str(e.value), r
    with pytest.raises(npb.PlaidError) as e:
        npb.MmapIndex.load(path)
    assert e.value.status == 1


def test_range_handles_refuse_directory_append_and_delete(npb, oracle, corpus, written, tmp_path):
    import shutil
    path = str(tmp_path / "ix")
    shutil.copytree(written, path)
    ix = corpus["ix"]
    D = ix.num_documents

    def dir_bytes():
        return {f: open(os.path.join(path, f), "rb").read() for f in sorted(os.listdir(path))}
    files = dir_bytes()
    codec = npb.ResidualCodec(NBITS, ix.centroids, ix.bucket_cutoffs)
    try:
        for (b, e), status in (((300, D), 4), ((0, 600), 1)):
            h = npb.MmapIndex.load_range(path, b, e)
            try:
                with pytest.raises(npb.PlaidError) as err:
                    h.delete([b + 1], index_dir=path)
                assert err.value.status == status, (b, e)
                with pytest.raises(npb.PlaidError) as err:
                    h.append(corpus["docs"][900:903], codec, index_dir=path)
                assert err.value.status == status, (b, e)
                assert h.num_documents() == e - b and dir_bytes() == files
            finally:
                h.close()
    finally:
        codec.close()
