"""Incremental append (pb_index_append*, MmapIndex::update_append + reload, index.rs:1675): after every append the live
handle equals a fresh pb_index_open of the concatenated arrays -- accessors, inverted file, decompression, search ids
and scores bit for bit, and the work counters, which show that the filter's constants (vmin, wmax, max_doclen) match
too -- and the CPU oracle on the concatenated index.  The directory side reproduces update_index's file changes."""
import json
import os
import sys
import threading

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from ivf_merge import merge_ivf  # noqa: E402

pytestmark = pytest.mark.gpu

NBITS, K, DIM = 2, 256, 128
COUNTERS = ("n_exact_docs", "n_exact_pairs", "n_recheck_docs", "n_filter_docs")
PARAMS = [dict(top_k=10, n_ivf_probe=8, n_full_scores=256),
          dict(top_k=5, n_ivf_probe=4, n_full_scores=64, centroid_batch_size=100),
          dict(top_k=10, n_ivf_probe=8, n_full_scores=256, centroid_score_threshold=None)]


@pytest.fixture(scope="module")
def npb():
    import next_plaid_b200 as m
    m.build_library()
    if m.device_count() < 1:
        pytest.fail("GPU tests need an H100; the library has no CPU fallback")
    return m


@pytest.fixture(scope="module")
def corpus(oracle):
    """2238 ragged docs encoded by the oracle with one fixed codec (K = 256 centroids drawn from the corpus)."""
    docs = oracle.synthetic_corpus(2238, 40, dim=DIM, seed=51, ragged=True)
    flat = np.concatenate(docs, 0)
    rng = np.random.default_rng(2)
    cent = flat[rng.choice(len(flat), K, replace=False)].copy()
    art = oracle.prepare_codec_artifacts(docs, cent, NBITS, 3)
    codes, packed, dl = oracle.encode_documents(docs, art, NBITS)
    off = np.zeros(len(dl) + 1, np.int64)
    np.cumsum(dl, out=off[1:])
    qs, _ = oracle.synthetic_queries(docs, 6, nq=32, seed=8)
    qs += oracle.synthetic_queries(docs[1500:], 2, nq=32, seed=9)[0]      # aimed at appended docs
    return dict(docs=docs, art=art, codes=codes, packed=packed, dl=dl, off=off, qs=qs)


def _prefix(c, D):
    t = int(c["off"][D])
    return c["codes"][:t], c["packed"][:t], c["dl"][:D]


def _open(npb, oracle, art, codes, packed, dl, with_ivf=True):
    ivf, lens = oracle.build_ivf(codes, dl, K) if with_ivf else (None, None)
    return npb.MmapIndex.from_arrays(art.centroids, art.bucket_weights, codes, packed, dl, ivf, lens, NBITS)


def _oracle_index(oracle, art, codes, packed, dl):
    ivf, lens = oracle.build_ivf(codes, dl, K)
    return oracle.Index(art.centroids, art.bucket_weights, art.bucket_cutoffs, codes, packed, dl, ivf, lens, NBITS)


def _search(ix, npb, qs, kw, subset=None):
    res = ix.search_batch(qs, npb.SearchParameters(**kw), subset=subset)
    w = ix.last_work_counters()
    return [(r.passage_ids.tolist(), r.scores.tobytes()) for r in res], {k: w[k] for k in COUNTERS}


def _set_paths(ix, on):
    ix.set_scores_tc(on)
    ix.set_fast_exact(on)
    ix.set_fast_approx(1 if on else 0)


def _check_same(npb, oracle, app, fresh, oix, qs, ids):
    """app (appended) == fresh (opened on the concatenation) == the oracle on the concatenation."""
    assert app.num_documents() == fresh.num_documents() == oix.num_documents
    assert app.num_embeddings() == fresh.num_embeddings() == oix.num_embeddings
    assert app.avg_doclen() == fresh.avg_doclen()
    a_ivf, a_len = app.export_ivf()
    assert np.array_equal(a_ivf, oix.ivf) and np.array_equal(a_len, oix.ivf_lengths)
    ea, la = app.decompress_documents(ids)
    ef, lf = fresh.decompress_documents(ids)
    assert np.array_equal(la, lf) and np.array_equal(ea, ef)
    want = [oracle.get_document_embeddings(oix, d) for d in ids if d < oix.num_documents]
    if want and sum(len(w) for w in want):
        assert np.array_equal(ea, np.concatenate(want, 0))
    subset = sorted(set(range(0, oix.num_documents, 3)) | set(range(max(oix.num_documents - 40, 0), oix.num_documents)))
    for on in (True, False):
        _set_paths(app, on)
        _set_paths(fresh, on)
        for kw in PARAMS:
            for sub in (None, subset):
                ra, ca = _search(app, npb, qs, kw, sub)
                rf, cf = _search(fresh, npb, qs, kw, sub)
                assert ra == rf, (kw, on, sub is not None)
                assert ca == cf, (kw, on, sub is not None, ca, cf)
                if on:
                    po = oracle.SearchParameters(**kw)
                    for q, (pid, sc) in zip(qs, ra):
                        w = oracle.search_one(oix, q, po, subset=sub)
                        assert pid == w.passage_ids.tolist() and sc == w.scores.astype(np.float32).tobytes(), kw
    _set_paths(app, True)


@pytest.mark.parametrize("with_ivf,reserve", [(True, False), (False, False), (True, True)],
                         ids=["ivf_given", "ivf_built_on_device", "reserved"])
def test_appends_match_a_fresh_open(npb, oracle, corpus, with_ivf, reserve):
    c = corpus
    D = 1500
    app = _open(npb, oracle, c["art"], *_prefix(c, D), with_ivf=with_ivf)
    try:
        if reserve:
            app.reserve(len(c["dl"]), int(c["off"][-1]))
        prev_ivf, prev_len = app.export_ivf()
        for n in (1, 0, 37, 700):
            t0, t1 = int(c["off"][D]), int(c["off"][D + n])
            got = app.append_encoded(c["codes"][t0:t1], c["packed"][t0:t1], c["dl"][D:D + n])
            assert got == list(range(D, D + n))
            merged = merge_ivf(prev_ivf, prev_len, c["codes"][t0:t1], c["dl"][D:D + n], D, K)
            D += n
            codes, packed, dl = _prefix(c, D)
            oix = _oracle_index(oracle, c["art"], codes, packed, dl)
            assert np.array_equal(merged[0], oix.ivf) and np.array_equal(merged[1], oix.ivf_lengths)
            fresh = _open(npb, oracle, c["art"], codes, packed, dl, with_ivf=with_ivf)
            try:
                _check_same(npb, oracle, app, fresh, oix, c["qs"], [0, 777, 1499, D - 1, D - n, D + 5])
            finally:
                fresh.close()
            prev_ivf, prev_len = app.export_ivf()
    finally:
        app.close()


def test_filter_constants_move(npb, oracle, corpus):
    # new docs whose residuals push max |w| up (every dim in the largest-|weight| bucket) and min |c + w| down (per dim
    # the bucket closest to -c), one longer than any doc so far: parity (and equal work counters) still hold
    c = corpus
    art = c["art"]
    D = 1500
    codes0, packed0, dl0 = _prefix(c, D)
    app = _open(npb, oracle, art, codes0, packed0, dl0)
    try:
        rng = np.random.default_rng(4)
        w = art.bucket_weights
        far = int(np.argmax(np.abs(w)))
        long_len = int(dl0.max()) + 9
        n_codes = rng.integers(0, K, 3 + long_len)
        near = np.argmin(np.abs(art.centroids[n_codes][:, :, None] + w[None, None, :]), axis=2)
        buckets = near.copy()
        buckets[:2] = far
        # packed rows with these per-dim buckets: quantize each bucket's own weight
        rows = oracle.quantize_residuals(w[buckets].astype(np.float32), art.bucket_cutoffs, NBITS)
        dl_new = np.array([2, 1, long_len], np.int64)

        def wnorms(codes, packed):
            # |w| and the pre-normalisation |c + w| per token; a value's bits are its bucket bit-reversed, MSB-first
            bits = np.unpackbits(packed, axis=1).reshape(len(codes), DIM, NBITS).astype(np.int64)
            wv = w[(bits << np.arange(NBITS)).sum(2)].astype(np.float64)
            return np.linalg.norm(wv, axis=1), np.linalg.norm(art.centroids[codes] + wv, axis=1)
        w_old, v_old = wnorms(codes0, packed0)
        w_new, v_new = wnorms(n_codes, rows)
        assert w_new.max() > w_old.max() and v_new.min() < v_old.min() and long_len > dl0.max()
        app.append_encoded(n_codes, rows, dl_new)
        codes, packed, dl = np.concatenate([codes0, n_codes]), np.concatenate([packed0, rows]), np.concatenate([dl0, dl_new])
        oix = _oracle_index(oracle, art, codes, packed, dl)
        fresh = _open(npb, oracle, art, codes, packed, dl)
        try:
            _check_same(npb, oracle, app, fresh, oix, c["qs"], [0, D, D + 1, D + 2])
        finally:
            fresh.close()
    finally:
        app.close()


def test_device_encode(npb, oracle, corpus):
    c = corpus
    art = c["art"]
    D = 1500
    app = _open(npb, oracle, art, *_prefix(c, D))
    codec = npb.ResidualCodec(NBITS, art.centroids, art.bucket_cutoffs)
    try:
        new = c["docs"][D:D + 300]
        assert app.append(new, codec) == list(range(D, D + 300))
        t0, t1 = int(c["off"][D]), int(c["off"][D + 300])
        flat = np.concatenate(new, 0)
        gc, gp = codec.encode_chunk(flat)
        assert np.array_equal(gc, c["codes"][t0:t1]) and np.array_equal(gp, c["packed"][t0:t1])
        emb, lens = app.decompress_documents(list(range(D, D + 300)))
        assert np.array_equal(lens, c["dl"][D:D + 300])
        assert np.array_equal(emb, oracle.decompress(art.centroids, art.bucket_weights, NBITS, c["packed"][t0:t1],
                                                     c["codes"][t0:t1]))
        codes, packed, dl = _prefix(c, D + 300)
        fresh = _open(npb, oracle, art, codes, packed, dl)
        try:
            _check_same(npb, oracle, app, fresh, _oracle_index(oracle, art, codes, packed, dl), c["qs"], [3, D, D + 299])
        finally:
            fresh.close()
    finally:
        codec.close()
        app.close()


def _snapshot(app, npb, qs):
    return (app.num_documents(), app.num_embeddings(), [a.tolist() for a in app.export_ivf()],
            _search(app, npb, qs, PARAMS[0]))


def test_rejections_change_nothing(npb, oracle, corpus):
    import torch
    c = corpus
    art = c["art"]
    D = 1500
    codes0, packed0, dl0 = _prefix(c, D)
    app = _open(npb, oracle, art, codes0, packed0, dl0)
    try:
        before = _snapshot(app, npb, c["qs"])
        t1 = int(c["off"][D + 5])
        bad = c["codes"][int(c["off"][D]):t1].copy()
        bad[-1] = K
        with pytest.raises(npb.PlaidError) as e:
            app.append_encoded(bad, c["packed"][int(c["off"][D]):t1], c["dl"][D:D + 5])
        assert e.value.status == 1
        assert _snapshot(app, npb, c["qs"]) == before
        other = art.centroids.copy()
        other[7, 3] = np.nextafter(other[7, 3], np.float32(2))
        codec = npb.ResidualCodec(NBITS, other, art.bucket_cutoffs)
        with pytest.raises(npb.PlaidError) as e:
            app.append(c["docs"][D:D + 5], codec)
        codec.close()
        assert e.value.status == 1
        nocut = npb.ResidualCodec(NBITS, art.centroids)
        with pytest.raises(npb.PlaidError) as e:
            app.append(c["docs"][D:D + 5], nocut)
        nocut.close()
        assert e.value.status == 1
        assert _snapshot(app, npb, c["qs"]) == before
    finally:
        app.close()
    # a member of a shard group
    a, b = _open(npb, oracle, art, *_prefix(c, 10)), _open(npb, oracle, art, *_prefix(c, 10))
    g = npb.ShardGroup([a, b])
    try:
        with pytest.raises(npb.PlaidError) as e:
            a.append_encoded(c["codes"][:3], c["packed"][:3], [3])
        assert e.value.status == 4 and a.num_documents() == 10
        with pytest.raises(npb.PlaidError) as e:
            a.reserve(100, 10_000)
        assert e.value.status == 4
    finally:
        g.close()
    # a handle on the caller's residual array
    dev = torch.device("cuda", 0)
    codes, packed, dl = _prefix(c, 100)
    t = {k: torch.from_numpy(np.ascontiguousarray(v)).to(dev) for k, v in dict(
        cen=art.centroids, w=art.bucket_weights, codes=codes, res=packed, dl=dl).items()}
    ad = npb.MmapIndex.from_device_pointers(DIM, NBITS, K, 100, len(codes), t["cen"].data_ptr(), t["w"].data_ptr(),
                                            t["codes"].data_ptr(), t["res"].data_ptr(), t["dl"].data_ptr(), None, None,
                                            adopt_residuals=True)
    try:
        with pytest.raises(npb.PlaidError) as e:
            ad.append_encoded(c["codes"][:3], c["packed"][:3], [3])
        assert e.value.status == 4 and ad.num_documents() == 100 and ad.num_embeddings() == len(codes)
    finally:
        ad.close()


def test_directory_append(npb, oracle, tmp_path):
    docs = oracle.synthetic_corpus(5610, 40, dim=DIM, seed=61, ragged=True)
    path = str(tmp_path / "ix")
    gpu = npb.create_index(docs[:2500], path, nbits=NBITS, num_partitions=K, batch_size=1000, seed=7)
    gpu.close()
    base = oracle.load_index(path)
    codec = npb.ResidualCodec(NBITS, base.centroids, base.bucket_cutoffs)
    live = npb.MmapIndex.load(path)
    qs, _ = oracle.synthetic_queries(docs, 6, nq=32, seed=4)

    def chunk(i):
        with open(os.path.join(path, f"doclens.{i}.json")) as f:
            dl = json.load(f)
        with open(os.path.join(path, f"{i}.metadata.json")) as f:
            return dl, json.load(f)

    def check(n_docs, chunk_docs):
        ix = oracle.load_index(path)
        flat = np.concatenate(docs[:n_docs], 0)
        codes = oracle.compress_into_codes(flat, base.centroids)
        assert ix.num_documents == n_docs and np.array_equal(ix.codes, codes)
        assert np.array_equal(ix.residuals, oracle.quantize_residuals(oracle.residuals_of(flat, base.centroids, codes),
                                                                      base.bucket_cutoffs, NBITS))
        ivf, lens = oracle.build_ivf(codes, ix.doc_lengths, K)
        assert np.array_equal(ix.ivf, ivf) and np.array_equal(ix.ivf_lengths, lens)
        off = 0
        for i, nd in enumerate(chunk_docs):
            dl, meta = chunk(i)
            assert len(dl) == nd and meta == dict(num_documents=nd, num_embeddings=sum(dl), embedding_offset=off), i
            off += sum(dl)
        assert not os.path.exists(os.path.join(path, f"{len(chunk_docs)}.codes.npy"))
        assert not [f for f in os.listdir(path) if f.startswith("merged_") or f.endswith(".tmp")]
        loaded = npb.MmapIndex.load(path)
        try:
            for kw in PARAMS[:2]:
                a = live.search_batch(qs, npb.SearchParameters(**kw))
                b = loaded.search_batch(qs, npb.SearchParameters(**kw))
                for q, x, y in zip(qs, a, b):
                    w = oracle.search_one(ix, q, oracle.SearchParameters(**kw))
                    assert x.passage_ids.tolist() == y.passage_ids.tolist() == w.passage_ids.tolist(), kw
                    assert np.array_equal(x.scores, w.scores) and np.array_equal(y.scores, w.scores), kw
        finally:
            loaded.close()

    try:
        for f in ("merged_codes.npy", "merged_residuals.manifest.json"):
            open(os.path.join(path, f), "w").write("stale")
        steps = [(2500, 1700, 1000, [1000, 1000, 1500, 700]),     # last chunk 500 < 2000 takes the first batch
                 (4200, 1400, 2000, [1000, 1000, 1500, 2100]),    # 700 + 1400
                 (5600, 10, 1000, [1000, 1000, 1500, 2100, 10])]  # last chunk has >= 2000 docs: a new chunk
        for d0, n, bs, chunks in steps:
            meta0 = json.load(open(os.path.join(path, "metadata.json")))
            new_tok = sum(d.shape[0] for d in docs[d0:d0 + n])
            assert live.append(docs[d0:d0 + n], codec, index_dir=path, batch_size=bs) == list(range(d0, d0 + n))
            meta = json.load(open(os.path.join(path, "metadata.json")))
            assert meta["num_chunks"] == len(chunks) and meta["num_documents"] == d0 + n
            assert meta["num_embeddings"] == meta0["num_embeddings"] + new_tok
            assert meta["avg_doclen"] == (meta0["avg_doclen"] * d0 + new_tok) / (d0 + n)     # update.rs:1089-1094
            assert (meta["nbits"], meta["num_partitions"], meta["embedding_dim"]) == (NBITS, K, DIM)
            check(d0 + n, chunks)
        # a directory that does not hold the handle's documents is refused before anything is written
        meta = open(os.path.join(path, "metadata.json")).read()
        other = npb.MmapIndex.load(path)
        other.append(docs[:2], codec)
        with pytest.raises(npb.PlaidError) as e:
            other.append(docs[2:4], codec, index_dir=path)
        other.close()
        assert e.value.status == 1 and open(os.path.join(path, "metadata.json")).read() == meta
    finally:
        codec.close()
        live.close()


@pytest.mark.parametrize("lanes", [1, 2])
def test_searches_see_all_or_nothing_of_an_append(npb, oracle, corpus, lanes):
    c = corpus
    D, n = 1500, 700
    qs = (c["qs"] * 2)[:16]                                  # >= 16 queries so that 2 lanes engage
    kw = PARAMS[0]
    app = _open(npb, oracle, c["art"], *_prefix(c, D))
    post = _open(npb, oracle, c["art"], *_prefix(c, D + n))
    try:
        app.set_lanes(lanes)
        before = _search(app, npb, qs, kw)[0]
        after = _search(post, npb, qs, kw)[0]
        assert before != after
        seen, errs, done = [], [], threading.Event()

        def searcher():
            try:
                extra = 3
                while extra > 0:
                    if done.is_set():
                        extra -= 1
                    seen.append(_search(app, npb, qs, kw)[0])
            except Exception as e:  # noqa: BLE001 - reported below
                errs.append(e)
        ths = [threading.Thread(target=searcher) for _ in range(2)]
        [t.start() for t in ths]
        t0, t1 = int(c["off"][D]), int(c["off"][D + n])
        app.append_encoded(c["codes"][t0:t1], c["packed"][t0:t1], c["dl"][D:D + n])
        done.set()
        [t.join() for t in ths]
        assert not errs, errs
        assert all(s == before or s == after for s in seen)
        assert seen.count(after) >= 6 and _search(app, npb, qs, kw)[0] == after   # 3 per thread start after it
    finally:
        app.close()
        post.close()
