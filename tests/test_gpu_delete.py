"""Incremental delete (pb_index_delete, MmapIndex::delete + reload, index.rs:1805 / delete.rs:43): after every delete
the live handle equals a fresh pb_index_open of the filtered arrays -- accessors, inverted file, decompression, search
ids and scores bit for bit, and the work counters, which show that the filter's constants (vmin, wmax, max_doclen) match
too -- and the CPU oracle on the filtered index.  The directory side reproduces delete_from_index's file changes."""
import json
import os
import sys
import threading

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from ivf_delete import delete_ivf, keep_mask  # noqa: E402
from test_gpu_append import (DIM, K, NBITS, PARAMS, _check_same, _oracle_index, _search,  # noqa: E402
                             _snapshot)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def npb():
    import next_plaid_b200 as m
    m.build_library()
    if m.device_count() < 1:
        pytest.fail("GPU tests need an H100; the library has no CPU fallback")
    return m


@pytest.fixture(scope="module")
def corpus(oracle):
    """1600 ragged docs encoded by the oracle with one fixed codec (K = 256 centroids drawn from the corpus)."""
    docs = oracle.synthetic_corpus(1600, 40, dim=DIM, seed=71, ragged=True)
    flat = np.concatenate(docs, 0)
    rng = np.random.default_rng(12)
    cent = flat[rng.choice(len(flat), K, replace=False)].copy()
    art = oracle.prepare_codec_artifacts(docs, cent, NBITS, 3)
    codes, packed, dl = oracle.encode_documents(docs, art, NBITS)
    qs, _ = oracle.synthetic_queries(docs, 8, nq=32, seed=18)
    return dict(docs=docs, art=art, codes=codes, packed=packed, dl=dl, qs=qs)


class Live:
    """the arrays a handle should hold: the corpus with documents deleted (and appended) as the handle was"""

    def __init__(self, c, D):
        self.codes, self.packed, self.dl = c["codes"][:int(c["dl"][:D].sum())], c["packed"][:int(c["dl"][:D].sum())], c["dl"][:D]

    def delete(self, ids):
        docs, toks = keep_mask(self.dl, ids)
        self.codes, self.packed, self.dl = self.codes[toks], self.packed[toks], self.dl[docs]

    def append(self, codes, packed, dl):
        self.codes = np.concatenate([self.codes, codes])
        self.packed = np.concatenate([self.packed, packed])
        self.dl = np.concatenate([self.dl, dl])


def _open(npb, oracle, art, codes, packed, dl, with_ivf=True, base=0):
    ivf, lens = oracle.build_ivf(codes, dl, K) if with_ivf else (None, None)
    return npb.MmapIndex.from_arrays(art.centroids, art.bucket_weights, codes, packed, dl, ivf, lens, NBITS,
                                     doc_id_base=base)


def _compare(npb, oracle, c, ix, live, ids=None, with_ivf=True):
    D = len(live.dl)
    oix = _oracle_index(oracle, c["art"], live.codes, live.packed, live.dl)
    fresh = _open(npb, oracle, c["art"], live.codes, live.packed, live.dl, with_ivf=with_ivf)
    try:
        _check_same(npb, oracle, ix, fresh, oix, c["qs"], ids if ids is not None else [0, D // 2, max(D - 1, 0), D + 3])
    finally:
        fresh.close()


def _patterns(D, rng):
    return {
        "scattered": np.concatenate([rng.choice(D, 120, replace=False), [-1, -(1 << 40), D, D + 7, 5, 5]]),
        "oldest": np.arange(100),                        # max_documents eviction
        "newest": np.arange(D - 100, D),                 # rollback of a failed add: moves nothing
        "one": np.array([777]),
        "every_other": np.arange(0, D, 2),
    }


@pytest.mark.parametrize("with_ivf", [True, False], ids=["ivf_given", "ivf_built_on_device"])
@pytest.mark.parametrize("pattern", ["scattered", "oldest", "newest", "one", "every_other"])
def test_delete_matches_a_fresh_open(npb, oracle, corpus, monkeypatch, pattern, with_ivf):
    monkeypatch.setenv("PB_DELETE_WINDOW_TOKENS", "200")     # a few docs per window: many window boundaries
    c = corpus
    D = 1500
    live = Live(c, D)
    ix = _open(npb, oracle, c["art"], live.codes, live.packed, live.dl, with_ivf=with_ivf)
    try:
        ids = _patterns(D, np.random.default_rng(3))[pattern]
        prev = ix.export_ivf()
        n = ix.delete(ids)
        want = len(set(i for i in ids.tolist() if 0 <= i < D))
        assert n == want
        assert all(np.array_equal(a, b) for a, b in zip(ix.export_ivf(), delete_ivf(*prev, ids, D)))
        live.delete(ids)
        _compare(npb, oracle, c, ix, live, with_ivf=with_ivf)
    finally:
        ix.close()


@pytest.mark.parametrize("window", ["1", None], ids=["one_doc_windows", "default_window"])
def test_window_sizes(npb, oracle, corpus, monkeypatch, window):
    if window is None:
        monkeypatch.delenv("PB_DELETE_WINDOW_TOKENS", raising=False)
    else:
        monkeypatch.setenv("PB_DELETE_WINDOW_TOKENS", window)
    c = corpus
    live = Live(c, 1500)
    ix = _open(npb, oracle, c["art"], live.codes, live.packed, live.dl)
    try:
        ids = np.random.default_rng(9).choice(1500, 300, replace=False)
        assert ix.delete(ids) == 300
        live.delete(ids)
        _compare(npb, oracle, c, ix, live)
    finally:
        ix.close()


def test_delete_nothing_changes_nothing(npb, oracle, corpus):
    c = corpus
    live = Live(c, 1500)
    ix = _open(npb, oracle, c["art"], live.codes, live.packed, live.dl)
    try:
        before = _snapshot(ix, npb, c["qs"])
        for ids in ([], [-3, 1500, 1 << 50]):
            assert ix.delete(ids) == 0
            assert _snapshot(ix, npb, c["qs"]) == before
    finally:
        ix.close()


def test_delete_all_then_append(npb, oracle, corpus):
    c = corpus
    live = Live(c, 1500)
    ix = _open(npb, oracle, c["art"], live.codes, live.packed, live.dl)
    try:
        assert ix.delete(range(1500)) == 1500
        assert ix.num_documents() == 0 and ix.num_embeddings() == 0 and ix.avg_doclen() == 0.0
        iv, ln = ix.export_ivf()
        assert len(iv) == 0 and not ln.any()
        for r in ix.search_batch(c["qs"], npb.SearchParameters(**PARAMS[0])):
            assert len(r.passage_ids) == 0
        # an append onto the emptied handle behaves as one onto a fresh open of an empty index
        t = int(c["dl"][:60].sum())
        assert ix.append_encoded(c["codes"][:t], c["packed"][:t], c["dl"][:60]) == list(range(60))
        _compare(npb, oracle, c, ix, Live(c, 60))
    finally:
        ix.close()


def test_deleting_the_docs_that_hold_the_constants(npb, oracle, corpus):
    # the tokens with the smallest |c + w| and the largest |w|, and the longest doc, go: vmin rises, wmax and
    # max_doclen fall, and the work counters still equal a fresh open's
    c = corpus
    art = c["art"]
    live = Live(c, 1500)
    ix = _open(npb, oracle, art, live.codes, live.packed, live.dl)
    try:
        w = art.bucket_weights
        bits = np.unpackbits(live.packed, axis=1).reshape(len(live.codes), DIM, NBITS).astype(np.int64)
        wv = w[(bits << np.arange(NBITS)).sum(2)].astype(np.float64)
        tok_doc = np.repeat(np.arange(1500), live.dl)
        vdoc = tok_doc[np.argmin(np.linalg.norm(art.centroids[live.codes] + wv, axis=1))]
        wdoc = tok_doc[np.argmax(np.linalg.norm(wv, axis=1))]
        ldoc = int(np.argmax(live.dl))
        ids = sorted({int(vdoc), int(wdoc), ldoc})
        assert ix.delete(ids) == len(ids)
        live.delete(ids)
        assert live.dl.max() <= c["dl"][:1500].max()
        _compare(npb, oracle, c, ix, live)
    finally:
        ix.close()


def test_append_delete_cycles(npb, oracle, corpus, monkeypatch):
    monkeypatch.setenv("PB_DELETE_WINDOW_TOKENS", "500")
    c = corpus
    off = np.zeros(len(c["dl"]) + 1, np.int64)
    np.cumsum(c["dl"], out=off[1:])
    live = Live(c, 1000)
    ix = _open(npb, oracle, c["art"], live.codes, live.packed, live.dl, with_ivf=False)
    rng = np.random.default_rng(21)
    nxt = 1000
    try:
        for step in range(4):
            n = 150
            t0, t1 = int(off[nxt]), int(off[nxt + n])
            ix.append_encoded(c["codes"][t0:t1], c["packed"][t0:t1], c["dl"][nxt:nxt + n])
            live.append(c["codes"][t0:t1], c["packed"][t0:t1], c["dl"][nxt:nxt + n])
            nxt += n
            D = len(live.dl)
            ids = rng.choice(D, 90, replace=False) if step % 2 == 0 else np.arange(D - 40, D)
            assert ix.delete(ids) == len(ids)
            live.delete(ids)
            _compare(npb, oracle, c, ix, live, with_ivf=False)
    finally:
        ix.close()


def test_delete_with_a_doc_id_base(npb, oracle, corpus):
    c = corpus
    base = 5000
    live = Live(c, 600)
    ix = _open(npb, oracle, c["art"], live.codes, live.packed, live.dl, base=base)
    try:
        local = np.array([0, 17, 300, 599])
        # global ids are base + local; local ids below the base are outside the handle
        assert ix.delete(np.concatenate([local + base, [3, 599]])) == 4
        live.delete(local)
        fresh = _open(npb, oracle, c["art"], live.codes, live.packed, live.dl, base=base)
        try:
            assert ix.num_documents() == fresh.num_documents() == 596
            assert all(np.array_equal(a, b) for a, b in zip(ix.export_ivf(), fresh.export_ivf()))
            for kw in PARAMS:
                assert _search(ix, npb, c["qs"], kw) == _search(fresh, npb, c["qs"], kw)
        finally:
            fresh.close()
    finally:
        ix.close()


def test_rejections_change_nothing(npb, oracle, corpus, tmp_path):
    import torch
    c = corpus
    art = c["art"]
    # a member of a shard group
    a, b = Live(c, 10), Live(c, 10)
    ha = _open(npb, oracle, art, a.codes, a.packed, a.dl)
    hb = _open(npb, oracle, art, b.codes, b.packed, b.dl)
    g = npb.ShardGroup([ha, hb])
    try:
        # a group member searches only together with its peers: its arrays are checked through the accessors
        arrays = (ha.num_documents(), ha.num_embeddings(), [x.tolist() for x in ha.export_ivf()])
        with pytest.raises(npb.PlaidError) as e:
            ha.delete([1, 2])
        assert e.value.status == 4
        assert (ha.num_documents(), ha.num_embeddings(), [x.tolist() for x in ha.export_ivf()]) == arrays
    finally:
        g.close()
    ha.close()
    hb.close()
    # a handle on the caller's residual array
    dev = torch.device("cuda", 0)
    live = Live(c, 100)
    t = {k: torch.from_numpy(np.ascontiguousarray(v)).to(dev) for k, v in dict(
        cen=art.centroids, w=art.bucket_weights, codes=live.codes, res=live.packed, dl=live.dl).items()}
    ad = npb.MmapIndex.from_device_pointers(DIM, NBITS, K, 100, len(live.codes), t["cen"].data_ptr(), t["w"].data_ptr(),
                                            t["codes"].data_ptr(), t["res"].data_ptr(), t["dl"].data_ptr(), None, None,
                                            adopt_residuals=True)
    try:
        before = _snapshot(ad, npb, c["qs"][:4])
        with pytest.raises(npb.PlaidError) as e:
            ad.delete([3])
        assert e.value.status == 4 and _snapshot(ad, npb, c["qs"][:4]) == before
    finally:
        ad.close()
    # an index directory: with a non-zero doc_id_base, and one that does not hold the handle's documents
    path = str(tmp_path / "ix")
    npb.create_index(c["docs"][:300], path, nbits=NBITS, num_partitions=K, batch_size=100, seed=7).close()

    def dir_bytes():
        return {f: open(os.path.join(path, f), "rb").read() for f in sorted(os.listdir(path))}
    files = dir_bytes()
    loaded = npb.MmapIndex.load(path)
    base = oracle.load_index(path)
    shifted = npb.MmapIndex.from_arrays(base.centroids, base.bucket_weights, base.codes, base.residuals,
                                        base.doc_lengths, base.ivf, base.ivf_lengths, NBITS, doc_id_base=1000)
    try:
        before = _snapshot(shifted, npb, c["qs"][:4])
        with pytest.raises(npb.PlaidError) as e:
            shifted.delete([1001], index_dir=path)
        assert e.value.status == 4 and _snapshot(shifted, npb, c["qs"][:4]) == before and dir_bytes() == files
        loaded.delete([5])                                   # the handle no longer matches the directory
        before = _snapshot(loaded, npb, c["qs"][:4])
        with pytest.raises(npb.PlaidError) as e:
            loaded.delete([6], index_dir=path)
        assert e.value.status == 1 and _snapshot(loaded, npb, c["qs"][:4]) == before and dir_bytes() == files
    finally:
        shifted.close()
        loaded.close()


def test_directory_delete(npb, oracle, tmp_path):
    docs = oracle.synthetic_corpus(3100, 40, dim=DIM, seed=81, ragged=True)
    path = str(tmp_path / "ix")
    npb.create_index(docs[:2600], path, nbits=NBITS, num_partitions=K, batch_size=1000, seed=7).close()
    base = oracle.load_index(path)
    qs, _ = oracle.synthetic_queries(docs, 6, nq=32, seed=14)
    # start-from-scratch and buffer files as the reference keeps them: embeddings of every doc, and of the last 5
    emb = np.concatenate(docs[:2600], 0).astype(np.float32)
    np.save(os.path.join(path, "embeddings.npy"), emb)
    json.dump([int(d.shape[0]) for d in docs[:2600]], open(os.path.join(path, "embeddings_lengths.json"), "w"))
    np.save(os.path.join(path, "buffer.npy"), np.concatenate(docs[2595:2600], 0).astype(np.float32))
    json.dump([int(d.shape[0]) for d in docs[2595:2600]], open(os.path.join(path, "buffer_lengths.json"), "w"))
    json.dump({"num_docs": 5}, open(os.path.join(path, "buffer_info.json"), "w"))
    live_docs = list(range(2600))                       # original doc index of each current doc
    chunk_docs = [1000, 1000, 600]
    chunk_off = [0, sum(d.shape[0] for d in docs[:1000]), sum(d.shape[0] for d in docs[:2000])]
    live = npb.MmapIndex.load(path)

    def read(i, name):
        return open(os.path.join(path, name.format(i)), "rb").read()

    try:
        for f in ("merged_codes.npy", "merged_residuals.manifest.json"):
            open(os.path.join(path, f), "w").write("stale")
        steps = [("inside one chunk", [3, 10, 999]),
                 ("across chunks", [0, 1500, 2100, 2593, 2596]),
                 ("a whole chunk", list(range(1993, 2592)))]       # chunk 2 (all of it now) plus the end of chunk 1
        for name, ids in steps:
            untouched = {}
            cut = np.cumsum([0] + chunk_docs)
            for i in range(len(chunk_docs)):
                if not any(cut[i] <= d < cut[i + 1] for d in ids):
                    untouched[i] = [read(i, n) for n in ("{}.codes.npy", "{}.residuals.npy", "doclens.{}.json",
                                                         "{}.metadata.json")]
            assert live.delete(ids, index_dir=path) == len(ids), name
            gone = set(live_docs[d] for d in ids)
            live_docs = [d for d in live_docs if d not in gone]
            for i in range(len(chunk_docs)):
                chunk_docs[i] -= sum(1 for d in ids if cut[i] <= d < cut[i + 1])
            D = len(live_docs)
            # chunk files against the filtered arrays; embedding_offset unchanged; untouched chunks byte for byte
            flat = np.concatenate([docs[d] for d in live_docs], 0)
            codes = oracle.compress_into_codes(flat, base.centroids)
            res = oracle.quantize_residuals(oracle.residuals_of(flat, base.centroids, codes), base.bucket_cutoffs, NBITS)
            t = 0
            for i, nd in enumerate(chunk_docs):
                dl = json.load(open(os.path.join(path, f"doclens.{i}.json")))
                meta = json.load(open(os.path.join(path, f"{i}.metadata.json")))
                assert len(dl) == nd and meta == dict(num_documents=nd, num_embeddings=sum(dl),
                                                      embedding_offset=chunk_off[i]), (name, i)
                assert np.array_equal(np.load(os.path.join(path, f"{i}.codes.npy")), codes[t:t + sum(dl)])
                assert np.array_equal(np.load(os.path.join(path, f"{i}.residuals.npy")), res[t:t + sum(dl)])
                t += sum(dl)
                if i in untouched:
                    assert [read(i, n) for n in ("{}.codes.npy", "{}.residuals.npy", "doclens.{}.json",
                                                 "{}.metadata.json")] == untouched[i], (name, i)
            meta = json.load(open(os.path.join(path, "metadata.json")))
            assert meta["num_chunks"] == 3 and meta["num_documents"] == D and meta["num_embeddings"] == len(flat)
            assert meta["avg_doclen"] == len(flat) / D                           # delete.rs:240-244
            assert (meta["nbits"], meta["num_partitions"], meta["embedding_dim"]) == (NBITS, K, DIM)
            assert not [f for f in os.listdir(path) if f.startswith("merged_") or f.endswith(".tmp")]
            # embeddings.npy: docs by id; buffer.npy: the last 5 docs of the index before each delete
            e = np.load(os.path.join(path, "embeddings.npy"))
            assert np.array_equal(e, flat.astype(np.float32))
            assert json.load(open(os.path.join(path, "embeddings_lengths.json"))) == [int(docs[d].shape[0]) for d in live_docs]
            buf = [d for d in range(2595, 2600) if d in live_docs]
            if name == "inside one chunk":
                assert json.load(open(os.path.join(path, "buffer_info.json"))) == {"num_docs": 5}
            if name == "across chunks":                                       # buffer ids 2592..2596 of 2597 docs
                assert json.load(open(os.path.join(path, "buffer_lengths.json"))) == [int(docs[d].shape[0]) for d in buf]
                assert np.array_equal(np.load(os.path.join(path, "buffer.npy")), np.concatenate([docs[d] for d in buf], 0))
                assert json.load(open(os.path.join(path, "buffer_info.json"))) == {"num_docs": 3}
            if name == "a whole chunk":                                       # every buffered doc deleted
                assert not [f for f in os.listdir(path) if f.startswith("buffer")]
            # the directory loads and searches like the live handle and the oracle
            oix = oracle.load_index(path)
            assert np.array_equal(oix.codes, codes) and oix.num_documents == D
            assert all(np.array_equal(a, b) for a, b in zip(live.export_ivf(), (oix.ivf, oix.ivf_lengths)))
            loaded = npb.MmapIndex.load(path)
            try:
                for kw in PARAMS[:2]:
                    a = live.search_batch(qs, npb.SearchParameters(**kw))
                    b = loaded.search_batch(qs, npb.SearchParameters(**kw))
                    for q, x, y in zip(qs, a, b):
                        w = oracle.search_one(oix, q, oracle.SearchParameters(**kw))
                        assert x.passage_ids.tolist() == y.passage_ids.tolist() == w.passage_ids.tolist(), (name, kw)
                        assert np.array_equal(x.scores, w.scores) and np.array_equal(y.scores, w.scores), (name, kw)
            finally:
                loaded.close()
        assert chunk_docs == [996, 997, 0]
        # an append goes into the emptied last chunk, which has < 2000 docs (update.rs:799-827)
        codec = npb.ResidualCodec(NBITS, base.centroids, base.bucket_cutoffs)
        try:
            D = len(live_docs)
            assert live.append(docs[2600:3100], codec, index_dir=path, batch_size=1000) == list(range(D, D + 500))
        finally:
            codec.close()
        meta = json.load(open(os.path.join(path, "metadata.json")))
        assert meta["num_chunks"] == 3 and meta["num_documents"] == D + 500
        assert len(json.load(open(os.path.join(path, "doclens.2.json")))) == 500
        assert json.load(open(os.path.join(path, "2.metadata.json")))["embedding_offset"] == chunk_off[2]
        oix = oracle.load_index(path)
        loaded = npb.MmapIndex.load(path)
        try:
            assert all(np.array_equal(a, b) for a, b in zip(loaded.export_ivf(), (oix.ivf, oix.ivf_lengths)))
            assert _search(loaded, npb, qs, PARAMS[0]) == _search(live, npb, qs, PARAMS[0])
        finally:
            loaded.close()
    finally:
        live.close()


@pytest.mark.parametrize("lanes", [1, 2])
def test_searches_see_all_or_nothing_of_a_delete(npb, oracle, corpus, lanes):
    c = corpus
    qs = (c["qs"] * 2)[:16]                                  # >= 16 queries so that 2 lanes engage
    kw = PARAMS[0]
    live = Live(c, 1500)
    ix = _open(npb, oracle, c["art"], live.codes, live.packed, live.dl)
    ids = np.random.default_rng(31).choice(1500, 400, replace=False)
    live.delete(ids)
    post = _open(npb, oracle, c["art"], live.codes, live.packed, live.dl)
    try:
        ix.set_lanes(lanes)
        before = _search(ix, npb, qs, kw)[0]
        after = _search(post, npb, qs, kw)[0]
        assert before != after
        seen, errs, done = [], [], threading.Event()

        def searcher():
            try:
                extra = 3
                while extra > 0:
                    if done.is_set():
                        extra -= 1
                    seen.append(_search(ix, npb, qs, kw)[0])
            except Exception as e:  # noqa: BLE001 - reported below
                errs.append(e)
        ths = [threading.Thread(target=searcher) for _ in range(2)]
        [t.start() for t in ths]
        assert ix.delete(ids) == 400
        done.set()
        [t.join() for t in ths]
        assert not errs, errs
        assert all(s == before or s == after for s in seen)
        assert seen.count(after) >= 6 and _search(ix, npb, qs, kw)[0] == after
    finally:
        ix.close()
        post.close()
