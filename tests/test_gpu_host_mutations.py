"""Appends and deletes on mutable host-tier handles (PB_OPEN_HOST_RESIDUALS | PB_OPEN_HOST_MUTABLE, DESIGN.md 4r): the
packed rows live in pinned host segments that grow in place.  After every mutation the handle must equal a fresh open
of the resulting arrays -- ids, scores, work counters, staging stats, decompression, exhaustive scores and the inverted
file -- and searching must read the rows through the segment table, also with segments of 256 bytes, where rows and
documents straddle segments."""
import ctypes
import filecmp
import os
import shutil
import sys
import threading

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_gpu_shape_edges import _codec_index, _queries_from  # noqa: E402

pytestmark = pytest.mark.gpu

NBITS, K, DIM = 2, 256, 128
COUNTERS = ("n_exact_docs", "n_exact_pairs", "n_recheck_docs", "n_filter_docs")
PARAMS = [dict(top_k=10, n_ivf_probe=8, n_full_scores=256),
          dict(top_k=5, n_ivf_probe=4, n_full_scores=64, centroid_batch_size=100)]


@pytest.fixture(scope="module")
def npb():
    import next_plaid_b200 as m
    m.build_library()
    if m.device_count() < 1:
        pytest.fail("GPU tests need an H100; the library has no CPU fallback")
    return m


@pytest.fixture(scope="module")
def corpus(oracle):
    """1600 ragged docs (dim 128, 2 bits) encoded by the oracle with one codec"""
    docs = oracle.synthetic_corpus(1600, 40, dim=DIM, seed=61, ragged=True)
    flat = np.concatenate(docs, 0)
    cent = flat[np.random.default_rng(2).choice(len(flat), K, replace=False)].copy()
    art = oracle.prepare_codec_artifacts(docs, cent, NBITS, 3)
    codes, packed, dl = oracle.encode_documents(docs, art, NBITS)
    qs, _ = oracle.synthetic_queries(docs, 6, nq=32, seed=8)
    qs += oracle.synthetic_queries(docs[1200:], 2, nq=32, seed=9)[0]
    return dict(docs=docs, art=art, codes=codes, packed=packed, dl=np.asarray(dl, np.int64), qs=qs, nbits=NBITS)


@pytest.fixture(scope="module")
def corpus48(oracle):
    """dim 48 at 1 bit: 6-byte rows, which straddle 256- and 4096-byte segments"""
    rng = np.random.default_rng(48)
    ix = _codec_index(oracle, 128, rng.integers(5, 60, 700), dim=48, nbits=1, seed=48)
    qs = _queries_from(oracle, ix, rng.integers(0, 700, 8).tolist(), [32, 8, 17, 32, 1, 24, 32, 5], 4)
    return dict(ix=ix, codes=ix.codes, packed=ix.residuals, dl=np.asarray(ix.doc_lengths, np.int64), qs=qs, nbits=1)


def _arrays(c):
    a = c["art"] if "art" in c else c["ix"]
    return a.centroids, a.bucket_weights


def _open(npb, oracle, c, codes, packed, dl, **kw):
    cen, w = _arrays(c)
    ivf, lens = oracle.build_ivf(codes, dl, len(cen))
    return npb.MmapIndex.from_arrays(cen, w, codes, packed, dl, ivf, lens, c["nbits"], **kw)


def _search(h, npb, qs, kw):
    res = h.search_batch(qs, npb.SearchParameters(**kw))
    w = h.last_work_counters()
    return [(r.passage_ids.tolist(), r.scores.tobytes()) for r in res], {k: w[k] for k in COUNTERS}, \
        h.last_staging_stats()["bytes"]


def _state(h, npb, qs, ids):
    out = [h.num_documents(), h.num_embeddings(), [a.tolist() for a in h.export_ivf()]]
    out += [_search(h, npb, qs, kw) for kw in PARAMS]
    e, l = h.decompress_documents(ids)
    out += [e.tobytes(), l.tolist()]
    if h.num_documents():
        out.append(h.exhaustive_scores(qs[:4]).tobytes())
    return out


def _equals_fresh(npb, oracle, c, h, codes, packed, dl, ids=(0, 5)):
    """h equals a fresh host-tier open (staging stats included) and a fresh resident open (all but the stats)"""
    ids = [i for i in ids if i < len(dl)] + [len(dl) - 1, len(dl) + 3]
    host = _open(npb, oracle, c, codes, packed, dl, host_residuals=True)
    res = _open(npb, oracle, c, codes, packed, dl)
    try:
        got = _state(h, npb, c["qs"], ids)
        assert got == _state(host, npb, c["qs"], ids)
        strip = lambda s: [x if not isinstance(x, tuple) else x[:2] for x in s]  # noqa: E731
        assert strip(got) == strip(_state(res, npb, c["qs"], ids))
    finally:
        host.close()
        res.close()


def _cat(c, parts):
    """codes, packed, dl of the docs listed (ranges of the corpus, in order)"""
    off = np.concatenate([[0], np.cumsum(c["dl"])])
    docs = np.concatenate([np.arange(a, b) for a, b in parts]) if parts else np.zeros(0, np.int64)
    tok = np.concatenate([np.arange(off[d], off[d + 1]) for d in docs] + [np.zeros(0, np.int64)]).astype(np.int64)
    return c["codes"][tok], c["packed"][tok], c["dl"][docs]


@pytest.mark.parametrize("seg", [256, 4096])
@pytest.mark.parametrize("which", ["dim128", "dim48"])
def test_tiny_segments_equal_resident_and_oracle(npb, oracle, corpus, corpus48, monkeypatch, seg, which):
    c = corpus if which == "dim128" else corpus48
    monkeypatch.setenv("PB_HOST_SEGMENT_BYTES", str(seg))
    h = _open(npb, oracle, c, c["codes"], c["packed"], c["dl"], host_residuals=True, mutable=True)
    try:
        assert h.memory_usage()["host_bytes"] == c["packed"].size
        _equals_fresh(npb, oracle, c, h, c["codes"], c["packed"], c["dl"], ids=(0, 3, 77, 401))
        if which == "dim48":
            ix = c["ix"]
            for q, (ids, sc) in zip(c["qs"], _search(h, npb, c["qs"], PARAMS[0])[0]):
                w = oracle.search_one(ix, q, oracle.SearchParameters(**PARAMS[0]))
                assert ids == w.passage_ids.tolist() and sc == w.scores.astype(np.float32).tobytes()
    finally:
        h.close()


@pytest.mark.parametrize("seg", [256, 4096])
@pytest.mark.parametrize("how", ["encoded_host", "encoded_device", "codec_host", "codec_device"])
def test_appends_equal_a_fresh_open(npb, oracle, corpus, monkeypatch, seg, how):
    import torch
    c = corpus
    monkeypatch.setenv("PB_HOST_SEGMENT_BYTES", str(seg))
    D = 1000
    h = _open(npb, oracle, c, *_cat(c, [(0, D)]), host_residuals=True, mutable=True)
    codec = npb.ResidualCodec(NBITS, c["art"].centroids, c["art"].bucket_cutoffs) if how.startswith("codec") else None
    L = npb.load_library()
    try:
        for n in (1, 0, 37, 300):
            codes, packed, dl = _cat(c, [(D, D + n)])
            if how == "encoded_host":
                assert h.append_encoded(codes, packed, dl) == list(range(D, D + n))
            elif how == "codec_host":
                assert h.append(c["docs"][D:D + n], codec) == list(range(D, D + n))
            else:
                dev = torch.device("cuda", 0)
                t_dl = torch.from_numpy(np.ascontiguousarray(dl)).to(dev)
                first = ctypes.c_int64()
                if how == "encoded_device":
                    t_c = torch.from_numpy(np.ascontiguousarray(codes, np.int64)).to(dev)
                    t_r = torch.from_numpy(np.ascontiguousarray(packed)).to(dev)
                    st = L.pb_index_append_encoded(h._h, t_c.data_ptr(), t_r.data_ptr(), t_dl.data_ptr(), n, 1,
                                                   ctypes.byref(first))
                else:
                    flat = np.concatenate(c["docs"][D:D + n], 0) if n else np.zeros((1, DIM), np.float32)
                    t_x = torch.from_numpy(np.ascontiguousarray(flat, np.float32)).to(dev)
                    st = L.pb_index_append(h._h, codec._h, t_x.data_ptr(), t_dl.data_ptr(), n, 1, None, 0,
                                           ctypes.byref(first))
                torch.cuda.synchronize()
                assert st == 0 and first.value == D
            D += n
            _equals_fresh(npb, oracle, c, h, *_cat(c, [(0, D)]), ids=(0, 999, D - n))
        assert h.memory_usage()["host_bytes"] % seg == 0 and h.memory_usage()["host_bytes"] >= c["packed"][:1].size
    finally:
        if codec:
            codec.close()
        h.close()


def test_reserve_then_append_adds_no_pinned_bytes(npb, oracle, corpus, monkeypatch):
    c = corpus
    monkeypatch.setenv("PB_HOST_SEGMENT_BYTES", "4096")
    h = _open(npb, oracle, c, *_cat(c, [(0, 1000)]), host_residuals=True, mutable=True)
    try:
        codes, packed, dl = _cat(c, [(0, 1600)])
        h.reserve(1600, len(codes))
        held = h.memory_usage()["host_bytes"]
        assert held >= packed.size and held % 4096 == 0
        h.append_encoded(*_cat(c, [(1000, 1600)]))
        assert h.memory_usage()["host_bytes"] == held
        _equals_fresh(npb, oracle, c, h, codes, packed, dl, ids=(0, 1000, 1599))
    finally:
        h.close()


DELETES = {"scattered": lambda D, rng: sorted(rng.choice(D, D // 7, replace=False).tolist()),
           "oldest": lambda D, rng: list(range(60)),
           "newest": lambda D, rng: list(range(D - 60, D)),
           "none": lambda D, rng: [D + 5, -1],
           "all": lambda D, rng: list(range(D))}


@pytest.mark.parametrize("pattern", list(DELETES))
def test_deletes_equal_a_fresh_open(npb, oracle, corpus, monkeypatch, pattern):
    c = corpus
    monkeypatch.setenv("PB_HOST_SEGMENT_BYTES", "256")
    monkeypatch.setenv("PB_DELETE_WINDOW_TOKENS", "500")
    D = 1200
    h = _open(npb, oracle, c, *_cat(c, [(0, D)]), host_residuals=True, mutable=True)
    try:
        held = h.memory_usage()["host_bytes"]
        gone = DELETES[pattern](D, np.random.default_rng(5))
        assert h.delete(gone) == len([g for g in gone if 0 <= g < D])
        keep = [(d, d + 1) for d in range(D) if d not in set(gone)]
        _equals_fresh(npb, oracle, c, h, *_cat(c, keep), ids=(0, 59, 600))
        assert h.memory_usage()["host_bytes"] == held                      # capacity is kept
        base = h.num_documents()
        h.append_encoded(*_cat(c, [(1200, 1300)]))                           # then an append, also to an emptied handle
        _equals_fresh(npb, oracle, c, h, *_cat(c, keep + [(1200, 1300)]), ids=(0, base, base + 99))
    finally:
        h.close()


def test_interleaved_appends_and_deletes_track_a_resident_handle(npb, oracle, corpus, monkeypatch):
    c = corpus
    monkeypatch.setenv("PB_HOST_SEGMENT_BYTES", "4096")
    monkeypatch.setenv("PB_DELETE_WINDOW_TOKENS", "3000")
    rng = np.random.default_rng(11)
    h = _open(npb, oracle, c, *_cat(c, [(0, 400)]), host_residuals=True, mutable=True)
    r = _open(npb, oracle, c, *_cat(c, [(0, 400)]))
    nxt = 400
    try:
        for step in range(8):
            if step % 2 == 0 and nxt < 1600:
                n = int(rng.integers(1, 200))
                part = _cat(c, [(nxt, min(nxt + n, 1600))])
                nxt = min(nxt + n, 1600)
                assert h.append_encoded(*part) == r.append_encoded(*part)
            else:
                gone = rng.choice(h.num_documents(), int(rng.integers(1, 80)), replace=False).tolist()
                assert h.delete(gone) == r.delete(gone)
            ids = [0, h.num_documents() // 2, h.num_documents() - 1]
            got, want = _state(h, npb, c["qs"], ids), _state(r, npb, c["qs"], ids)
            strip = lambda s: [x if not isinstance(x, tuple) else x[:2] for x in s]  # noqa: E731
            assert strip(got) == strip(want), step
    finally:
        h.close()
        r.close()


def test_bad_calls_change_nothing(npb, oracle, corpus):
    c = corpus
    h = _open(npb, oracle, c, *_cat(c, [(0, 800)]), host_residuals=True, mutable=True)
    other = npb.ResidualCodec(NBITS, c["art"].centroids + 1.0, c["art"].bucket_cutoffs)
    try:
        before = _state(h, npb, c["qs"], [0, 799])
        held = h.memory_usage()["host_bytes"]
        codes, packed, dl = _cat(c, [(800, 900)])
        bad = codes.copy()
        bad[-1] = K                                                       # a code outside [0, K)
        with pytest.raises(npb.PlaidError) as e:
            h.append_encoded(bad, packed, dl)
        assert e.value.status == 1
        with pytest.raises(npb.PlaidError) as e:
            h.append(c["docs"][800:900], other)                           # the codec's centroids differ
        assert e.value.status == 1
        assert _state(h, npb, c["qs"], [0, 799]) == before
        assert h.memory_usage()["host_bytes"] >= held
        h.append_encoded(codes, packed, dl)                               # the handle still works
        _equals_fresh(npb, oracle, c, h, *_cat(c, [(0, 900)]))
    finally:
        other.close()
        h.close()


def test_searches_see_all_or_nothing(npb, oracle, corpus, monkeypatch):
    c = corpus
    monkeypatch.setenv("PB_HOST_SEGMENT_BYTES", "4096")
    h = _open(npb, oracle, c, *_cat(c, [(0, 1000)]), host_residuals=True, mutable=True)
    states = []
    for parts in ([(0, 1000)], [(0, 1300)], [(0, 1000), (1001, 1300)]):
        f = _open(npb, oracle, c, *_cat(c, parts))
        states.append(_search(f, npb, c["qs"][:8], PARAMS[0])[0])
        f.close()
    stop, seen, errors = threading.Event(), [], []

    def reader():
        try:
            while not stop.is_set():
                seen.append(h.search_batch(c["qs"][:8], npb.SearchParameters(**PARAMS[0])))
        except Exception as e:  # pragma: no cover - reported below
            errors.append(e)
    t = threading.Thread(target=reader)
    t.start()
    try:
        h.append_encoded(*_cat(c, [(1000, 1300)]))
        h.delete([1000])
    finally:
        stop.set()
        t.join()
    try:
        assert not errors and seen
        for res in seen:
            assert [(r.passage_ids.tolist(), r.scores.tobytes()) for r in res] in states
    finally:
        h.close()


def test_directory_files_equal_a_resident_handle(npb, oracle, tmp_path, monkeypatch):
    docs = oracle.synthetic_corpus(1500, 40, dim=DIM, seed=71, ragged=True)
    base_dir = str(tmp_path / "base")
    npb.create_index(docs[:1200], base_dir, nbits=NBITS, num_partitions=K, batch_size=500, seed=7).close()
    dirs = {k: str(tmp_path / k) for k in ("host", "res")}
    for d in dirs.values():
        shutil.copytree(base_dir, d)
    monkeypatch.setenv("PB_HOST_SEGMENT_BYTES", "4096")
    hs = {"host": npb.MmapIndex.load(dirs["host"], host_residuals=True, mutable=True),
          "res": npb.MmapIndex.load(dirs["res"])}
    base = oracle.load_index(base_dir)
    codec = npb.ResidualCodec(NBITS, base.centroids, base.bucket_cutoffs)
    try:
        for k, h in hs.items():
            h.append(docs[1200:1500], codec, index_dir=dirs[k], batch_size=500)
            h.delete([3, 700, 1210, 1499], index_dir=dirs[k])
            h.append_encoded(*[np.asarray(a) for a in codec.encode_chunk(np.concatenate(docs[:2], 0))],
                             [len(docs[0]), len(docs[1])])
        names = sorted(os.listdir(dirs["res"]))
        assert names == sorted(os.listdir(dirs["host"]))
        for n in names:
            assert filecmp.cmp(os.path.join(dirs["res"], n), os.path.join(dirs["host"], n), shallow=False), n
        qs, _ = oracle.synthetic_queries(docs, 4, nq=32, seed=3)
        a = hs["host"].search_batch(qs, npb.SearchParameters(**PARAMS[0]))
        b = hs["res"].search_batch(qs, npb.SearchParameters(**PARAMS[0]))
        assert [(r.passage_ids.tolist(), r.scores.tobytes()) for r in a] == \
               [(r.passage_ids.tolist(), r.scores.tobytes()) for r in b]
    finally:
        codec.close()
        for h in hs.values():
            h.close()


def _dir(npb, oracle, tmp_path, corpus, D=1200):
    path = str(tmp_path / "ix")
    npb.create_index(corpus["docs"][:D], path, nbits=NBITS, num_partitions=K, batch_size=400, seed=7).close()
    return path


def _results(h, npb, qs, kw):
    return [(r.passage_ids.tolist(), r.scores.tobytes()) for r in h.search_batch(qs, npb.SearchParameters(**kw))]


def _same_handles(npb, a, b, qs):
    for kw in PARAMS:
        assert _results(a, npb, qs, kw) == _results(b, npb, qs, kw)
    assert a.num_documents() == b.num_documents() and a.num_embeddings() == b.num_embeddings()
    ids = [0, a.num_documents() // 2, a.num_documents() - 1]
    ea, la = a.decompress_documents(ids)
    eb, lb = b.decompress_documents(ids)
    assert np.array_equal(ea, eb) and np.array_equal(la, lb)


def _mutate(npb, oracle, h, c, path):
    """a codec append, an encoded append, a delete across both, another codec append"""
    base = oracle.load_index(path)
    codec = npb.ResidualCodec(NBITS, base.centroids, base.bucket_cutoffs)
    try:
        h.append(c["docs"][1200:1400], codec)
        new = c["docs"][1400:1450]
        codes, packed = codec.encode_chunk(np.concatenate(new, 0))
        h.append_encoded(codes, packed, [len(d) for d in new])
        h.delete([1, 500, 1250, 1399, 1420])
        h.append(c["docs"][1450:1500], codec)
    finally:
        codec.close()


def _every_replica_serves(npb, rep, one, qs):
    """searches cut over every replica, and decompression on replica 1: a whole call goes to the least-loaded replica
    (ties to replica 0), so it is issued while a one-slice search holds replica 0"""
    R = rep.replica_layout()[0]
    many = (qs * (32 * R // len(qs) + 1))[:32 * R]
    rep.replica_stats(reset=True)
    for kw in PARAMS:
        assert _results(rep, npb, many, kw) == _results(one, npb, many, kw)
    calls, queries = rep.replica_stats(reset=True)
    assert (calls > 0).all() and (queries > 0).all(), (calls, queries)
    ids = list(range(0, rep.num_documents(), 7))
    want = one.decompress_documents(ids)
    few = qs[:8]
    stop, errors = threading.Event(), []

    def searcher():                  # one search thread: every search ties at zero load and goes to replica 0
        try:
            while not stop.is_set():
                rep.search_batch(few, npb.SearchParameters(**PARAMS[0]))
        except Exception as e:  # pragma: no cover - reported below
            errors.append(e)
    t = threading.Thread(target=searcher)
    t.start()
    try:
        for _ in range(2000):
            e, l = rep.decompress_documents(ids)
            assert np.array_equal(e, want[0]) and np.array_equal(l, want[1])
            if rep.replica_stats()[0][1] > 0:                    # only a decompression can have gone to replica 1
                break
    finally:
        stop.set()
        t.join()
    assert not errors
    assert rep.replica_stats()[0][1] > 0, rep.replica_stats()


@pytest.mark.parametrize("devices,shards", [([0, 0], 1), ([0, 0, 0, 0], 2)], ids=["R2S1", "R2S2"])
def test_replica_set_equals_a_single_handle(npb, oracle, corpus, tmp_path, monkeypatch, devices, shards):
    c = corpus
    monkeypatch.setenv("PB_HOST_SEGMENT_BYTES", "4096")
    monkeypatch.setenv("PB_DELETE_WINDOW_TOKENS", "3000")
    path = _dir(npb, oracle, tmp_path, c)
    one = npb.MmapIndex.load(path, host_residuals=True, mutable=True)
    rep = npb.MmapIndex.load_replicas(path, devices, shards=shards, host_residuals=True, mutable=True)
    try:
        held = one.memory_usage()["host_bytes"]
        assert rep.memory_usage()["host_bytes"] == held                      # one store per rank, counted once
        _every_replica_serves(npb, rep, one, c["qs"])
        for h in (one, rep):
            _mutate(npb, oracle, h, c, path)
        assert one.memory_usage()["host_bytes"] > held
        if shards == 1:
            assert rep.memory_usage()["host_bytes"] == one.memory_usage()["host_bytes"]
        else:                                        # each rank's store holds its own rows: the same total, two tails
            assert rep.memory_usage()["host_bytes"] >= held
        _every_replica_serves(npb, rep, one, c["qs"])
        if shards == 1:                              # a deployment refuses reserve (it would split the capacity)
            rep.reserve(rep.num_documents() + 100, rep.num_embeddings() + 10_000)
            one.reserve(one.num_documents() + 100, one.num_embeddings() + 10_000)
            assert rep.memory_usage()["host_bytes"] == one.memory_usage()["host_bytes"]
        base = oracle.load_index(path)
        codec = npb.ResidualCodec(NBITS, base.centroids, base.bucket_cutoffs)
        try:
            for h in (one, rep):
                h.append(c["docs"][1500:1600], codec)
                h.delete(list(range(0, h.num_documents(), 9)))
        finally:
            codec.close()
        _every_replica_serves(npb, rep, one, c["qs"])
    finally:
        one.close()
        rep.close()


def _group_state(npb, grp, qs):
    return (_results(grp, npb, qs, PARAMS[0]), _results(grp, npb, qs, PARAMS[1]),
            [(s.num_documents(), s.num_embeddings(), s.memory_usage()) for s in grp.shards])


def test_deployment_and_shard_group(npb, oracle, corpus, tmp_path, monkeypatch):
    c = corpus
    monkeypatch.setenv("PB_HOST_SEGMENT_BYTES", "4096")
    path = _dir(npb, oracle, tmp_path, c)
    one = npb.MmapIndex.load(path)
    dep = npb.MmapIndex.load_devices(path, [0, 0], host_residuals=True, mutable=True)
    grp = npb.ShardGroup([npb.MmapIndex.load_shard(path, r, 2, host_residuals=True, mutable=True) for r in range(2)])
    try:
        for h in (one, dep):
            _mutate(npb, oracle, h, c, path)
        _same_handles(npb, dep, one, c["qs"])
        base = oracle.load_index(path)
        codec = npb.ResidualCodec(NBITS, base.centroids, base.bucket_cutoffs)
        try:
            grp.append(c["docs"][1200:1400], codec)
            new = c["docs"][1400:1450]
            codes, packed = codec.encode_chunk(np.concatenate(new, 0))
            grp.append_encoded(codes, packed, [len(d) for d in new])
            grp.delete([1, 500, 1250, 1399, 1420])
            grp.append(c["docs"][1450:1500], codec)
        finally:
            codec.close()
        for kw in PARAMS:
            assert _results(grp, npb, c["qs"], kw) == _results(one, npb, c["qs"], kw)
        # the rebalance refuses host-tier ranks, on a deployment and on a group, and changes nothing
        before = (_results(dep, npb, c["qs"], PARAMS[0]), dep.num_documents(), dep.num_embeddings(),
                  dep.memory_usage(), dep.shard_layout()[0].tolist())
        with pytest.raises(npb.PlaidError) as e:
            dep.rebalance_sharded()
        assert e.value.status == 4
        assert (_results(dep, npb, c["qs"], PARAMS[0]), dep.num_documents(), dep.num_embeddings(),
                dep.memory_usage(), dep.shard_layout()[0].tolist()) == before
        before = _group_state(npb, grp, c["qs"])
        with pytest.raises(npb.PlaidError) as e:
            grp.rebalance()
        assert e.value.status == 4
        assert _group_state(npb, grp, c["qs"]) == before
    finally:
        one.close()
        dep.close()
        grp.close()


def test_mutable_needs_host_residuals_and_plain_host_still_refuses(npb, oracle, corpus):
    c = corpus
    with pytest.raises(npb.PlaidError) as e:
        _open(npb, oracle, c, *_cat(c, [(0, 100)]), mutable=True)
    assert e.value.status == 1
    h = _open(npb, oracle, c, *_cat(c, [(0, 100)]), host_residuals=True)
    try:
        with pytest.raises(npb.PlaidError) as e:
            h.append_encoded(*_cat(c, [(100, 110)]))
        assert e.value.status == 4
        assert h.memory_usage()["host_bytes"] == _cat(c, [(0, 100)])[1].size
    finally:
        h.close()
