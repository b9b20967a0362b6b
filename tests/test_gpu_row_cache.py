"""The device row cache of host-tier handles (pb_index_set_row_cache / pb_index_fill_row_cache, DESIGN.md 4s): search
staging copies a cached doc's rows device to device instead of over PCIe.  Results, counts and every work counter must
be the same with the cache off, partly filled and full, and equal a resident handle and the oracle; fills must take the
docs tests/row_cache.py restates; mutations must keep the cache consistent with a fresh open."""
import os
import sys
import threading

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import row_cache  # noqa: E402
from test_gpu_shape_edges import _codec_index, _queries_from  # noqa: E402

pytestmark = pytest.mark.gpu

NBITS, K, DIM = 2, 256, 128
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
    """1600 ragged docs (dim 128, 2 bits: 32-byte rows, the uint4 form) encoded by the oracle with one codec"""
    docs = oracle.synthetic_corpus(1600, 40, dim=DIM, seed=61, ragged=True)
    flat = np.concatenate(docs, 0)
    cent = flat[np.random.default_rng(2).choice(len(flat), K, replace=False)].copy()
    art = oracle.prepare_codec_artifacts(docs, cent, NBITS, 3)
    codes, packed, dl = oracle.encode_documents(docs, art, NBITS)
    ix = oracle.Index(art.centroids, art.bucket_weights, art.bucket_cutoffs, codes, packed, np.asarray(dl, np.int64),
                      *oracle.build_ivf(codes, dl, K), NBITS)
    qs, _ = oracle.synthetic_queries(docs, 6, nq=32, seed=8)
    qs += oracle.synthetic_queries(docs[1200:], 2, nq=32, seed=9)[0]
    return dict(docs=docs, art=art, ix=ix, qs=qs)


def _corpus48(oracle, nbits, seed):
    rng = np.random.default_rng(seed)
    ix = _codec_index(oracle, 128, rng.integers(5, 60, 700), dim=48, nbits=nbits, seed=seed)
    qs = _queries_from(oracle, ix, rng.integers(0, 700, 8).tolist(), [32, 8, 17, 32, 1, 24, 32, 5], 4)
    return dict(ix=ix, qs=qs)


@pytest.fixture(scope="module")
def corpora(oracle, corpus):
    """dim 128 at 2 bits, dim 48 at 2 bits (12-byte rows, the uint32_t form), dim 48 at 1 bit (6-byte rows, the
    unsigned short form)"""
    return {"d128b2": corpus, "d48b2": _corpus48(oracle, 2, 482), "d48b1": _corpus48(oracle, 1, 481)}


def _open(npb, oracle, ix, docs=None, **kw):
    """a handle of the docs listed of the oracle index ix (all by default)"""
    off = np.concatenate([[0], np.cumsum(ix.doc_lengths)]).astype(np.int64)
    d = np.arange(len(ix.doc_lengths)) if docs is None else np.asarray(docs, np.int64)
    tok = np.concatenate([np.arange(off[i], off[i + 1]) for i in d] + [np.zeros(0, np.int64)]).astype(np.int64)
    codes, packed, dl = np.asarray(ix.codes)[tok], np.asarray(ix.residuals)[tok], np.asarray(ix.doc_lengths)[d]
    ivf, lens = oracle.build_ivf(codes, dl, len(ix.centroids))
    return npb.MmapIndex.from_arrays(ix.centroids, ix.bucket_weights, codes, packed, dl, ivf, lens, ix.nbits, **kw)


def _res(out):
    return [(r.passage_ids.tolist(), r.scores.tobytes()) for r in out]


def _calls(h, npb, qs, ids):
    """every search form's ids, scores and counts with all its work counters, and decompression"""
    out = []
    for kw in PARAMS:
        out.append((_res(h.search_batch(qs, npb.SearchParameters(**kw))), h.last_work_counters()))
    res, tr = h.search_batch(qs, npb.SearchParameters(**PARAMS[0]), trace=True)
    out.append((_res(res), [k.tolist() for k in tr.kept], [e.tobytes() for e in tr.kept_exact], h.last_work_counters()))
    n = h.num_documents()
    subsets = [None if i % 3 == 0 else list(range(i % 5, n, 3)) for i in range(len(qs))]
    ps = [npb.SearchParameters(**PARAMS[i % 2]) for i in range(len(qs))]
    out.append((_res(h.search_batch_params(qs, ps, subsets)), h.last_work_counters()))
    out.append(h.decompress_documents(ids)[0].tobytes())
    return out


def _threads(h, npb, qs):
    """pb_search from one thread per query, coalesced into shared batches"""
    h.set_coalescing(8, max_wait_us=2000)
    got = [None] * len(qs)

    def one(i):
        got[i] = _res([h.search(qs[i], npb.SearchParameters(**PARAMS[0]))])[0]
    th = [threading.Thread(target=one, args=(i,)) for i in range(len(qs))]
    for t in th:
        t.start()
    for t in th:
        t.join()
    h.set_coalescing(1)
    return got


@pytest.mark.parametrize("seg", [256, 4096])
@pytest.mark.parametrize("which", ["d128b2", "d48b2", "d48b1"])
def test_results_equal_at_every_cache_state(npb, oracle, corpora, monkeypatch, seg, which):
    c = corpora[which]
    ix, qs = c["ix"], c["qs"]
    monkeypatch.setenv("PB_HOST_SEGMENT_BYTES", str(seg))
    res = _open(npb, oracle, ix)
    h = _open(npb, oracle, ix, host_residuals=True)
    rows = int(np.asarray(ix.residuals).size)
    ids = [0, 3, 77, 401, len(ix.doc_lengths) - 1]
    try:
        want = _calls(res, npb, qs, ids)
        want_threads = _threads(res, npb, qs)
        for lanes in (1, 2):
            h.set_lanes(lanes)
            assert _calls(h, npb, qs, ids) == want                                   # the cache off
            h.set_row_cache(rows // 3)
            assert _calls(h, npb, qs, ids) == want                                   # on, empty: counting
            half = h.fill_row_cache()                                                # by the counts of those searches
            st = h.row_cache_stats()
            assert 0 < st["cached_docs"] == len(half) and st["cached_bytes"] <= rows // 3
            assert _calls(h, npb, qs, ids) == want
            h.set_row_cache(rows)
            assert len(h.fill_row_cache(range(len(ix.doc_lengths)))) == len(ix.doc_lengths)
            assert h.row_cache_stats()["cached_bytes"] == rows
            h.row_cache_stats(reset=True)
            assert _calls(h, npb, qs, ids) == want
            st = h.row_cache_stats()
            assert st["hit_docs"] == st["staged_docs"] > 0                          # every staged doc came from the cache
            assert _threads(h, npb, qs) == want_threads
            h.set_row_cache(0)
        for q, (got_ids, got_sc) in zip(qs, want[0][0]):
            w = oracle.search_one(ix, q, oracle.SearchParameters(**PARAMS[0]))
            assert got_ids == w.passage_ids.tolist() and got_sc == w.scores.astype(np.float32).tobytes()
    finally:
        h.close()
        res.close()


def test_fill_by_counts_and_hits_follow_the_traces(npb, oracle, corpus):
    ix, qs = corpus["ix"], corpus["qs"]
    h = _open(npb, oracle, ix, host_residuals=True)
    D, pk = len(ix.doc_lengths), np.asarray(ix.residuals).shape[1]
    try:
        h.set_row_cache(40_000)
        kept = []
        for i, kw in enumerate(PARAMS + PARAMS[:1]):                   # traced searches, no fill in between
            _, tr = h.search_batch(qs[i:], npb.SearchParameters(**kw), trace=True)
            kept += tr.kept
        st = h.row_cache_stats(reset=True)
        assert st["staged_docs"] == sum(len(k) for k in kept) and st["hit_docs"] == 0 and st["cached_docs"] == 0
        counts = row_cache.keep_counts(kept, D)
        want, used = row_cache.fit_or_skip(row_cache.order_by_counts(counts), ix.doc_lengths, pk, 40_000)
        got = h.fill_row_cache()
        assert got.tolist() == want.tolist()
        st = h.row_cache_stats()
        assert (st["cached_docs"], st["cached_bytes"], st["dead_bytes"], st["budget_bytes"]) == (len(want), used, 0, 40_000)
        # the counts were reset: a fill by counts right away caches nothing
        assert h.fill_row_cache().tolist() == [] and h.row_cache_stats()["cached_docs"] == 0
        h.fill_row_cache(want)
        cached = set(want.tolist())
        for kw in PARAMS:
            h.row_cache_stats(reset=True)
            _, tr = h.search_batch(qs, npb.SearchParameters(**kw), trace=True)
            hit = [d for k in tr.kept for d in k.tolist() if d in cached]
            st = h.row_cache_stats()
            assert st["staged_docs"] == sum(len(k) for k in tr.kept)
            assert st["hit_docs"] == len(hit) and st["hit_bytes"] == int(np.asarray(ix.doc_lengths)[hit].sum()) * pk
    finally:
        h.close()


def test_fill_with_ids_fits_or_skips(npb, oracle, corpus):
    ix = corpus["ix"]
    h = _open(npb, oracle, ix, host_residuals=True)
    D, pk, dl = len(ix.doc_lengths), np.asarray(ix.residuals).shape[1], np.asarray(ix.doc_lengths)
    try:
        before = h.memory_usage()
        h.set_row_cache(int(dl[:50].sum()) * pk)
        ids = [D + 3, 7, -1, 1000, 7, 5] + list(range(100, 200)) + [2 * D, 9]
        want, _ = row_cache.fit_or_skip(row_cache.order_of_ids(ids, D), dl, pk, int(dl[:50].sum()) * pk)
        got = h.fill_row_cache(ids)
        assert got.tolist() == want.tolist() and 0 < len(want) < len(row_cache.order_of_ids(ids, D))  # some skipped
        assert h.row_cache_stats()["cached_docs"] == len(want)
        big = int(np.argmax(dl))
        h.set_row_cache(int(dl[big]) * pk - 1)                       # smaller than one doc: nothing of it is cached
        assert h.row_cache_stats()["cached_docs"] == 0               # the lower budget emptied the cache
        assert big not in h.fill_row_cache([big]).tolist()
        assert h.fill_row_cache([D, -5]).tolist() == [] and h.row_cache_stats()["cached_bytes"] == 0
        h.set_row_cache(0)
        assert h.memory_usage() == before
    finally:
        h.close()


def _sequence(npb, docs, codec, pk, ops):
    """appends (encoded and with a codec), deletes (scattered, oldest, all) and an append under a filled cache.  After
    each, ops["results"](kw) must equal ops["want"](live, kw) for the corpus docs `live` the handle holds, and the
    cache's cached_docs and dead_bytes must follow the deleted cached docs.  ops: set(budget), fill(ids), stats(),
    append(embeddings), append_encoded(codes, packed, lengths), delete(ids), results(kw), want(live, kw)."""
    live = list(range(1000))                       # the corpus doc of each current id
    ops["set"](10 ** 9)
    cached = set(ops["fill"](list(range(0, 1000, 2))))
    assert cached == set(range(0, 1000, 2))
    dead = 0

    def check():
        for kw in PARAMS:
            assert ops["results"](kw) == ops["want"](live, kw)
        st = ops["stats"]()
        assert (st["cached_docs"], st["dead_bytes"]) == (len(cached & set(live)), dead * pk), (st, dead)

    def encoded(a, b):
        codes, packed = codec.encode_chunk(np.concatenate(docs[a:b], 0))
        return np.asarray(codes), np.asarray(packed), [len(d) for d in docs[a:b]]
    ops["append_encoded"](*encoded(1000, 1100))
    live += list(range(1000, 1100))
    check()
    ops["append"](docs[1100:1200])
    live += list(range(1100, 1200))
    check()
    for pattern in ("scattered", "oldest", "all"):
        n = len(live)
        gone = {"scattered": list(range(3, n, 7)), "oldest": list(range(40)), "all": list(range(n))}[pattern]
        dead += sum(len(docs[live[i]]) for i in gone if live[i] in cached)
        ops["delete"](gone)
        drop = set(gone)
        live = [d for i, d in enumerate(live) if i not in drop]
        check()
    ops["append_encoded"](*encoded(1200, 1300))
    live += list(range(1200, 1300))
    check()


def test_mutations_under_a_filled_cache(npb, oracle, corpus, monkeypatch):
    monkeypatch.setenv("PB_HOST_SEGMENT_BYTES", "256")
    monkeypatch.setenv("PB_DELETE_WINDOW_TOKENS", "500")
    ix, art = corpus["ix"], corpus["art"]
    h = _open(npb, oracle, ix, range(1000), host_residuals=True, mutable=True)
    codec = npb.ResidualCodec(NBITS, art.centroids, art.bucket_cutoffs)

    def want(live, kw):
        f = _open(npb, oracle, ix, live, host_residuals=True)
        try:
            return _res(f.search_batch(corpus["qs"], npb.SearchParameters(**kw)))
        finally:
            f.close()
    try:
        ops = dict(set=h.set_row_cache, fill=lambda ids: h.fill_row_cache(ids).tolist(), stats=h.row_cache_stats,
                   append=lambda e: h.append(e, codec), append_encoded=h.append_encoded, delete=h.delete,
                   results=lambda kw: _res(h.search_batch(corpus["qs"], npb.SearchParameters(**kw))), want=want)
        _sequence(npb, corpus["docs"], codec, DIM * NBITS // 8, ops)
        held = h.memory_usage()["device_bytes"]
        h.set_row_cache(0)
        assert h.memory_usage()["device_bytes"] < held and h.row_cache_stats()["budget_bytes"] == 0
    finally:
        codec.close()
        h.close()


@pytest.mark.parametrize("kind", ["group", "deployment", "R2S1", "R2S2"])
def test_mutations_on_groups_deployments_and_replicas(npb, oracle, corpus, tmp_path, monkeypatch, kind):
    """the same sequence on mutable host-tier ranks of a ShardGroup or a deployment, and on replica sets, compared with a
    single mutable host-tier handle (no cache) that takes the same mutations"""
    monkeypatch.setenv("PB_HOST_SEGMENT_BYTES", "4096")
    monkeypatch.setenv("PB_DELETE_WINDOW_TOKENS", "3000")
    path = str(tmp_path / "ix")
    npb.create_index(corpus["docs"][:1000], path, nbits=NBITS, num_partitions=K, batch_size=400, seed=7).close()
    kw = dict(host_residuals=True, mutable=True)
    if kind == "group":
        h = npb.ShardGroup([npb.MmapIndex.load_shard(path, r, 2, **kw) for r in range(2)])
    elif kind == "deployment":
        h = npb.MmapIndex.load_devices(path, [0, 0], **kw)
    else:
        h = npb.MmapIndex.load_replicas(path, [0, 0] if kind == "R2S1" else [0, 0, 0, 0],
                                        shards=1 if kind == "R2S1" else 2, **kw)
    one = npb.MmapIndex.load(path, **kw)
    base = oracle.load_index(path)
    codec = npb.ResidualCodec(NBITS, base.centroids, base.bucket_cutoffs)
    copies = 2 if kind.startswith("R2") else 1
    parts = h.shards if kind == "group" else [h]

    def both(name):
        def call(*a):
            getattr(one, name)(*(a if name != "append" else (a[0], codec)))
            return getattr(h, name)(*(a if name != "append" else (a[0], codec)))
        return call

    def fill(ids):
        got = np.concatenate([p.fill_row_cache(ids) for p in parts]).tolist()
        assert len(got) == copies * len(ids) and got == got[:len(ids)] * copies
        return got[:len(ids)]

    def stats():
        st = [p.row_cache_stats() for p in parts]
        return {k: sum(s[k] for s in st) // copies for k in ("cached_docs", "dead_bytes")}
    try:
        ops = dict(set=lambda b: [p.set_row_cache(b) for p in parts], fill=fill, stats=stats,
                   append=both("append"), append_encoded=both("append_encoded"), delete=both("delete"),
                   results=lambda kw: _res(h.search_batch(corpus["qs"], npb.SearchParameters(**kw))),
                   want=lambda live, kw: _res(one.search_batch(corpus["qs"], npb.SearchParameters(**kw))))
        _sequence(npb, corpus["docs"], codec, DIM * NBITS // 8, ops)
        held = [p.memory_usage()["device_bytes"] for p in parts]
        for p in parts:
            p.set_row_cache(0)
        assert all(p.memory_usage()["device_bytes"] < b for p, b in zip(parts, held))
    finally:
        codec.close()
        h.close()
        one.close()


def test_fills_during_concurrent_searches(npb, oracle, corpus):
    ix, qs = corpus["ix"], corpus["qs"]
    h = _open(npb, oracle, ix, host_residuals=True)
    dl, pk = np.asarray(ix.doc_lengths), np.asarray(ix.residuals).shape[1]
    try:
        want = {i: _res(h.search_batch(qs[i:i + 4], npb.SearchParameters(**PARAMS[i % 2]))) for i in range(8)}
        h.set_row_cache(int(dl.sum()) * pk // 2)
        sets = [list(range(0, len(dl), 2)), list(range(len(dl) - 1, 0, -3))]
        stop, errors, seen = threading.Event(), [], [0] * 8

        def reader(i):
            try:
                while not stop.is_set():
                    got = _res(h.search_batch(qs[i:i + 4], npb.SearchParameters(**PARAMS[i % 2])))
                    assert got == want[i]
                    seen[i] += 1
            except Exception as e:  # pragma: no cover - reported below
                errors.append(e)
        th = [threading.Thread(target=reader, args=(i,)) for i in range(8)]
        for t in th:
            t.start()
        try:
            for k in range(12):
                assert len(h.fill_row_cache(sets[k % 2])) > 0
        finally:
            stop.set()
            for t in th:
                t.join()
        assert not errors, errors[:1]
        assert all(seen)
    finally:
        h.close()


def test_refusals_leave_the_handle_unchanged(npb, oracle, corpus):
    import torch
    ix, qs, art = corpus["ix"], corpus["qs"], corpus["art"]
    D = 100
    codes, packed, dl = [np.asarray(a)[:int(np.sum(ix.doc_lengths[:D]))] for a in (ix.codes, ix.residuals)] + \
        [np.asarray(ix.doc_lengths[:D], np.int64)]
    t = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in dict(
        cen=art.centroids, w=art.bucket_weights, codes=codes, res=packed, dl=dl).items()}
    adopt = npb.MmapIndex.from_device_pointers(DIM, NBITS, K, D, len(codes), t["cen"].data_ptr(), t["w"].data_ptr(),
                                               t["codes"].data_ptr(), t["res"].data_ptr(), t["dl"].data_ptr(), None,
                                               None, adopt_residuals=True)
    res = _open(npb, oracle, ix)
    host = _open(npb, oracle, ix, host_residuals=True)
    p = npb.SearchParameters(**PARAMS[0])
    try:
        for h in (adopt, res, host):
            mem, want = h.memory_usage(), _res(h.search_batch(qs, p))
            if h is not host:
                with pytest.raises(npb.PlaidError) as e:
                    h.set_row_cache(1 << 20)
                assert e.value.status == 4
            with pytest.raises(npb.PlaidError) as e:
                h.set_row_cache(-1)
            assert e.value.status == 1
            with pytest.raises(npb.PlaidError) as e:                 # no budget: a fill is refused
                h.fill_row_cache()
            assert e.value.status == (1 if h is host else 4)
            assert h.memory_usage() == mem and _res(h.search_batch(qs, p)) == want
            assert h.row_cache_stats()["budget_bytes"] == 0
        mem = host.memory_usage()
        host.set_row_cache(1 << 20)
        assert host.memory_usage()["device_bytes"] > mem["device_bytes"]
        host.fill_row_cache(range(50))
        filled = host.memory_usage()
        with pytest.raises(npb.PlaidError) as e:
            host.set_row_cache(-5)
        assert e.value.status == 1 and host.memory_usage() == filled and host.row_cache_stats()["cached_docs"] == 50
        host.set_row_cache(0)
        assert host.memory_usage() == mem
        st = host.row_cache_stats()
        assert (st["budget_bytes"], st["cached_docs"], st["cached_bytes"]) == (0, 0, 0)
    finally:
        adopt.close()
        res.close()
        host.close()
