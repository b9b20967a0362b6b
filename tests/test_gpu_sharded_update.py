"""Appends and deletes on a doc-sharded deployment (pb_index_delete_sharded, pb_index_append_sharded,
pb_index_append_encoded_sharded), with G handles on device 0 in an in-process shard group.  After every change each rank
equals a fresh pb_index_open of its expected range of the changed index (accessors, inverted file with its base,
decompression, work counters of a group search), and group searches equal a single handle changed by pb_index_delete /
pb_index_append_encoded and the CPU oracle on the changed index.  A directory changed through a group of load_shard
handles is byte-identical to one changed through pb_index_load and the single-handle calls."""
import filecmp
import os
import shutil
import sys
import threading

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import sharded_update as su  # noqa: E402
from ivf_delete import delete_ivf  # noqa: E402
from ivf_slice import ivf_slice  # noqa: E402
from test_gpu_append import COUNTERS, DIM, K, NBITS, PARAMS, _oracle_index  # noqa: E402

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
    """1800 ragged docs encoded with one fixed codec, and 400 more to append"""
    docs = oracle.synthetic_corpus(2200, 40, dim=DIM, seed=71, ragged=True)
    flat = np.concatenate(docs, 0)
    rng = np.random.default_rng(3)
    cent = flat[rng.choice(len(flat), K, replace=False)].copy()
    art = oracle.prepare_codec_artifacts(docs, cent, NBITS, 3)
    codes, packed, dl = oracle.encode_documents(docs, art, NBITS)
    qs, _ = oracle.synthetic_queries(docs, 5, nq=32, seed=12)
    qs += oracle.synthetic_queries(docs[1700:], 2, nq=32, seed=13)[0]
    return dict(docs=docs, art=art, codes=codes, packed=packed, dl=np.asarray(dl, np.int64), qs=qs)


class State:
    """the whole index as arrays (codes, packed residuals, doc lengths, ivf, ivf_lengths), changed in numpy"""

    def __init__(self, oracle, art, codes, packed, dl):
        self.art, self.codes, self.packed, self.dl = art, codes, packed, np.asarray(dl, np.int64)
        self.ivf, self.lens = oracle.build_ivf(codes, self.dl, K)

    @property
    def off(self):
        return np.concatenate([[0], np.cumsum(self.dl)]).astype(np.int64)

    def delete(self, ids):
        D = len(self.dl)
        gone = su.deleted_set(ids, D)
        keep = ~np.isin(np.arange(D), gone)
        tok = np.repeat(keep, self.dl)
        self.ivf, self.lens = delete_ivf(self.ivf, self.lens, gone, D)
        self.codes, self.packed, self.dl = self.codes[tok], self.packed[tok], self.dl[keep]

    def append(self, codes, packed, dl):
        from ivf_merge import merge_ivf
        self.ivf, self.lens = merge_ivf(self.ivf, self.lens, codes, dl, len(self.dl), K)
        self.codes = np.concatenate([self.codes, codes])
        self.packed = np.concatenate([self.packed, packed])
        self.dl = np.concatenate([self.dl, np.asarray(dl, np.int64)])

    def open_range(self, npb, b, e):
        off = self.off
        iv, ln = ivf_slice(self.ivf, self.lens, b, e)
        return npb.MmapIndex.from_arrays(self.art.centroids, self.art.bucket_weights, self.codes[off[b]:off[e]],
                                         self.packed[off[b]:off[e]], self.dl[b:e], iv, ln, NBITS, doc_id_base=b)

    def oracle_index(self, oracle):
        return _oracle_index(oracle, self.art, self.codes, self.packed, self.dl)


def _search_all(grp, npb, qs, kw, subset=None):
    res = grp.search_batch(qs, npb.SearchParameters(**kw), subset=subset)
    counters = [{k: s.last_work_counters()[k] for k in COUNTERS} for s in grp.shards]
    return [(r.passage_ids.tolist(), r.scores.tobytes()) for r in res], counters


def _check(npb, oracle, grp, st, bounds, single, qs):
    """every rank == a fresh open of its range; group searches == fresh group == single handle == oracle"""
    D = len(st.dl)
    assert bounds[0] == 0 and bounds[-1] == D
    fresh = [st.open_range(npb, int(bounds[r]), int(bounds[r + 1])) for r in range(len(grp.shards))]
    fgrp = npb.ShardGroup(fresh)
    try:
        for r, (s, f) in enumerate(zip(grp.shards, fresh)):
            assert s.num_documents() == f.num_documents() == bounds[r + 1] - bounds[r], r
            assert s.num_embeddings() == f.num_embeddings(), r
            assert s.avg_doclen() == f.avg_doclen(), r
            a, b = s.export_ivf(), f.export_ivf()         # global ids: the new base shows here
            assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]), r
            if f.num_documents():
                ids = sorted({int(bounds[r]), int(bounds[r + 1]) - 1, (int(bounds[r]) + int(bounds[r + 1])) // 2})
                ea, la = s.decompress_documents(ids)
                ef, lf = f.decompress_documents(ids)
                assert np.array_equal(la, lf) and np.array_equal(ea, ef), r
        assert single.num_documents() == D
        oix = st.oracle_index(oracle)
        subset = sorted(set(range(0, D, 3)) | set(range(max(D - 30, 0), D)))
        for kw in PARAMS[:2]:
            for sub in (None, subset) if kw.get("centroid_batch_size") else (None,):
                got, cnt = _search_all(grp, npb, qs, kw, sub)
                want, fcnt = _search_all(fgrp, npb, qs, kw, sub)
                assert got == want, (kw, sub is not None)
                assert cnt == fcnt, (kw, cnt, fcnt)
                res = single.search_batch(qs, npb.SearchParameters(**kw), subset=sub)
                assert got == [(r.passage_ids.tolist(), r.scores.tobytes()) for r in res], kw
                po = oracle.SearchParameters(**kw)
                for q, (pid, sc) in zip(qs, got):
                    w = oracle.search_one(oix, q, po, subset=sub)
                    assert pid == w.passage_ids.tolist() and sc == w.scores.astype(np.float32).tobytes(), kw
    finally:
        fgrp.close()


def _setup(npb, oracle, c, D, bounds):
    st = State(oracle, c["art"], c["codes"][:int(np.sum(c["dl"][:D]))], c["packed"][:int(np.sum(c["dl"][:D]))],
               c["dl"][:D])
    grp = npb.ShardGroup([st.open_range(npb, int(bounds[r]), int(bounds[r + 1])) for r in range(len(bounds) - 1)])
    single = st.open_range(npb, 0, D)
    return st, grp, single


def _patterns(D, bounds, rng):
    return [("scattered_invalid", np.concatenate([rng.choice(D, D // 9, replace=False), [-3, D, D + 7, 5, 5]])),
            ("oldest", np.arange(0, int(bounds[1]))),                  # empties rank 0
            ("newest", np.arange(D - 150, D)),
            ("across_a_boundary", np.arange(int(bounds[1]) - 20, int(bounds[1]) + 20)),
            ("every_other", np.arange(0, D, 2)),
            ("none", np.array([-1, D], np.int64)),
            ("all", np.arange(D))]


@pytest.mark.parametrize("G", [2, 3, 8])
def test_delete_patterns(npb, oracle, corpus, G):
    c = corpus
    D = 1800
    bounds0 = np.array([g * D // G for g in range(G)] + [D], np.int64)      # make_shard's split
    for name, ids in _patterns(D, bounds0, np.random.default_rng(G)):
        st, grp, single = _setup(npb, oracle, c, D, bounds0)
        try:
            n = grp.delete(ids)
            want = len(su.deleted_set(ids, D))
            assert n == want and all(x == want for x in grp.all_results), name
            assert single.delete(ids) == want
            st.delete(ids)
            _check(npb, oracle, grp, st, su.delete_bounds(bounds0, ids), single, c["qs"])
        finally:
            grp.close()
            single.close()


@pytest.mark.parametrize("G", [2, 3, 8])
def test_append_delete_cycles(npb, oracle, corpus, G):
    c = corpus
    D = 1500
    bounds = np.array([g * D // G for g in range(G)] + [D], np.int64)
    st, grp, single = _setup(npb, oracle, c, D, bounds)
    codec = npb.ResidualCodec(NBITS, c["art"].centroids, c["art"].bucket_cutoffs)
    off = np.concatenate([[0], np.cumsum(c["dl"])]).astype(np.int64)
    rng = np.random.default_rng(9)
    nxt = D
    try:
        for step, n in enumerate((120, 0, 90)):
            t0, t1 = int(off[nxt]), int(off[nxt + n])
            Dt = len(st.dl)
            if step % 2 == 0:                                             # encoded
                got = grp.append_encoded(c["codes"][t0:t1], c["packed"][t0:t1], c["dl"][nxt:nxt + n])
                single.append_encoded(c["codes"][t0:t1], c["packed"][t0:t1], c["dl"][nxt:nxt + n])
            else:                                                         # encoded on the device
                got = grp.append(c["docs"][nxt:nxt + n], codec)
                single.append(c["docs"][nxt:nxt + n], codec)
            assert got == list(range(Dt, Dt + n)) and all(x == Dt for x in grp.all_results)
            st.append(c["codes"][t0:t1], c["packed"][t0:t1], c["dl"][nxt:nxt + n])
            nxt += n
            bounds = bounds.copy()
            bounds[-1] += n
            _check(npb, oracle, grp, st, bounds, single, c["qs"])
            ids = rng.choice(len(st.dl), 60, replace=False)
            assert grp.delete(ids) == single.delete(ids) == 60
            st.delete(ids)
            bounds = su.delete_bounds(bounds, ids)
            _check(npb, oracle, grp, st, bounds, single, c["qs"])
        # device-encoded append into an emptied last rank
        last = np.arange(int(bounds[-2]), int(bounds[-1]))
        grp.delete(last)
        single.delete(last)
        st.delete(last)
        bounds = su.delete_bounds(bounds, last)
        assert grp.shards[-1].num_documents() == 0
        got = grp.append(c["docs"][nxt:nxt + 30], codec)
        single.append(c["docs"][nxt:nxt + 30], codec)
        t0, t1 = int(off[nxt]), int(off[nxt + 30])
        st.append(c["codes"][t0:t1], c["packed"][t0:t1], c["dl"][nxt:nxt + 30])
        bounds[-1] += 30
        _check(npb, oracle, grp, st, bounds, single, c["qs"])
    finally:
        codec.close()
        grp.close()
        single.close()


def _state(grp):
    return [(s.num_documents(), s.num_embeddings(), s.export_ivf()[0].tobytes(), s.export_ivf()[1].tobytes())
            for s in grp.shards]


def test_rejections_change_nothing_on_any_rank(npb, oracle, corpus, tmp_path):
    import next_plaid_b200 as m
    c = corpus
    D = 900
    bounds = np.array([0, 400, 900], np.int64)
    st, grp, single = _setup(npb, oracle, c, D, bounds)
    single.close()
    try:
        before = _state(grp)

        def expect(status, call):
            errs = [None, None]

            def run(r):
                try:
                    call(r, grp.shards[r])
                except m.PlaidError as e:
                    errs[r] = e
            ths = [threading.Thread(target=run, args=(r,)) for r in range(2)]
            [t.start() for t in ths]
            [t.join() for t in ths]
            assert all(e is not None and e.status == status for e in errs), errs
            assert _state(grp) == before
            return errs

        L = m.load_library()
        import ctypes as C

        def delete(ids_by_rank, dir_by_rank=(None, None)):
            def call(r, s):
                ids = np.asarray(ids_by_rank[r], np.int64)
                n = C.c_int64()
                d = dir_by_rank[r]
                m.index._check(L.pb_index_delete_sharded(s._h, m.index._ptr(ids), len(ids),
                                                         None if d is None else os.fsencode(d), C.byref(n)))
            return call
        # different id lists per rank; index_dir on only one rank
        expect(1, delete(([1, 2], [1, 3])))
        expect(1, delete(([1, 2], [1, 2]), (None, str(tmp_path))))
        # codec mismatch on the last rank: every rank reports rank 1's status and names it
        other = np.random.default_rng(0).standard_normal((K, DIM)).astype(np.float32)
        bad = npb.ResidualCodec(NBITS, other, c["art"].bucket_cutoffs)
        try:
            docs = c["docs"][900:905]
            dl = np.array([d.shape[0] for d in docs], np.int64)
            flat = np.concatenate(docs, 0).astype(np.float32)

            def app(r, s):
                first = C.c_int64()
                m.index._check(L.pb_index_append_sharded(s._h, bad._h if r == 1 else None,
                                                         m.index._ptr(flat) if r == 1 else None, m.index._ptr(dl),
                                                         len(dl), 0, None, 1000, C.byref(first)))
            errs = expect(1, app)
            assert all("rank 1" in str(e) for e in errs), errs
        finally:
            bad.close()
    finally:
        grp.close()
    # a group whose ranges do not tile [0, D): both handles have base 0
    a = st.open_range(npb, 0, 400)
    b = st.open_range(npb, 0, 400)
    g2 = npb.ShardGroup([a, b])
    try:
        before = _state(g2)
        with pytest.raises(m.PlaidError) as e:
            g2.delete([1, 2])
        assert e.value.status == 1 and _state(g2) == before
        with pytest.raises(m.PlaidError):
            g2.append_encoded(c["codes"][:5], c["packed"][:5], [5])
        assert _state(g2) == before
    finally:
        g2.close()


def test_adopted_residual_member_is_refused(npb, oracle, corpus):
    import next_plaid_b200 as m
    import torch
    c = corpus
    st = State(oracle, c["art"], c["codes"][:int(np.sum(c["dl"][:300]))], c["packed"][:int(np.sum(c["dl"][:300]))],
               c["dl"][:300])
    off = st.off
    a = st.open_range(npb, 0, 150)
    iv, ln = ivf_slice(st.ivf, st.lens, 150, 300)
    dev = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in dict(
        cen=st.art.centroids.astype(np.float32), w=st.art.bucket_weights.astype(np.float32),
        codes=st.codes[off[150]:].astype(np.int64), res=st.packed[off[150]:].astype(np.uint8),
        dl=st.dl[150:].astype(np.int64), ivf=iv.astype(np.int64), lens=ln.astype(np.int32)).items()}
    b = npb.MmapIndex.from_device_pointers(DIM, NBITS, K, 150, int(off[300] - off[150]), dev["cen"].data_ptr(),
                                           dev["w"].data_ptr(), dev["codes"].data_ptr(), dev["res"].data_ptr(),
                                           dev["dl"].data_ptr(), dev["ivf"].data_ptr(), dev["lens"].data_ptr(),
                                           doc_id_base=150, adopt_residuals=True)
    g = npb.ShardGroup([a, b])
    try:
        before = _state(g)
        with pytest.raises(m.PlaidError) as e:
            g.delete([1, 200])
        assert e.value.status == 4 and _state(g) == before
    finally:
        g.close()
        torch.cuda.synchronize()


@pytest.mark.parametrize("W", [2, 3, 8])
def test_directory_through_a_load_shard_group(npb, oracle, tmp_path, W):
    docs = oracle.synthetic_corpus(3300, 40, dim=DIM, seed=91, ragged=True)
    a, b = str(tmp_path / "a"), str(tmp_path / "b")
    npb.create_index(docs[:2600], a, nbits=NBITS, num_partitions=K, batch_size=1000, seed=7).close()
    shutil.copytree(a, b)
    base = oracle.load_index(a)
    codec = npb.ResidualCodec(NBITS, base.centroids, base.bucket_cutoffs)
    qs, _ = oracle.synthetic_queries(docs, 5, nq=32, seed=15)
    grp = npb.ShardGroup([npb.MmapIndex.load_shard(a, r, W) for r in range(W)])
    single = npb.MmapIndex.load(b)

    def same_files():
        fa, fb = sorted(os.listdir(a)), sorted(os.listdir(b))
        assert fa == fb
        for f in fa:
            assert filecmp.cmp(os.path.join(a, f), os.path.join(b, f), shallow=False), f

    try:
        rng = np.random.default_rng(4)
        steps = [("delete", rng.choice(2600, 300, replace=False)), ("append", (2600, 3000)),
                 ("delete", np.arange(700, 1200)), ("append", (3000, 3300))]
        for kind, arg in steps:
            if kind == "delete":
                assert grp.delete(arg, index_dir=a) == single.delete(arg, index_dir=b)
            else:
                got = grp.append(docs[arg[0]:arg[1]], codec, index_dir=a, batch_size=250)
                assert got == single.append(docs[arg[0]:arg[1]], codec, index_dir=b, batch_size=250)
            same_files()
            p = npb.SearchParameters(top_k=10, n_ivf_probe=8, n_full_scores=256)
            want = [(r.passage_ids.tolist(), r.scores.tobytes()) for r in single.search_batch(qs, p)]
            got = [(r.passage_ids.tolist(), r.scores.tobytes()) for r in grp.search_batch(qs, p)]
            assert got == want, kind
            # reloading the directory with fresh bounds searches the same
            re = npb.ShardGroup([npb.MmapIndex.load_shard(a, r, W) for r in range(W)])
            try:
                assert [(r.passage_ids.tolist(), r.scores.tobytes()) for r in re.search_batch(qs, p)] == want
            finally:
                re.close()
        # a directory that does not hold D_total documents: refused on every rank, nothing changes
        c = str(tmp_path / "c")
        npb.create_index(docs[:500], c, nbits=NBITS, num_partitions=K, batch_size=1000, seed=7).close()
        snap = [(s.num_documents(), s.export_ivf()[0].tobytes()) for s in grp.shards]
        with pytest.raises(npb.PlaidError) as e:
            grp.delete([1, 2], index_dir=c)
        assert e.value.status == 1
        assert [(s.num_documents(), s.export_ivf()[0].tobytes()) for s in grp.shards] == snap
    finally:
        codec.close()
        grp.close()
        single.close()


def test_readers_see_each_rank_before_or_after(npb, oracle, corpus):
    c = corpus
    D = 1800
    bounds = np.array([0, 600, 1200, 1800], np.int64)
    st, grp, single = _setup(npb, oracle, c, D, bounds)
    single.close()
    ids = np.arange(0, D, 3)
    after_bounds = su.delete_bounds(bounds, ids)
    def snap(s):                                  # one read: the inverted file with its base and lengths
        iv, ln = s.export_ivf()
        return iv.tobytes() + ln.tobytes()
    before = [snap(s) for s in grp.shards]
    st.delete(ids)
    after = []
    for r in range(3):
        f = st.open_range(npb, int(after_bounds[r]), int(after_bounds[r + 1]))
        after.append(snap(f))
        f.close()
    stop, seen, bad = threading.Event(), [], []

    def reader(r):
        s = grp.shards[r]
        while not stop.is_set():
            x = snap(s)
            if x not in (before[r], after[r]):
                bad.append(r)
            seen.append(x == after[r])

    ths = [threading.Thread(target=reader, args=(r,)) for r in range(3)]
    try:
        [t.start() for t in ths]
        assert grp.delete(ids) == len(ids)
    finally:
        stop.set()
        [t.join() for t in ths]
        grp.close()
    assert not bad
