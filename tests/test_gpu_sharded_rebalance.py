"""Rebalancing a doc-sharded deployment on the device (pb_index_rebalance_sharded), with G handles on device 0 in an
in-process shard group.  After every rebalance each rank equals a fresh pb_index_open of its new range (accessors,
inverted file with its base, decompression, work counters of a group search), and group searches equal a single
handle and the CPU oracle (_check of the sharded-update tests).  Refusals change no rank; a group of load_shard handles
ends up equal to load_range of its new bounds and leaves the directory untouched; unsorted inverted files follow the
rank-order concatenation rule of tests/sharded_rebalance.py."""
import os
import sys
import threading

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import sharded_rebalance as sr  # noqa: E402
import sharded_update as su  # noqa: E402
from ivf_slice import ivf_slice, shard_bounds  # noqa: E402
from test_gpu_append import DIM, K, NBITS  # noqa: E402
from test_gpu_sharded_update import State, _check, corpus, npb  # noqa: E402,F401 - fixtures

pytestmark = pytest.mark.gpu


def _group(npb, st, bounds):
    return npb.ShardGroup([st.open_range(npb, int(bounds[r]), int(bounds[r + 1])) for r in range(len(bounds) - 1)])


def _state(c, oracle, D):
    n = int(np.sum(c["dl"][:D]))
    return State(oracle, c["art"], c["codes"][:n], c["packed"][:n], c["dl"][:D])


def _skewed(D, G):
    """rank 0 empty, ranks 1 .. G - 2 five docs each, the rest on the last rank"""
    return np.array([0, 0] + [5 * g for g in range(1, G - 1)] + [D], np.int64)


def _rebalance(grp, bounds=None):
    got = grp.rebalance(bounds)
    assert all(np.array_equal(x, got) for x in grp.all_results)
    return got


@pytest.mark.parametrize("G", [2, 3, 5])
def test_skewed_to_balanced(npb, oracle, corpus, G):
    c = corpus
    D = 1500
    st = _state(c, oracle, D)
    b0 = _skewed(D, G)
    assert len(b0) == G + 1 and b0[1] == 0
    grp, single = _group(npb, st, b0), st.open_range(npb, 0, D)
    try:
        got = _rebalance(grp)
        assert np.array_equal(got, shard_bounds(st.dl, G)), got
        _check(npb, oracle, grp, st, got, single, c["qs"])
    finally:
        grp.close()
        single.close()


def test_explicit_bounds(npb, oracle, corpus):
    c = corpus
    D, G = 1500, 4
    st = _state(c, oracle, D)
    bounds = np.array([0, 375, 750, 1125, 1500], np.int64)
    grp, single = _group(npb, st, bounds), st.open_range(npb, 0, D)
    try:
        for want in ([0, 1300, 1400, 1450, 1500],        # rank 0 takes docs of ranks 1, 2 and 3
                     [0, 1300, 1300, 1450, 1500],        # rank 1 emptied
                     [0, 0, 0, 1500, 1500],              # everything on rank 2
                     [0, 10, 20, 30, 1500],              # from rank 2 to the last rank and back down
                     None):                              # back to balanced
            got = _rebalance(grp, want)
            assert np.array_equal(got, shard_bounds(st.dl, G) if want is None else want), (want, got)
            _check(npb, oracle, grp, st, got, single, c["qs"])
    finally:
        grp.close()
        single.close()


def test_interleaved_with_updates(npb, oracle, corpus):
    c = corpus
    D, G = 1200, 3
    st = _state(c, oracle, D)
    bounds = np.array([0, 400, 800, 1200], np.int64)
    grp, single = _group(npb, st, bounds), st.open_range(npb, 0, D)
    off = np.concatenate([[0], np.cumsum(c["dl"])]).astype(np.int64)
    nxt = D
    rng = np.random.default_rng(5)

    def append(n):
        nonlocal nxt, bounds
        t0, t1 = int(off[nxt]), int(off[nxt + n])
        grp.append_encoded(c["codes"][t0:t1], c["packed"][t0:t1], c["dl"][nxt:nxt + n])
        single.append_encoded(c["codes"][t0:t1], c["packed"][t0:t1], c["dl"][nxt:nxt + n])
        st.append(c["codes"][t0:t1], c["packed"][t0:t1], c["dl"][nxt:nxt + n])
        nxt += n
        bounds = bounds.copy()
        bounds[-1] += n
        _check(npb, oracle, grp, st, bounds, single, c["qs"])

    try:
        for n in (200, 150, 250):
            append(n)
        bounds = _rebalance(grp)
        assert np.array_equal(bounds, shard_bounds(st.dl, G))
        _check(npb, oracle, grp, st, bounds, single, c["qs"])
        ids = rng.choice(len(st.dl), 120, replace=False)
        assert grp.delete(ids) == single.delete(ids) == 120
        st.delete(ids)
        bounds = su.delete_bounds(bounds, ids)
        _check(npb, oracle, grp, st, bounds, single, c["qs"])
        append(180)
        bounds = _rebalance(grp)
        assert np.array_equal(bounds, shard_bounds(st.dl, G))
        _check(npb, oracle, grp, st, bounds, single, c["qs"])
    finally:
        grp.close()
        single.close()


def _snap(grp):
    return [(s.num_documents(), s.num_embeddings(), s.export_ivf()[0].tobytes(), s.export_ivf()[1].tobytes())
            for s in grp.shards]


def _expect(grp, status, bounds_by_rank):
    """each rank calls with its own bounds; every rank must fail with `status` and no rank may change"""
    import next_plaid_b200 as m
    before = _snap(grp)
    errs = [None] * len(grp.shards)

    def run(r):
        try:
            grp.shards[r].rebalance_sharded(bounds_by_rank[r])
        except m.PlaidError as e:
            errs[r] = e
    ths = [threading.Thread(target=run, args=(r,)) for r in range(len(grp.shards))]
    [t.start() for t in ths]
    [t.join() for t in ths]
    assert all(e is not None and e.status == status for e in errs), errs
    assert _snap(grp) == before


def test_noop_and_refusals(npb, oracle, corpus):
    import torch
    c = corpus
    D, G = 900, 3
    st = _state(c, oracle, D)
    bounds = np.array([0, 200, 650, 900], np.int64)
    grp, single = _group(npb, st, bounds), st.open_range(npb, 0, D)
    try:
        before = _snap(grp)
        assert np.array_equal(_rebalance(grp, bounds), bounds) and _snap(grp) == before
        for bad in ([1, 200, 650, 900], [0, 200, 650, 899], [0, 200, 650, 901], [0, 650, 200, 900]):
            _expect(grp, 1, [bad] * G)
        _expect(grp, 1, [[0, 300, 600, 900], [0, 300, 600, 900], [0, 300, 601, 900]])   # ranks disagree
        _expect(grp, 1, [None, None, [0, 300, 600, 900]])
        _check(npb, oracle, grp, st, bounds, single, c["qs"])
    finally:
        grp.close()
        single.close()
    # a member on the caller's residual array
    off = st.off
    a = st.open_range(npb, 0, 450)
    iv, ln = ivf_slice(st.ivf, st.lens, 450, 900)
    dev = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in dict(
        cen=st.art.centroids.astype(np.float32), w=st.art.bucket_weights.astype(np.float32),
        codes=st.codes[off[450]:].astype(np.int64), res=st.packed[off[450]:].astype(np.uint8),
        dl=st.dl[450:].astype(np.int64), ivf=iv.astype(np.int64), lens=ln.astype(np.int32)).items()}
    b = npb.MmapIndex.from_device_pointers(DIM, NBITS, K, 450, int(off[900] - off[450]), dev["cen"].data_ptr(),
                                           dev["w"].data_ptr(), dev["codes"].data_ptr(), dev["res"].data_ptr(),
                                           dev["dl"].data_ptr(), dev["ivf"].data_ptr(), dev["lens"].data_ptr(),
                                           doc_id_base=450, adopt_residuals=True)
    g = npb.ShardGroup([a, b])
    try:
        _expect(g, 4, [None, None])
        _expect(g, 4, [[0, 300, 900]] * 2)
    finally:
        g.close()
        torch.cuda.synchronize()


@pytest.mark.parametrize("W", [2, 3])
def test_directory_group_equals_load_range(npb, oracle, tmp_path, W):
    docs = oracle.synthetic_corpus(2600, 40, dim=DIM, seed=93, ragged=True)
    a = str(tmp_path / "a")
    npb.create_index(docs[:2000], a, nbits=NBITS, num_partitions=K, batch_size=700, seed=7).close()
    base = oracle.load_index(a)
    codec = npb.ResidualCodec(NBITS, base.centroids, base.bucket_cutoffs)
    qs, _ = oracle.synthetic_queries(docs, 5, nq=32, seed=17)
    grp = npb.ShardGroup([npb.MmapIndex.load_shard(a, r, W) for r in range(W)])
    p = npb.SearchParameters(top_k=10, n_ivf_probe=8, n_full_scores=256)

    def files():
        return {f: open(os.path.join(a, f), "rb").read() for f in sorted(os.listdir(a))}

    try:
        grp.append(docs[2000:2600], codec, index_dir=a, batch_size=250)   # all onto the last rank
        single = npb.MmapIndex.load(a)
        want = [(r.passage_ids.tolist(), r.scores.tobytes()) for r in single.search_batch(qs, p)]
        single.close()
        assert [(r.passage_ids.tolist(), r.scores.tobytes()) for r in grp.search_batch(qs, p)] == want
        snap = files()
        b = _rebalance(grp)
        assert files() == snap
        for r, s in enumerate(grp.shards):
            f = npb.MmapIndex.load_range(a, int(b[r]), int(b[r + 1]))
            try:
                x, y = s.export_ivf(), f.export_ivf()
                assert np.array_equal(x[0], y[0]) and np.array_equal(x[1], y[1]), r
                assert s.num_embeddings() == f.num_embeddings()
                if f.num_documents():
                    ids = sorted({int(b[r]), int(b[r + 1]) - 1, (int(b[r]) + int(b[r + 1])) // 2})
                    ea, la = s.decompress_documents(ids)
                    ef, lf = f.decompress_documents(ids)
                    assert np.array_equal(la, lf) and np.array_equal(ea, ef), r
            finally:
                f.close()
        assert [(r.passage_ids.tolist(), r.scores.tobytes()) for r in grp.search_batch(qs, p)] == want
        fresh = npb.ShardGroup([npb.MmapIndex.load_shard(a, r, W) for r in range(W)])
        try:
            assert [(r.passage_ids.tolist(), r.scores.tobytes()) for r in fresh.search_batch(qs, p)] == want
        finally:
            fresh.close()
    finally:
        codec.close()
        grp.close()


def test_unsorted_inverted_file(npb, oracle, corpus):
    c = corpus
    D, G = 1200, 3
    st = _state(c, oracle, D)
    rng = np.random.default_rng(11)
    off = np.concatenate([[0], np.cumsum(st.lens)]).astype(np.int64)
    st.ivf = np.concatenate([rng.permutation(st.ivf[off[k]:off[k + 1]]) for k in range(K)]).astype(np.int64)
    old = np.array([0, 100, 300, 1200], np.int64)
    grp = _group(npb, st, old)
    try:
        for new in ([0, 700, 1000, 1200], None):
            ranks = []
            for r, s in enumerate(grp.shards):
                iv, ln = s.export_ivf()
                ranks.append((iv - int(old[r]), ln))
            new = _rebalance(grp, new)
            for r, s in enumerate(grp.shards):
                want = sr.rank_ivf(ranks, old, new, r, K)
                iv, ln = s.export_ivf()
                assert np.array_equal(iv - int(new[r]), want[0]) and np.array_equal(ln, want[1]), r
            # the same lists through a fresh open of each range
            cat = sr.global_lists(ranks, old, K)
            st.ivf, st.lens = cat
            for r, s in enumerate(grp.shards):
                f = st.open_range(npb, int(new[r]), int(new[r + 1]))
                try:
                    x, y = s.export_ivf(), f.export_ivf()
                    assert np.array_equal(x[0], y[0]) and np.array_equal(x[1], y[1]), r
                    if f.num_documents():
                        ids = [int(new[r]), int(new[r + 1]) - 1]
                        assert all(np.array_equal(u, v) for u, v in zip(s.decompress_documents(ids),
                                                                       f.decompress_documents(ids)))
                finally:
                    f.close()
            old = new
    finally:
        grp.close()
