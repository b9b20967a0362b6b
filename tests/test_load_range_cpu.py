"""CPU checks for loading a document range of an index directory (pb_index_load_range) and the token-balanced shard
bounds (pb_index_dir_shard_bounds): the numpy restatement of the inverted-file slice, the bounds rule, and the loader's
error contract, which needs no device because every check comes before the device is touched."""
import json
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from ivf_slice import ivf_slice, shard_bounds  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def npb():
    import next_plaid_b200 as m
    m.build_library()
    return m


@pytest.fixture(scope="module")
def index_dir(oracle, tmp_path_factory):
    docs = oracle.synthetic_corpus(120, 12, dim=32, seed=3, ragged=True)
    ix = oracle.create_index(docs, nbits=4, seed=1, num_partitions=16)
    d = tmp_path_factory.mktemp("ix")
    oracle.write_index(ix, str(d), chunk_docs=50)          # three chunks: docs 0-49, 50-99, 100-119
    return str(d), ix


def _lists(ivf, lens):
    off = np.concatenate([[0], np.cumsum(lens)])
    return [ivf[off[c]:off[c + 1]].tolist() for c in range(len(lens))]


def _scrambled_ivf(ix, rng):
    """An inverted file that is not the rebuild of the codes: lists shuffled, extra valid ids, duplicates."""
    parts = []
    for lst in _lists(ix.ivf, ix.ivf_lengths):
        extra = rng.integers(0, ix.num_documents, int(rng.integers(0, 4))).tolist()
        lst = lst + extra + lst[:1]
        rng.shuffle(lst)
        parts.append(lst)
    return np.array([x for p in parts for x in p], np.int64), np.array([len(p) for p in parts], np.int32)


def test_slices_of_a_partition_give_back_the_lists(oracle):
    rng = np.random.default_rng(7)
    docs = oracle.synthetic_corpus(90, 10, dim=32, seed=4, ragged=True)
    ix = oracle.create_index(docs, nbits=2, seed=2, num_partitions=32)
    D = ix.num_documents
    for ivf, lens in ((ix.ivf, ix.ivf_lengths), _scrambled_ivf(ix, rng)):
        for cuts in ([], [45], [0, 1, 89, 90], sorted(rng.choice(np.arange(1, D), 6, replace=False).tolist()),
                     list(range(1, D))):
            bounds = [0] + list(cuts) + [D]
            # each list in file order within a shard, shards in order: the list itself when it is sorted (a rebuild)
            want = [sorted(lst, key=lambda x: np.searchsorted(bounds, x, "right")) for lst in _lists(ivf, lens)]
            if ivf is ix.ivf:
                assert want == _lists(ivf, lens)
            got = [[] for _ in want]
            for b, e in zip(bounds[:-1], bounds[1:]):
                sl, sll = ivf_slice(ivf, lens, b, e)
                assert sll.dtype == np.int32 and sll.sum() == len(sl)
                assert all(0 <= x < e - b for x in sl.tolist())
                for c, lst in enumerate(_lists(sl, sll)):
                    got[c] += [x + b for x in lst]
            assert got == want


def test_slice_of_the_rebuild_is_the_rebuild_of_the_slice(oracle):
    docs = oracle.synthetic_corpus(90, 10, dim=32, seed=5, ragged=True)
    ix = oracle.create_index(docs, nbits=4, seed=3, num_partitions=32)
    D, K = ix.num_documents, ix.num_centroids
    for b, e in ((0, D), (0, 1), (10, 10), (17, 60), (D - 1, D), (30, D)):
        t0, t1 = int(ix.doc_offsets[b]), int(ix.doc_offsets[e])
        want = oracle.build_ivf(ix.codes[t0:t1], ix.doc_lengths[b:e], K)
        got = ivf_slice(ix.ivf, ix.ivf_lengths, b, e)
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]), (b, e)


def _layout_dir(path, chunks):
    """A directory with only what the bounds read: metadata.json and one doclens file per chunk."""
    os.makedirs(path, exist_ok=True)
    for i, dl in enumerate(chunks):
        with open(os.path.join(path, f"doclens.{i}.json"), "w") as f:
            json.dump([int(x) for x in dl], f)
    with open(os.path.join(path, "metadata.json"), "w") as f:
        json.dump({"num_chunks": len(chunks), "nbits": 4, "num_embeddings": int(sum(sum(c) for c in chunks))}, f)
    return path


def _check_bounds(npb, path, doclens, world):
    got = npb.shard_bounds(path, world)
    want = shard_bounds(doclens, world)
    assert got.tolist() == want.tolist(), (world, got, want)
    D, N = len(doclens), int(np.sum(doclens))
    assert got[0] == 0 and got[-1] == D and np.all(np.diff(got) >= 0)
    off = np.concatenate([[0], np.cumsum(doclens)]).astype(np.int64)
    mx = int(np.max(doclens)) if D else 0
    for r in range(world):
        assert off[got[r + 1]] - off[got[r]] <= N / world + mx


def test_shard_bounds(npb, tmp_path):
    rng = np.random.default_rng(11)
    cases = {
        "ragged": [rng.integers(1, 300, 500), rng.integers(1, 300, 400), rng.integers(1, 30, 7)],
        "with_empty_docs_and_chunk": [rng.integers(0, 5, 40), [], rng.integers(0, 50, 25)],
        "one_long_doc": [[1, 1, 5000, 1, 1, 1]],
        "no_tokens": [[0, 0, 0], [0]],
        "no_docs": [[]],
    }
    for name, chunks in cases.items():
        path = _layout_dir(str(tmp_path / name), chunks)
        doclens = np.concatenate([np.asarray(c, np.int64) for c in chunks])
        for world in (1, 2, 3, 4, 7, 8, len(doclens) + 3):
            _check_bounds(npb, path, doclens, world)
    # world > D gives empty shards; world = 1 the whole directory
    b = npb.shard_bounds(str(tmp_path / "one_long_doc"), 10)
    assert b[-1] == 6 and len(b) == 11
    assert npb.shard_bounds(str(tmp_path / "ragged"), 1).tolist() == [0, 907]


def test_shard_bounds_of_a_written_index(npb, index_dir):
    path, ix = index_dir
    for world in (1, 2, 3, 8):
        _check_bounds(npb, path, ix.doc_lengths, world)


def test_shard_bounds_errors(npb, index_dir, tmp_path):
    for world in (0, -1):
        with pytest.raises(npb.PlaidError) as e:
            npb.shard_bounds(index_dir[0], world)
        assert e.value.status == 1
    with pytest.raises(npb.PlaidError) as e:
        npb.shard_bounds(str(tmp_path / "missing"), 2)
    assert e.value.status == 3 and "metadata.json" in str(e.value)


def _status(npb, fn):
    with pytest.raises(npb.PlaidError) as e:
        fn()
    return e.value.status, str(e.value)


def test_bad_ranges_are_refused_before_the_device(npb, index_dir):
    path, ix = index_dir
    D = ix.num_documents
    for b, e in ((-1, 5), (5, 4), (0, D + 1), (D + 1, D + 2), (-3, -1)):
        st, msg = _status(npb, lambda: npb.MmapIndex.load_range(path, b, e))
        assert st == 1, (b, e, msg)
    for rank, world in ((2, 2), (-1, 2), (0, 0)):
        st, msg = _status(npb, lambda: npb.MmapIndex.load_shard(path, rank, world))
        assert st == 1, (rank, world, msg)


def test_well_formed_range_reaches_the_device(npb, index_dir):
    path, ix = index_dir
    for b, e in ((0, ix.num_documents), (50, 100), (60, 60), (119, 120)):
        if npb.device_count() > 0:
            gpu = npb.MmapIndex.load_range(path, b, e)
            assert gpu.num_documents() == e - b
            gpu.close()
        else:
            st, msg = _status(npb, lambda: npb.MmapIndex.load_range(path, b, e))
            assert st == 2, msg                              # PB_ERR_CUDA: parsed fine, no device, no fallback


def _copy(src, dst):
    shutil.copytree(src, dst)
    return str(dst)


def _truncate(path, name):
    f = os.path.join(path, name)
    data = open(f, "rb").read()
    open(f, "wb").write(data[:len(data) - 64])


def _edit_npy(path, name, fn):
    p = os.path.join(path, name)
    np.save(p, fn(np.load(p)))


def _edit_meta(path, key, fn):
    p = os.path.join(path, "metadata.json")
    meta = json.load(open(p))
    meta[key] = fn(meta[key])
    json.dump(meta, open(p, "w"))


MALFORMED = {
    "truncated_chunk_1": lambda p: _truncate(p, "1.residuals.npy"),
    "truncated_chunk_2": lambda p: _truncate(p, "2.codes.npy"),
    "ivf_lengths_off_by_one": lambda p: _edit_npy(p, "ivf_lengths.npy", lambda a: a + (np.arange(len(a)) == 0)),
    "ivf_lengths_f8": lambda p: _edit_npy(p, "ivf_lengths.npy", lambda a: a.astype(np.float64)),
    "num_embeddings": lambda p: _edit_meta(p, "num_embeddings", lambda v: v + 5),
    "nbits_3": lambda p: _edit_meta(p, "nbits", lambda v: 3),
    "codes_i4": lambda p: _edit_npy(p, "0.codes.npy", lambda a: a.astype(np.int32)),
    "missing_doclens": lambda p: os.remove(os.path.join(p, "doclens.2.json")),
    "missing_ivf": lambda p: os.remove(os.path.join(p, "ivf.npy")),
}


@pytest.mark.parametrize("fault", sorted(MALFORMED))
def test_malformed_directory_same_status_as_load(npb, index_dir, tmp_path, fault):
    path = _copy(index_dir[0], tmp_path / "ix")
    MALFORMED[fault](path)
    want = _status(npb, lambda: npb.MmapIndex.load(path))
    assert want[0] in (1, 3), want
    # ranges inside the first chunk never read chunks 1 and 2, yet their faults are refused all the same
    for b, e in ((0, 120), (0, 10), (10, 50), (55, 101), (119, 120), (30, 30)):
        assert _status(npb, lambda: npb.MmapIndex.load_range(path, b, e)) == want, (fault, b, e)
    for world in (2, 3):
        for rank in range(world):
            assert _status(npb, lambda: npb.MmapIndex.load_shard(path, rank, world)) == want, (fault, rank)


def test_header_compiles_as_plain_c(tmp_path):
    src = tmp_path / "h.c"
    src.write_text('#include "plaid_b200.h"\n'
                   'pb_status (*f0)(const char *, int32_t, int64_t, int64_t, pb_index **) = pb_index_load_range;\n'
                   'pb_status (*f1)(const char *, int32_t, int64_t *) = pb_index_dir_shard_bounds;\n')
    for std in ("c99", "c11"):
        r = subprocess.run(["cc", f"-std={std}", "-pedantic-errors", "-Wall", "-Werror", "-c", str(src), "-I",
                            os.path.join(ROOT, "include"), "-o", str(tmp_path / "h.o")], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
