"""pb_pool_embeddings on the device against the CPU restatement of pool_document_embeddings (pool_oracle.c), bit for
bit: every output row's f32 bits and every pooled length, over the built widths, pool factors, the lengths where the
length rule and the kernels' 64-token tiles switch, multi-wave batches, degenerate documents, host and device memory,
and concurrent callers.  One end-to-end case appends the pooled device buffer to an index and searches it."""
import ctypes as C
import os
import sys
import threading

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import pool_oracle  # noqa: E402

pytestmark = pytest.mark.gpu

LENGTHS = [0, 1, 2, 3, 31, 32, 33, 300, 512]


@pytest.fixture(scope="module")
def npb():
    import next_plaid_b200 as m
    m.build_library()
    if m.device_count() < 1:
        pytest.fail("GPU tests need an H100; the library has no CPU fallback")
    return m


def _docs(lengths, dim, seed):
    rng = np.random.default_rng(seed)
    out = []
    for n in lengths:
        x = rng.standard_normal((n, dim)).astype(np.float32)
        x /= np.maximum(np.linalg.norm(x, axis=1, keepdims=True), 1e-6)
        out.append(x.astype(np.float32))
    return out


def _same(got, want):
    assert len(got) == len(want)
    for i, (g, w) in enumerate(zip(got, want)):
        g = np.asarray(g)
        assert g.shape == w.shape, (i, g.shape, w.shape)
        assert np.array_equal(g.view(np.uint32), w.view(np.uint32)), i


@pytest.mark.parametrize("dim", [48, 96, 128])
@pytest.mark.parametrize("pf", [1, 2, 3, 4, 1000])
def test_lengths_and_factors(npb, dim, pf):
    docs = _docs(LENGTHS + LENGTHS[::-1], dim, seed=dim + pf)
    _same(npb.pool_document_embeddings(docs, pf), pool_oracle.pool_embeddings(docs, pf))


def test_pool_factor_none_returns_the_input(npb):
    docs = _docs([5, 40], 128, seed=3)
    _same(npb.pool_document_embeddings(docs, None), docs)


@pytest.mark.parametrize("pf", [2, 1000])
def test_long_document(npb, pf):
    docs = _docs([2100, 7, 300], 128, seed=5)
    _same(npb.pool_document_embeddings(docs, pf), pool_oracle.pool_embeddings(docs, pf))


def test_many_documents_over_several_waves(npb):
    """3600 ragged docs of 150-450 tokens: about 3 waves of the 1 GiB distance workspace"""
    from oracle import oracle
    docs = oracle.synthetic_corpus(3600, 300, dim=128, seed=17, ragged=True)
    rng = np.random.default_rng(1)
    for i in rng.choice(len(docs), 40, replace=False):      # a few short ones in between
        docs[i] = docs[i][:int(rng.integers(0, 5))]
    _same(npb.pool_document_embeddings(docs, 2), pool_oracle.pool_embeddings(docs, 2))


def _degenerate(dim):
    rng = np.random.default_rng(9)
    same = np.tile(rng.standard_normal((1, dim)).astype(np.float32), (70, 1))          # all distances 0: tie order
    dup = rng.standard_normal((6, dim)).astype(np.float32)[rng.integers(0, 6, size=90)]  # many duplicated tokens
    zero = rng.standard_normal((50, dim)).astype(np.float32)
    zero[rng.choice(50, 20, replace=False)] = 0                                          # zero vectors: distance 1
    opp = rng.standard_normal((41, dim)).astype(np.float32)
    opp[21:] = -opp[1:21]                                                                # opposite pairs: clamp at 2
    ints = rng.integers(-1, 2, size=(65, dim)).astype(np.float32)                        # many exact ties
    return [same, dup, zero, opp, ints, np.zeros((9, dim), np.float32)]


@pytest.mark.parametrize("pf", [2, 3, 1000])
def test_degenerate_documents(npb, pf):
    docs = _degenerate(128)
    _same(npb.pool_document_embeddings(docs, pf), pool_oracle.pool_embeddings(docs, pf))


def test_device_memory(npb):
    import torch
    docs = _docs([0, 3, 33, 300, 65, 129], 96, seed=21) + _degenerate(96)
    want = pool_oracle.pool_embeddings(docs, 2)
    got = npb.pool_document_embeddings([torch.from_numpy(d).cuda() for d in docs], 2)
    assert all(g.is_cuda for g in got)
    _same([g.cpu().numpy() for g in got], want)


def test_concurrent_callers(npb):
    batches = [_docs(list(np.random.default_rng(s).integers(0, 400, size=300)), 128, seed=s) for s in range(4)]
    want = [pool_oracle.pool_embeddings(b, 2) for b in batches]
    got, errs = [None] * 4, []

    def run(i):
        try:
            for _ in range(3):
                got[i] = npb.pool_document_embeddings(batches[i], 2)
        except Exception as e:    # noqa: BLE001 -- reported below
            errs.append(e)

    ts = [threading.Thread(target=run, args=(i,)) for i in range(4)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errs, errs
    for g, w in zip(got, want):
        _same(g, w)


def test_non_finite_input_is_refused_untouched(npb):
    import torch
    L = npb.load_library()
    docs = _docs([40, 40], 128, seed=2)
    flat = np.concatenate(docs, 0)
    lens = np.array([40, 40], np.int64)
    for bad in (np.nan, np.inf, -np.inf):
        x = flat.copy()
        x[57, 3] = bad
        out = np.full((42, 128), 7.0, np.float32)
        olens = np.full(2, -5, np.int64)
        st = L.pb_pool_embeddings(0, x.ctypes.data_as(C.c_void_p), lens.ctypes.data_as(C.c_void_p), 2, 128, 2, 0,
                                  out.ctypes.data_as(C.c_void_p), olens.ctypes.data_as(C.c_void_p))
        assert st == npb.index.PB_ERR_INVALID
        assert (out == 7.0).all() and (olens == -5).all()
        dx = torch.from_numpy(x).cuda()
        dout = torch.full((42, 128), 7.0, device="cuda")
        torch.cuda.synchronize()
        st = L.pb_pool_embeddings(0, dx.data_ptr(), lens.ctypes.data_as(C.c_void_p), 2, 128, 2, 1, dout.data_ptr(),
                                  olens.ctypes.data_as(C.c_void_p))
        assert st == npb.index.PB_ERR_INVALID
        assert bool((dout == 7.0).all()) and (olens == -5).all()


def test_pool_then_append_on_device(npb, oracle):
    """encoder output on the device -> pb_pool_embeddings(PB_MEM_DEVICE) -> pb_index_append(PB_MEM_DEVICE): the index
    arrays and the search results equal the oracle's pool -> encode -> search on the same documents"""
    import torch
    NBITS, K, DIM, PF = 2, 256, 128, 2
    base = oracle.synthetic_corpus(1200, 40, dim=DIM, seed=71, ragged=True)
    new = oracle.synthetic_corpus(300, 90, dim=DIM, seed=72, ragged=True)
    flat = np.concatenate(base, 0)
    cent = flat[np.random.default_rng(2).choice(len(flat), K, replace=False)].copy()
    art = oracle.prepare_codec_artifacts(base, cent, NBITS, 3)
    codes, packed, dl = oracle.encode_documents(base, art, NBITS)
    ix = npb.MmapIndex.from_arrays(art.centroids, art.bucket_weights, codes, packed, dl,
                                   *oracle.build_ivf(codes, dl, K), NBITS)
    codec = npb.ResidualCodec(NBITS, art.centroids, art.bucket_cutoffs)
    L = npb.load_library()
    try:
        d_in = torch.from_numpy(np.concatenate(new, 0)).cuda()
        lens = np.array([d.shape[0] for d in new], np.int64)
        olens = np.array([npb.pooled_doc_length(int(n), PF) for n in lens], np.int64)
        d_out = torch.empty((int(olens.sum()), DIM), dtype=torch.float32, device="cuda")
        got_lens = np.zeros(len(new), np.int64)
        torch.cuda.synchronize()
        assert L.pb_pool_embeddings(0, d_in.data_ptr(), lens.ctypes.data_as(C.c_void_p), len(new), DIM, PF, 1,
                                    d_out.data_ptr(), got_lens.ctypes.data_as(C.c_void_p)) == 0, L.pb_last_error()
        assert np.array_equal(got_lens, olens)
        d_lens = torch.from_numpy(got_lens).cuda()
        torch.cuda.synchronize()
        first = C.c_int64()
        assert L.pb_index_append(ix._h, codec._h, d_out.data_ptr(), d_lens.data_ptr(), len(new), 1, None, 50_000,
                                 C.byref(first)) == 0, L.pb_last_error()
        assert first.value == len(base)

        pooled = pool_oracle.pool_embeddings(new, PF)
        all_docs = base + pooled
        codes2, packed2, dl2 = oracle.encode_documents(all_docs, art, NBITS)
        ivf2, lens2 = oracle.build_ivf(codes2, dl2, K)
        oix = oracle.Index(art.centroids, art.bucket_weights, art.bucket_cutoffs, codes2, packed2, dl2, ivf2, lens2,
                           NBITS)
        assert ix.num_documents() == oix.num_documents and ix.num_embeddings() == oix.num_embeddings
        a_ivf, a_len = ix.export_ivf()
        assert np.array_equal(a_ivf, oix.ivf) and np.array_equal(a_len, oix.ivf_lengths)
        ids = list(range(len(base) - 2, len(all_docs)))
        emb, el = ix.decompress_documents(ids)
        assert np.array_equal(emb, np.concatenate([oracle.get_document_embeddings(oix, d) for d in ids], 0))
        qs, _ = oracle.synthetic_queries(new, 6, nq=32, seed=5)
        params = dict(top_k=10, n_ivf_probe=8, n_full_scores=256)
        for q, r in zip(qs, ix.search_batch(qs, npb.SearchParameters(**params))):
            w = oracle.search_one(oix, q, oracle.SearchParameters(**params))
            assert r.passage_ids.tolist() == w.passage_ids.tolist()
            assert np.array_equal(r.scores, w.scores)
    finally:
        codec.close()
        ix.close()
