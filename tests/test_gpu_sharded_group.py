"""The doc-sharded protocol's merge kernels (k_merge_cut, k_merge_topk) on ONE GPU: G shard handles on
device 0 joined into an in-process shard group (pb_shard_group: peer copies behind a host barrier instead of
NCCL), searched together from G host threads.  Every rank's result must be bit-identical to the CPU oracle
searching the UNSHARDED index (SURVEY 8e strict mode; the NCCL transport runs the same kernels on the same
buffers, tests/gpu_sharded_check.py)."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import sharded_protocol as sp  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def npb():
    import next_plaid_b200 as m
    m.build_library()
    if m.device_count() < 1:
        pytest.fail("GPU tests need an H100; the library has no CPU fallback")
    return m


def _group(npb, oracle, ix, G):
    shards = []
    for g in range(G):
        sh, base = sp.make_shard(oracle, ix, g, G)
        shards.append(npb.MmapIndex.from_arrays(sh.centroids, sh.bucket_weights, sh.codes, sh.residuals,
                                                sh.doc_lengths, sh.ivf, sh.ivf_lengths, sh.nbits, device=0,
                                                doc_id_base=base))
    return npb.ShardGroup(shards)


def _check(oracle, ix, grp, qs, pg, po, subset=None):
    res = grp.search_batch(qs, pg, subset=subset)
    for r, per_rank in enumerate(grp.all_results):          # every rank holds the same global answer
        for a, b in zip(per_rank, res):
            assert a.passage_ids.tolist() == b.passage_ids.tolist() and np.array_equal(a.scores, b.scores), r
    for q, got in zip(qs, res):
        want = oracle.search_one(ix, q, po, subset=subset)
        assert got.passage_ids.tolist() == want.passage_ids.tolist()
        assert np.array_equal(got.scores, want.scores)


@pytest.fixture(scope="module")
def corpus(oracle):
    docs = oracle.synthetic_corpus(3000, 40, dim=128, seed=31, ragged=True)
    ix = oracle.create_index(docs, nbits=4, seed=5, num_partitions=512)
    qs, _ = oracle.synthetic_queries(docs, 12, nq=32, seed=6)
    return docs, ix, qs


@pytest.mark.parametrize("G", [2, 3, 8])
def test_group_equals_unsharded_oracle(npb, oracle, corpus, G):
    docs, ix, qs = corpus
    grp = _group(npb, oracle, ix, G)
    try:
        for cbs in (100_000, 128):                               # dense and batched variants
            kw = dict(top_k=10, n_ivf_probe=8, n_full_scores=256, centroid_batch_size=cbs)
            _check(oracle, ix, grp, qs, npb.SearchParameters(**kw), oracle.SearchParameters(**kw))
        kw = dict(top_k=50, n_ivf_probe=4, n_full_scores=64, centroid_batch_size=128)   # top_k > n_full_scores/4
        _check(oracle, ix, grp, qs, npb.SearchParameters(**kw), oracle.SearchParameters(**kw))
        # subset with the batched variant (candidate intersection only, search.rs:542-545)
        kw = dict(top_k=10, n_ivf_probe=8, n_full_scores=256, centroid_batch_size=128)
        _check(oracle, ix, grp, qs, npb.SearchParameters(**kw), oracle.SearchParameters(**kw),
               subset=list(range(0, 3000, 3)))
    finally:
        grp.close()


def test_group_ties_across_shards(npb, oracle):
    """Duplicated documents in different shards tie on the approximate AND the exact score: the global cut
    and the final order must fall back to the global doc id exactly as the unsharded stable sorts do."""
    base = oracle.synthetic_corpus(300, 24, dim=128, seed=41, ragged=False)
    docs = [base[i % 300] for i in range(1200)]                 # every doc four times, one copy per shard of G=4
    ix = oracle.create_index(docs, nbits=4, seed=6, num_partitions=128)
    qs, _ = oracle.synthetic_queries(docs, 8, nq=32, seed=7)
    grp = _group(npb, oracle, ix, 4)
    try:
        for nfs, k in ((64, 10), (32, 20), (400, 40)):
            kw = dict(top_k=k, n_ivf_probe=8, n_full_scores=nfs, centroid_batch_size=64)
            _check(oracle, ix, grp, qs, npb.SearchParameters(**kw), oracle.SearchParameters(**kw))
    finally:
        grp.close()


def test_group_with_an_empty_shard_and_mixed_query_lengths(npb, oracle):
    docs = oracle.synthetic_corpus(900, 30, dim=64, seed=51, ragged=True)
    ix = oracle.create_index(docs, nbits=2, seed=8, num_partitions=128)
    qs = [oracle.synthetic_queries(docs, 1, nq=n, seed=60 + n)[0][0] for n in (1, 7, 32, 33, 48, 64)]
    G = 3
    grp = _group(npb, oracle, ix, G)
    try:
        kw = dict(top_k=10, n_ivf_probe=4, n_full_scores=128, centroid_batch_size=64)
        _check(oracle, ix, grp, qs, npb.SearchParameters(**kw), oracle.SearchParameters(**kw))
        # subset that leaves the middle shard without any eligible doc
        sub = list(range(0, 300)) + list(range(600, 900, 2))
        _check(oracle, ix, grp, qs, npb.SearchParameters(**kw), oracle.SearchParameters(**kw), subset=sub)
    finally:
        grp.close()
