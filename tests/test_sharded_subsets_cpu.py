"""The global eligibility of tests/sharded_subsets.py equals the unsharded oracle on CPU: for random doc partitions
(empty ranks included) and subsets of every kind, the OR of the ranks' eligible rows scaled by the deployment's D gives
exactly the cells the oracle probes on the whole index."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import sharded_subsets as ss  # noqa: E402


def _shard(oracle, ix, d0, d1):
    t0, t1 = int(ix.doc_offsets[d0]), int(ix.doc_offsets[d1])
    codes, res, dl = ix.codes[t0:t1], ix.residuals[t0:t1], ix.doc_lengths[d0:d1]
    ivf, ivf_lengths = oracle.build_ivf(codes, dl, ix.num_centroids)
    return oracle.Index(ix.centroids, ix.bucket_weights, ix.bucket_cutoffs, codes, res, dl, ivf, ivf_lengths, ix.nbits)


@pytest.fixture(scope="module")
def corpus(oracle):
    docs = oracle.synthetic_corpus(600, 24, dim=64, seed=17, ragged=True)
    ix = oracle.create_index(docs, nbits=2, seed=5, num_partitions=128)
    qs = [oracle.synthetic_queries(docs, 1, nq=n, seed=40 + n)[0][0] for n in (1, 8, 32, 33)]
    return ix, qs


@pytest.mark.parametrize("seed", range(4))
@pytest.mark.parametrize("thr", [None, 0.3])
def test_or_of_local_rows_gives_the_unsharded_cells(oracle, corpus, seed, thr):
    ix, qs = corpus
    D = ix.num_documents
    rng = np.random.default_rng(seed)
    G = int(rng.integers(2, 6))
    cuts = np.sort(rng.integers(0, D + 1, G - 1))
    bounds = [0] + cuts.tolist() + [D]                      # random partition; equal cuts leave a rank empty
    shards = [_shard(oracle, ix, bounds[r], bounds[r + 1]) for r in range(G)]
    subsets = [[], [D + 3, -2], sorted(rng.choice(D, 5, replace=False).tolist()),
               list(range(bounds[1], D, 3)) or [0], list(range(1, D, 40)),
               rng.integers(-5, D + 5, 200).tolist()]          # duplicates and out-of-range ids
    for subset in subsets:
        for q in qs:
            p = oracle.SearchParameters(top_k=10, n_ivf_probe=4, n_full_scores=64, centroid_score_threshold=thr)
            _, tr = oracle.search_one(ix, q, p, subset=subset, trace=True)
            got = ss.sharded_cells(oracle, shards, bounds[:-1], q, ix.centroids, subset, 4, thr)
            assert got.tolist() == tr.cells.tolist(), (G, bounds, len(subset), q.shape)


def test_local_rows_partition_the_eligible_set(oracle, corpus):
    ix, _ = corpus
    D, K = ix.num_documents, ix.num_centroids
    bounds = [0, 150, 150, 420, D]
    shards = [_shard(oracle, ix, bounds[r], bounds[r + 1]) for r in range(4)]
    subset = list(range(100, 200))
    rows = [ss.local_eligible(s, b, subset, K) for s, b in zip(shards, bounds[:-1])]
    assert not rows[1].any() and not rows[3].any()            # an empty rank, a rank without subset docs
    whole = ss.local_eligible(ix, 0, subset, K)
    assert np.array_equal(np.logical_or.reduce(rows), whole)
    assert ss.probe_width(4, D, len(subset), int(whole.sum())) == min(4 * D // 100, int(whole.sum()))
