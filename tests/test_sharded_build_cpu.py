"""The plan of pb_create_index_sharded (tests/sharded_build.py) against pb_create_index's single-process arrays, over
many random splits of a corpus into ranks (empty ranks, one-document ranks, chunks over three or more ranks, rank
boundaries on chunk edges): the ranks' fit points reassemble the fit sample in order, their seed entries the seed
table, their held-out rows the held-out matrix in order, each chunk writer's rows the chunk, and every rank's
positioned pieces the inverted file oracle.build_ivf gives for the whole corpus."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import sharded_build as sb  # noqa: E402


def _splits(rng, D, W):
    cuts = np.sort(rng.integers(0, D + 1, W - 1))
    return np.concatenate([[0], cuts, [D]]).astype(np.int64)


def _cases():
    out = []
    for seed in range(10):
        rng = np.random.default_rng(seed)
        D = int(rng.integers(1, 300))
        W = int(rng.integers(1, 7))
        out.append((seed, D, _splits(rng, D, W), int(rng.integers(1, 60))))
    # named shapes: an empty rank and a chunk over three ranks; one-document ranks; boundaries on chunk edges
    out.append((100, 200, np.array([0, 30, 30, 45, 60, 200]), 50))
    out.append((101, 7, np.array([0, 1, 2, 3, 4, 5, 6, 7]), 3))
    out.append((102, 240, np.array([0, 80, 160, 240]), 40))
    out.append((103, 240, np.array([0, 0, 240, 240]), 40))
    return out


def _single_process(lens, seed, parts):
    """pb_create_index's arrays for the whole corpus, as its steps build them from one embedding array (here each
    token's row is its global token id): the fit sample, the seed rows and the held-out rows"""
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    emb = np.arange(off[-1], dtype=np.int64)
    D = len(lens)
    sdocs = sb.shuffled_prefix(D, sb.kmeans_sample_docs(D), seed)
    samples = np.concatenate([emb[off[d]:off[d + 1]] for d in sdocs])
    K = min(parts, len(samples)) if parts > 0 else sb.num_partitions(D, len(samples) / len(sdocs), len(samples))
    if len(samples) > K * 256:
        samples = samples[sb.shuffled_prefix(len(samples), K * 256, seed ^ 0x5BD1E995)]
    seeds = samples[sb.lcg_seeds(len(samples), K, seed)]
    cdocs = sb.shuffled_prefix(D, sb.codec_sample_docs(D), seed + 1)
    want, held = sb.heldout_tokens(int(off[-1])), []
    for d in reversed(cdocs):
        if len(held) >= want:
            break
        held += emb[off[d]:off[d] + min(want - len(held), int(lens[d]))].tolist()
    return dict(fit=samples.tolist(), K=K, seed_rows=seeds.tolist(), held=held)


@pytest.mark.parametrize("seed,D,base,bs", _cases())
def test_plan_pieces_reassemble_the_single_process_arrays(oracle, seed, D, base, bs):
    rng = np.random.default_rng(1000 + seed)
    lens = rng.integers(0, 12, D).astype(np.int64)
    lens[0] = max(int(lens[0]), 1)                       # at least one token
    W = len(base) - 1
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    tokb = off[base]
    parts = int(rng.choice([0, 4, 16]))
    p = sb.plan(lens, seed, parts)
    want = _single_process(lens, seed, parts)

    # k-means: fit points in global fit order, the seed table completed by the all-reduce
    shares = [sb.rank_share(p, tokb, r) for r in range(W)]
    for r, (fit, _, _) in enumerate(shares):
        assert all(tokb[r] <= t < tokb[r + 1] for t in fit)
    assert sorted(t for f, _, _ in shares for t in f) == sorted(want["fit"])
    merged = sorted((t for f, _, _ in shares for t in f), key=want["fit"].index)
    assert merged == want["fit"]
    table = {}
    for r, (fit, seeds, _) in enumerate(shares):
        for k, j in seeds.items():
            assert k not in table                          # one owner per seed: the sum of zero-padded tables is exact
            table[k] = fit[j]
    assert p["K"] == want["K"]
    assert [table[k] for k in range(p["K"])] == want["seed_rows"]

    # codec training: the trainer's reassembly is the held-out matrix in order
    assert sb.trainer_rows(p, tokb, [h for _, _, h in shares]) == want["held"]

    # chunk files: each writer's rows are the chunk's rows
    moves = sb.chunk_moves(base, bs)
    n_chunks = -(-D // bs)
    writers = {}
    for r in range(W):
        for c in sb.chunks_written(base, r, D, bs):
            assert c not in writers
            writers[c] = r
    assert sorted(writers) == list(range(n_chunks))
    for c, w in writers.items():
        d0, d1 = c * bs, min(D, c * bs + bs)
        rows = list(range(off[d0], off[min(d1, base[w + 1])]))
        for r in range(W):                                 # heads received, in rank order
            if r in moves and moves[r][0] == w and base[r] < d1:
                rows += list(range(off[base[r]], off[moves[r][1]]))
        assert rows == list(range(off[d0], off[d1])), (c, w)

    # inverted file: each rank's local lists at their offsets give oracle.build_ivf's lists
    K = 8
    codes = rng.integers(0, K, int(off[-1])).astype(np.int64)
    ivf, ivf_len = oracle.build_ivf(codes, lens, K)
    out = np.full(len(ivf), -1, np.int64)
    local = []
    for r in range(W):
        li, ll = oracle.build_ivf(codes[tokb[r]:tokb[r + 1]], lens[base[r]:base[r + 1]], K)
        local.append((li + base[r], ll))
    for r in range(W):
        src = 0
        li, ll = local[r]
        for k_off, n in sb.ivf_pieces([l for _, l in local], r):
            assert out[k_off:k_off + n].tolist() == [-1] * n           # pieces do not overlap
            out[k_off:k_off + n] = li[src:src + n]
            src += n
    assert np.array_equal(out, ivf)
    assert np.array_equal(np.sum([l for _, l in local], 0), ivf_len)
