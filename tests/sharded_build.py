"""numpy restatement of pb_create_index_sharded's plan (DESIGN §4n): which rank contributes which k-means fit point,
seed and held-out row, which chunk rows go from which rank to which chunk writer, and where each rank's pieces land in
ivf.npy.  Every rank computes the same plan from the global doc lengths; tests/test_sharded_build_cpu.py reassembles
the pieces and checks them against pb_create_index's single-process arrays."""
import math

import numpy as np

M64 = (1 << 64) - 1


def splitmix64(s):
    s = (s + 0x9E3779B97F4A7C15) & M64
    z = s
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return s, z ^ (z >> 31)


def shuffled_prefix(n, take, seed):
    """the first `take` entries of a seeded Fisher-Yates shuffle of 0..n-1 (builder.cpp)"""
    p, s = list(range(n)), seed & M64
    for i in range(min(take, n)):
        s, z = splitmix64(s)
        j = i + z % (n - i)
        p[i], p[j] = p[j], p[i]
    return p[:min(take, n)]


def lcg_seeds(n, K, seed):
    """pb_kmeans_fit's initial centroids: K distinct fit points (partial Fisher-Yates with a 64-bit LCG)"""
    a, c = 6364136223846793005, 1442695040888963407
    s, p = (seed * a + c) & M64, list(range(n))
    for i in range(K):
        s = (s * a + c) & M64
        j = i + (s >> 11) % (n - i)
        p[i], p[j] = p[j], p[i]
    return p[:K]


def kmeans_sample_docs(D):
    return min(int(1.0 + 16.0 * math.sqrt(120.0 * D)), D)


def num_partitions(D, avg, n_stok):
    return max(1, min(int(2.0 ** math.floor(math.log2(16.0 * math.sqrt(avg * D)))), n_stok))


def codec_sample_docs(D):
    return max(1, min(int(16.0 * math.sqrt(120.0 * D)), D))


def heldout_tokens(N):
    return int(min(0.05 * N, 50000.0))


def plan(lens, seed, parts=0, mpp=256):
    """The global plan: fit points as global token ids in fit order, K, the seeds (fit indices), and the held-out
    pieces (first global token, rows) in pb_create_index's order."""
    lens = [int(x) for x in lens]
    D = len(lens)
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    sdocs = shuffled_prefix(D, kmeans_sample_docs(D), seed)
    rows = [int(off[d]) + t for d in sdocs for t in range(lens[d])]       # the sample's tokens in sample order
    n_stok = len(rows)
    K = min(parts, n_stok) if parts > 0 else num_partitions(D, n_stok / len(sdocs), n_stok)
    fit = rows
    if n_stok > K * mpp:
        fit = [rows[i] for i in shuffled_prefix(n_stok, K * mpp, seed ^ 0x5BD1E995)]
    seeds = lcg_seeds(len(fit), K, seed)
    cdocs = shuffled_prefix(D, codec_sample_docs(D), seed + 1)
    want, got, held = heldout_tokens(int(off[-1])), 0, []
    for d in reversed(cdocs):
        if got >= want:
            break
        take = min(want - got, lens[d])
        got += take
        if take:
            held.append((int(off[d]), take))
    return dict(off=off, fit=fit, K=K, seeds=seeds, held=held)


def owner(bounds, x):
    """the rank whose [bounds[r], bounds[r + 1]) holds x (empty ranks hold nothing)"""
    return int(np.searchsorted(bounds, x, side="right")) - 1


def rank_share(p, tokb, r):
    """Rank r's contributions: its fit points (global tokens, in global fit order), its seed table entries
    {k: index into its fit points}, and its held-out rows (global tokens, in held-out order)."""
    mine = [i for i, t in enumerate(p["fit"]) if owner(tokb, t) == r]
    pos = {i: j for j, i in enumerate(mine)}
    seeds = {k: pos[i] for k, i in enumerate(p["seeds"]) if i in pos}
    held = [t0 + t for t0, n in p["held"] if owner(tokb, t0) == r for t in range(n)]
    return [p["fit"][i] for i in mine], seeds, held


def trainer_rows(p, tokb, shares):
    """What the trainer (rank 0) reassembles from every rank's held-out rows, received per source in rank order."""
    cur = [0] * (len(tokb) - 1)
    out = []
    for t0, n in p["held"]:
        r = owner(tokb, t0)
        out += shares[r][cur[r]:cur[r] + n]
        cur[r] += n
    return out


def chunk_moves(base, bs):
    """Per rank, its head -- the docs [base[r], end) of a chunk begun on an earlier rank -- and that chunk's writer
    (the rank holding its first doc): {r: (writer, end)}.  Every other chunk is written by the rank it starts in."""
    out = {}
    for r in range(len(base) - 1):
        if base[r] == base[r + 1] or base[r] % bs == 0:
            continue
        c0 = base[r] // bs * bs
        out[r] = (owner(base, c0), min(c0 + bs, base[r + 1]))
    return out


def chunks_written(base, r, D, bs):
    """the chunks rank r writes: those whose first doc it holds"""
    if base[r] == base[r + 1]:
        return []
    return list(range(-(-base[r] // bs), -(-base[r + 1] // bs)))


def ivf_pieces(lengths, r):
    """Rank r's pieces of ivf.npy from every rank's [K] list lengths (rows in rank order): for each centroid with a
    non-empty local list, (element offset in the file's payload, count).  List k of the file is the ranks' lists of k
    in rank order."""
    L = np.asarray(lengths, np.int64)
    start = np.concatenate([[0], np.cumsum(L.sum(0))])
    before = L[:r].sum(0)
    return [(int(start[k] + before[k]), int(L[r, k])) for k in range(L.shape[1]) if L[r, k]]
