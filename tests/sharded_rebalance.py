"""numpy restatement of pb_index_rebalance_sharded (include/plaid_b200.h) on a doc-sharded deployment whose rank r holds
documents [old[r], old[r + 1]) with its own inverted file (local ids).

Plan: the piece from rank s to rank r is docs [max(old[s], new[r]), min(old[s + 1], new[r + 1])); rank r keeps its
overlap with itself.  Inverted file: each sender splits its lists stably by destination, ids rebased to the piece's
first doc; each receiver concatenates, per centroid and in source-rank order, its sources' pieces with the piece's
first doc in its new range added.  That is the slice [new[r], new[r + 1]) of the deployment's global lists (the ranks'
lists rebased and concatenated in rank order), which for sorted lists is ivf_slice of the global inverted file.
Balanced bounds: each rank offers, per boundary, the least doc of its closed range [old[s], old[s + 1]] whose global
token offset qualifies; the least offer wins."""
import numpy as np


def plan(old, new):
    """{(s, r): (lo, hi)}: the non-empty global doc ranges that go from rank s to rank r"""
    W = len(old) - 1
    out = {}
    for s in range(W):
        for r in range(W):
            lo, hi = max(int(old[s]), int(new[r])), min(int(old[s + 1]), int(new[r + 1]))
            if lo < hi:
                out[(s, r)] = (lo, hi)
    return out


def split_ivf(ivf, lens, base, new):
    """a sender's lists (local ids, base = its old[s]) split by destination: {r: (entries rebased to the piece's first
    doc, per-centroid counts)}, each list's order kept"""
    ivf = np.asarray(ivf, np.int64) + base
    lens = np.asarray(lens, np.int64)
    cen = np.repeat(np.arange(len(lens)), lens)
    out = {}
    for r in range(len(new) - 1):
        keep = (ivf >= new[r]) & (ivf < new[r + 1])
        if keep.any():
            out[r] = (ivf[keep] - max(base, int(new[r])), np.bincount(cen[keep], minlength=len(lens)))
    return out


def rank_ivf(rank_lists, old, new, r, K):
    """rank r's new inverted file from every rank's (ivf, lens) before the call: per centroid its sources' pieces in
    source order, ids + (piece start - new[r])"""
    segs = []
    for s, (iv, ln) in enumerate(rank_lists):
        pieces = split_ivf(iv, ln, int(old[s]), new)
        if r in pieces:
            e, cnt = pieces[r]
            start = max(int(old[s]), int(new[r]))
            segs.append((e + (start - int(new[r])), cnt))
    per_c = [[] for _ in range(K)]
    for e, cnt in segs:
        off = np.concatenate([[0], np.cumsum(cnt)])
        for c in range(K):
            per_c[c].append(e[off[c]:off[c + 1]])
    lists = [np.concatenate(x) if x else np.zeros(0, np.int64) for x in per_c]
    return (np.concatenate(lists).astype(np.int64) if lists else np.zeros(0, np.int64),
            np.array([len(x) for x in lists], np.int32))


def global_lists(rank_lists, old, K):
    """the deployment's global inverted file: per centroid the ranks' lists, ids + old[s], in rank order"""
    per_c = [[] for _ in range(K)]
    for s, (iv, ln) in enumerate(rank_lists):
        off = np.concatenate([[0], np.cumsum(np.asarray(ln, np.int64))])
        iv = np.asarray(iv, np.int64)
        for c in range(K):
            per_c[c].append(iv[off[c]:off[c + 1]] + int(old[s]))
    lists = [np.concatenate(x) for x in per_c]
    return np.concatenate(lists).astype(np.int64), np.array([len(x) for x in lists], np.int32)


def balanced_bounds(doclens_by_rank):
    """the distributed token-balanced bounds: rank s knows its doc lengths and, from the first exchange, every rank's D
    and N; its offer for boundary r is the least d in [old[s], old[s + 1]] with (tok[s] + off_s[d - old[s]]) W >= N r"""
    W = len(doclens_by_rank)
    D = [len(x) for x in doclens_by_rank]
    N = [int(np.sum(x)) for x in doclens_by_rank]
    old = np.concatenate([[0], np.cumsum(D)]).astype(np.int64)
    tok = np.concatenate([[0], np.cumsum(N)]).astype(np.int64)
    D_total, N_total = int(old[-1]), int(tok[-1])
    offers = np.full((W, W + 1), D_total, np.int64)
    for s, dl in enumerate(doclens_by_rank):
        off = np.concatenate([[0], np.cumsum(np.asarray(dl, np.int64))])
        for r in range(1, W):
            j = int(np.searchsorted((tok[s] + off) * W, N_total * r, side="left"))
            if j <= D[s]:
                offers[s, r] = old[s] + j
    b = offers.min(axis=0)
    b[0], b[W] = 0, D_total
    return b
