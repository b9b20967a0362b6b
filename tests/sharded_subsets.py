"""Executable specification of the global eligibility a doc-sharded deployment computes for a subset (DESIGN.md 4k).
Each rank marks the centroids of the subset's docs in its own range; the OR of those rows over the ranks is the
unsharded eligible set, so every rank derives the same count, the same n_ivf_probe scaled by the deployment's D and
the same cells (search.rs:350-382, 417-425).  The CUDA path does the same with one all-gather of the rows and an OR on
the device (k_eligible_bits, k_or_ranks)."""
import numpy as np


def local_eligible(shard, base, subset, K):
    """bool [K]: the codes of the subset's docs in [base, base + D) of this shard (other ids mark nothing)"""
    row = np.zeros(K, bool)
    D = shard.num_documents
    for g in subset:
        d = int(g) - base
        if 0 <= d < D:
            row[shard.codes[int(shard.doc_offsets[d]):int(shard.doc_offsets[d + 1])]] = True
    return row


def global_eligible(shards, bases, subset, K):
    """the OR over the ranks' rows: what every rank holds after the exchange"""
    out = np.zeros(K, bool)
    for sh, b in zip(shards, bases):
        out |= local_eligible(sh, b, subset, K)
    return out


def probe_width(n_ivf_probe, D_total, subset_len, n_eligible):
    """n_probe_eff = clamp(max(n_ivf_probe * D / len, n_ivf_probe), <= |eligible|) in integer arithmetic; len is the
    raw list length (duplicates and out-of-range ids counted)"""
    scaled = n_ivf_probe * D_total // subset_len if subset_len > 0 else n_ivf_probe
    return min(max(scaled, n_ivf_probe), n_eligible)


def dense_cells(S, eligible, n_probe_eff, threshold=None):
    """the dense variant's cells of one query from its centroid scores S [nq, K] (fp32): every eligible centroid when
    n_probe_eff covers them, else each token's n_probe_eff best eligible centroids (ties to the lower id); then the
    threshold on the best token score"""
    elig = np.flatnonzero(eligible)
    if len(elig) == 0:
        return np.zeros(0, np.int64)
    if n_probe_eff >= len(elig):
        cells = elig
    else:
        sel = set()
        for row in S:
            order = np.lexsort((elig, -row[elig].astype(np.float64)))[:n_probe_eff]
            sel.update(elig[order].tolist())
        cells = np.array(sorted(sel), np.int64)
    if threshold is not None and len(cells) and S.shape[0]:
        cells = cells[S[:, cells].max(0) >= np.float32(threshold)]
    return cells.astype(np.int64)


def sharded_cells(oracle, shards, bases, q, C, subset, n_ivf_probe, threshold=None):
    """every rank's cells for one query with a subset, from the exchanged rows and the deployment's D"""
    K = C.shape[0]
    D_total = sum(s.num_documents for s in shards)
    elig = global_eligible(shards, bases, subset, K)
    n = probe_width(n_ivf_probe, D_total, len(subset), int(elig.sum()))
    return dense_cells(oracle.centroid_scores(q, C), elig, n, threshold)
