"""numpy restatement of pb_index_load_range's shard of an index directory (include/plaid_b200.h): the inverted file is
ivf.npy's lists filtered to the doc range in file order with ids rebased -- a slice, not a rebuild from the shard's
codes -- and the token-balanced bounds of pb_index_dir_shard_bounds."""
import numpy as np


def ivf_slice(ivf, ivf_lengths, b, e):
    """Per centroid the entries of its list with b <= id < e, in file order, minus b; and their counts."""
    ivf = np.asarray(ivf, np.int64)
    lens = np.asarray(ivf_lengths, np.int64)
    cen = np.repeat(np.arange(len(lens)), lens)
    keep = (ivf >= b) & (ivf < e)
    return ivf[keep] - b, np.bincount(cen[keep], minlength=len(lens)).astype(np.int32)


def shard_arrays(ix, b, e):
    """What pb_index_open is given for docs [b, e) of the oracle index `ix`: (codes, residuals, doc_lengths, ivf,
    ivf_lengths); doc_id_base is b."""
    t0, t1 = int(ix.doc_offsets[b]), int(ix.doc_offsets[e])
    ivf, lens = ivf_slice(ix.ivf, ix.ivf_lengths, b, e)
    return ix.codes[t0:t1], ix.residuals[t0:t1], ix.doc_lengths[b:e], ivf, lens


def shard_bounds(doc_lengths, world):
    """bounds[r] = min { d : doc_off[d] * world >= N * r } for 0 < r < world, bounds[0] = 0, bounds[world] = D."""
    off = np.concatenate([[0], np.cumsum(np.asarray(doc_lengths, np.int64))]).astype(object)
    D, N = len(off) - 1, off[-1]
    out = [0]
    for r in range(1, world):
        out.append(next(d for d in range(D + 1) if off[d] * world >= N * r))
    return np.array(out + [D], np.int64)
