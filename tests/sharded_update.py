"""numpy restatement of pb_index_delete_sharded / pb_index_append_sharded (include/plaid_b200.h) on a doc-sharded
deployment whose rank r holds documents [bounds[r], bounds[r + 1]) with that range's slice of the inverted file.

Delete: rank r removes the ids in its range and renumbers its survivors locally (delete_ivf on its own slice); its base
drops by the documents removed below it.  Append: the documents go to the last rank (merge_ivf on its slice, ids from
its local D).  Either way each rank's patch must equal the slice of the global patch (delete_ivf / merge_ivf of the
whole inverted file) over the rank's new range."""
import numpy as np

from ivf_delete import delete_ivf
from ivf_merge import merge_ivf
from ivf_slice import ivf_slice  # noqa: F401 - also used by the tests


def deleted_set(doc_ids, D):
    """the distinct ids of an index of D documents among doc_ids, sorted"""
    ids = np.asarray(doc_ids, np.int64).reshape(-1)
    return np.unique(ids[(ids >= 0) & (ids < D)])


def delete_bounds(bounds, doc_ids):
    """the ranks' new bounds: bounds[r] minus the deleted documents below it (the base shift)"""
    b = np.asarray(bounds, np.int64)
    return b - np.searchsorted(deleted_set(doc_ids, int(b[-1])), b, side="left")


def rank_delete(ivf, ivf_lengths, bounds, r, doc_ids):
    """rank r's inverted file after its local delete: its slice, its own ids, renumbered locally"""
    b, e = int(bounds[r]), int(bounds[r + 1])
    iv, ln = ivf_slice(ivf, ivf_lengths, b, e)
    mine = deleted_set(doc_ids, e)
    return delete_ivf(iv, ln, mine[mine >= b] - b, e - b)


def global_delete_slices(ivf, ivf_lengths, bounds, doc_ids):
    """the slices of the global delete_ivf over the new bounds"""
    D = int(bounds[-1])
    giv, gln = delete_ivf(ivf, ivf_lengths, deleted_set(doc_ids, D), D)
    nb = delete_bounds(bounds, doc_ids)
    return [ivf_slice(giv, gln, int(nb[r]), int(nb[r + 1])) for r in range(len(nb) - 1)]


def rank_append(ivf, ivf_lengths, bounds, new_codes, new_doc_lengths, K):
    """the last rank's inverted file after an append: merge_ivf on its slice with local ids from its own D"""
    b, e = int(bounds[-2]), int(bounds[-1])
    iv, ln = ivf_slice(ivf, ivf_lengths, b, e)
    return merge_ivf(iv, ln, new_codes, new_doc_lengths, e - b, K)


def global_append_slice(ivf, ivf_lengths, bounds, new_codes, new_doc_lengths, K):
    """the last rank's slice of the global merge_ivf (ids D_total ..), over its grown range"""
    D = int(bounds[-1])
    giv, gln = merge_ivf(ivf, ivf_lengths, new_codes, new_doc_lengths, D, K)
    return ivf_slice(giv, gln, int(bounds[-2]), D + len(new_doc_lengths))
