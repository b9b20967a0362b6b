"""numpy restatement of the inverted-file patch of delete_from_index (next-plaid/src/delete.rs:196-237), the reference
side of pb_index_delete's filter-and-renumber: deleted ids leave every list, and a survivor's new id is its old one
minus the number of deleted ids below it.  Only ids of the index count as deleted (0 <= id < num_documents, each once):
the reference's shift also counts negative ids it was asked for, which would renumber the inverted file without
renumbering the chunks."""
import numpy as np


def delete_ivf(ivf, ivf_lengths, doc_ids, num_documents):
    """(ivf <i8, ivf_lengths <i4) after deleting doc_ids from an index of num_documents documents"""
    ivf = np.asarray(ivf, np.int64)
    ids = np.asarray(doc_ids, np.int64).reshape(-1)
    deleted = set(ids[(ids >= 0) & (ids < num_documents)].tolist())
    sorted_deleted = np.array(sorted(deleted), np.int64)
    data, lengths = [], []
    off = 0
    for n in np.asarray(ivf_lengths, np.int64).tolist():
        kept = 0
        for d in ivf[off:off + n].tolist():
            if d in deleted:
                continue
            data.append(d - int(np.searchsorted(sorted_deleted, d, side="left")))   # partition_point(< d)
            kept += 1
        lengths.append(kept)
        off += n
    return np.array(data, np.int64), np.array(lengths, np.int32)


def keep_mask(doc_lengths, doc_ids):
    """(kept docs, kept tokens) as boolean masks, for filtering the per-doc and per-token arrays"""
    dl = np.asarray(doc_lengths, np.int64)
    ids = np.asarray(doc_ids, np.int64).reshape(-1)
    docs = ~np.isin(np.arange(len(dl)), ids)
    return docs, np.repeat(docs, dl)
