"""numpy restatement of the inverted-file merge of update_index (next-plaid/src/update.rs:1000-1067), the reference
side of pb_index_append's merge: every list is sorted and de-duplicated literally, as the reference does, without
relying on the new ids being larger than the old ones."""
import numpy as np


def merge_ivf(old_ivf, old_lengths, new_codes, new_doc_lengths, old_D, K):
    """(ivf <i8, ivf_lengths <i4) after appending docs with these codes as ids old_D, old_D + 1, ..."""
    old_ivf = np.asarray(old_ivf, np.int64)
    old_lengths = np.asarray(old_lengths, np.int32)
    new_codes = np.asarray(new_codes, np.int64)
    # update.rs:1000-1009: centroid -> new pids, in doc order
    partition_pids = {}
    pos = 0
    for pid, n in enumerate(np.asarray(new_doc_lengths, np.int64).tolist(), start=old_D):
        for code in new_codes[pos:pos + n].tolist():
            partition_pids.setdefault(code, []).append(pid)
        pos += n
    # update.rs:1033-1039: old offsets
    old_offsets = np.zeros(len(old_lengths) + 1, np.int64)
    np.cumsum(old_lengths, out=old_offsets[1:])
    data, lengths = [], []
    for c in range(K):                                   # update.rs:1045-1067
        start = int(old_offsets[c]) if c < len(old_lengths) else 0
        n = int(old_lengths[c]) if c < len(old_lengths) else 0
        pids = old_ivf[start:start + n].tolist() if n > 0 and start + n <= len(old_ivf) else []
        pids.extend(partition_pids.get(c, []))
        pids = sorted(set(pids))                         # sort_unstable + dedup
        lengths.append(len(pids))
        data.extend(pids)
    return np.array(data, np.int64), np.array(lengths, np.int32)
