"""numpy restatement of which documents a fill of the device row cache takes (pb_index_fill_row_cache, DESIGN.md 4s).

By counts: every doc kept at least once by search staging since the last such fill, most kept first, ties by ascending
id.  With ids: the caller's ids in its order, ids outside the handle's range and repeats ignored.  Either way each doc
is taken when its rows (length x packed bytes) still fit the budget, and skipped otherwise."""
import numpy as np


def keep_counts(kept_lists, n_docs, base=0):
    """per doc of [base, base + n_docs), how many of the given kept lists (one per query and call) hold it"""
    c = np.zeros(n_docs, np.int64)
    for ids in kept_lists:
        np.add.at(c, np.asarray(ids, np.int64) - base, 1)
    return c


def order_by_counts(counts):
    """docs with a nonzero count, by count descending, then id ascending"""
    d = np.nonzero(np.asarray(counts))[0]
    return d[np.lexsort((d, -np.asarray(counts)[d]))]


def order_of_ids(ids, n_docs, base=0):
    """the ids in [base, base + n_docs) as local docs, first occurrences only, in the given order"""
    seen, out = set(), []
    for i in ids:
        d = int(i) - base
        if 0 <= d < n_docs and d not in seen:
            seen.add(d)
            out.append(d)
    return np.array(out, np.int64)


def fit_or_skip(order, lengths, packed, budget):
    """(docs taken in order, row bytes they use): each doc whose rows still fit the budget"""
    taken, used = [], 0
    for d in order:
        b = int(lengths[d]) * packed
        if used + b <= budget:
            taken.append(int(d))
            used += b
    return np.array(taken, np.int64), used
