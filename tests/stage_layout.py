"""numpy restatement of the slot layout the exact stage of a host-tier handle (PB_OPEN_HOST_RESIDUALS) runs in
(next-plaid_b200/csrc/k_stage.cuh, DESIGN.md 4j).

After the cut, query b of a sub-batch of B keeps nkept[b] <= Mcap docs kept[b][j] with the token prefix tokp[b][0..nkept]
of their lengths.  Slot s = b * Mcap + j stands for kept doc j of query b:
  soff[s]        staged offset of the slot: base_b + tokp[b][min(j, nkept[b])], base_b = the tokens the queries before b
                 keep; soff[B * Mcap] = the total.  Empty slots take the next query's base, so soff[s + 1] - soff[s] is
                 the length of every slot.
  kept_s[s]      s: the kernels' doc_off[kept[j]] becomes soff[s]
  staged rows    rows doc_off[d] .. doc_off[d + 1] of doc d = kept[b][j] at soff[s] ..
  map back       a list of slots (the kept list itself, or the filter's survivors) -> kept.flat[slot]
"""
import numpy as np


def layout(nkept, tokp, Mcap):
    """(soff int64 [B * Mcap + 1], kept_s uint32 [B * Mcap]) from nkept [B] and tokp [B][Mcap + 1]"""
    nkept = np.asarray(nkept, np.int64)
    tokp = np.asarray(tokp, np.int64)
    B = len(nkept)
    totals = tokp[np.arange(B), nkept]
    base = np.concatenate([[0], np.cumsum(totals)])
    j = np.arange(Mcap)
    soff = np.empty(B * Mcap + 1, np.int64)
    for b in range(B):
        soff[b * Mcap:(b + 1) * Mcap] = base[b] + tokp[b, np.minimum(j, nkept[b])]
    soff[B * Mcap] = base[B]
    return soff, np.arange(B * Mcap, dtype=np.uint32)


def stage(rows, doc_off, kept, nkept, soff, Mcap):
    """the staged copy of rows (any per-token array, first axis = token) for the kept docs"""
    out = np.zeros((int(soff[-1]),) + rows.shape[1:], rows.dtype)
    for b in range(len(nkept)):
        for j in range(nkept[b]):
            d = kept[b * Mcap + j]
            s = b * Mcap + j
            out[soff[s]:soff[s] + doc_off[d + 1] - doc_off[d]] = rows[doc_off[d]:doc_off[d + 1]]
    return out


def unstage(slots, nkept, Mcap, kept_flat):
    """slot ids -> doc ids for the first nkept[b] entries of each query's row of `slots` (in place on a copy)"""
    out = np.array(slots, copy=True)
    for b in range(len(nkept)):
        row = out[b * Mcap:b * Mcap + nkept[b]]
        row[:] = kept_flat[row]
    return out
