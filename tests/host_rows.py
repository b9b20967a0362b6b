"""numpy restatement of the pinned row store of a host-tier handle (HostRows in next-plaid_b200/csrc/engine.cu,
DESIGN.md 4r) and of how a delete compacts it.

The packed rows (`packed` bytes per token) are one byte array cut into segments of S = 2^shift bytes:
  byte b          is at segment b >> shift, offset b & (S - 1)
  pieces(b, n)    the (segment, offset in segment, offset in range, length) runs of bytes [b, b + n), split at every
                  segment boundary; a row or a document may straddle two segments, an aligned 2-, 4- or 16-byte load
                  unit never does (S is a multiple of 16)
  open(n)         segments of S bytes, the last exactly as long as the rows need
  grow(want)      the short last segment replaced by a full one, then full segments added up to ceil(want / S)

A delete keeps the docs not deleted, in order, at new offsets new_off[j] <= old_off[kept[j]].  From the first deleted
doc on, the survivors are cut into windows: runs of survivors whose rows fit `window` tokens (a longer doc is a window
of its own).  Each window's rows are gathered from their old offsets into a staging buffer and written back at
new_off[j0] .. new_off[j1], one copy per segment piece of that destination range, windows in ascending order.
"""
import numpy as np


def pieces(b, n, shift):
    """[(segment, offset in segment, offset in range, length)] of bytes [b, b + n)"""
    S = 1 << shift
    out, done = [], 0
    while done < n:
        o = (b + done) & (S - 1)
        m = min(n - done, S - o)
        out.append(((b + done) >> shift, o, done, m))
        done += m
    return out


def open_sizes(n, shift):
    """segment lengths of a store opened on n bytes"""
    S = 1 << shift
    return [min(S, n - o) for o in range(0, n, S)]


def grow_sizes(sizes, want, shift):
    """segment lengths after capacity for `want` bytes"""
    S = 1 << shift
    if want <= sum(sizes):
        return list(sizes)
    return [S] * (-(-want // S))


def write(segs, b, data, shift):
    for k, o, r, m in pieces(b, len(data), shift):
        segs[k][o:o + m] = data[r:r + m]


def read(segs, b, n, shift):
    out = np.empty(n, np.uint8)
    for k, o, r, m in pieces(b, n, shift):
        out[r:r + m] = segs[k][o:o + m]
    return out


def store(rows, shift):
    """the segments of a store opened on rows (uint8 [N, packed])"""
    flat = np.ascontiguousarray(rows, np.uint8).reshape(-1)
    return [flat[o:o + m].copy() for o, m in zip(range(0, len(flat), 1 << shift), open_sizes(len(flat), shift))]


def delete_plan(doc_lengths, deleted, window):
    """(kept, old_off, new_off, windows [(j0, j1)]) of deleting the doc ids `deleted`"""
    dl = np.asarray(doc_lengths, np.int64)
    old_off = np.concatenate([[0], np.cumsum(dl)])
    gone = np.zeros(len(dl), bool)
    gone[list(deleted)] = True
    kept = np.flatnonzero(~gone)
    new_off = np.concatenate([[0], np.cumsum(dl[kept])])
    wins = []
    if gone.any():
        first = int(np.argmax(gone))                     # survivors before the first deleted doc keep their rows
        j0 = first
        while j0 < len(kept):
            j1 = j0 + 1
            while j1 < len(kept) and new_off[j1 + 1] - new_off[j0] <= window:
                j1 += 1
            wins.append((j0, j1))
            j0 = j1
    return kept, old_off, new_off, wins


def compact(segs, doc_lengths, deleted, window, packed, shift):
    """the store after the delete, in place, window by window as the library runs it"""
    kept, old_off, new_off, wins = delete_plan(doc_lengths, deleted, window)
    for j0, j1 in wins:
        stage = np.concatenate([read(segs, int(old_off[d]) * packed, int(old_off[d + 1] - old_off[d]) * packed, shift)
                                for d in kept[j0:j1]] + [np.zeros(0, np.uint8)])
        write(segs, int(new_off[j0]) * packed, stage, shift)
    return segs, int(new_off[-1])
