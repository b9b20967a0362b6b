"""numpy restatement of a5's pruned first pass (next-plaid_b200/csrc/k_approx16.cuh, DESIGN.md 4b).

One query of nq tokens over a 16-bit score table T [K, nq] (code units) and candidates given as lists of distinct codes:
  L(d)     = sum_q max_{c in d} T[c, q]                                   the first-pass score (k_approx16)
  live(c)  = any_q T[c, q] >= f[q]                                        (k_a5_live)
  U(d)     = sum_q max(max_{c in d, live(c)} T[c, q] (0 if none), f[q] - 1 (0 if f[q] = 0))   (k_a5_bound)
  select(keys, N, W) = N-th largest key minus W (0 when fewer than N keys)  (k_select_u32)
Dense:  band = {d : L(d) >= select(L, M, W)}.
Pruned: theta1 = select(U, M1, 0); R1 = {U >= theta1}; tau1 = select(L over R1, M, W) (the threshold, band included);
        R2 = {tau1 <= U < theta1}; band = {d in R1 + R2 : L(d) >= select(L over R1 + R2, M, W)}.
"""
import numpy as np


def first_pass(T, docs):
    return np.array([int(T[d].max(0).sum()) if len(d) else 0 for d in docs], np.int64)


def bound(T, docs, f):
    f = np.asarray(f, np.int64)
    live = (T >= f[None, :]).any(1)
    dead = np.maximum(f - 1, 0)
    out = []
    for d in docs:
        d = np.asarray(d, np.int64)
        lv = d[live[d]] if len(d) else d
        m = T[lv].max(0) if len(lv) else np.zeros(T.shape[1], np.int64)
        out.append(int(np.maximum(m, dead).sum()))
    return np.array(out, np.int64), int(sum(int(live[np.asarray(d, np.int64)].sum()) for d in docs if len(d)))


def select(keys, N, W):
    keys = np.asarray(keys, np.int64)
    if len(keys) < N or N <= 0:
        return 0
    tau = int(np.sort(keys)[::-1][N - 1])
    return max(tau - W, 0)


def dense_band(L, M, W):
    return set(np.flatnonzero(L >= select(L, M, W)).tolist())


def pruned_band(L, U, M, M1, W):
    """(band, |R1| + |R2|); L is read only on R1 and R2"""
    theta1 = select(U, M1, 0)
    r1 = np.flatnonzero(U >= theta1)
    tau1 = select(L[r1], M, W)
    r2 = np.flatnonzero((U >= tau1) & (U < theta1))
    r = np.concatenate([r1, r2])
    thr = select(L[r], M, W)
    return set(r[L[r] >= thr].tolist()), len(r)
