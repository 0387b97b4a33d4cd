"""numpy restatement of the conformal predictive distribution (csrc/cpd.cu, train.ScoreDistribution): the fp32 score
and its -0 canonicalisation, the sorted table and its row layout, the row a query reads, the tail counts, the p-value
and the quantile at any level.

``table`` / ``tail`` / ``quantile`` are the vectorised forms (one lexsort, ``np.searchsorted`` on both sides);
``table_brute`` / ``tail_brute`` / ``quantile_brute`` sort every group with Python's sort and count by comparing.  The
``defect`` switches break one rule each, so the CPU tests can show that the GPU tests' bit-equality would catch it:
  "swap_ge_gt"   the counts of s >= c and s > c are swapped
  "no_plus1"     the p-value is #{s >= c} / (m + 1)
  "k_n"          k = ceil(m tau) instead of ceil((m + 1) tau)
  "no_fallback"  an in-range entry always reads its own row (an empty or small one too)
  "row_shift"    entry g reads row g + 1
"""
import math

import numpy as np


def scores(y, yhat):
    """[n] fp32 scores (float)y - yhat, -0 -> +0."""
    s = (np.asarray(y, dtype=np.int64).astype(np.float32) - np.asarray(yhat, dtype=np.float32)).astype(np.float32)
    s[s == 0] = np.float32(0.0)
    return s


def table(y, yhat, group, n_groups):
    """-> (scores fp32 [ptr[-1]], ptr int64 [G + 2]): rows 0 .. G-1 the sorted scores of each group, then row G all
    of them sorted; group None: the global row only (rows 0 .. G-1 empty)."""
    s = scores(y, yhat)
    G = int(n_groups)
    if group is None:
        return np.sort(s), np.concatenate([np.zeros(G + 1, np.int64), [s.size]]).astype(np.int64)
    g = np.asarray(group, dtype=np.int64)
    cnt = np.bincount(g, minlength=G)[:G]
    ptr = np.concatenate([[0], np.cumsum(cnt), [2 * s.size]]).astype(np.int64)
    return np.concatenate([s[np.lexsort((s, g))], np.sort(s)]).astype(np.float32), ptr


def table_brute(y, yhat, group, n_groups):
    s = scores(y, yhat).tolist()
    G = int(n_groups)
    rows = [[] for _ in range(G)]
    if group is not None:
        for v, gi in zip(s, np.asarray(group, dtype=np.int64).tolist()):
            rows[gi].append(v)
    rows = [sorted(r) for r in rows] + [sorted(s)]
    ptr = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int64)
    return np.array([v for r in rows for v in r], dtype=np.float32), ptr


def rows_of(ptr, min_count, group, Q, defect=None):
    """The row each of Q queries reads: g iff 0 <= g < G and n_g >= min_count, else G."""
    G = ptr.size - 2
    g = np.full(Q, -1, np.int64) if group is None else np.asarray(group, dtype=np.int64).reshape(-1)
    ok = (g >= 0) & (g < G)
    gi = np.where(ok, g, 0)
    if defect != "no_fallback":
        ok &= (ptr[gi + 1] - ptr[gi]) >= min_count
    r = np.where(ok, g, G)
    if defect == "row_shift":
        r = np.where(ok, np.minimum(r + 1, G), r)
    return r


def thresholds(yhat, x=None, y=None):
    """c [Q, S] fp32: fl(x - yhat), or fl((float)y - yhat) for labels (S = 1), -0 -> +0."""
    yh = np.asarray(yhat, dtype=np.float32).reshape(-1, 1)
    v = (np.asarray(y, dtype=np.int64).astype(np.float32).reshape(-1, 1) if x is None
         else np.asarray(x, dtype=np.float32).reshape(yh.shape[0], -1))
    with np.errstate(invalid="ignore"):
        c = (v - yh).astype(np.float32)
    c[c == 0] = np.float32(0.0)
    return c


def tail(tab, ptr, min_count, yhat, group, x=None, y=None, defect=None):
    """-> (ge, gt [Q, S] int32, row [Q] int32): #{s >= c} and #{s > c} in the row each query reads."""
    c = thresholds(yhat, x, y)
    Q, S = c.shape
    r = rows_of(ptr, min_count, group, Q, defect)
    ge = np.empty((Q, S), np.int32)
    gt = np.empty((Q, S), np.int32)
    for row in np.unique(r):
        sel = r == row
        a = tab[ptr[row]:ptr[row + 1]]
        ge[sel] = a.size - np.searchsorted(a, c[sel], side="left")
        gt[sel] = a.size - np.searchsorted(a, c[sel], side="right")
    if defect == "swap_ge_gt":
        ge, gt = gt, ge
    return ge, gt, r.astype(np.int32)


def tail_brute(tab, ptr, min_count, yhat, group, x=None, y=None):
    c = thresholds(yhat, x, y)
    Q, S = c.shape
    r = rows_of(ptr, min_count, group, Q)
    ge = np.empty((Q, S), np.int32)
    gt = np.empty((Q, S), np.int32)
    for q in range(Q):
        a = tab[ptr[r[q]]:ptr[r[q] + 1]].tolist()
        for j in range(S):
            ge[q, j] = sum(1 for v in a if v >= c[q, j])
            gt[q, j] = sum(1 for v in a if v > c[q, j])
    return ge, gt, r.astype(np.int32)


def probabilities(ge, gt, row, ptr):
    """(lo, hi) float64: gt / (m + 1), (ge + 1) / (m + 1), m the size of the row read."""
    m1 = (ptr[row.astype(np.int64) + 1] - ptr[row.astype(np.int64)] + 1).astype(np.float64).reshape(-1, 1)
    return gt / m1, (ge + 1) / m1


def pvalues(tab, ptr, min_count, yhat, group, y, defect=None):
    ge, gt, row = tail(tab, ptr, min_count, yhat, group, y=y, defect=defect)
    m1 = (ptr[row.astype(np.int64) + 1] - ptr[row.astype(np.int64)] + 1).astype(np.float64)
    return (ge[:, 0] + (0 if defect == "no_plus1" else 1)) / m1


def k_of(m, tau, defect=None):
    return max(1, math.ceil(m * tau if defect == "k_n" else (m + 1) * tau))


def quantile(tab, ptr, min_count, yhat, group, levels, defect=None):
    """-> fp32 [Q, L]: fl(yhat + s_(k)) with the own-row rule of the calibration, +inf where row G has no k-th score."""
    yh = np.asarray(yhat, dtype=np.float32).reshape(-1)
    Q, G = yh.size, ptr.size - 2
    g = np.full(Q, -1, np.int64) if group is None else np.asarray(group, dtype=np.int64).reshape(-1)
    out = np.empty((Q, len(levels)), np.float32)
    n = int(ptr[G + 1] - ptr[G])
    for li, tau in enumerate(levels):
        kg = k_of(n, tau, defect)
        own_k = {}
        for r in range(G):
            m = int(ptr[r + 1] - ptr[r])
            k = k_of(m, tau, defect)
            if (m > 0 and k <= m and m >= min_count) or (defect == "no_fallback" and m > 0):
                own_k[r] = min(k, m)
        for q in range(Q):
            r = int(g[q])
            if defect == "row_shift" and 0 <= r < G:
                r += 1
            if 0 <= r < G and r in own_k:
                s = tab[ptr[r] + own_k[r] - 1]
            elif kg <= n:
                s = tab[ptr[G] + kg - 1]
            else:
                out[q, li] = np.inf
                continue
            out[q, li] = np.float32(yh[q] + s)
    return out


def quantile_brute(tab, ptr, min_count, yhat, group, levels):
    """The same from the §8m rule, row by row with Python numbers (the float add in fp32)."""
    yh = np.asarray(yhat, dtype=np.float32).reshape(-1)
    G = ptr.size - 2
    rows = [tab[ptr[r]:ptr[r + 1]].tolist() for r in range(G + 1)]
    out = np.empty((yh.size, len(levels)), np.float32)
    for q in range(yh.size):
        g = -1 if group is None else int(np.asarray(group).reshape(-1)[q])
        for li, tau in enumerate(levels):
            row = rows[g] if 0 <= g < G else None
            if row is not None:
                m = len(row)
                k = max(1, math.ceil((m + 1) * tau))
                if not (m > 0 and k <= m and m >= min_count):
                    row = None
            if row is None:
                row = rows[G]
                k = max(1, math.ceil((len(row) + 1) * tau))
            out[q, li] = np.inf if k > len(row) else np.float32(np.float32(yh[q]) + np.float32(row[k - 1]))
    return out


def make_set(rng, n, n_groups, kind, score_kind="normal"):
    """A synthetic held-out set: y int64, yhat [n] fp32, group int64.  kind: "uniform", "sparse" (many empty groups),
    "zipf" (one group holds 90 %); score_kind: "normal", "ties" (a small integer set, +-0), "extreme" (subnormals,
    +-1e30 and ties), "top_byte" (keys sharing their top byte: scores in [1, 2)), "equal" (one score)."""
    if kind == "uniform":
        g = rng.integers(0, n_groups, n)
    elif kind == "sparse":
        live = rng.choice(n_groups, size=max(1, n_groups // 8), replace=False)
        g = live[rng.integers(0, live.size, n)]
    elif kind == "zipf":
        g = np.where(rng.random(n) < 0.9, n_groups // 2, rng.integers(0, n_groups, n))
    else:
        raise ValueError(kind)
    y = rng.integers(0, 2000, n).astype(np.int64)
    if score_kind == "normal":
        yhat = y + rng.normal(0, 100, n)
    elif score_kind == "ties":
        yhat = y - rng.integers(-3, 4, n)
    elif score_kind == "top_byte":
        y = np.zeros(n, np.int64)
        yhat = -(1.0 + rng.random(n))
    elif score_kind == "equal":
        yhat = y - 7.0
    else:
        pool = np.array([0.0, -0.0, 1e-40, -1e-40, 1e30, -1e30, 1.0, -1.0, 2.5], dtype=np.float32)
        y = rng.integers(0, 3, n).astype(np.int64)
        yhat = pool[rng.integers(0, pool.size, n)]
        yhat = np.where(rng.random(n) < 0.3, y.astype(np.float32), yhat)
    return y, np.asarray(yhat, dtype=np.float32), g.astype(np.int64)
