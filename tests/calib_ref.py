"""numpy restatement of the conformal calibration (csrc/calib.cu, train.Calibration): the fp32 score and its -0
canonicalisation, the k rule, the own-or-global fallback, the apply and the running max.

``offsets`` is the vectorised form (one lexsort per level); ``offsets_brute`` sorts every group on its own.  The
``defect`` switches break one rule each, so the CPU tests can show that the GPU tests' bit-equality would catch it:
  "k_n"          k = ceil(n tau) instead of ceil((n + 1) tau)
  "no_fallback"  a group without its own offset gets 0 instead of the global one
  "running_min"  the monotone apply takes a running min
  "row_shift"    the apply reads row g + 1 for group g
"""
import math

import numpy as np


def scores(y, yhat):
    """[n, T] fp32 scores (float)y - yhat, -0 -> +0."""
    yf = np.asarray(y, dtype=np.int64).astype(np.float32)
    yh = np.asarray(yhat, dtype=np.float32).reshape(yf.shape[0], -1)
    s = (yf[:, None] - yh).astype(np.float32)
    s[s == 0] = np.float32(0.0)
    return s


def k_of(m, tau, defect=None):
    x = m * tau if defect == "k_n" else (m + 1) * tau
    return max(1, math.ceil(x))


def own_of(m, tau, min_count, is_global, defect=None):
    return m > 0 and k_of(m, tau, defect) <= m and (is_global or m >= min_count)


def offsets(y, yhat, group, n_groups, taus, min_count=1, defect=None):
    """-> (off [G+1, T] fp32, count [G+1] int32, own [G+1, T] int8); group None: one global group."""
    s = scores(y, yhat)
    n, T = s.shape
    G = int(n_groups)
    g = np.full(n, G, dtype=np.int64) if group is None else np.asarray(group, dtype=np.int64)
    count = np.zeros(G + 1, dtype=np.int32)
    if group is not None:
        count[:G] = np.bincount(g, minlength=G)[:G]
    count[G] = n
    ptr = np.concatenate([[0], np.cumsum(count[:G].astype(np.int64))])
    off = np.zeros((G + 1, T), dtype=np.float32)
    own = np.zeros((G + 1, T), dtype=np.int8)
    for t, tau in enumerate(taus):
        col = s[:, t]
        kg = k_of(n, tau, defect)
        glob = np.partition(col, kg - 1)[kg - 1] if kg <= n else np.float32(np.nan)
        srt = col[np.lexsort((col, g))] if group is not None else None
        for r in range(G + 1):
            m = int(count[r])
            if own_of(m, tau, min_count, r == G, defect):
                k = k_of(m, tau, defect)
                off[r, t] = glob if r == G else srt[ptr[r] + k - 1]
                own[r, t] = 1
            else:
                off[r, t] = np.float32(0.0) if defect == "no_fallback" else glob
    return off, count, own


def offsets_brute(y, yhat, group, n_groups, taus, min_count=1):
    """The same by sorting every group's scores with Python's sort."""
    s = scores(y, yhat)
    n, T = s.shape
    G = int(n_groups)
    members = [[] for _ in range(G)]
    if group is not None:
        for i, gi in enumerate(np.asarray(group, dtype=np.int64).tolist()):
            members[gi].append(i)
    members.append(list(range(n)))
    off = np.zeros((G + 1, T), dtype=np.float32)
    own = np.zeros((G + 1, T), dtype=np.int8)
    for t, tau in enumerate(taus):
        rows = [sorted(s[idx, t].tolist()) for idx in members]
        k = max(1, math.ceil((n + 1) * tau))
        glob = rows[G][k - 1]
        for r, v in enumerate(rows):
            m = len(v)
            k = max(1, math.ceil((m + 1) * tau))
            if m > 0 and k <= m and (r == G or m >= min_count):
                off[r, t], own[r, t] = v[k - 1], 1
            else:
                off[r, t] = glob
    return off, np.array([len(v) for v in members], dtype=np.int32), own


def apply(yhat, group, off, monotone=False, live=None, defect=None):
    """fp32 yhat [Q, T] + off[g] (g outside [0, rows - 1): the last row), then the running max; rows >= live kept."""
    out = np.array(yhat, dtype=np.float32, copy=True)
    flat = out.ndim == 1
    if flat:
        out = out[:, None]
    Q = out.shape[0]
    q = Q if live is None else min(Q, int(live))
    if off is not None:
        off = np.asarray(off, dtype=np.float32)
        rows = off.shape[0]
        g = np.full(Q, rows - 1, dtype=np.int64) if group is None else np.asarray(group, dtype=np.int64).copy()
        g[(g < 0) | (g >= rows - 1)] = rows - 1
        if defect == "row_shift":
            g = np.minimum(g + 1, rows - 1)
        out[:q] = (out[:q] + off[g[:q]]).astype(np.float32)
    if monotone:
        acc = np.fmin.accumulate if defect == "running_min" else np.fmax.accumulate
        out[:q] = acc(out[:q], axis=1)
    return out[:, 0] if flat else out


def roundtrip_slack(y, yhat):
    """r of the in-sample coverage bound: graphs with fl(yhat + fl(y - yhat)) < y, per level [T]."""
    yf = np.asarray(y, dtype=np.int64).astype(np.float32)
    yh = np.asarray(yhat, dtype=np.float32).reshape(yf.shape[0], -1)
    s = (yf[:, None] - yh).astype(np.float32)
    return ((yh + s).astype(np.float32) < yf[:, None]).sum(axis=0)


def make_set(rng, n, T, n_groups, kind, score_kind="normal"):
    """A synthetic calibration set: y int64, yhat [n, T] fp32, group int64.  kind: "uniform", "sparse" (many empty
    groups), "zipf" (one group holds 90 %); score_kind: "normal", "ties" (a small integer set, +-0), "extreme"
    (subnormals, +-1e30 and ties)."""
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
        yhat = (y[:, None] + rng.normal(0, 100, (n, T))).astype(np.float32)
    elif score_kind == "ties":
        yhat = (y[:, None] - rng.integers(-3, 4, (n, T))).astype(np.float32)
    else:
        pool = np.array([0.0, -0.0, 1e-40, -1e-40, 1e30, -1e30, 1.0, -1.0, 2.5], dtype=np.float32)
        y = rng.integers(0, 3, n).astype(np.int64)
        yhat = pool[rng.integers(0, pool.size, (n, T))]
        yhat = np.where(rng.random((n, T)) < 0.3, y[:, None].astype(np.float32), yhat).astype(np.float32)
    return y, yhat.astype(np.float32), g.astype(np.int64)
