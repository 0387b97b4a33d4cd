"""numpy restatement of the score window (train.ScoreDistribution.insert / evict, csrc/cpd.cu pert_cpd_merge): the
log, the update of the table by a merge with the fit of the change, and the growth of the entry rows.

``Window`` keeps the log (y, yhat, entry, ts) in insertion order and a table it updates with ``merge`` (the vectorised
form: the rows of both tables concatenated and sorted, or the delta's values removed by count through sorted ranks);
``table()`` is the fit of ``tests/cpd_ref.table`` over the log, the contract the GPU tests hold the update to.
``merge_brute`` updates row by row with Python lists (``list.remove`` for a removal).  The ``defect`` switches break
one rule each, so the CPU tests can show that the GPU tests' bit-equality would catch it:
  "skip_global"   an evict leaves row G as it was
  "old_g_at_gold" after growth, old row G lands in row G_old instead of row G_new
  "remove_all"    a removal drops every copy of an evicted value instead of its count
  "unstable"      the log split keeps the surviving rows in reverse order
"""
import numpy as np

from tests import cpd_ref as R


def old_row(r, G_old, G_new, defect=None):
    """The old row output row r reads, or -1 (an empty old row)."""
    if r < G_old:
        return r
    if defect == "old_g_at_gold":
        return G_old if r == G_old else -1
    return G_old if r == G_new else -1


def _rows(tab, ptr):
    return [tab[ptr[r]:ptr[r + 1]] for r in range(ptr.size - 1)]


def _pack(rows):
    ptr = np.concatenate([[0], np.cumsum([r.size for r in rows])]).astype(np.int64)
    tab = np.concatenate(rows).astype(np.float32) if rows else np.zeros(0, np.float32)
    return tab, ptr


def _keys(a):
    """The order-preserving uint32 keys of fp32 values (calib.cuh's map)."""
    u = np.asarray(a, dtype=np.float32).view(np.uint32)
    return np.where(u & 0x80000000, ~u, u | 0x80000000).astype(np.uint32)


def remove_sorted(a, d, defect=None):
    """The sorted multiset a minus the sorted multiset d (d within a): each value loses its count in d."""
    if d.size == 0:
        return a.copy()
    ka, kd = _keys(a), _keys(d)
    if defect == "remove_all":
        return a[~np.isin(ka, kd)]
    # rank of every element of a in its run of equal values; it is dropped iff rank < the value's count in d
    rank = np.arange(a.size) - np.searchsorted(ka, ka, side="left")
    c = np.searchsorted(kd, ka, side="right") - np.searchsorted(kd, ka, side="left")
    if (np.searchsorted(ka, kd, side="right") - np.searchsorted(ka, kd, side="left")
            < np.searchsorted(kd, kd, side="right") - np.searchsorted(kd, kd, side="left")).any():
        raise ValueError("the delta holds a value more often than the table")
    return a[rank >= c]


def merge(tab, ptr, dtab, dptr, sign, defect=None):
    """-> (tab, ptr) of the old table (G_old = ptr.size - 2) plus / minus the delta (G_new = dptr.size - 2)."""
    G_old, G_new = ptr.size - 2, dptr.size - 2
    if G_new < G_old:
        raise ValueError("G_new < G_old")
    old, dl = _rows(tab, ptr), _rows(dtab, dptr)
    out = []
    for r in range(G_new + 1):
        ro = old_row(r, G_old, G_new, defect)
        a = old[ro] if ro >= 0 else np.zeros(0, np.float32)
        if sign > 0:
            row = np.sort(np.concatenate([a, dl[r]]).astype(np.float32), kind="stable")
        elif defect == "skip_global" and r == G_new:
            row = a.copy()
        else:
            row = remove_sorted(a, dl[r], defect)
        out.append(row)
    return _pack(out)


def merge_brute(tab, ptr, dtab, dptr, sign):
    G_old, G_new = ptr.size - 2, dptr.size - 2
    old = [tab[ptr[r]:ptr[r + 1]].tolist() for r in range(G_old + 1)]
    out = []
    for r in range(G_new + 1):
        ro = old_row(r, G_old, G_new)
        row = list(old[ro]) if ro >= 0 else []
        d = dtab[dptr[r]:dptr[r + 1]].tolist()
        if sign > 0:
            row = sorted(row + d)
        else:
            for v in d:
                row.remove(v)                 # ValueError when the table lacks it
        out.append(np.array(row, dtype=np.float32))
    return _pack(out)


class Window:
    """The log and the table of one distribution (``group`` False: by="global", the global row only)."""

    def __init__(self, y, yhat, entry, ts, n_groups, group=True, defect=None, brute=False):
        self.G, self.group, self.defect, self.brute = int(n_groups), group, defect, brute
        self.log = [np.asarray(a, dtype=t).copy() for a, t in
                    zip((y, yhat, entry, ts), (np.int64, np.float32, np.int64, np.int64))]
        self.tab, self.ptr = self._fit(*self.log[:3], self.G)

    def _fit(self, y, yhat, entry, G):
        if self.brute:
            return R.table_brute(y, yhat, entry if self.group else None, G if self.group else 0)
        return R.table(y, yhat, entry if self.group else None, G if self.group else 0)

    def _merge(self, dtab, dptr, sign):
        if self.brute:
            return merge_brute(self.tab, self.ptr, dtab, dptr, sign)
        return merge(self.tab, self.ptr, dtab, dptr, sign, self.defect)

    def table(self):
        """The fit over the surviving log: what the updated table must equal."""
        return self._fit(*self.log[:3], self.G)

    def insert(self, y, yhat, entry, ts, n_groups=None):
        G_new = self.G if n_groups is None or not self.group else int(n_groups)
        if G_new < self.G:
            raise ValueError("n_groups shrinks the table")
        d = [np.asarray(a, dtype=t) for a, t in zip((y, yhat, entry, ts), (np.int64, np.float32, np.int64, np.int64))]
        dtab, dptr = self._fit(*d[:3], G_new)
        self.tab, self.ptr = self._merge(dtab, dptr, 1)
        self.G = G_new
        self.log = [np.concatenate([a, b]) for a, b in zip(self.log, d)]

    def evict(self, before):
        drop = self.log[3] < before
        k = int(drop.sum())
        if k == 0:
            return 0
        if k == drop.size:
            raise ValueError("the window would be empty")
        dtab, dptr = self._fit(*(a[drop] for a in self.log[:3]), self.G)
        self.tab, self.ptr = self._merge(dtab, dptr, -1)
        keep = np.flatnonzero(~drop)
        if self.defect == "unstable":
            keep = keep[::-1]
        self.log = [a[keep] for a in self.log]
        return k
