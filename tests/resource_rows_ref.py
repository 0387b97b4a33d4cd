"""Host restatement of a live store's resource rows (DESIGN.md section 8e): the list L of rows in arrival order and what
each update does to it.  The store after any sequence of updates must equal the constructor fed L."""
import numpy as np


class ResourceRows:
    """L as three host columns (timestamps, microservices, float64 values [n, 8]) over a fixed n_ms."""

    def __init__(self, art):
        self.art, self.n_ms = art, int(art["n_ms"])
        self.ts = np.array([t for t, _ in art["resource_index"]], dtype=np.int64)
        self.ms = np.array([m for _, m in art["resource_index"]], dtype=np.int64)
        self.vals = np.asarray(art["resource_values"], dtype=np.float64).reshape(-1, 8)

    def keys(self, ts=None, ms=None):
        return (self.ts if ts is None else ts) * self.n_ms + (self.ms if ms is None else ms)

    def _keep(self, keep):
        self.ts, self.ms, self.vals = self.ts[keep], self.ms[keep], self.vals[keep]

    def evict(self, cut):
        """L = [r in L : ts(r) >= cut]; returns the number of rows removed."""
        n = self.ts.size
        if cut is not None:
            self._keep(self.ts >= cut)
        return n - self.ts.size

    def append(self, ts, ms, vals, cut=None):
        """L += batch."""
        self.ts, self.ms = np.concatenate([self.ts, ts]), np.concatenate([self.ms, ms])
        self.vals = np.concatenate([self.vals, np.asarray(vals, dtype=np.float64).reshape(-1, 8)])
        self.evict(cut)

    def delete(self, ts, ms, cut=None):
        """L = [r in L : key(r) not in K]; returns the number of rows removed, by key and by the cut."""
        n = self.ts.size
        self._keep(~np.isin(self.keys(), self.keys(ts, ms)))
        self.evict(cut)
        return n - self.ts.size

    def replace(self, ts, ms, vals, cut=None):
        """L = [r in L : key(r) not in K] + [the last batch row of each key in K, in input order]."""
        k = self.keys(ts, ms)
        _, first_of_reversed = np.unique(k[::-1], return_index=True)
        last = np.sort(k.size - 1 - first_of_reversed)
        self._keep(~np.isin(self.keys(), k))
        self.append(ts[last], ms[last], np.asarray(vals, dtype=np.float64).reshape(-1, 8)[last], cut)

    def rebuild(self, device="cuda"):
        from pert_gnn_kdd23_b200.store import PatternStore

        art = dict(self.art, resource_index=list(zip(self.ts.tolist(), self.ms.tolist())), resource_values=self.vals)
        return PatternStore.from_artifacts(art, device)
