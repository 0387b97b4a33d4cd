"""Host mirror of rawtable.ResourceSampleWindow: every open key's samples as a list in arrival order, late samples
counted and dropped, and the statistics of a set of keys from the numpy oracle (oracle.raw_table_oracle._group_stats)
over those lists."""
import numpy as np

from oracle.raw_table_oracle import _group_stats

I64_MIN = -(1 << 63)


class SampleWindowRef:
    def __init__(self, n_ms):
        self.n_ms = n_ms
        self.samples = {}                                # key -> [(cpu, mem)] in arrival order
        self.sealed = I64_MIN

    def add(self, ts, ms, cpu, mem):
        """-> (sorted touched keys, late count)."""
        touched, late = set(), 0
        for t, m, c, u in zip(ts, ms, cpu, mem):
            if int(t) < self.sealed:
                late += 1
                continue
            key = int(t) * self.n_ms + int(m)
            self.samples.setdefault(key, []).append((float(c), float(u)))
            touched.add(key)
        return sorted(touched), late

    def seal(self, before):
        if before <= self.sealed:
            return
        self.sealed = before
        self.samples = {k: v for k, v in self.samples.items() if k // self.n_ms >= before}

    def keys(self):
        return sorted(self.samples)

    def stats(self, keys):
        """(index int64 [n, 2], values float64 [n, 8]) of ``keys`` in the given order."""
        keys = list(keys)
        n = np.array([len(self.samples[k]) for k in keys], dtype=np.int64)
        gid = np.repeat(np.arange(len(keys)), n)
        v = np.array([s for k in keys for s in self.samples[k]], dtype=np.float64).reshape(-1, 2)
        with np.errstate(invalid="ignore"):                # inf - inf in the Kahan fold, as pandas
            vals = np.concatenate([_group_stats(v[:, j].copy(), gid, len(keys)) for j in (0, 1)], axis=1)
        k = np.array(keys, dtype=np.int64)
        return np.stack([k // self.n_ms, k % self.n_ms], 1), vals
