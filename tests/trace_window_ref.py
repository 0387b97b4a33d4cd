"""Numpy restatement of a live pattern store under PatternStore.append_traces and PatternStore.evict_traces: a state
machine over ordered dicts.

State: ``patterns`` {runtime id: (key bytes, representative rows)} in pattern order; ``entries`` {entry: {runtime id:
trace count}} in each entry's key order; ``traces`` {traceid: (entry, runtime id, bucket, y)} in trace-table order;
``next_rt``, the number of runtime ids ever issued, and ``n_ent``.

* ``append(cols)`` groups the chunk on its own (``trace_chunk_ref.group_traces``), matches its runtimes by key rows
  against the live patterns, and merges it by the append rules: a known runtime keeps its id, representative and graph;
  new runtimes get ``next_rt + j`` in order of their smallest traceid and their patterns go after the live ones in the
  chunk's insertion order; traces follow in the chunk's iteration order; each entry keeps its keys in order, then takes
  the runtimes new to it in order of first appearance.  A runtime whose pattern was evicted is new again.
* ``evict(before)`` drops the traces with bucket < before, the (entry, runtime) keys left without a trace and the
  patterns left without a key, and returns the remap of the old trace positions.
* ``store_dicts(kind)`` gives the constructor's (runtime2graph, entry2runtimes, tr2data), the graphs built from the
  representatives' rows as ``TraceGroups.graphs`` builds them."""
import numpy as np

from tests import trace_chunk_ref as R

KEY_COLS = ("um", "dm", "interface")
REP_COLS = ("um", "dm", "interface", "rpctype", "timestamp", "rpcid", "rt")


class TraceWindow:
    def __init__(self):
        self.patterns, self.by_key, self.entries, self.traces = {}, {}, {}, {}
        self.next_rt = self.n_ent = 0

    def append(self, cols):
        """Takes a chunk (dict of int64 columns, whole traces, traceids new to the state); -> its traces' positions."""
        r = R.group_traces(cols)
        rp, perm = r["row_ptr"], r["perm"]
        c = {k: np.asarray(cols[k], dtype=np.int64)[perm] for k in REP_COLS}
        key_of = lambda t: np.stack([c[k][rp[t]:rp[t + 1]] for k in KEY_COLS], 1).tobytes()   # noqa: E731
        rep = {int(rt): int(t) for rt, t in zip(r["ins_runtime"], r["rep_trace"])}
        gid, new = {}, 0
        for rt in range(len(rep)):                                   # chunk runtime ids: by smallest traceid
            key = key_of(rep[rt])
            if key in self.by_key:
                gid[rt] = self.by_key[key]
            else:
                gid[rt], new = self.next_rt + new, new + 1
        for rt in r["ins_runtime"]:                                  # new patterns in the chunk's insertion order
            g = gid[int(rt)]
            if g >= self.next_rt:
                t = rep[int(rt)]
                key = key_of(t)
                self.patterns[g] = (key, {k: c[k][rp[t]:rp[t + 1]] for k in REP_COLS})
                self.by_key[key] = g
        self.next_rt += new
        T0 = len(self.traces)
        for t in r["order"]:                                         # the chunk's iteration order
            e, g = int(r["entry"][t]), gid[int(r["runtime"][t])]
            self.traces[int(r["trace_id"][t])] = (e, g, int(r["bucket"][t]), int(r["y"][t]))
            mix = self.entries.setdefault(e, {})
            mix[g] = mix.get(g, 0) + 1
            self.n_ent = max(self.n_ent, e + 1)
        return range(T0, len(self.traces))

    def evict(self, before):
        """Drops the traces with bucket < before; -> remap (int64 [T_old]: new position or -1)."""
        keep = np.array([v[2] >= before for v in self.traces.values()], dtype=bool)
        remap = np.where(keep, np.cumsum(keep) - 1, -1).astype(np.int64)
        for tid, kept in zip(list(self.traces), keep):
            if kept:
                continue
            e, g, _, _ = self.traces.pop(tid)
            self.entries[e][g] -= 1
            if self.entries[e][g] == 0:
                del self.entries[e][g]
        alive = {g for mix in self.entries.values() for g in mix}
        for g in [g for g in self.patterns if g not in alive]:
            del self.by_key[self.patterns.pop(g)[0]]
        return remap

    # ---- views -------------------------------------------------------------------------------------------------------
    def entry2runtimes(self):
        """{e: {runtime id: count / total}} for every e < n_ent (fp64 probabilities; {} for an entry without traces)."""
        out = {}
        for e in range(self.n_ent):
            mix = self.entries.get(e, {})
            total = sum(mix.values())
            out[e] = {g: n / total for g, n in mix.items()}
        return out

    def tr2data(self):
        return {tid: {"entry_id": e, "runtime_id": g, "timestamp": np.int64(b), "y": y}
                for tid, (e, g, b, y) in self.traces.items()}

    def pair_counts(self):
        """(cnt [pairs], tot [n_ent]) in the store's pair order (entries ascending, each in key order)."""
        cnt = [n for e in range(self.n_ent) for n in self.entries.get(e, {}).values()]
        tot = [sum(self.entries.get(e, {}).values()) for e in range(self.n_ent)]
        return np.array(cnt, dtype=np.int64), np.array(tot, dtype=np.int64)

    def trace_patterns(self):
        """Pattern index of every trace, trace-table order."""
        index = {g: i for i, g in enumerate(self.patterns)}
        return np.array([index[g] for _, g, _, _ in self.traces.values()], dtype=np.int64)

    def key_rows(self):
        """(rows [3, R'], ptr [n_pat + 1]): the representatives' (um, dm, interface) rows, pattern order."""
        reps = [rows for _, rows in self.patterns.values()]
        ptr = np.concatenate([[0], np.cumsum([len(r["um"]) for r in reps])]).astype(np.int64)
        rows = np.stack([np.concatenate([r[k] for r in reps]) if reps else np.zeros(0, np.int64) for k in KEY_COLS])
        return rows, ptr

    def store_dicts(self, kind, device="cuda"):
        """(runtime2graph, entry2runtimes, tr2data) of the constructor; needs at least one pattern."""
        ids = list(self.patterns)
        reps = [self.patterns[g][1] for g in ids]
        cols = {k: np.concatenate([r[k] for r in reps]) for k in REP_COLS}
        lens = np.array([len(r["um"]) for r in reps], dtype=np.int64)
        res = {"row_ptr": np.concatenate([[0], np.cumsum(lens)]), "perm": np.arange(int(lens.sum())),
               "rep_trace": np.arange(len(ids)), "ins_runtime": np.array(ids, dtype=np.int64)}
        pg, ids = R.rep_graphs(cols, res, kind, device)
        return {g: pg.pattern(k) for k, g in enumerate(ids)}, self.entry2runtimes(), self.tr2data()
