"""Trace grouping on the GPU: processed span table -> runtime patterns, entry pattern mixes, trace labels.

The body of the reference's preprocess.py main() after get_df() (:269-381) -- which traces share a runtime pattern,
each entry's pattern probabilities, each trace's label and timestamp bucket, and the representative trace whose rows
become the pattern's graph -- computed over the whole table at once by csrc/tracegroup.cu.  ``TraceGroups`` keeps the
results on the device; its converters return the reference's artefacts (``tr2data``, ``entry2runtimes`` and, through
pertgraph, the graphs of ``runtime2{span,pert}graph_map``) and ``PatternStore.from_trace_groups`` builds the store
straight from the device arrays.  There is no CPU fallback: without the CUDA library the calls raise.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib
from . import pertgraph

COLUMNS = ("traceid", "timestamp", "rpcid", "um", "dm", "interface", "rpctype", "rt", "entryid")
GATHERED = pertgraph.COLUMNS + ("rpcid", "rt")          # row order of pert_trace_group_gather's output

P = C.c_void_p


class _SpanTable(C.Structure):
    _fields_ = [("R", C.c_longlong)] + [(k, P) for k in COLUMNS]


class _Groups(C.Structure):
    _fields_ = [(k, P) for k in ("row_ptr", "perm", "trace_id", "bucket", "y", "entry", "runtime", "order",
                                 "ent_trace_ptr", "ent_pair_ptr", "pair_runtime", "pair_prob", "occurrences",
                                 "ins_runtime", "rep_trace", "runtime_ins", "rep_ptr", "sizes")]


class TraceGroups:
    """Device tensors of a grouped span table.  Traces t = 0..T-1 in ascending traceid:
      trace_id, bucket, y [T] int64; entry, runtime [T] int32; row_ptr [T+1] / perm [R] int32 (rows of trace t, file
      order); order [T] int32 = trace at iteration position p (entries ascending, traceids ascending: tr2data's key
      order).
    Runtimes (ids 0.. in order of their smallest traceid): occurrences [n_rt]; ins_runtime [n_rt] = runtime ids in the
      order the reference inserts them into runtime2*graph_map; rep_trace [n_rt] = their representative traces;
      runtime_ins [n_rt] = insertion index of every runtime id.
    Entries 0..n_ent-1: ent_trace_ptr [n_ent+1] into ``order``; ent_pair_ptr [n_ent+1] into pair_runtime / pair_prob
      [n_pairs] (entry2runtimes[e] in key order, fp64)."""

    def __init__(self, table, t, status):
        self._table, self.status = table, status          # table: the device columns (kept for graphs())
        for k, v in t.items():
            setattr(self, k, v)

    def __len__(self):
        return int(self.trace_id.shape[0])

    @property
    def n_runtimes(self):
        return int(self.ins_runtime.shape[0])

    def check(self):
        """Synchronising check of the status word: a traceid or entryid outside [0, 2^31), or a trace whose rows
        disagree on entryid, raises PertGnnError."""
        code = int(self.status.item())
        if code != 0:
            _lib.check(code, "trace grouping (traceid / entryid out of [0, 2^31) or a trace under two entries)")
        return self

    def tr2data(self):
        """preprocess.py:304-309: {traceid: {entry_id, runtime_id, timestamp (np.int64), y (0-dim int64 tensor)}} in
        the reference's key order."""
        o = self.order.long()
        tid, ent, rt, ts, y = (a.cpu().numpy() for a in (self.trace_id[o], self.entry[o], self.runtime[o],
                                                          self.bucket[o], self.y[o]))
        return {int(k): {"entry_id": int(e), "runtime_id": int(r), "timestamp": np.int64(s), "y": torch.tensor(int(v))}
                for k, e, r, s, v in zip(tid, ent, rt, ts, y)}

    def entry2runtimes(self):
        """preprocess.py:310-316, :371-375: {entry: {runtime_id: count / total}}, entries ascending (entries without
        traces left out), runtimes in the reference's key order, float64 probabilities."""
        ptr, rt, pr = (a.cpu().numpy() for a in (self.ent_pair_ptr, self.pair_runtime, self.pair_prob))
        return {e: {int(r): float(p) for r, p in zip(rt[ptr[e]:ptr[e + 1]], pr[ptr[e]:ptr[e + 1]])}
                for e in range(len(ptr) - 1) if ptr[e + 1] > ptr[e]}

    def occurrences_by_insertion(self):
        """``occurences`` of runtime2*graph_map (:336, :342) in insertion order."""
        return self.occurrences[self.ins_runtime.long()]

    def representative_rows(self):
        """(host int64 [8, R'] rows of GATHERED, rep_ptr [n_rt+1]): the representatives' rows in insertion order, file
        order inside each -- the only rows that cross to the host."""
        return self._rows.cpu().numpy(), self.rep_ptr.cpu().numpy().astype(np.int64)

    def graphs(self, kind="pert"):
        """-> (PertGraphs, runtime_ids): the graphs of runtime2{kind}graph_map in insertion order, built from the
        representatives' rows by the host row filters (pertgraph.clean_span_tables_flat, misc.py:87-105, :138-142) and
        the CUDA graph builder.  A representative whose rows are all removed by the filters raises PertGnnError (the
        reference fails on edge_index.max() of an empty tensor)."""
        rows, rep_ptr = self.representative_rows()
        cols = dict(zip(GATHERED, rows))
        keep, new_ptr, roots = pertgraph.clean_span_tables_flat(cols, rep_ptr)
        ids = self.ins_runtime.cpu().numpy().astype(np.int64)
        empty = np.flatnonzero(np.diff(new_ptr) == 0)
        if empty.size:
            raise _lib.PertGnnError(f"runtime {int(ids[empty[0]])}: the row filters (misc.py:87-105) leave its "
                                    "representative trace without rows")
        flat = rows[:len(pertgraph.COLUMNS)][:, keep]
        g = pertgraph.build_pert_graphs_flat(flat, new_ptr, roots, self.trace_id.device, kind).check()
        return g, [int(r) for r in ids]


def _column(v, dev):
    t = v if torch.is_tensor(v) else torch.from_numpy(np.ascontiguousarray(v, dtype=np.int64))
    t = t.to(device=dev, dtype=torch.int64).contiguous()
    return t.reshape(-1)


def group_traces(columns, device="cuda", hash_bits=64):
    """``columns``: dict of the nine COLUMNS (int64 arrays or CUDA tensors, one row per span, file order) -> TraceGroups.
    ``hash_bits`` narrows the runtime hash (1..64); only tests lower it, to force collisions.
    Host synchronisations: (1) the largest traceid and entryid (sizes the per-traceid count array and the entry
    tables), (2) the number of traces T, (3) the numbers of runtimes, (entry, runtime) pairs and representative rows
    R' -- each a read of a few integers that sizes the next outputs.  Errors found on the device go to the status word
    (``check()``): call it before trusting the result."""
    dev = torch.device(device)
    if dev.type != "cuda":
        raise _lib.PertGnnError("group_traces needs a CUDA device (no CPU fallback)")
    with torch.cuda.device(dev):
        cols = {k: _column(columns[k], dev) for k in COLUMNS}
        R = int(cols["traceid"].shape[0])
        if R == 0:
            raise _lib.PertGnnError("group_traces: the span table is empty")
        if any(int(c.shape[0]) != R for c in cols.values()):
            raise ValueError("group_traces: columns of different lengths")
        tab = _SpanTable(R, *(cols[k].data_ptr() for k in COLUMNS))
        st = _lib.stream()
        L = _lib.lib()
        i32 = dict(dtype=torch.int32, device=dev)
        status = torch.zeros(1, **i32)
        maxes = torch.empty(2, **i32)
        _lib.check(L.pert_trace_group_range(C.byref(tab), maxes.data_ptr(), status.data_ptr(), st),
                   "pert_trace_group_range")
        max_tid, max_ent = (int(v) for v in maxes.cpu())                            # sync 1
        if max_tid < 0 or max_ent < 0:
            _lib.check(int(status.item()), "trace grouping (no row with a traceid and entryid in [0, 2^31))")
            raise _lib.PertGnnError("group_traces: no valid row")
        n_keys, n_ent = max_tid + 1, max_ent + 1
        ws = torch.empty(int(L.pert_trace_group_workspace_bytes(R, n_keys, -1, 0)), dtype=torch.uint8, device=dev)
        key_ptr, key_trace = torch.empty(n_keys + 1, **i32), torch.empty(n_keys + 1, **i32)
        _lib.check(L.pert_trace_group_keys(C.byref(tab), n_keys, key_ptr.data_ptr(), key_trace.data_ptr(),
                                           ws.data_ptr(), ws.numel(), st), "pert_trace_group_keys")
        T = int(key_trace[n_keys].item())                                          # sync 2
        nbytes = int(L.pert_trace_group_workspace_bytes(R, n_keys, T, n_ent))
        if nbytes < 0:
            raise _lib.PertGnnError(f"group_traces: {n_ent} entries x {T} traces exceed the entry sort's table")
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        i64, f64 = dict(dtype=torch.int64, device=dev), dict(dtype=torch.float64, device=dev)
        t = {"row_ptr": torch.empty(T + 1, **i32), "perm": torch.empty(R, **i32), "trace_id": torch.empty(T, **i64),
             "bucket": torch.empty(T, **i64), "y": torch.empty(T, **i64), "entry": torch.empty(T, **i32),
             "runtime": torch.empty(T, **i32), "order": torch.empty(T, **i32),
             "ent_trace_ptr": torch.empty(n_ent + 1, **i32), "ent_pair_ptr": torch.empty(n_ent + 1, **i32),
             "pair_runtime": torch.empty(T, **i32), "pair_prob": torch.empty(T, **f64),
             "occurrences": torch.empty(T, **i32), "ins_runtime": torch.empty(T, **i32),
             "rep_trace": torch.empty(T, **i32), "runtime_ins": torch.empty(T, **i32),
             "rep_ptr": torch.empty(T + 1, **i32), "sizes": torch.empty(3, **i64)}
        out = _Groups(*(t[k].data_ptr() for k, _ in _Groups._fields_))
        _lib.check(L.pert_trace_group_build(C.byref(tab), n_keys, T, n_ent, int(hash_bits), key_ptr.data_ptr(),
                                            key_trace.data_ptr(), C.byref(out), ws.data_ptr(), ws.numel(),
                                            status.data_ptr(), st), "pert_trace_group_build")
        n_rt, n_pairs, R2 = (int(v) for v in t.pop("sizes").cpu())                 # sync 3
        for k in ("occurrences", "ins_runtime", "rep_trace", "runtime_ins"):
            t[k] = t[k][:n_rt]
        for k in ("pair_runtime", "pair_prob"):
            t[k] = t[k][:n_pairs]
        t["rep_ptr"] = t["rep_ptr"][:n_rt + 1]
        rows = torch.empty(len(GATHERED), R2, **i64)
        _lib.check(L.pert_trace_group_gather(C.byref(tab), t["perm"].data_ptr(), t["row_ptr"].data_ptr(),
                                             t["rep_trace"].data_ptr(), t["rep_ptr"].data_ptr(), n_rt, R2,
                                             rows.data_ptr(), st), "pert_trace_group_gather")
        t["_rows"] = rows
    return TraceGroups(cols, t, status)
