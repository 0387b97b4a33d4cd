"""Plain numpy restatement of the reference's preprocess.py main() after get_df() (:269-381), without the graphs:
what tr2data, entry2runtimes and the key order / occurrences of runtime2{span,pert}graph_map hold for a processed span
table.  The test reference for tracegroup.group_traces on tables too large for the reference's pandas loop.

  (1) traces in ascending traceid, rows of a trace in file order;
  (2) bucket = min(timestamp) // 30000 * 30000 (get_tr2ts_map, :32-41);
  (3) y = max |rt| (:290-292);
  (4) runtime id = Series.factorize of the " ".join of a trace's um_dm_interface strings over ascending traceids
      (:280-293): equal exactly when the (um, dm, interface) sequences are equal;
  (5) iteration order = entries ascending, traceids ascending inside an entry (:295-299); the representative of a
      runtime is the first trace of it in that order, runtimes are inserted into the graph maps in that order, and
      occurrences count all its traces;
  (6) entry2runtimes[e] = {runtime: count / total} in order of first appearance inside the entry (:310-316, :371-375).
"""
import numpy as np

BUCKET = 30000


def group_traces(cols):
    """``cols``: dict of int64 arrays (traceid, timestamp, um, dm, interface, rt, entryid; file order).  -> dict:
    trace_id [T] ascending; entry, runtime, bucket, y [T] in that order; order [T] = trace indices in iteration order;
    occurrences [n_rt] by runtime id; ins_runtime [n_rt] = runtime ids in insertion order; rep_trace [n_rt] =
    representative trace index in insertion order; row_ptr [T+1] / perm [R] = rows grouped by trace;
    entry2runtimes = {entry: {runtime: prob}} with the reference's key order.  Raises ValueError for a trace whose
    rows disagree on entryid."""
    tid = np.asarray(cols["traceid"], dtype=np.int64)
    perm = np.argsort(tid, kind="stable")
    trace_id, first, counts = np.unique(tid[perm], return_index=True, return_counts=True)
    T = trace_id.shape[0]
    row_ptr = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    g = {k: np.asarray(cols[k], dtype=np.int64)[perm] for k in ("timestamp", "um", "dm", "interface", "rt", "entryid")}
    starts = row_ptr[:-1]
    bucket = np.minimum.reduceat(g["timestamp"], starts) // BUCKET * BUCKET
    y = np.maximum.reduceat(np.abs(g["rt"]), starts)
    emin, emax = np.minimum.reduceat(g["entryid"], starts), np.maximum.reduceat(g["entryid"], starts)
    if (emin != emax).any():
        raise ValueError(f"trace {int(trace_id[np.flatnonzero(emin != emax)[0]])} has rows under two entries")
    entry = emin
    triples = np.stack([g["um"], g["dm"], g["interface"]], axis=1)
    ids, runtime = {}, np.empty(T, dtype=np.int64)
    for t in range(T):                                                   # factorize in ascending traceid
        key = triples[row_ptr[t]:row_ptr[t + 1]].tobytes()
        runtime[t] = ids.setdefault(key, len(ids))
    order = np.lexsort((np.arange(T), entry))                            # entries ascending, then traceid
    occurrences = np.bincount(runtime, minlength=len(ids))
    _, first_pos = np.unique(runtime[order], return_index=True)
    ins_pos = np.sort(first_pos)
    rep_trace = order[ins_pos]
    e2r = {}
    for e in np.unique(entry):
        ts = order[entry[order] == e]
        rts = runtime[ts]
        u, fp, cnt = np.unique(rts, return_index=True, return_counts=True)
        k = np.argsort(fp)
        total = int(ts.shape[0])
        e2r[int(e)] = {int(r): int(c) / total for r, c in zip(u[k], cnt[k])}
    return {"trace_id": trace_id, "entry": entry, "runtime": runtime, "bucket": bucket, "y": y, "order": order,
            "occurrences": occurrences, "ins_runtime": runtime[rep_trace], "rep_trace": rep_trace, "row_ptr": row_ptr,
            "perm": perm, "entry2runtimes": e2r}


def tr2data(res):
    """The reference's tr2data dict (:304-309) from ``group_traces``'s result: keys in iteration order."""
    import torch

    out = {}
    for t in res["order"]:
        out[int(res["trace_id"][t])] = {"entry_id": int(res["entry"][t]), "runtime_id": int(res["runtime"][t]),
                                        "timestamp": np.int64(res["bucket"][t]), "y": torch.tensor(int(res["y"][t]))}
    return out
