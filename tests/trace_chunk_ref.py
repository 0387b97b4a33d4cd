"""Chunk-ordered restatement of the trace grouping (oracle/trace_group_oracle.py) for PatternStore.append_traces.

A store after appends of chunks 1..c holds what the constructor builds from the grouping of the concatenated table in
which the chunk leads every order: traces are ordered by (chunk, traceid) (runtime ids by factorize in that order),
the iteration order is (chunk, entry, traceid), and representatives, insertion order and each entry's key order follow
the iteration order as before.  ``group_traces(cols, chunk)`` is the oracle's function with that optional per-row
chunk column; without it the result is the oracle's.  ``rep_graphs`` builds the representatives' graphs the way
TraceGroups.graphs does, and ``store_dicts`` the constructor's inputs."""
import numpy as np

from oracle import trace_group_oracle as O

BUCKET = O.BUCKET


def group_traces(cols, chunk=None):
    """``cols`` as for ``oracle.trace_group_oracle.group_traces``; ``chunk``: int array, one per row (whole traces per
    chunk).  -> that function's dict (traces in (chunk, traceid) order) plus ``trace_chunk`` [T].  ValueError for a
    trace whose rows disagree on entryid or chunk."""
    tid = np.asarray(cols["traceid"], dtype=np.int64)
    ch = np.zeros_like(tid) if chunk is None else np.asarray(chunk, dtype=np.int64)
    perm = np.lexsort((tid, ch))                                         # stable: file order inside a trace
    st, sc = tid[perm], ch[perm]
    new = np.ones(tid.shape[0], dtype=bool)
    new[1:] = (st[1:] != st[:-1]) | (sc[1:] != sc[:-1])
    starts = np.flatnonzero(new)
    trace_id, trace_chunk = st[starts], sc[starts]
    if np.unique(trace_id).shape[0] != trace_id.shape[0]:
        raise ValueError("a traceid has rows in two chunks")
    T = trace_id.shape[0]
    row_ptr = np.concatenate([starts, [tid.shape[0]]]).astype(np.int64)
    g = {k: np.asarray(cols[k], dtype=np.int64)[perm] for k in ("timestamp", "um", "dm", "interface", "rt", "entryid")}
    bucket = np.minimum.reduceat(g["timestamp"], starts) // BUCKET * BUCKET
    y = np.maximum.reduceat(np.abs(g["rt"]), starts)
    emin, emax = np.minimum.reduceat(g["entryid"], starts), np.maximum.reduceat(g["entryid"], starts)
    if (emin != emax).any():
        raise ValueError(f"trace {int(trace_id[np.flatnonzero(emin != emax)[0]])} has rows under two entries")
    entry = emin
    triples = np.stack([g["um"], g["dm"], g["interface"]], axis=1)
    ids, runtime = {}, np.empty(T, dtype=np.int64)
    for t in range(T):                                                   # factorize in (chunk, traceid) order
        key = triples[row_ptr[t]:row_ptr[t + 1]].tobytes()
        runtime[t] = ids.setdefault(key, len(ids))
    order = np.lexsort((np.arange(T), entry, trace_chunk))              # chunk, entry, traceid
    occurrences = np.bincount(runtime, minlength=len(ids))
    _, first_pos = np.unique(runtime[order], return_index=True)
    rep_trace = order[np.sort(first_pos)]
    e2r = {}
    for e in np.unique(entry):
        ts = order[entry[order] == e]
        rts = runtime[ts]
        u, fp, cnt = np.unique(rts, return_index=True, return_counts=True)
        k = np.argsort(fp)
        total = int(ts.shape[0])
        e2r[int(e)] = {int(r): int(c) / total for r, c in zip(u[k], cnt[k])}
    return {"trace_id": trace_id, "trace_chunk": trace_chunk, "entry": entry, "runtime": runtime, "bucket": bucket,
            "y": y, "order": order, "occurrences": occurrences, "ins_runtime": runtime[rep_trace],
            "rep_trace": rep_trace, "row_ptr": row_ptr, "perm": perm, "entry2runtimes": e2r}


def rep_graphs(cols, res, kind, device="cuda"):
    """-> (PertGraphs, runtime ids): the graphs of the representatives ``res`` names, insertion order, through the
    host row filters and the CUDA builder (TraceGroups.graphs' path)."""
    from pert_gnn_kdd23_b200 import pertgraph

    rp, perm = res["row_ptr"], res["perm"]
    rows = np.concatenate([perm[rp[t]:rp[t + 1]] for t in res["rep_trace"]])
    lens = np.array([rp[t + 1] - rp[t] for t in res["rep_trace"]], dtype=np.int64)
    ptr = np.concatenate([[0], np.cumsum(lens)])
    c = {k: np.asarray(cols[k], dtype=np.int64)[rows] for k in ("um", "dm", "interface", "rpctype", "timestamp",
                                                                   "rpcid", "rt")}
    c["endTimestamp"] = c["timestamp"] + np.abs(c["rt"])
    keep, new_ptr, roots = pertgraph.clean_span_tables_flat(c, ptr)
    flat = np.stack([c[k] for k in pertgraph.COLUMNS])[:, keep]
    g = pertgraph.build_pert_graphs_flat(flat, new_ptr, roots, device, kind).check()
    return g, [int(r) for r in res["ins_runtime"]]


def store_dicts(cols, res, kind, device="cuda"):
    """(runtime2graph, entry2runtimes, tr2data) of the constructor for ``res``."""
    pg, ids = rep_graphs(cols, res, kind, device)
    return {rt: pg.pattern(k) for k, rt in enumerate(ids)}, res["entry2runtimes"], O.tr2data(res)
