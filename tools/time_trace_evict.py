"""Cost of evicting the oldest bucket of traces from a live store: PatternStore.evict_traces against regrouping the
surviving traces and rebuilding the store, and a steady-state window loop.

Table: make_random_trace_table with --stores traces (default 10^5 and 10^6) over 10 buckets of 30 s, the workload of
tools/time_trace_append.py.  Arms, alternated, --reps times each after a warm-up repetition:
  * evict:   PatternStore.evict_traces(30000) on a store built from the table (the build is not timed);
  * rebuild: group_traces + PatternStore.from_trace_groups over the traces with bucket >= 30000, what a caller runs
             without evict_traces.
Both are timed with a host clock around work that ends in a device synchronise.  Inside the evict arm the count
(pert_ingest_evict_count) and apply (pert_ingest_evict_apply) kernels are timed by CUDA events around their calls;
the rest of the call is the size read, the read of the host copies and the host glue, of which the rebuild of
``trace_keys`` (a Python list, filtered with ``itertools.compress``) is timed on its own, beside what a list of the
surviving device traceids would cost (``tolist``).  The apply kernels' bytes
(every array they read and write, from the sizes) over their time are reported as a share of 3.35 TB/s.
Window loop (--loop-steps): append a 10^4-trace chunk of the next bucket, then evict the oldest bucket.
Prints the card name and power limit, then one JSON line per store size: median and [min, max] of every number, in ms.

    python tools/time_trace_evict.py [--stores 100000 1000000] [--reps 5] [--loop-steps 6]
"""
import argparse
import itertools
import json
import statistics
import time

import numpy as np
import torch

from measure import HBM_BYTES_PER_S, Probe, card, host_ms

BUCKET = 30000
CHUNK = 10_000


def stats(xs):
    return {"median": round(statistics.median(xs), 3), "range": [round(min(xs), 3), round(max(xs), 3)]}


def apply_bytes(old, new, attr_cols):
    """Bytes pert_ingest_evict_apply reads and writes: every old item's flags and fields, every kept item's output.
    old / new: (traces, pairs, patterns, nodes, edges, key rows)."""
    T, P, n_pat, N, E, K = old
    T2, P2, n_pat2, N2, E2, K2 = new
    trace = T * (8 + 4 + 8 + 8 + 4 + 8 + 4 + 8) + T2 * (4 + 8 + 8 + 4 + 8)      # flags, 5 fields, pattern map, remap
    pair = P * (8 + 4 + 4 + 4 + 4) + P2 * (4 + 4 + 4 + 4)                         # flags, cnt, ev, ent_pat, map, total
    pat = n_pat * (8 + 4 * 3) + n_pat * 4 + (n_pat2 + 1) * 12
    node = N * (8 + 8 + 8 + 1) + N2 * (8 + 8 + 1)                                # owner pattern flags, ms, depth, last
    edge = E * (8 + 8 + 8 * attr_cols) + E2 * (8 + 8 * attr_cols)
    key = K * (8 + 24) + K2 * 24
    return trace + pair + pat + node + edge + key


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--stores", type=int, nargs="+", default=[100_000, 1_000_000])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--loop-steps", type=int, default=6)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    from pert_gnn_kdd23_b200 import _lib, tracegroup
    from pert_gnn_kdd23_b200.store import PatternStore
    from pert_gnn_kdd23_b200.synthetic import make_random_trace_table

    print("card:", card())
    L = _lib.lib()
    probe = Probe()
    L.pert_ingest_evict_count = probe.cuda("count", L.pert_ingest_evict_count)
    L.pert_ingest_evict_apply = probe.cuda("apply", L.pert_ingest_evict_apply)
    group = tracegroup.group_traces
    res = ([], np.zeros((0, 8)))
    for n in args.stores:
        n_loop = args.loop_steps * CHUNK
        cols = make_random_trace_table(7, n + n_loop, n_patterns=max(2000, n // 50))
        tid, inv = np.unique(cols["traceid"], return_inverse=True)
        is_loop = np.zeros(tid.shape[0], dtype=bool)
        is_loop[np.random.default_rng(n).permutation(tid.shape[0])[:n_loop]] = True
        row_loop = is_loop[inv]
        t_min = np.full(tid.shape[0], np.iinfo(np.int64).max)
        np.minimum.at(t_min, inv, cols["timestamp"])
        t_bucket = t_min // BUCKET * BUCKET
        dev_cols = lambda m: {k: torch.from_numpy(v[m]).cuda() for k, v in cols.items()}   # noqa: E731
        base = dev_cols(~row_loop)
        survivors = dev_cols(~row_loop & (t_bucket[inv] >= BUCKET))
        build = lambda c: PatternStore.from_trace_groups(group(c).check(), "span", *res, "cuda", n_ms=4096)  # noqa
        rows = {"evict": [], "rebuild": []}
        parts, bw, evicted = [], [], []
        for r in range(args.reps + 1):                   # repetition 0 warms every shape up
            for arm in (("evict", "rebuild") if r % 2 == 0 else ("rebuild", "evict")):
                if arm == "evict":
                    s = build(base)
                    old = (len(s), int(s._ingest.cnt.shape[0]), len(s.rt_ids), s._ingest.n_nodes, s._ingest.n_edges,
                           int(s._ingest.rows.shape[1]))
                    keys = list(s.trace_keys)
                    probe.take()
                    remap, dt = host_ms(lambda: s.evict_traces(BUCKET))
                    p = probe.take()
                    new = (len(s), int(s._ingest.cnt.shape[0]), len(s.rt_ids), s._ingest.n_nodes, s._ingest.n_edges,
                           int(s._ingest.rows.shape[1]))
                    t1 = time.perf_counter()         # the trace_keys rebuild evict_traces does, on its own
                    list(itertools.compress(keys, (remap >= 0).view(np.uint8).tobytes()))
                    p["trace_keys"] = (time.perf_counter() - t1) * 1e3
                    t1 = time.perf_counter()         # what a list of the device traceids would cost instead
                    s._ingest.trace_tid.cpu().numpy().tolist()
                    p["traceid_tolist"] = (time.perf_counter() - t1) * 1e3
                    if r:
                        rows["evict"].append(dt)
                        parts.append(p)
                        bw.append(apply_bytes(old, new, s.attr_cols) / (p["apply"] * 1e-3) / HBM_BYTES_PER_S)
                        evicted.append(int((remap < 0).sum()))
                    del s
                else:
                    dt = host_ms(lambda: build(survivors))[1]
                    if r:
                        rows["rebuild"].append(dt)
                    probe.take()
        out = {"store_traces": n, "evicted_traces": stats(evicted), "evict_ms": stats(rows["evict"]),
               "rebuild_ms": stats(rows["rebuild"]),
               "speedup_median": round(statistics.median(rows["rebuild"]) / statistics.median(rows["evict"]), 2)}
        for k in ("count", "apply", "trace_keys", "traceid_tolist"):
            out[k + "_ms"] = stats([p[k] for p in parts])
        out["rest_of_call_ms"] = stats([d - p["count"] - p["apply"] for d, p in zip(rows["evict"], parts)])
        out["apply_share_of_hbm"] = stats(bw)
        # ---- window loop: append a chunk of the next bucket, evict the oldest bucket
        s = build(base)
        loop_tid = tid[is_loop]
        step_ms = []
        for k in range(args.loop_steps):
            sel = np.isin(cols["traceid"], loop_tid[k * CHUNK:(k + 1) * CHUNK])
            host = {c: v[sel].copy() for c, v in cols.items()}
            host["timestamp"] += 300000 + k * BUCKET - t_min[inv[sel]]       # every chunk trace in the next bucket
            chunk = {c: torch.from_numpy(v).cuda() for c, v in host.items()}
            dt = host_ms(lambda: (s.append_traces(chunk), s.evict_traces((k + 1) * BUCKET)))[1]
            if k:                                        # step 0 builds the runtime table
                step_ms.append(dt)
        probe.take()
        out["loop_store_traces_end"] = len(s)
        out["loop_step_ms"] = stats(step_ms)
        print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
