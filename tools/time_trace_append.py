"""Cost of appending a chunk of traces to a live store: PatternStore.append_traces against regrouping the whole table.

Table: make_random_trace_table with --stores traces (default 10^5 and 10^6) plus one 10^4-trace chunk per repetition,
all drawn from the same pattern law; the store holds the first part, every chunk is a fresh random set of traces, 1 %
of which carry a runtime the store has never seen (the share of the chunk's runtimes that are new is printed).
Arms, alternated, --reps times each:
  * append:  PatternStore.append_traces(chunk) on a store built from the base table (the build is not timed);
  * rebuild: group_traces + PatternStore.from_trace_groups over the base table and the chunk, what a caller runs
             without append_traces.
Both are timed with a host clock around work that ends in a device synchronise.  Inside the append arm the stages are
split out: the chunk's group_traces, the match (pert_ingest_match) and merge (pert_ingest_merge) kernels by CUDA
events around their calls, and the host row filters and graph build of the new representatives by a host clock.
Prints the card name and power limit, then one JSON line per store size: median and [min, max] of every number, in ms.

    python tools/time_trace_append.py [--stores 100000 1000000] [--reps 5]
"""
import argparse
import json
import statistics

import numpy as np
import torch

from measure import Probe, card, host_ms

CHUNK = 10_000


def stats(xs):
    return {"median": round(statistics.median(xs), 3), "range": [round(min(xs), 3), round(max(xs), 3)]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--stores", type=int, nargs="+", default=[100_000, 1_000_000])
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    from pert_gnn_kdd23_b200 import _lib, pertgraph, tracegroup
    from pert_gnn_kdd23_b200.store import PatternStore
    from pert_gnn_kdd23_b200.synthetic import make_random_trace_table

    print("card:", card())
    L = _lib.lib()
    probe = Probe()
    L.pert_ingest_match = probe.cuda("match", L.pert_ingest_match)
    L.pert_ingest_merge = probe.cuda("merge", L.pert_ingest_merge)
    pertgraph.clean_span_tables_flat = probe.clock("host_filters", pertgraph.clean_span_tables_flat)
    pertgraph.build_pert_graphs_flat = probe.clock("graph_build", pertgraph.build_pert_graphs_flat)
    group = tracegroup.group_traces
    res = ([], np.zeros((0, 8)))
    for n in args.stores:
        cols = make_random_trace_table(7, n + (args.reps + 1) * CHUNK, n_patterns=max(2000, n // 50))
        tid = np.unique(cols["traceid"])
        perm = np.random.default_rng(n).permutation(tid.shape[0])
        chunk_of = np.full(int(tid.max()) + 1, -1)
        chunk_of[tid[perm[:n]]] = 0
        for r in range(args.reps + 1):
            chunk_of[tid[perm[n + r * CHUNK:n + (r + 1) * CHUNK]]] = r + 1
        row_chunk = chunk_of[cols["traceid"]]
        # 1 % of every chunk's traces get a runtime no other trace has: their first row's interface is made unique
        fresh = np.isin(cols["traceid"], tid[perm[n:]][::100])
        idx = np.flatnonzero(fresh)
        first = idx[np.unique(cols["traceid"][idx], return_index=True)[1]]
        cols["interface"][first] = 1_000_000 + cols["traceid"][first]
        base = {k: v[row_chunk == 0] for k, v in cols.items()}
        dev_cols = lambda m: {k: torch.from_numpy(v[m]).cuda() for k, v in cols.items()}   # noqa: E731
        rows = {"append": [], "rebuild": []}
        parts, new_share = [], []
        for r in range(args.reps + 1):                   # repetition 0 warms every shape up
            chunk = dev_cols(row_chunk == r + 1)
            whole = dev_cols((row_chunk == 0) | (row_chunk == r + 1))
            for arm in (("append", "rebuild") if r % 2 == 0 else ("rebuild", "append")):
                if arm == "append":
                    s = PatternStore.from_trace_groups(group(base).check(), "span", *res, "cuda", n_ms=4096)
                    s.append_traces(chunk)                  # builds the runtime table: a store's first append
                    s = PatternStore.from_trace_groups(group(base).check(), "span", *res, "cuda", n_ms=4096)
                    s._ingest.insert(0, 64)                 # the table as a store that has appended before has it
                    n_pat = len(s.rt_ids)
                    probe.take()
                    tracegroup.group_traces = probe.clock("group_chunk", group)
                    dt = host_ms(lambda: s.append_traces(chunk))[1]
                    tracegroup.group_traces = group
                    p = probe.take()
                    n_c = group(chunk).n_runtimes
                    if r:
                        rows["append"].append(dt)
                        parts.append(p)
                        new_share.append((len(s.rt_ids) - n_pat) / n_c)
                else:
                    dt = host_ms(lambda: PatternStore.from_trace_groups(group(whole).check(), "span", *res, "cuda",
                                                                        n_ms=4096))[1]
                    if r:
                        rows["rebuild"].append(dt)
                    probe.take()
        out = {"store_traces": n, "chunk_traces": CHUNK, "new_runtime_share": stats(new_share),
               "append_ms": stats(rows["append"]), "rebuild_ms": stats(rows["rebuild"]),
               "speedup_median": round(statistics.median(rows["rebuild"]) / statistics.median(rows["append"]), 2)}
        for k in ("group_chunk", "match", "host_filters", "graph_build", "merge"):
            out[k + "_ms"] = stats([p.get(k, 0.0) for p in parts])
        print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
