"""Time the trace grouping (tracegroup.group_traces) and the whole table -> pattern store path on a seeded processed
span table (synthetic.make_random_trace_table), with CUDA events after warm-up.  Prints one JSON line.

  python tools/time_trace_groups.py --traces 1000000 --rows 20 40 --iters 5

Stages: "group" = group_traces (upload of the nine columns excluded: they start on the device), "graphs" = the
representatives' rows -> host row filters -> CUDA graph build (TraceGroups.graphs), "store" =
PatternStore.from_trace_groups (includes its own graph build).  Every stage ends in a device read, so event times are
wall times of the stage.  Algorithmic bytes of "group" (the least HBM traffic of the method, counted from R rows and T
traces; int64 columns, int32 indices):
  rows:   traceid read 3x (range, count, fill)                            24 B
          slot write + read, perm write (group by traceid)                12 B
          perm + timestamp, rt, entryid, um, dm, interface (reductions)   52 B
          perm + um, dm, interface of the trace and of its runtime's
          first member (row-by-row comparison)                           2 x 28 B
  traces: ~30 int32 / int64 words per trace across the tables and outputs 160 B
and the share of the 3.35 TB/s HBM3 data-sheet bandwidth of the H100 SXM they imply.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

PEAK_BYTES_S = 3.35e12
ROW_BYTES = 24 + 12 + 52 + 2 * 28
TRACE_BYTES = 160


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        name, power = (s.strip() for s in q.stdout.strip().split(","))
    except Exception as e:                                    # the card name still comes from the runtime
        name, power = torch.cuda.get_device_name(), f"unknown ({type(e).__name__})"
    return name, power


def timed(fn, iters):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2 * iters)]
    out = None
    for i in range(iters):
        ev[2 * i].record()
        out = fn()
        ev[2 * i + 1].record()
    torch.cuda.synchronize()
    ms = [ev[2 * i].elapsed_time(ev[2 * i + 1]) for i in range(iters)]
    return out, float(np.median(ms)), ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--traces", type=int, default=1_000_000)
    ap.add_argument("--rows", type=int, nargs=2, default=(20, 40))
    ap.add_argument("--patterns", type=int, default=20000)
    ap.add_argument("--entries", type=int, default=64)
    ap.add_argument("--kind", default="span", choices=("span", "pert"))
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--seed", type=int, default=1)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_trace_groups needs a CUDA device")
    from pert_gnn_kdd23_b200.store import PatternStore
    from pert_gnn_kdd23_b200.tracegroup import group_traces

    t0 = time.perf_counter()
    host = make(a)
    gen_s = time.perf_counter() - t0
    cols = {k: torch.from_numpy(v).cuda() for k, v in host.items()}
    R = int(cols["traceid"].shape[0])
    buckets = np.unique(host["timestamp"] // 30000 * 30000)
    res_index = [(int(b), ms) for b in buckets for ms in range(64)]
    res_vals = np.random.default_rng(a.seed).random((len(res_index), 8))
    for _ in range(a.warmup):
        g = group_traces(cols).check()
        PatternStore.from_trace_groups(g, a.kind, res_index, res_vals, "cuda")
    torch.cuda.synchronize()
    g, group_ms, group_all = timed(lambda: group_traces(cols).check(), a.iters)
    _, graphs_ms, _ = timed(lambda: g.graphs(a.kind), a.iters)
    store, store_ms, _ = timed(lambda: PatternStore.from_trace_groups(g, a.kind, res_index, res_vals, "cuda"),
                               a.iters)
    T, n_rt = len(g), g.n_runtimes
    R2 = int(g.rep_ptr[-1])
    name, power = card()
    alg = ROW_BYTES * R + TRACE_BYTES * T
    print(json.dumps({
        "card": name, "power_limit": power, "rows": R, "traces": T, "runtimes": n_rt, "rep_rows": R2,
        "entries": int(g.ent_trace_ptr.shape[0]) - 1, "kind": a.kind,
        "group_ms": round(group_ms, 3), "group_ms_all": [round(x, 3) for x in group_all],
        "graphs_ms": round(graphs_ms, 3), "store_ms": round(store_ms, 3),
        "table_to_store_ms": round(group_ms + store_ms, 3),
        "group_rows_per_s": R / (group_ms * 1e-3), "table_to_store_rows_per_s": R / ((group_ms + store_ms) * 1e-3),
        "group_alg_bytes": alg, "group_alg_GBps": alg / (group_ms * 1e-3) / 1e9,
        "group_share_of_3.35TBps": alg / (group_ms * 1e-3) / PEAK_BYTES_S,
        "store_traces": len(store), "generate_s_cpu": round(gen_s, 1),
    }))


def make(a):
    from pert_gnn_kdd23_b200.synthetic import make_random_trace_table

    return make_random_trace_table(a.seed, a.traces, rows=tuple(a.rows), n_patterns=a.patterns, n_entries=a.entries)


if __name__ == "__main__":
    main()
