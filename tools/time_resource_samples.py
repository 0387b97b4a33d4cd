"""Cost of aggregating raw resource samples into the open buckets' statistics: ResourceSampleWindow.add of one new
bucket against recomputing the statistics of every open sample.

Window: n_ms = 30000 microservices, 1-8 samples per (bucket, ms) key, W open buckets (--open, default 1 and 4); the
timed call adds one new bucket of the same shape (about 1.35e5 samples, as CUDA tensors).  Arms, alternating, --reps
times each after one warm-up round, each from the same window (``add`` swaps in new arrays and leaves the old ones
untouched, so every rep starts from the same state):
  * add:     ResourceSampleWindow.add (including its one device -> host read), CUDA events around the call;
  * rebuild: the resource part of process_raw over every open sample plus the new bucket, on device-resident columns:
             the stable (timestamp, ms) sort, pert_raw_resource_groups, the read of the group count, the per-group
             value sorts and pert_raw_resource_stats; CUDA events around it;
  * pandas:  groupby(["timestamp", "msname"]).agg(["max", "min", "mean", "median"]) over the same samples on the host,
             a wall clock around it.
Every timed add is checked bit for bit (NaN-aware) against the rebuild's rows of the keys it touched.  `merge_ms` is
the time of the window's merge kernels (k_win_keys, k_win_fold, k_win_runs; torch.profiler, one add in a run of its
own) and `merge_bw` the bytes they must move -- the old window read (8 B key, 4 B offset and 80 B fold state per key,
16 B per sample), the new one written, the batch's sorted values and fold inputs read (40 B per sample) -- over that
time, as a fraction of the H100 SXM data-sheet 3.35 TB/s; the same profile gives every window kernel's time (merge,
scans, flags, emit), the torch sorts' and all device time of the add (the rest of ``add_ms`` is host work and the two
device -> host reads).  Prints the card name, power limit and SM clocks read in
the same run, then one JSON line per window size (with --json, also into that file).

    python tools/time_resource_samples.py [--open 1 4] [--reps 5] [--json results.json]
"""
import argparse
import copy
import json
import statistics
import time

import numpy as np
import torch

from measure import HBM_BYTES_PER_S, card, timed

B, N_MS = 30000, 30000


def bucket(rng, b):
    cnt = rng.integers(1, 9, N_MS)
    ts = np.full(int(cnt.sum()), b * B, dtype=np.int64)
    ms = np.repeat(np.arange(N_MS), cnt)
    perm = rng.permutation(ts.size)
    cpu, mem = rng.random(ts.size), rng.random(ts.size)
    cpu[rng.random(ts.size) < 0.02] = np.nan
    return ts, ms[perm], cpu, mem


def rebuild(ts, ms, cpu, mem):
    """process_raw's resource statistics of device columns -> (keys [G], values [G, 8])."""
    from pert_gnn_kdd23_b200 import _lib

    L, st, dev = _lib.lib(), _lib.stream(), ts.device
    K = int(ts.shape[0])
    p1 = torch.sort(ms, stable=True).indices
    perm = p1[torch.sort(ts[p1], stable=True).indices].contiguous()
    i32, i64 = dict(dtype=torch.int32, device=dev), dict(dtype=torch.int64, device=dev)
    gflag, gptr, has_res = torch.empty(K + 1, **i32), torch.empty(K + 1, **i32), torch.empty(N_MS, **i32)
    g_ts, g_ms, ng, status = torch.empty(K, **i64), torch.empty(K, **i64), torch.empty(1, **i64), torch.zeros(1, **i32)
    ws = torch.empty(int(L.pert_raw_resource_workspace_bytes(K)), dtype=torch.uint8, device=dev)
    _lib.check(L.pert_raw_resource_groups(K, ts.data_ptr(), ms.data_ptr(), perm.data_ptr(), N_MS, gflag.data_ptr(),
                                          has_res.data_ptr(), gptr.data_ptr(), g_ts.data_ptr(), g_ms.data_ptr(),
                                          ng.data_ptr(), ws.data_ptr(), ws.numel(), status.data_ptr(), st), "groups")
    G = int(ng.item())
    gid = gflag[1:] - 1
    srt = []
    for u in (cpu, mem):
        s = torch.sort(u[perm], stable=True)
        srt.append(s.values[torch.sort(gid[s.indices], stable=True).indices].contiguous())
    vals = torch.empty(G, 8, dtype=torch.float64, device=dev)
    _lib.check(L.pert_raw_resource_stats(G, perm.data_ptr(), gptr.data_ptr(), cpu.data_ptr(), mem.data_ptr(),
                                         srt[0].data_ptr(), srt[1].data_ptr(), vals.data_ptr(), st), "stats")
    return g_ts[:G] * N_MS + g_ms[:G], vals


def pandas_stats(ts, ms, cpu, mem):
    import pandas as pd

    df = pd.DataFrame({"timestamp": ts, "msname": ms, "instance_cpu_usage": cpu, "instance_memory_usage": mem})
    return df.groupby(["timestamp", "msname"]).agg(["max", "min", "mean", "median"])


def same_bits(a, b):
    return torch.equal(torch.isnan(a), torch.isnan(b)) and torch.equal(a.nan_to_num(7).view(torch.int64),
                                                                       b.nan_to_num(7).view(torch.int64))


def merge_kernel_ms(win, batch):
    from torch.profiler import ProfilerActivity, profile

    w = copy.copy(win)
    w.t = dict(win.t)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        w.add(*batch)
        torch.cuda.synchronize()
    ev = prof.key_averages()
    merge = sum(e.device_time_total for e in ev if any(k in e.key for k in ("k_win_keys", "k_win_fold", "k_win_runs")))
    window = sum(e.device_time_total for e in ev if "k_win_" in e.key or "k_scan_" in e.key)
    sorts = sum(e.device_time_total for e in ev if "sort" in e.key.lower() or "radix" in e.key.lower())
    return merge / 1e3, window / 1e3, sorts / 1e3, sum(e.device_time_total for e in ev) / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--open", type=int, nargs="+", default=[1, 4])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--json", help="also write the card and every result to this file")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    from pert_gnn_kdd23_b200.rawtable import ResourceSampleWindow

    print(f"card: {card(sm_clock=True)}", flush=True)
    results = []
    for W in a.open:
        rng = np.random.default_rng(W)
        win = ResourceSampleWindow(N_MS, "cuda")
        host = [bucket(rng, b) for b in range(W)]
        for h in host:
            win.add(*(torch.from_numpy(c).cuda() for c in h))
        new = bucket(rng, W)
        allh = [np.concatenate([h[j] for h in host] + [new[j]]) for j in range(4)]
        alld = [torch.from_numpy(c).cuda() for c in allh]
        batch = [torch.from_numpy(c).cuda() for c in new]
        U, S, k = win.n_keys, win.n_samples, int(new[0].size)

        def do_add():
            w = copy.copy(win)
            w.t = dict(win.t)
            return w.add(*batch)

        times = {"add": [], "rebuild": [], "pandas": []}
        for rep in range(a.reps + 1):
            rows, t_add = timed(do_add)
            (keys, vals), t_reb = timed(lambda: rebuild(*alld))
            t0 = time.perf_counter()
            pandas_stats(*allh)
            t_pd = (time.perf_counter() - t0) * 1e3
            got_keys = rows.index[:, 0] * N_MS + rows.index[:, 1]
            pos = torch.searchsorted(keys, got_keys)
            assert torch.equal(keys[pos], got_keys) and same_bits(rows.values, vals[pos]), "add != rebuild"
            if rep:                                       # rep 0 is the warm-up
                for name, t in (("add", t_add), ("rebuild", t_reb), ("pandas", t_pd)):
                    times[name].append(t)
        med = {n: statistics.median(v) for n, v in times.items()}
        U2, S2 = U + N_MS, S + k                          # the new bucket's keys are all new
        merge_ms, window_ms, sort_ms, device_ms = merge_kernel_ms(win, batch)
        nbytes = 92 * (U + U2) + 16 * (S + S2) + 40 * k
        r = {"open_buckets": W, "open_keys": U, "open_samples": S, "new_samples": k,
             "add_ms": round(med["add"], 3), "rebuild_ms": round(med["rebuild"], 3), "pandas_ms": round(med["pandas"], 1),
             "add_vs_rebuild": round(med["rebuild"] / med["add"], 2), "merge_ms": round(merge_ms, 4),
             "window_kernels_ms": round(window_ms, 4), "sort_kernels_ms": round(sort_ms, 4),
             "add_device_ms": round(device_ms, 4), "merge_bytes": nbytes,
             "merge_bw": round(nbytes / (merge_ms * 1e-3) / HBM_BYTES_PER_S, 3) if merge_ms else None,
             "reps": a.reps, "all_ms": {n: [round(x, 3) for x in v] for n, v in times.items()}}
        results.append(r)
        print(json.dumps(r), flush=True)
    if a.json:
        with open(a.json, "w") as f:
            json.dump({"card": card(sm_clock=True), "results": results}, f, indent=1)


if __name__ == "__main__":
    main()
