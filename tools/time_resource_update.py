"""Cost of one resource update of a live store: PatternStore.append_resources against rebuilding the resource state.

Table: n_ms = 30000 microservices, one row per microservice and 30 s bucket, --rows rows in all (default 10^6 and
10^7: 33 and 333 buckets); every update brings k = 30000 rows (one bucket).  Workloads:
  * in_order: the next bucket, rows in random order;
  * late:     the same with a random 10 % of the rows moved into older buckets;
  * evict:    the next bucket plus the eviction of the oldest one, in one call.
Arms:
  * append:  PatternStore.append_resources (batch sort, count, one size read, merge);
  * rebuild: the device rebuild a caller would otherwise run -- torch.sort(stable) of all surviving keys, a gather of
             the values, ms_has_res by bincount and store.asof_index;
  * host:    (10^6 rows only) the host constructor PatternStore(...) on the list of surviving rows, what a new store
             costs.
Every arm starts from the same table (restored outside the timed window), after warm-up; the arms alternate, --reps
times each, timed with CUDA events (the host arm with a host clock around a synchronised call).  `merge` is the kernel
time of pert_store_resources_merge alone (CUDA events around repeated calls on the same inputs), and `merge_bw` the
bytes it must move -- old plus new rows, 40 B each in the table and 12 B in the index, read and written -- over that
time, as a fraction of the H100 SXM data-sheet 3.35 TB/s.  Also checks once per workload that the append equals the
device rebuild bit for bit.  Prints the card name and power limit, then one JSON line per (rows, workload).

    python tools/time_resource_update.py [--rows 1000000 10000000] [--reps 5]
"""
import argparse
import ctypes as C
import json
import statistics

import numpy as np
import torch

from measure import HBM_BYTES_PER_S, card, host_ms, timed

B, N_MS, K = 30000, 30000, 30000


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, nargs="+", default=[1_000_000, 10_000_000])
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    from pert_gnn_kdd23_b200 import _lib
    from pert_gnn_kdd23_b200.store import PatternStore, asof_index
    from pert_gnn_kdd23_b200.synthetic import make_trace_artifacts

    print(f"card: {card()}", flush=True)
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(0)
    art = make_trace_artifacts(7)
    art.update(resource_index=[], resource_values=np.zeros((0, 8)), n_ms=N_MS)
    for rows in a.rows:
        n_b = rows // N_MS
        store = PatternStore.from_artifacts(art, dev)
        order = torch.randperm(n_b * N_MS, device=dev, generator=g)
        store.append_resources(torch.stack([(order // N_MS) * B, order % N_MS], 1),
                               torch.rand(n_b * N_MS, 8, device=dev, generator=g))
        base = {k: store.t[k].clone() for k in ("res_keys", "res_vals", "ms_has_res")}
        base_asof = {k: v.clone() for k, v in store.asof_t.items()}
        n = store.desc.n_res

        def restore():
            for k, v in base.items():
                store.t[k] = v.clone()
                setattr(store.desc, k, store.t[k].data_ptr())
            store.desc.n_res = n
            store._set_asof(*(base_asof[k].clone() for k in ("ms_ptr", "ts", "row")))

        for workload in ("in_order", "late", "evict"):
            ms1 = torch.randperm(N_MS, device=dev, generator=g)
            ts1 = torch.full((K,), n_b * B, dtype=torch.int64, device=dev)
            if workload == "late":
                late = torch.rand(K, device=dev, generator=g) < 0.1
                ts1 = torch.where(late, torch.randint(0, n_b, (K,), device=dev, generator=g) * B, ts1)
            idx1, v1 = torch.stack([ts1, ms1], 1), torch.rand(K, 8, device=dev, generator=g)
            cut = B if workload == "evict" else None

            def append():
                store.append_resources(idx1, v1, evict_before=cut)

            def rebuild():
                keys = torch.cat([base["res_keys"], ts1 * N_MS + ms1])
                vals = torch.cat([base["res_vals"], v1])
                if cut is not None:
                    keep = keys >= cut * N_MS
                    keys, vals = keys[keep], vals[keep]
                sk, perm = torch.sort(keys, stable=True)
                return sk, vals[perm], (torch.bincount(sk % N_MS, minlength=N_MS) > 0).to(torch.uint8), \
                    asof_index(sk, N_MS)

            # correctness at the timed size, and warm-up of both arms
            restore()
            append()
            sk, sv, has, (ptr, ts, row) = rebuild()
            for got, want in ((store.t["res_keys"], sk), (store.t["res_vals"], sv), (store.t["ms_has_res"], has),
                              (store.asof_t["ms_ptr"], ptr), (store.asof_t["ts"], ts), (store.asof_t["row"], row)):
                assert torch.equal(got, want)
            del sk, sv, has, ptr, ts, row
            times = {"append": [], "rebuild": []}
            host_list = None
            if rows <= 1_000_000:
                times["host"] = []
                ks = base["res_keys"].cpu().numpy()
                h_ts = np.concatenate([ks // N_MS, ts1.cpu().numpy()])
                h_ms = np.concatenate([ks % N_MS, ms1.cpu().numpy()])
                host_vals = np.concatenate([base["res_vals"].double().cpu().numpy(), v1.double().cpu().numpy()])
                if cut is not None:                          # the constructor gets the surviving rows only
                    keep = h_ts >= cut
                    h_ts, h_ms, host_vals = h_ts[keep], h_ms[keep], host_vals[keep]
                host_list = list(zip(h_ts.tolist(), h_ms.tolist()))
            for r in range(a.reps):
                restore()
                times["append"].append(timed(append)[1])
                times["rebuild"].append(timed(rebuild)[1])
                if host_list is not None:
                    times["host"].append(host_ms(lambda: PatternStore(
                        art["runtime2graph"], art["entry2runtimes"], host_list, host_vals, art["tr2data"], dev,
                        n_ms=N_MS))[1])
            # kernel time of the merge alone: the count once, then the merge repeated on the same inputs
            restore()
            nk, perm = torch.sort(ts1 * N_MS + ms1, stable=True)
            grp = torch.sort(torch.remainder(nk, N_MS), stable=True)[1].to(torch.int32)
            ms_ptr = torch.empty(N_MS + 1, dtype=torch.int32, device=dev)
            seg = torch.empty(2 * N_MS, dtype=torch.int32, device=dev)
            sizes = torch.empty(3, dtype=torch.int64, device=dev)
            L = _lib.lib()
            _lib.check(L.pert_store_resources_count(C.byref(store.desc), C.byref(store.asof_desc), nk.data_ptr(),
                                                    grp.data_ptr(), K, cut if cut is not None else -(1 << 63),
                                                    ms_ptr.data_ptr(), seg.data_ptr(), sizes.data_ptr(),
                                                    _lib.stream()), "count")
            p, q, n_out = sizes.tolist()
            out = [torch.empty(n_out, dtype=torch.int64, device=dev), torch.empty(n_out, 8, device=dev),
                   torch.empty(N_MS, dtype=torch.uint8, device=dev), torch.empty(n_out, dtype=torch.int64, device=dev),
                   torch.empty(n_out, dtype=torch.int32, device=dev)]

            def merge():
                _lib.check(L.pert_store_resources_merge(
                    C.byref(store.desc), C.byref(store.asof_desc), nk.data_ptr(), perm.data_ptr(), v1.data_ptr(),
                    grp.data_ptr(), K, ms_ptr.data_ptr(), seg.data_ptr(), p, q, n_out, *(t.data_ptr() for t in out),
                    _lib.stream()), "merge")

            merge()
            t_merge = timed(merge, 20)[1]
            moved = 2 * (n + K) * 52
            res = {"rows": n, "k": K, "workload": workload,
                   **{f"{k}_ms_median": round(statistics.median(v), 3) for k, v in times.items()},
                   **{f"{k}_ms_min": round(min(v), 3) for k, v in times.items()},
                   "merge_kernel_ms": round(t_merge, 4), "merge_bytes": moved,
                   "merge_bw_frac_of_3.35TBps": round(moved / (t_merge * 1e-3) / HBM_BYTES_PER_S, 3),
                   "append_vs_rebuild": round(statistics.median(times["rebuild"]) / statistics.median(times["append"]),
                                              2)}
            print(json.dumps(res), flush=True)
        del store, base, base_asof
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
