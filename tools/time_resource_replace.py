"""Cost of replacing and deleting resource rows of a live store: PatternStore.append_resources(replace=True) and
delete_resources against a plain append of the same rows and against rebuilding the resource state.

Table: n_ms = 30000 microservices, one row per microservice and 30 s bucket, --rows rows in all (default 10^6 and
10^7: 33 and 333 buckets); every update names k = 30000 keys.  Workloads:
  * replace:       the newest bucket again (every key present), rows in random order;
  * replace_late:  the same with a random 10 % of the rows moved into older buckets;
  * delete:        delete_resources of the newest bucket's keys;
  * replace_evict: replace plus the eviction of the oldest bucket, in one call.
Arms, alternating, --reps times each after warm-up, each from the same table (restored outside the timed window) and
timed with CUDA events around the call:
  * update:  the workload's call;
  * append:  a plain append_resources of the same rows (with the same cut);
  * rebuild: the device rebuild a caller would otherwise run -- a keep-last dedupe of the batch, torch.isin to drop the
             old rows of its keys, torch.sort(stable) of all surviving keys, a gather of the values, ms_has_res by
             bincount and store.asof_index.
`merge` is the kernel time of pert_store_resources_update_merge alone (CUDA events around repeated calls on the same
inputs), and `merge_bw` the bytes it must move -- the old and inserted rows read and the rows written, 40 B each in
the table and 12 B in the index -- over that time, as a fraction of the H100 SXM data-sheet 3.35 TB/s.  Checks once per
workload that the update equals the device rebuild bit for bit.  Prints the card name and power limit, then one JSON
line per (rows, workload).

    python tools/time_resource_replace.py [--rows 1000000 10000000] [--reps 5]
"""
import argparse
import ctypes as C
import json
import statistics

import torch

from measure import HBM_BYTES_PER_S, card, timed

B, N_MS, K = 30000, 30000, 30000


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, nargs="+", default=[1_000_000, 10_000_000])
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    import numpy as np

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

        for workload in ("replace", "replace_late", "delete", "replace_evict"):
            ms1 = torch.randperm(N_MS, device=dev, generator=g)
            ts1 = torch.full((K,), (n_b - 1) * B, dtype=torch.int64, device=dev)
            if workload == "replace_late":
                late = torch.rand(K, device=dev, generator=g) < 0.1
                ts1 = torch.where(late, torch.randint(0, n_b - 1, (K,), device=dev, generator=g) * B, ts1)
            idx1, v1 = torch.stack([ts1, ms1], 1), torch.rand(K, 8, device=dev, generator=g)
            cut = B if workload == "replace_evict" else None
            insert = workload != "delete"

            def update():
                if insert:
                    store.append_resources(idx1, v1, evict_before=cut, replace=True)
                else:
                    store.delete_resources(idx1, evict_before=cut)

            def append():
                store.append_resources(idx1, v1, evict_before=cut)

            def rebuild():
                k1 = ts1 * N_MS + ms1
                sk1, p1 = torch.sort(k1, stable=True)
                last = torch.ones(K, dtype=torch.bool, device=dev)
                last[:-1] = sk1[1:] != sk1[:-1]
                keep = ~torch.isin(base["res_keys"], sk1[last])
                keys, vals = base["res_keys"][keep], base["res_vals"][keep]
                if insert:
                    pick = torch.sort(p1[last])[0]
                    keys, vals = torch.cat([keys, k1[pick]]), torch.cat([vals, v1[pick]])
                if cut is not None:
                    keep = keys >= cut * N_MS
                    keys, vals = keys[keep], vals[keep]
                sk, perm = torch.sort(keys, stable=True)
                return sk, vals[perm], (torch.bincount(sk % N_MS, minlength=N_MS) > 0).to(torch.uint8), \
                    asof_index(sk, N_MS)

            # correctness at the timed size, and warm-up of every arm
            restore()
            update()
            sk, sv, has, (ptr, ts, row) = rebuild()
            for got, want in ((store.t["res_keys"], sk), (store.t["res_vals"], sv), (store.t["ms_has_res"], has),
                              (store.asof_t["ms_ptr"], ptr), (store.asof_t["ts"], ts), (store.asof_t["row"], row)):
                assert torch.equal(got, want), workload
            del sk, sv, has, ptr, ts, row
            restore()
            append()
            times = {"update": [], "append": [], "rebuild": []}
            for _ in range(a.reps):
                restore()
                times["update"].append(timed(update)[1])
                restore()
                times["append"].append(timed(append)[1])
                times["rebuild"].append(timed(rebuild)[1])
            # kernel time of the merge alone: the count once (as _update_resources prepares it), the merge repeated
            restore()
            L = _lib.lib()
            nk, perm = torch.sort(ts1 * N_MS + ms1, stable=True)
            last = torch.ones(K, dtype=torch.bool, device=dev)
            last[:-1] = nk[1:] != nk[:-1]
            dk = nk[last]
            dgrp = torch.sort(torch.remainder(dk, N_MS), stable=True)[1].to(torch.int32)
            nd = int(dk.shape[0])
            ik, iperm, igrp, k = (dk, perm[last], dgrp, nd) if insert else (dk[:0], perm[:0], dgrp[:0], 0)
            cnt = torch.empty(2 * (nd + 1), dtype=torch.int32, device=dev)
            ms_ptr = torch.empty(N_MS + 1, dtype=torch.int32, device=dev)
            seg = torch.empty(3 * N_MS + 1, dtype=torch.int32, device=dev)
            sizes = torch.empty(4, dtype=torch.int64, device=dev)
            _lib.check(L.pert_store_resources_update_count(
                C.byref(store.desc), C.byref(store.asof_desc), dk.data_ptr(), dgrp.data_ptr(), nd, ik.data_ptr(),
                igrp.data_ptr(), k, cut if cut is not None else -(1 << 63), cnt.data_ptr(), ms_ptr.data_ptr(),
                seg.data_ptr(), sizes.data_ptr(), _lib.stream()), "count")
            p, q, n_out, n_dropped = sizes.tolist()
            out = [torch.empty(n_out, dtype=torch.int64, device=dev), torch.empty(n_out, 8, device=dev),
                   torch.empty(N_MS, dtype=torch.uint8, device=dev), torch.empty(n_out, dtype=torch.int64, device=dev),
                   torch.empty(n_out, dtype=torch.int32, device=dev)]

            def merge():
                _lib.check(L.pert_store_resources_update_merge(
                    C.byref(store.desc), C.byref(store.asof_desc), dk.data_ptr(), dgrp.data_ptr(), cnt.data_ptr(), nd,
                    ik.data_ptr(), iperm.data_ptr(), v1.data_ptr(), igrp.data_ptr(), k, ms_ptr.data_ptr(),
                    seg.data_ptr(), p, q, n_dropped, n_out, *(t.data_ptr() for t in out), _lib.stream()), "merge")

            merge()
            t_merge = timed(merge, 20)[1]
            moved = (n + k + n_out) * 52
            med = {key: statistics.median(v) for key, v in times.items()}
            res = {"rows": n, "k": K, "workload": workload,
                   **{f"{key}_ms_median": round(m, 3) for key, m in med.items()},
                   **{f"{key}_ms_range": [round(min(v), 3), round(max(v), 3)] for key, v in times.items()},
                   "merge_kernel_ms": round(t_merge, 4), "merge_bytes": moved,
                   "merge_bw_frac_of_3.35TBps": round(moved / (t_merge * 1e-3) / HBM_BYTES_PER_S, 3),
                   "update_vs_append": round(med["update"] / med["append"], 2),
                   "rebuild_vs_update": round(med["rebuild"] / med["update"], 2)}
            print(json.dumps(res), flush=True)
            del out, cnt
        del store, base, base_asof
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
