"""Times rawtable.process_raw (dictionary-encoded raw rows -> processed span and resource tables on the GPU) and,
optionally, the reference's get_df() on the same rows written as CSV.

  python tools/time_raw_tables.py --traces 1000000            # GPU: process_raw at ~3e7 rows, device bytes per row
  python tools/time_raw_tables.py --traces 20000 --reference <checkout>   # CPU: the reference's get_df() on CSVs

process_raw is timed with CUDA events around the whole call (host-to-device copies of the encoded columns
included, CSV parsing excluded: the table is generated already encoded), after one warm-up call; read_raw (the host
parse) is timed separately when --reference writes CSVs.  Peak device memory above the input columns gives the bytes
per raw row and, from it, the largest table that fits in 80 GB.
"""
import argparse
import importlib.util
import json
import os
import sys
import tempfile
import time
import warnings

import numpy as np

from measure import timed
from pert_gnn_kdd23_b200.rawtable import CALL_COLUMNS, RESOURCE_COLUMNS
from pert_gnn_kdd23_b200.synthetic import make_random_raw_tables


def time_gpu(raw, reps):
    import torch

    from pert_gnn_kdd23_b200.rawtable import process_raw

    process_raw(raw, "cuda").check()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    ms = []
    for _ in range(reps):
        p, t = timed(lambda: process_raw(raw, "cuda"))
        ms.append(t)
        kept = len(p.check())
        del p
    peak = torch.cuda.max_memory_allocated() - base
    R = len(raw)
    return {"rows": R, "kept_rows": kept, "process_raw_ms": sorted(ms), "device_bytes_per_row": peak / R,
            "rows_fitting_80GB": int(80e9 / (peak / R)), "gpu": torch.cuda.get_device_name()}


def write_csvs(raw, work):
    """The encoded table as raw CSV files (two call-graph files, one resource file)."""
    import pandas as pd

    os.makedirs(os.path.join(work, "data", "MSCallGraph"))
    os.makedirs(os.path.join(work, "data", "MSResource"))
    cols = {}
    for k in CALL_COLUMNS:
        v = raw.calls[k]
        if k in ("timestamp", "rt"):
            cols[k] = v
        else:
            d = np.array(raw.dicts["ms" if k in ("um", "dm") else k], dtype=object)
            cols[k] = d[v]
    df = pd.DataFrame(cols)
    half = len(df) // 2
    df.iloc[:half].to_csv(os.path.join(work, "data", "MSCallGraph", "a.csv"))
    df.iloc[half:].to_csv(os.path.join(work, "data", "MSCallGraph", "b.csv"))
    r = {k: raw.resources[k] for k in RESOURCE_COLUMNS}
    r["msname"] = np.array(raw.dicts["ms"], dtype=object)[r["msname"]]
    pd.DataFrame(r).to_csv(os.path.join(work, "data", "MSResource", "r.csv"), index=False)


def time_reference(raw, ref):
    import pandas as pd

    from pert_gnn_kdd23_b200.rawtable import read_raw

    pd.set_option("future.infer_string", False)
    warnings.simplefilter("ignore")
    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as work:
        write_csvs(raw, work)
        os.makedirs(os.path.join(work, "processed"))
        t = time.perf_counter()
        read_raw([os.path.join(work, "data", "MSCallGraph", f) for f in ("a.csv", "b.csv")],
                 [os.path.join(work, "data", "MSResource", "r.csv")])
        t_read = time.perf_counter() - t
        os.chdir(work)
        sys.path.insert(0, ref)
        try:
            spec = importlib.util.spec_from_file_location("_ref_preprocess", os.path.join(ref, "preprocess.py"))
            mod = importlib.util.module_from_spec(spec)
            spec.loader.exec_module(mod)
            devnull = open(os.devnull, "w")
            out, err = sys.stdout, sys.stderr
            sys.stdout = sys.stderr = devnull
            t = time.perf_counter()
            try:
                mod.get_df()
            finally:
                sys.stdout, sys.stderr = out, err
            t_ref = time.perf_counter() - t
        finally:
            os.chdir(cwd)
            sys.path.remove(ref)
    return {"rows": len(raw), "read_raw_s": t_read, "reference_get_df_s": t_ref, "cpus": os.cpu_count()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--traces", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--reference", default=None, help="checkout of the reference: time its get_df() on the CPU")
    a = ap.parse_args()
    raw = make_random_raw_tables(11, a.traces)
    res = time_reference(raw, a.reference) if a.reference else time_gpu(raw, a.reps)
    res["traces"] = a.traces
    print(json.dumps(res))


if __name__ == "__main__":
    main()
