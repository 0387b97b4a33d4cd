"""Generates tests/golden/ref_preprocess.npz by RUNNING THE REFERENCE's preprocess.main() (needs pandas, joblib, tqdm
and a checkout of handasontam/PERT-GNN-KDD23 named by the environment variable PERT_GNN_REFERENCE).

synthetic.make_trace_table(SEED) is written to processed/processed_df.csv and processed/processed_resource_df.csv in a
temporary working directory, so get_df() (:191-266) takes its "already processed" branch and main() (:269-381) runs
on exactly that table.  Stored, from the files main() writes:
  tr2data           (:304-309) key order, entry_id, runtime_id, timestamp, y
  entry2runtimes    (:310-316, :371-375) entry key order, runtime key order per entry, float64 probabilities
  runtime2{span,pert}graph_map (:317-367) insertion order, occurences, num_nodes and the graph tensors, concatenated
The table is regenerated from the seed by the tests (make_trace_table is deterministic).
Usage:  PERT_GNN_REFERENCE=<checkout> python oracle/gen_golden_preprocess.py
"""
import importlib.util
import os
import sys
import tempfile
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from pert_gnn_kdd23_b200.synthetic import make_trace_table  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "ref_preprocess.npz")
SEED = 5
# interface before rpctype: misc.py:178 takes .loc[:, ["interface", "rpctype"]].values of a single-dtype frame
CSV_COLUMNS = ("traceid", "timestamp", "rpcid", "um", "interface", "dm", "rpctype", "rt", "entryid")


def _concat(graphs, key, axis):
    return np.concatenate([g[key].numpy() for g in graphs], axis=axis)


def main():
    import joblib
    import pandas as pd
    import torch

    pd.set_option("future.infer_string", False)          # map_consecutive_ids writes int codes into the Series
    warnings.simplefilter("ignore")
    ref = os.environ["PERT_GNN_REFERENCE"]
    d = make_trace_table(SEED)
    cols = d["columns"]
    res = pd.DataFrame([(t, m) for t, m in d["resource_index"]], columns=["timestamp", "msname"])
    for j in range(d["resource_values"].shape[1]):
        res[f"v{j}"] = d["resource_values"][:, j]
    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as work:
        os.makedirs(os.path.join(work, "processed"))
        pd.DataFrame({c: cols[c] for c in CSV_COLUMNS}).to_csv(os.path.join(work, "processed", "processed_df.csv"),
                                                              index=False)
        res.to_csv(os.path.join(work, "processed", "processed_resource_df.csv"), index=False)
        os.chdir(work)
        sys.path.insert(0, ref)
        try:
            spec = importlib.util.spec_from_file_location("_ref_preprocess", os.path.join(ref, "preprocess.py"))
            mod = importlib.util.module_from_spec(spec)
            spec.loader.exec_module(mod)
            mod.main()
            tr2data = torch.load("processed/tr2data.pt", weights_only=False)
            e2r = joblib.load("processed/entry2runtimes.joblib")
            gmaps = {k: torch.load(f"processed/runtime2{k}graph_map.pt", weights_only=False) for k in ("span", "pert")}
        finally:
            os.chdir(cwd)
            sys.path.remove(ref)
    out = {"seed": np.int64(SEED)}
    keys = list(tr2data)
    out["tr_keys"] = np.array(keys, dtype=np.int64)
    for f in ("entry_id", "runtime_id", "timestamp"):
        out[f"tr_{f}"] = np.array([tr2data[k][f] for k in keys], dtype=np.int64)
    assert all(type(tr2data[k]["timestamp"]) is np.int64 for k in keys)
    assert all(tr2data[k]["y"].dtype == torch.int64 and tr2data[k]["y"].dim() == 0 for k in keys)
    out["tr_y"] = np.array([int(tr2data[k]["y"]) for k in keys], dtype=np.int64)
    out["e2r_entries"] = np.array(list(e2r), dtype=np.int64)
    out["e2r_ptr"] = np.concatenate([[0], np.cumsum([len(v) for v in e2r.values()])]).astype(np.int64)
    out["e2r_runtime"] = np.array([r for v in e2r.values() for r in v], dtype=np.int64)
    out["e2r_prob"] = np.array([p for v in e2r.values() for p in v.values()], dtype=np.float64)
    for kind, gm in gmaps.items():
        gs = list(gm.values())
        out[f"{kind}_runtime"] = np.array(list(gm), dtype=np.int64)
        out[f"{kind}_occurences"] = np.array([g["occurences"] for g in gs], dtype=np.int64)
        out[f"{kind}_num_nodes"] = np.array([g["num_nodes"] for g in gs], dtype=np.int64)
        out[f"{kind}_node_ptr"] = np.concatenate([[0], np.cumsum([g["ms_id"].shape[0] for g in gs])]).astype(np.int64)
        out[f"{kind}_edge_ptr"] = np.concatenate([[0], np.cumsum([g["edge_index"].shape[1] for g in gs])]).astype(
            np.int64)
        out[f"{kind}_ms_id"] = _concat(gs, "ms_id", 0).reshape(-1).astype(np.int64)
        out[f"{kind}_node_depth"] = _concat(gs, "node_depth", 0)
        out[f"{kind}_edge_index"] = _concat(gs, "edge_index", 1)
        out[f"{kind}_edge_attr"] = _concat(gs, "edge_attr", 0)
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, os.path.getsize(OUT), "bytes;", len(keys), "traces,", len(gmaps["span"]), "runtimes")


if __name__ == "__main__":
    main()
