"""Generates tests/golden/ref_pert.npz by RUNNING THE REFERENCE's GraphConstruct (needs pandas and a checkout
of handasontam/PERT-GNN-KDD23 named by the environment variable PERT_GNN_REFERENCE).

For every table of synthetic.make_span_tables(SEED) it builds the DataFrame preprocess.py:296-318 would pass and calls,
from the reference's misc.py itself:
  GraphConstruct.__init__  -> get_root_spanID (:138-142) and drop_wrong_edges (:87-105)
  get_pert_edge_index      -> edge_index, edge_attr, node_depth, sorted_span_id          (:221-370)
  get_span_edge_index      -> edge_index, node_depth, edge_attr, sorted_unique_ms        (:190-219)
Stored per trace t: the surviving row indices (`t{t}_keep`), the root (`t{t}_root`) and the four outputs.  The raw
tables are regenerated from the seed by the tests (synthetic.make_span_tables is deterministic).
Usage:  PERT_GNN_REFERENCE=<checkout> python oracle/gen_golden_pert.py
"""
import importlib.util
import os
import sys
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from pert_gnn_kdd23_b200.synthetic import make_span_tables  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "ref_pert.npz")
SEED, N_TRACES = 11, 24
COLS = ("timestamp", "rpcid", "um", "interface", "dm", "rpctype", "rt", "endTimestamp")   # interface before rpctype:
# misc.py:178 takes .loc[:, ["interface", "rpctype"]].values of a single-dtype frame (a negative-stride view otherwise)


def load_reference_misc():
    spec = importlib.util.spec_from_file_location("_ref_misc", os.path.join(os.environ["PERT_GNN_REFERENCE"], "misc.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def main():
    import pandas as pd

    warnings.simplefilter("ignore")                      # SettingWithCopyWarning inside drop_wrong_edges
    misc = load_reference_misc()
    tables = make_span_tables(SEED, N_TRACES)
    n_ms = 40
    resource_df = pd.DataFrame(np.zeros((n_ms, 8)), index=np.arange(n_ms))
    out = {"seed": np.int64(SEED), "n_traces": np.int64(len(tables))}
    for t, tab in enumerate(tables):
        df = pd.DataFrame({c: tab[c] for c in COLS})
        df["row"] = np.arange(len(df))
        gc = misc.GraphConstruct(df, resource_df, np.arange(n_ms))
        ei, ea, _x, nd, span = gc.get_pert_edge_index()
        out[f"t{t}_keep"] = gc.trace_span_df_no_duplicates["row"].values.astype(np.int64)
        out[f"t{t}_root"] = np.int64(gc.root_span)
        out[f"t{t}_edge_index"] = ei.numpy()
        out[f"t{t}_edge_attr"] = ea.numpy()
        out[f"t{t}_node_depth"] = nd.numpy()
        out[f"t{t}_ms_id"] = np.asarray(span, dtype=np.int64)
        gs = misc.GraphConstruct(df, resource_df, np.arange(n_ms))
        sei, _sx, snd, sea, _sdur, sms = gs.get_span_edge_index()
        out[f"t{t}_span_edge_index"] = sei.numpy()
        out[f"t{t}_span_edge_attr"] = sea.numpy()
        out[f"t{t}_span_node_depth"] = snd.numpy()
        out[f"t{t}_span_ms_id"] = np.asarray(sms, dtype=np.int64)
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, os.path.getsize(OUT), "bytes;", len(tables), "traces")


if __name__ == "__main__":
    main()
