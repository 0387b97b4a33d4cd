"""Generates tests/golden/ref_loop.npz by RUNNING THE REFERENCE's own code (needs a checkout of
handasontam/PERT-GNN-KDD23 named by the environment variable PERT_GNN_REFERENCE).

What runs, from the reference's pert_gnn.py itself (oracle/ref_loop.py extracts the function definitions at run time):
  get_data_list -> get_entry_data -> get_x / get_cat_X / get_edge_index / ... (:40-188)  on synthetic processed/ artefacts
  get_data_loader (:196-210), train (:213-251), test (:254-294)                            for EPOCHS epochs
with `torch_geometric` = compat/ shim (Data, DataLoader) and `model` = the CPU oracle (oracle/model_oracle.py; PyG
itself is not installable, see DESIGN.md section 6).  Stored:
  * every per-trace Data the reference's get_entry_data built (x, edge_index, edge_attr, cat_X, node_depth,
    pattern_num_nodes, pattern_probs, entry_id, y)  -> pins the device pattern store + feature join (SURVEY N1 / N4);
  * the batch composition of every step (the train loader shuffles), the initial weights, and per epoch the values
    train() / test() returned  -> pins the drop-in loop and the eval metrics (X1 / N3) end to end.
Usage:  PERT_GNN_REFERENCE=<checkout> python oracle/gen_golden_loop.py
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import ref_loop  # noqa: E402
from oracle.model_oracle import OracleSAGEDeterministic  # noqa: E402
from pert_gnn_kdd23_b200.synthetic import make_trace_artifacts  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "ref_loop.npz")
SEED, HIDDEN, LAYERS, BATCH, TAU, LR, EPOCHS = 7, 16, 3, 12, 0.5, 3e-3, 3
KEYS = ("x", "edge_index", "edge_attr", "cat_X", "node_depth", "pattern_num_nodes", "pattern_probs", "entry_id", "y")


def run(model_factory=None, device="cpu", artifacts=None, init_state=None):
    """-> dict of everything the fixture stores.  `model_factory(args) -> model` lets the CPU test re-run it."""
    art = artifacts or make_trace_artifacts(SEED)
    Rec, order = ref_loop.recording_loader()
    ns = ref_loop.load_namespace(art, None, None, device, BATCH, TAU, loader_cls=Rec)
    data_list = ns["get_data_list"](art["tr2data"], art["entry2runtimes"], art["runtime2graph"])
    for i, d in enumerate(data_list):
        d.tr_idx = torch.tensor(i)
    # model construction exactly as pert_gnn.py:324-343 derives its arguments
    num_features = ns["resource_df"].shape[1]
    unique_ms = np.unique([int(m) for g in art["runtime2graph"].values() for m in g["ms_id"].reshape(-1)])
    entry_id_max = max(int(d.entry_id) for d in data_list)
    if_max = max(int(d.edge_attr[:, 0].max()) for d in data_list)
    rpc_max = max(int(d.edge_attr[:, 1].max()) for d in data_list)
    margs = (num_features + 1, [int(unique_ms.max()) + 1], entry_id_max, if_max, rpc_max, HIDDEN, LAYERS, 0.0)
    torch.manual_seed(0)
    model = (model_factory or (lambda a: OracleSAGEDeterministic(*a)))(margs)
    if init_state is not None:
        model.load_state_dict(init_state)
    init = {k: v.detach().cpu().clone() for k, v in model.state_dict().items()}
    model = model.to(device)
    ns["model"] = model
    ns["optimizer"] = torch.optim.Adam(model.parameters(), lr=LR)
    torch.manual_seed(1234)                       # the train loader's shuffle (torch global RNG)
    train_loader, valid_loader, test_loader = ns["get_data_loader"](data_list)
    epochs = []
    for _ in range(EPOCHS):
        tr_loss, tr_mape = ns["train"](train_loader)
        v = ns["test"](valid_loader)
        t = ns["test"](test_loader)
        epochs.append([float(tr_loss), float(tr_mape)] + [float(z) for z in v] + [float(z) for z in t])
    return {"data_list": data_list, "order": order, "init": init, "epochs": np.array(epochs, dtype=np.float64),
            "model_args": margs}


def main():
    assert ref_loop.available(), "set PERT_GNN_REFERENCE to a checkout of handasontam/PERT-GNN-KDD23"
    r = run()
    out = {"epochs": r["epochs"], "n_traces": np.int64(len(r["data_list"])),
           "model_args": np.array([r["model_args"][0], r["model_args"][1][0], *r["model_args"][2:7]], dtype=np.int64),
           "hyper": np.array([SEED, HIDDEN, LAYERS, BATCH, EPOCHS], dtype=np.int64), "tau_lr": np.array([TAU, LR])}
    for i, d in enumerate(r["data_list"]):
        for k in KEYS:
            out[f"d{i}_{k}"] = d[k].numpy()
    flat = [np.array(b, dtype=np.int64) for b in r["order"]]
    out["order_flat"] = np.concatenate(flat)
    out["order_len"] = np.array([len(b) for b in flat], dtype=np.int64)
    for k, v in r["init"].items():
        out[f"w_{k}"] = v.numpy()
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    np.savez_compressed(OUT, **out)
    print("epochs [train_loss, train_mape, valid mae/mape/q, test mae/mape/q]:\n", r["epochs"])
    print("batches:", len(flat), "traces:", len(r["data_list"]), "->", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
