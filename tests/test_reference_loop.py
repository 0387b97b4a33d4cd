"""The drop-in claim, executed.

tests/golden/ref_loop.npz is what the REFERENCE'S OWN get_data_list / train / test functions returned when run through
`compat/`'s torch_geometric shim with the CPU oracle as `model` (oracle/gen_golden_loop.py).

GPU (-m gpu): the same loop -- `from model import SAGEDeterministic`,
`torch_geometric.data.Data`, `torch_geometric.loader.DataLoader` resolved through `compat/` exactly as
`PYTHONPATH=compat python pert_gnn.py` would -- on the reference-built per-trace Data of the fixture, same initial
weights, same batch composition, `torch.optim.Adam`; per-epoch train loss / MAPE and test MAE / MAPE / quantile loss
(pert_gnn.py:251,290-294) must match what the reference's loop returned with the oracle model."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "ref_loop.npz")
KEYS = ("x", "edge_index", "edge_attr", "cat_X", "node_depth", "pattern_num_nodes", "pattern_probs", "entry_id", "y")


def _golden():
    return np.load(GOLD)


def test_fixture_data_follows_the_reference_schema():
    """Schema of pert_gnn.py:163-173 on the reference-built Data (CPU, no reference needed)."""
    g = _golden()
    n = int(g["n_traces"])
    assert n == 72
    for i in (0, n - 1):
        x, ei, ea = g[f"d{i}_x"], g[f"d{i}_edge_index"], g[f"d{i}_edge_attr"]
        assert x.dtype == np.float32 and x.shape[1] == 9
        assert ei.dtype == np.int64 and ei.shape[0] == 2 and ea.shape == (ei.shape[1], 4)
        assert g[f"d{i}_cat_X"].shape == (x.shape[0], 1) and g[f"d{i}_node_depth"].shape == (x.shape[0], 1)
        assert g[f"d{i}_pattern_num_nodes"].dtype == np.float32 and g[f"d{i}_y"].shape == ()
        assert abs(float(g[f"d{i}_pattern_probs"].sum()) - 1.0) < 1e-6
        # missing-indicator column: stats are zero wherever the indicator is 1 (pert_gnn.py:44-66)
        assert np.all(x[x[:, 8] == 1.0, :8] == 0.0)


def _expand_rt_probs(d):
    """Per-node pattern probability, what pert_gnn.py:220-230 rebuilds on the host every step: pattern p's probability
    repeated over its nodes (pattern sizes read off pattern_num_nodes)."""
    pnn = d.pattern_num_nodes.reshape(-1)
    out, i, p = [], 0, 0
    while i < pnn.numel():
        sz = int(pnn[i])
        out.append(d.pattern_probs[p].expand(sz))
        i += sz
        p += 1
    assert p == d.pattern_probs.size(0)
    return torch.cat(out).reshape(-1, 1)


@pytest.mark.gpu
def test_dropin_loop_through_compat_matches_the_reference_run():
    compat = os.path.join(ROOT, "compat")
    sys.path.insert(0, compat)
    try:
        import importlib

        model_mod = importlib.import_module("model")                 # compat/model.py  (pert_gnn.py:12)
        from torch_geometric.data import Data                         # compat/torch_geometric (pert_gnn.py:2-3)
        from torch_geometric.loader import DataLoader
    finally:
        sys.path.remove(compat)
    assert model_mod.__file__.startswith(compat)
    g = _golden()
    n = int(g["n_traces"])
    ma = g["model_args"].tolist()
    seed, H, L, BATCH, EPOCHS = g["hyper"].tolist()
    tau, lr = g["tau_lr"].tolist()
    data_list = []
    for i in range(n):
        d = Data(**{k: torch.from_numpy(g[f"d{i}_{k}"]) for k in KEYS})
        d.rt_probs = _expand_rt_probs(d)
        data_list.append(d)
    device = torch.device("cuda:0")
    model = model_mod.SAGEDeterministic(ma[0], [ma[1]], ma[2], ma[3], ma[4], ma[5], ma[6], 0.0)
    model.load_state_dict({k[2:]: torch.from_numpy(g[k]) for k in g.files if k.startswith("w_")})
    model = model.to(device)
    optimizer = torch.optim.Adam(model.parameters(), lr=lr)
    # the loaders of pert_gnn.py:196-210, with the train order the reference's shuffle produced
    n_tr, n_va = int(n * 0.6), int(n * 0.8)
    order, lens = g["order_flat"].tolist(), g["order_len"].tolist()
    batches, o = [], 0
    for ln in lens:
        batches.append(order[o:o + ln])
        o += ln
    per_epoch = len(batches) // EPOCHS
    n_train_b = -(-n_tr // BATCH)
    n_valid_b = -(-(n_va - n_tr) // BATCH)

    def q_loss(y, yhat):                                               # pert_gnn.py:191-193
        e = y - yhat
        return torch.mean(torch.maximum(tau * e, (tau - 1) * e))

    def fwd(data):
        return model(data.x, data.cat_X, data.edge_index, data.edge_attr, data.pattern_num_nodes, data.rt_probs,
                     data.entry_id, data.batch)

    got = []
    for ep in range(EPOCHS):
        bs = batches[ep * per_epoch:(ep + 1) * per_epoch]
        model.train()
        total, mape = 0.0, 0.0
        for idx in bs[:n_train_b]:
            data = next(iter(DataLoader([data_list[i] for i in idx], batch_size=len(idx), shuffle=False))).to(device)
            optimizer.zero_grad()
            gp, _ = fwd(data)
            loss = q_loss(data.y.float(), gp.flatten())
            loss.backward()
            optimizer.step()
            total += float(loss) * data.num_graphs
            mape += float(((gp.flatten() - data.y).abs() / data.y).sum())
        row = [total / n_tr, mape / n_tr]
        model.eval()
        for part, cnt in ((bs[n_train_b:n_train_b + n_valid_b], n_va - n_tr), (bs[n_train_b + n_valid_b:], n - n_va)):
            mae = mp = q = 0.0
            with torch.no_grad():
                for idx in part:
                    data = next(iter(DataLoader([data_list[i] for i in idx], batch_size=len(idx)))).to(device)
                    gp, _ = fwd(data)
                    mae += float((gp.flatten() - data.y).abs().sum())
                    mp += float(((gp.flatten() - data.y).abs() / data.y).sum())
                    q += float(q_loss(data.y.float(), gp.flatten()) * data.y.shape[0])
            row += [mae / cnt, mp / cnt, q / cnt]
        got.append(row)
    got, ref = np.array(got), g["epochs"]
    rel = np.abs(got - ref) / np.abs(ref)
    log = os.environ.get("PERT_PARITY_LOG")
    if log:
        import json

        with open(log, "a") as f:
            f.write(json.dumps({"what": "dropin loop vs reference run (per epoch rel err)", "rel": rel.tolist()}) + "\n")
    assert rel[0].max() <= 2e-4, rel          # epoch 1: a handful of Adam steps
    assert rel.max() <= 2e-3, rel             # later epochs: Adam amplifies gradient rounding (see DESIGN.md section 6)
