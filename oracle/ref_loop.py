"""TEST INFRASTRUCTURE (not product): runs the REFERENCE'S OWN sample assembly and train / test loop.

The reference's `pert_gnn.py` is a script (argparse + file loads at import time), so it cannot be imported; this
harness parses it with `ast`, takes the function definitions it needs VERBATIM FROM THE FILE AT RUN TIME (nothing is
copied into this repository) --

  get_x :40-67, get_all_runtimes_id_probs :70-74, get_edge_attr :77-82, get_pattern_num_nodes :85-94,
  get_cat_X :97-99, get_node_depth :102-104, get_edge_index :107-119, transform_pattern_probs :122-131,
  get_entry_data :134-173, get_data_list :176-188, torch_quantile_loss :191-193, get_data_loader :196-210,
  train :213-251, test :254-294

-- and executes them in a namespace whose module-level globals (`args`, `device`, `resource_df`, `runtime2graph`,
`entry2runtimes`, `model`, `optimizer`) are synthetic stand-ins, with `torch_geometric` resolved to this repository's
`compat/` shim (`Data`, `DataLoader`).  So the reference's loop body really executes against the shim's
Data/Batch/DataLoader surface; the model is whatever the caller passes (the CPU oracle when generating goldens).

Only usable with a checkout of handasontam/PERT-GNN-KDD23 named by the environment variable PERT_GNN_REFERENCE; the
tests use the committed fixture tests/golden/ref_loop.npz produced by oracle/gen_golden_loop.py.
"""
import ast
import itertools
import os
import sys
import types
from functools import lru_cache

import numpy as np
import pandas as pd
import torch

REF_FILE = os.path.join(os.environ.get("PERT_GNN_REFERENCE", ""), "pert_gnn.py")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

FUNCS = ("get_x", "get_all_runtimes_id_probs", "get_edge_attr", "get_pattern_num_nodes", "get_cat_X",
         "get_node_depth", "get_edge_index", "transform_pattern_probs", "get_entry_data", "get_data_list",
         "torch_quantile_loss", "get_data_loader", "train", "test")


def available():
    return bool(os.environ.get("PERT_GNN_REFERENCE")) and os.path.exists(REF_FILE)


def _shim_modules():
    """`torch_geometric.data.Data` / `torch_geometric.loader.DataLoader` exactly as `PYTHONPATH=compat` resolves them."""
    compat = os.path.join(ROOT, "compat")
    for p in (compat, ROOT):
        if p not in sys.path:
            sys.path.insert(0, p)
    import torch_geometric.data as tg_data          # noqa: E402  (compat/torch_geometric)
    import torch_geometric.loader as tg_loader      # noqa: E402

    assert tg_data.__file__.startswith(compat), tg_data.__file__
    return tg_data.Data, tg_loader.DataLoader


class _NoBar:
    """tqdm stand-in: same iteration protocol, `set_description` swallowed (keeps test logs quiet)."""

    def __init__(self, it):
        self.it = it

    def __iter__(self):
        return iter(self.it)

    def set_description(self, *_a, **_k):
        pass


def load_namespace(artifacts, model, optimizer, device, batch_size, tau, loader_cls=None):
    """Namespace with the reference's functions compiled from its own source + synthetic module globals."""
    Data, DataLoader = _shim_modules()
    with open(REF_FILE) as f:
        tree = ast.parse(f.read(), REF_FILE)
    keep = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name in FUNCS]
    assert sorted(n.name for n in keep) == sorted(FUNCS), [n.name for n in keep]
    idx = pd.MultiIndex.from_tuples(artifacts["resource_index"], names=["timestamp", "msname"])
    resource_df = pd.DataFrame(artifacts["resource_values"], index=idx)
    ns = {
        "torch": torch, "np": np, "pd": pd, "itertools": itertools, "lru_cache": lru_cache, "tqdm": _NoBar,
        "Data": Data, "DataLoader": loader_cls or DataLoader,
        "args": types.SimpleNamespace(batch_size=batch_size, tau=tau),
        "device": torch.device(device), "resource_df": resource_df,
        "runtime2graph": artifacts["runtime2graph"], "entry2runtimes": artifacts["entry2runtimes"],
        "model": model, "optimizer": optimizer,
    }
    code = compile(ast.Module(body=keep, type_ignores=[]), REF_FILE, "exec")
    exec(code, ns)      # noqa: S102 -- the reference's own function bodies, from its own file
    return ns


def recording_loader():
    """DataLoader subclass (of the compat shim's) that records which dataset items went into every batch it yields, in
    order -- the reference shuffles the train loader with torch's global RNG (pert_gnn.py:201-203)."""
    _, DataLoader = _shim_modules()
    log = []

    class Rec(DataLoader):
        def __iter__(self):
            for b in super().__iter__():
                log.append(b.tr_idx.tolist())
                yield b

    return Rec, log
