"""Generates tests/golden/node_depth_*.npz by RUNNING THE REFERENCE's own code (needs a checkout of
handasontam/PERT-GNN-KDD23 named by the environment variable PERT_GNN_REFERENCE).  Row A9 of SURVEY.md section 8a -- the one piece of the hot-path scope whose reference
implementation is pure Python/numpy and importable here:
  misc.DFS.dfs_min_node_depth (misc.py:59-63), GraphConstruct.build_adj_list (:107-111),
  GraphConstruct.get_node_depth (:113-136), GraphConstruct.get_node_features (:144-175),
  and the torch.tensor(node_depth, dtype=torch.long) cast of misc.py:215 / :368.
Usage:  PERT_GNN_REFERENCE=<checkout> python oracle/gen_golden.py
"""
import os
import sys

import numpy as np
import pandas as pd
import torch

REF = os.environ.get("PERT_GNN_REFERENCE", "")
OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")


def main():
    sys.path.insert(0, REF)
    import misc  # the reference module itself

    sys.setrecursionlimit(20000)
    sys.path.insert(0, os.path.dirname(OUT.rstrip("/")).rsplit("/tests", 1)[0])
    from pert_gnn_kdd23_b200.synthetic import random_dag

    gc = object.__new__(misc.GraphConstruct)
    gc.n_features = 8
    gc.ms_with_resource = np.array([], dtype=np.int64)
    gc.resource_df = pd.DataFrame(np.zeros((0, 8)), index=pd.Index([], dtype=np.int64))

    rng = np.random.default_rng(20230806)
    cases = []
    specs = [(2, 1, 2), (5, 7, 3), (50, 150, 5), (200, 600, 8), (37, 90, 6), (300, 299, 40), (64, 400, 4)]
    for n, m, L in specs:
        ei, _ = random_dag(rng, n, m, L)
        cases.append((ei, n, 0))
    # unreachable nodes: root in the middle of the DAG; and a graph with a cycle (the relaxing DFS still terminates)
    ei, _ = random_dag(rng, 60, 150, 6)
    cases.append((ei, 60, int(ei[1, 0])))
    cyc = np.array([[0, 1, 2, 3, 1], [1, 2, 3, 1, 4]], dtype=np.int64)
    cases.append((cyc, 6, 0))
    os.makedirs(OUT, exist_ok=True)
    for i, (ei, n, root) in enumerate(cases):
        t_ei = torch.from_numpy(ei)
        adj = gc.build_adj_list(t_ei)
        raw = gc.get_node_depth(root, n, adj)                       # list with float('inf') for unreachable
        raw_int = np.array([-1 if np.isinf(x) else int(x) for x in raw], dtype=np.int32)
        _, node_depth = gc.get_node_features(np.arange(n), t_ei, root, n)
        nd_long = torch.tensor(node_depth, dtype=torch.long).numpy()   # misc.py:215
        np.savez(os.path.join(OUT, f"node_depth_{i}.npz"), edge_index=ei, num_nodes=n, root=root,
                 min_depth=raw_int, node_depth=nd_long)
        print(i, n, ei.shape[1], root, raw_int.max(), nd_long.sum())


if __name__ == "__main__":
    main()
