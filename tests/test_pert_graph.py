"""PERT-graph construction (SURVEY N2) against the REFERENCE'S OWN GraphConstruct.

tests/golden/ref_pert.npz holds what the reference's misc.py returned on synthetic.make_span_tables(11)
(oracle/gen_golden_pert.py): surviving rows, root, and per trace the PERT graph (edge_index, edge_attr, node_depth,
sorted_span_id) and the span graph (`--graph_type span`: edge_index, edge_attr, node_depth, sorted_unique_ms).
CPU tests pin the oracle restatement and the host row filters to it; the gpu tests compare the CUDA builder
bit for bit with the oracle (same canonical node numbering) and, up to relabelling, with the reference outputs."""
import os

import numpy as np
import pytest
import torch

from oracle import pert_graph_oracle as O
from pert_gnn_kdd23_b200.synthetic import make_span_tables

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "ref_pert.npz")


def _gold():
    g = np.load(GOLD)
    return g, make_span_tables(int(g["seed"]), int(g["n_traces"]))


def _cleaned(tab, keep):
    return {k: tab[k][keep] for k in tab}


def _oracle_graph(c, root):
    return O.pert_graph(c["um"], c["dm"], c["interface"], c["rpctype"], c["timestamp"], c["endTimestamp"], root)


# ------------------------------------------------------------------------------------------------- CPU
def test_oracle_matches_reference_graphconstruct():
    g, tabs = _gold()
    anomalies = 0
    for t, tab in enumerate(tabs):
        root = O.get_root_ms(tab)
        assert root == int(g[f"t{t}_root"])
        keep = O.drop_wrong_edges(tab, root)
        assert np.array_equal(keep, g[f"t{t}_keep"]), t
        anomalies += len(tab["um"]) - len(keep)
        ms, ei, ea, nd, _ = _oracle_graph(_cleaned(tab, keep), root)
        # shape law of the PERT graph (misc.py:238-302): nodes = 2 rows + distinct ms, edges = 4 rows
        assert ei.shape[1] == 4 * len(keep) and len(ms) == 2 * len(keep) + len(set(tab["um"][keep]) | set(tab["dm"][keep]))
        ref = O.canonical_form(g[f"t{t}_ms_id"], g[f"t{t}_edge_index"], g[f"t{t}_edge_attr"], g[f"t{t}_node_depth"])
        assert O.canonical_form(ms, ei, ea, nd) == ref, t
        assert nd.dtype == g[f"t{t}_node_depth"].dtype and nd.shape == g[f"t{t}_node_depth"].shape
    assert anomalies > 20          # the row filters are really exercised


def test_span_oracle_matches_reference_bit_for_bit():
    """misc.py:190-219 is fully specified (torch.unique sorted): the oracle equals the reference's tensors exactly."""
    g, tabs = _gold()
    for t, tab in enumerate(tabs):
        c = _cleaned(tab, g[f"t{t}_keep"])
        ms, ei, ea, nd, _ = O.span_graph(c["um"], c["dm"], c["interface"], c["rpctype"], int(g[f"t{t}_root"]))
        for k, v in (("ms_id", ms), ("edge_index", ei), ("edge_attr", ea), ("node_depth", nd)):
            w = g[f"t{t}_span_{k}"]
            assert v.dtype == w.dtype and np.array_equal(v, w), (t, k)


def test_host_row_filters_match_reference():
    from pert_gnn_kdd23_b200 import pertgraph

    g, tabs = _gold()
    for t, tab in enumerate(tabs):
        root = pertgraph.get_root_ms(tab)
        assert root == int(g[f"t{t}_root"])
        assert np.array_equal(pertgraph.drop_wrong_edges(tab, root), g[f"t{t}_keep"]), t
    # more tables than the fixture: numpy filters == loop oracle
    for seed in (1, 2, 3):
        for tab in make_span_tables(seed, 40, calls=(1, 60)):
            root = pertgraph.get_root_ms(tab)
            assert root == O.get_root_ms(tab)
            assert np.array_equal(pertgraph.drop_wrong_edges(tab, root), O.drop_wrong_edges(tab, root))


def test_flat_row_filters_equal_per_trace_filters():
    """clean_span_tables_flat (all traces at once, no Python loop) == get_root_ms + drop_wrong_edges per trace."""
    from pert_gnn_kdd23_b200 import pertgraph

    for seed, n, calls in ((11, 24, (1, 30)), (5, 60, (1, 80)), (6, 10, (200, 400))):
        tabs = make_span_tables(seed, n, calls=calls)
        row_ptr = np.concatenate([[0], np.cumsum([len(t["um"]) for t in tabs])])
        cols = {k: np.concatenate([t[k] for t in tabs]) for k in tabs[0]}
        keep, new_ptr, roots = pertgraph.clean_span_tables_flat(cols, row_ptr)
        exp_keep, exp_roots = [], []
        for t, tab in enumerate(tabs):
            r = pertgraph.get_root_ms(tab)
            exp_roots.append(r)
            exp_keep.append(pertgraph.drop_wrong_edges(tab, r) + row_ptr[t])
        assert np.array_equal(roots, np.array(exp_roots))
        assert np.array_equal(keep, np.concatenate(exp_keep))
        assert np.array_equal(np.diff(new_ptr), np.array([len(k) for k in exp_keep]))
    bad = {k: v.copy() for k, v in cols.items()}
    bad["timestamp"][int(np.argmax(np.abs(bad["rt"][:row_ptr[1]])))] += 10 ** 6      # trace 0 loses its root row
    with pytest.raises(IndexError):
        pertgraph.clean_span_tables_flat(bad, row_ptr)


def test_oracle_time_tie_rule():
    """Stable sort by time only (misc.py:290): equal times keep row order, a row's start before its end -- also for a
    zero-length call."""
    um = np.array([5, 5, 5])
    dm = np.array([1, 2, 3])
    z = np.zeros(3, dtype=np.int64)
    ms, ei, ea, nd, root = O.pert_graph(um, dm, z + 7, z + 2, np.array([10, 10, 10]), np.array([10, 12, 10]), 5)
    assert ms.tolist() == [5] * 7 + [1, 2, 3] and root == 0
    ev = ei[:, 6:].T.tolist()
    # order: start(1) end(1) start(2) start(3) end(3) end(2)
    assert ev == [[0, 7], [7, 2], [2, 8], [3, 9], [9, 5], [8, 6]]
    assert ea[6:, 2].tolist() == [1, 0, 1, 1, 0, 0]


def test_no_cpu_fallback_and_generator_contract():
    from pert_gnn_kdd23_b200 import _lib, pertgraph

    a, b = make_span_tables(4, 6), make_span_tables(4, 6)
    for ta, tb in zip(a, b):                                       # deterministic in the seed (goldens rely on it)
        assert all(np.array_equal(ta[k], tb[k]) for k in ta)
        assert np.array_equal(ta["endTimestamp"], ta["timestamp"] + np.abs(ta["rt"]))      # preprocess.py:263
        root = pertgraph.get_root_ms(ta)
        i = int(np.argmax(np.abs(ta["rt"])))
        assert ta["timestamp"][i] == ta["timestamp"].min() and ta["um"][i] == root          # misc.py:138-142
    c = _cleaned(a[0], pertgraph.drop_wrong_edges(a[0], pertgraph.get_root_ms(a[0])))
    for build in (pertgraph.build_pert_graphs, pertgraph.build_span_graphs):
        with pytest.raises(_lib.PertGnnError):
            build([c], [pertgraph.get_root_ms(a[0])], "cpu")        # the product path has no CPU implementation


# ------------------------------------------------------------------------------------------------- GPU
def _build(tables, roots):
    from pert_gnn_kdd23_b200 import pertgraph

    return pertgraph.build_pert_graphs(tables, roots, "cuda").check()


def _assert_equals_oracle(pg, tables, roots):
    for t, (c, root) in enumerate(zip(tables, roots)):
        ms, ei, ea, nd, rn = _oracle_graph(c, root)
        p = pg.pattern(t)
        assert p["num_nodes"] == len(ms)
        assert np.array_equal(p["ms_id"].cpu().numpy().reshape(-1), ms), t
        assert np.array_equal(p["edge_index"].cpu().numpy(), ei), t
        assert np.array_equal(p["edge_attr"].cpu().numpy(), ea), t
        assert np.array_equal(p["node_depth"].cpu().numpy(), nd), t
        assert int(pg.root_nid[t]) - int(pg.node_ptr[t]) == rn
        for k in ("ms_id", "edge_index", "edge_attr", "node_depth"):
            assert p[k].dtype == torch.int64


@pytest.mark.gpu
def test_cuda_pert_graphs_match_reference_and_oracle():
    g, tabs = _gold()
    cleaned = [_cleaned(tab, g[f"t{t}_keep"]) for t, tab in enumerate(tabs)]
    roots = [int(g[f"t{t}_root"]) for t in range(len(tabs))]
    pg = _build(cleaned, roots)
    _assert_equals_oracle(pg, cleaned, roots)
    for t in range(len(tabs)):
        p = {k: (v.cpu().numpy() if torch.is_tensor(v) else v) for k, v in pg.pattern(t).items()}
        ref = O.canonical_form(g[f"t{t}_ms_id"], g[f"t{t}_edge_index"], g[f"t{t}_edge_attr"], g[f"t{t}_node_depth"])
        assert O.canonical_form(p["ms_id"], p["edge_index"], p["edge_attr"], p["node_depth"]) == ref, t


@pytest.mark.gpu
def test_cuda_span_graphs_equal_reference_tensors():
    """`--graph_type span` (pert_gnn.py:32 default): the CUDA builder reproduces the reference's own tensors exactly."""
    from pert_gnn_kdd23_b200 import pertgraph

    g, tabs = _gold()
    cleaned = [_cleaned(tab, g[f"t{t}_keep"]) for t, tab in enumerate(tabs)]
    roots = [int(g[f"t{t}_root"]) for t in range(len(tabs))]
    sg = pertgraph.build_span_graphs(cleaned, roots, "cuda").check()
    for t in range(len(tabs)):
        p = sg.pattern(t)
        assert p["num_nodes"] == int(g[f"t{t}_span_edge_index"].max()) + 1      # preprocess.py:332
        for k in ("ms_id", "edge_index", "edge_attr", "node_depth"):
            got, want = p[k].cpu().numpy(), g[f"t{t}_span_{k}"]
            if k == "ms_id":
                got = got.reshape(-1)
            assert got.dtype == want.dtype and np.array_equal(got, want), (t, k)
    # ragged, long traces against the oracle
    tables, rts = [], []
    for seed, calls, nms in ((31, (1, 3), 10), (32, (300, 800), 300)):
        for tab in make_span_tables(seed, 5, n_ms=nms, calls=calls):
            root = pertgraph.get_root_ms(tab)
            keep = pertgraph.drop_wrong_edges(tab, root)
            if len(keep):
                tables.append(_cleaned(tab, keep))
                rts.append(root)
    sg = pertgraph.build_span_graphs(tables, rts, "cuda").check()
    for t, (c, root) in enumerate(zip(tables, rts)):
        ms, ei, ea, nd, rn = O.span_graph(c["um"], c["dm"], c["interface"], c["rpctype"], root)
        p = sg.pattern(t)
        assert np.array_equal(p["ms_id"].cpu().numpy().reshape(-1), ms) and np.array_equal(p["edge_index"].cpu().numpy(), ei)
        assert np.array_equal(p["edge_attr"].cpu().numpy(), ea) and np.array_equal(p["node_depth"].cpu().numpy(), nd)
        assert int(sg.root_nid[t]) - int(sg.node_ptr[t]) == rn


@pytest.mark.gpu
def test_cuda_pert_graphs_long_and_ragged_traces():
    """Raw tables -> host filters -> CUDA, ragged lengths from 1 row to > 600 rows (the > 48 KiB shared-memory path),
    many equal timestamps."""
    from pert_gnn_kdd23_b200 import pertgraph

    tables, roots = [], []
    for seed, calls, nms in ((21, (1, 4), 12), (22, (40, 200), 90), (23, (700, 900), 400)):
        for tab in make_span_tables(seed, 6, n_ms=nms, calls=calls):
            root = pertgraph.get_root_ms(tab)
            keep = pertgraph.drop_wrong_edges(tab, root)
            if len(keep) == 0:
                continue
            tables.append(_cleaned(tab, keep))
            roots.append(root)
    assert max(len(t["um"]) for t in tables) > 620 and min(len(t["um"]) for t in tables) <= 3
    pg = _build(tables, roots)
    _assert_equals_oracle(pg, tables, roots)
    # shape law
    rows = np.array([len(t["um"]) for t in tables])
    assert np.array_equal(np.diff(pg.edge_ptr), 4 * rows)
    dist = np.array([len(set(t["um"]) | set(t["dm"])) for t in tables])
    assert np.array_equal(np.diff(pg.node_ptr), 2 * rows + dist)


@pytest.mark.gpu
def test_cuda_pert_graph_errors():
    from pert_gnn_kdd23_b200 import _lib, pertgraph

    tab = make_span_tables(5, 1, anomalies=False)[0]
    root = pertgraph.get_root_ms(tab)
    c = _cleaned(tab, pertgraph.drop_wrong_edges(tab, root))
    pg = pertgraph.build_pert_graphs([c], [10 ** 9], "cuda")          # root absent: KeyError in the reference
    with pytest.raises(_lib.PertGnnError):
        pg.check()
    assert int(pg.root_nid[0]) == -1
    big = {k: np.zeros(pertgraph.MAX_ROWS + 1, dtype=np.int64) for k in pertgraph.COLUMNS}
    with pytest.raises(_lib.PertGnnError):
        pertgraph.build_pert_graphs([big], [0], "cuda")
    with pytest.raises(_lib.PertGnnError):
        pertgraph.build_pert_graphs([c], [root], "cpu")


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["pert", "span"])
def test_spans_to_training_batch_on_device(kind):
    """Span rows -> PERT patterns (CUDA) -> resident pattern store -> collated batch -> model forward, next to the
    same chain with the oracle's patterns collated on the host: identical batches, same predictions."""
    from pert_gnn_kdd23_b200 import pertgraph
    from pert_gnn_kdd23_b200.model import SAGEDeterministic
    from pert_gnn_kdd23_b200.store import PatternStore
    from pert_gnn_kdd23_b200.synthetic import make_trace_artifacts

    art = make_trace_artifacts(3, n_ms=40)
    tabs = make_span_tables(9, len(art["runtime2graph"]), n_ms=40)
    tables, roots = [], []
    for tab in tabs:
        root = pertgraph.get_root_ms(tab)
        tables.append(_cleaned(tab, pertgraph.drop_wrong_edges(tab, root)))
        roots.append(root)
    pg = pertgraph.build_pert_graphs(tables, roots, "cuda", kind=kind).check()
    art_dev, art_ora = dict(art), dict(art)
    art_dev["runtime2graph"], art_ora["runtime2graph"] = {}, {}
    for t, rt in enumerate(art["runtime2graph"]):
        p = pg.pattern(t)
        art_dev["runtime2graph"][rt] = p                 # CUDA tensors, as build_*_graphs returns them
        if kind == "pert":
            ms, ei, ea, nd, _ = _oracle_graph(tables[t], roots[t])
        else:
            c = tables[t]
            ms, ei, ea, nd, _ = O.span_graph(c["um"], c["dm"], c["interface"], c["rpctype"], roots[t])
        art_ora["runtime2graph"][rt] = {"edge_index": torch.from_numpy(ei), "edge_attr": torch.from_numpy(ea),
                                        "ms_id": torch.from_numpy(ms).reshape(-1, 1), "num_nodes": len(ms),
                                        "node_depth": torch.from_numpy(nd)}
    sa, sb = PatternStore.from_artifacts(art_dev, "cuda"), PatternStore.from_artifacts(art_ora, "cuda")
    # bulk ingest of the PertGraphs object (one D2H copy, vectorised last-occurrence flags) == per-pattern ingest
    sc = PatternStore.from_graphs(pg, list(art["runtime2graph"].keys()), art["entry2runtimes"], art["resource_index"],
                                  art["resource_values"], art["tr2data"], "cuda", n_ms=art.get("n_ms"))
    ids = list(range(16))
    ba, bb, bc = sa.assemble(ids), sb.assemble(ids), sc.assemble(ids)
    for k in ("x", "edge_index", "edge_attr", "cat_X", "node_depth", "batch", "ptr", "rt_probs"):
        assert torch.equal(ba[k], bb[k]), k
        assert torch.equal(bc[k], bb[k]), k
    torch.manual_seed(0)
    model = SAGEDeterministic(9, [40], 8, art["n_if"], art["n_rpc"], 32, 2, 0.0).cuda().eval()

    def run(b):                                         # the reference's call, pert_gnn.py:232-241
        with torch.no_grad():
            y = model(b.x, b.cat_X, b.edge_index, b.edge_attr, b.pattern_num_nodes, b.rt_probs, b.entry_id, b.batch)
        return y[0] if isinstance(y, (tuple, list)) else y

    ya, yb = run(ba), run(bb)
    assert ya.shape[0] == len(ids) and torch.isfinite(ya).all()
    assert torch.allclose(ya, yb, rtol=1e-5, atol=1e-6)      # same tensors in; float atomics order in the pool
