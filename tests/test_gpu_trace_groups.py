"""Trace grouping on the GPU (tracegroup.group_traces, csrc/tracegroup.cu) against the reference's own preprocessing
run (tests/golden/ref_preprocess.npz) and, on large random tables, against the numpy oracle; forced hash collisions,
determinism, errors, and the table -> store -> train-step path against the store built from the reference's dicts."""
import copy
import os

import numpy as np
import pytest
import torch

from oracle import pert_graph_oracle as PO
from oracle import trace_group_oracle as O
from pert_gnn_kdd23_b200.synthetic import make_random_trace_table, make_trace_table

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "ref_preprocess.npz")
FIELDS = ("trace_id", "row_ptr", "perm", "entry", "runtime", "bucket", "y", "order", "occurrences", "ins_runtime",
          "rep_trace", "runtime_ins", "ent_trace_ptr", "ent_pair_ptr", "pair_runtime", "pair_prob", "rep_ptr", "_rows")


def _group(cols, **kw):
    from pert_gnn_kdd23_b200.tracegroup import group_traces

    return group_traces(cols, "cuda", **kw).check()


def _assert_equals_oracle(g, r):
    h = lambda k: getattr(g, k).cpu().numpy()               # noqa: E731
    for k in ("trace_id", "row_ptr", "perm", "entry", "runtime", "bucket", "y", "order", "occurrences",
              "ins_runtime", "rep_trace"):
        assert np.array_equal(h(k).astype(np.int64), np.asarray(r[k], dtype=np.int64)), k
    assert np.array_equal(h("runtime_ins")[r["ins_runtime"]], np.arange(len(r["ins_runtime"])))
    e2r = g.entry2runtimes()
    assert list(e2r) == list(r["entry2runtimes"])
    for e, v in r["entry2runtimes"].items():
        assert list(e2r[e]) == list(v), e
        assert np.array_equal(np.array(list(e2r[e].values())).view(np.int64), np.array(list(v.values())).view(np.int64))


@pytest.fixture(scope="module")
def big():
    cols = make_random_trace_table(17, 200_000, rows=(4, 40), n_patterns=3000, long_rows=3000, n_long=3)
    return cols, O.group_traces(cols)


def test_fixture_bit_for_bit():
    from pert_gnn_kdd23_b200 import pertgraph

    gold = np.load(GOLD)
    d = make_trace_table(int(gold["seed"]))
    g = _group(d["columns"])
    _assert_equals_oracle(g, O.group_traces(d["columns"]))
    tr = g.tr2data()
    assert np.array_equal(np.array(list(tr)), gold["tr_keys"])
    for f in ("entry_id", "runtime_id", "timestamp"):
        assert np.array_equal(np.array([v[f] for v in tr.values()]), gold[f"tr_{f}"]), f
    assert all(type(v["timestamp"]) is np.int64 and v["y"].dtype == torch.int64 and v["y"].dim() == 0
               for v in tr.values())
    assert np.array_equal(np.array([int(v["y"]) for v in tr.values()]), gold["tr_y"])
    e2r = g.entry2runtimes()
    assert np.array_equal(np.array(list(e2r)), gold["e2r_entries"])
    assert np.array_equal(np.array([k for v in e2r.values() for k in v]), gold["e2r_runtime"])
    prob = np.array([p for v in e2r.values() for p in v.values()], dtype=np.float64)
    assert np.array_equal(prob.view(np.int64), gold["e2r_prob"].view(np.int64))
    assert np.array_equal(g.occurrences_by_insertion().cpu().numpy(), gold["span_occurences"])
    for kind in ("span", "pert"):
        pg, ids = g.graphs(kind)
        assert np.array_equal(np.array(ids), gold[f"{kind}_runtime"])
        npt, ept = gold[f"{kind}_node_ptr"], gold[f"{kind}_edge_ptr"]
        for k in range(len(ids)):
            p = {a: (v.cpu().numpy() if torch.is_tensor(v) else v) for a, v in pg.pattern(k).items()}
            assert p["num_nodes"] == gold[f"{kind}_num_nodes"][k]
            want = {"ms_id": gold[f"{kind}_ms_id"][npt[k]:npt[k + 1]],
                    "node_depth": gold[f"{kind}_node_depth"][npt[k]:npt[k + 1]],
                    "edge_index": gold[f"{kind}_edge_index"][:, ept[k]:ept[k + 1]],
                    "edge_attr": gold[f"{kind}_edge_attr"][ept[k]:ept[k + 1]]}
            if kind == "span":                                           # fully specified: the reference's tensors
                for a, w in want.items():
                    got = p[a].reshape(-1) if a == "ms_id" else p[a]
                    assert got.dtype == w.dtype and np.array_equal(got, w), (k, a)
            else:                                                        # node numbering is pandas order there
                ref = PO.canonical_form(want["ms_id"], want["edge_index"], want["edge_attr"], want["node_depth"])
                assert PO.canonical_form(p["ms_id"], p["edge_index"], p["edge_attr"], p["node_depth"]) == ref, k
    assert pertgraph.MAX_ROWS >= int(np.diff(g.rep_ptr.cpu().numpy()).max())


def test_scale_against_oracle(big):
    cols, r = big
    assert len(r["trace_id"]) == 200_000 and len(cols["um"]) > 3_000_000
    assert np.diff(r["row_ptr"]).max() > 2048 and len(r["ins_runtime"]) < len(r["trace_id"]) // 20
    _assert_equals_oracle(_group({k: torch.from_numpy(v).cuda() for k, v in cols.items()}), r)


def test_forced_hash_collisions_change_nothing(big):
    cols, r = big
    _assert_equals_oracle(_group(cols, hash_bits=3), r)


def test_deterministic():
    cols = make_random_trace_table(23, 30_000, rows=(1, 30), n_patterns=400)
    a, b = _group(cols), _group(cols)
    for k in FIELDS:
        assert torch.equal(getattr(a, k), getattr(b, k)), k


def test_errors_reported_not_faulted():
    from pert_gnn_kdd23_b200 import _lib
    from pert_gnn_kdd23_b200.tracegroup import group_traces

    d = make_trace_table(5)["columns"]
    mixed = {k: v.copy() for k, v in d.items()}
    mixed["entryid"][np.flatnonzero(mixed["traceid"] == mixed["traceid"][0])[-1]] += 1     # one trace, two entries
    for bad in (-1, 2 ** 31):
        out = {k: v.copy() for k, v in d.items()}
        out["traceid"][7] = bad
        with pytest.raises(_lib.PertGnnError):
            group_traces(out, "cuda").check()
    with pytest.raises(_lib.PertGnnError):
        group_traces(mixed, "cuda").check()
    with pytest.raises(_lib.PertGnnError):
        group_traces({k: np.zeros(0, dtype=np.int64) for k in d}, "cuda")
    with pytest.raises(_lib.PertGnnError):
        group_traces(d, "cpu")
    # a runtime whose representative loses every row to the filters (one self-loop row)
    lone = {k: np.concatenate([v, v[:1]]) for k, v in d.items()}
    lone["traceid"][-1], lone["um"][-1], lone["dm"][-1] = d["traceid"].max() + 5, 3, 3
    g = _group(lone)
    with pytest.raises(_lib.PertGnnError, match="runtime"):
        g.graphs("span")
    torch.cuda.synchronize()


@pytest.mark.parametrize("kind", ["span", "pert"])
def test_table_to_store_to_train_step(kind):
    """PatternStore.from_trace_groups == PatternStore(runtime2graph, entry2runtimes, ..., tr2data) built from the
    converters: identical batches through StoreLoader, equal losses through GraphedTrainStep."""
    from pert_gnn_kdd23_b200.model import SAGEDeterministic
    from pert_gnn_kdd23_b200.store import PatternStore, StoreLoader
    from pert_gnn_kdd23_b200.train import FlatParams, FusedAdam, GraphedTrainStep

    d = make_trace_table(5)
    g = _group(d["columns"])
    sa = PatternStore.from_trace_groups(g, kind, d["resource_index"], d["resource_values"], "cuda")
    pg, ids = g.graphs(kind)
    r2g = {rt: pg.pattern(k) for k, rt in enumerate(ids)}
    sb = PatternStore(r2g, g.entry2runtimes(), d["resource_index"], d["resource_values"], g.tr2data(), "cuda")
    assert sa.trace_keys == sb.trace_keys and sa.rt_ids == sb.rt_ids and sa.n_ms == sb.n_ms
    for k in sb.t:
        assert torch.equal(sa.t[k], sb.t[k]), k
    ids_all = list(range(len(sb)))
    la, lb = StoreLoader(sa, ids_all, 64), StoreLoader(sb, ids_all, 64)
    torch.manual_seed(0)
    ma = SAGEDeterministic(9, [d["n_ms"]], 6, 32, 6, 32, 2, 0.0).cuda()
    mb = copy.deepcopy(ma)
    sta = GraphedTrainStep(ma, FusedAdam(FlatParams(ma), lr=1e-3), 0.5)
    stb = GraphedTrainStep(mb, FusedAdam(FlatParams(mb), lr=1e-3), 0.5)
    n = 0
    for ba, bb in zip(la, lb):
        for key in ("x", "edge_index", "edge_attr", "cat_X", "node_depth", "pattern_num_nodes", "rt_probs",
                    "pattern_probs", "batch", "ptr", "entry_id", "y"):
            assert torch.equal(ba[key], bb[key]), key
        lossa, lossb = sta(ba), stb(bb)
        assert torch.isfinite(lossa).all()
        torch.testing.assert_close(lossa, lossb, rtol=1e-5, atol=0)
        n += 1
    sa.check()
    sb.check()
    assert n == len(la) >= 4
