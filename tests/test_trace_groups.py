"""Trace grouping (preprocess.py main() after get_df(), :269-381) on the CPU: the numpy oracle against the REFERENCE'S
OWN preprocessing run (tests/golden/ref_preprocess.npz, oracle/gen_golden_preprocess.py on synthetic.make_trace_table),
the generators' determinism, and the host-side argument checks of the C-ABI."""
import ctypes
import os

import numpy as np
import pytest

from oracle import trace_group_oracle as O
from pert_gnn_kdd23_b200.synthetic import make_random_trace_table, make_trace_table

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "ref_preprocess.npz")


def _gold():
    g = np.load(GOLD)
    return g, make_trace_table(int(g["seed"]))


def test_oracle_equals_reference_preprocessing():
    g, d = _gold()
    r = O.group_traces(d["columns"])
    tr = O.tr2data(r)
    assert np.array_equal(np.array(list(tr), dtype=np.int64), g["tr_keys"])                 # key order
    for f in ("entry_id", "runtime_id", "timestamp"):
        assert np.array_equal(np.array([v[f] for v in tr.values()], dtype=np.int64), g[f"tr_{f}"]), f
    assert all(type(v["timestamp"]) is np.int64 and v["y"].dim() == 0 for v in tr.values())
    assert np.array_equal(np.array([int(v["y"]) for v in tr.values()]), g["tr_y"])
    e2r = r["entry2runtimes"]
    assert np.array_equal(np.array(list(e2r)), g["e2r_entries"])
    assert np.array_equal(np.array([k for v in e2r.values() for k in v]), g["e2r_runtime"])
    prob = np.array([p for v in e2r.values() for p in v.values()], dtype=np.float64)
    assert np.array_equal(prob.view(np.int64), g["e2r_prob"].view(np.int64))               # float64 bit for bit
    for kind in ("span", "pert"):
        assert np.array_equal(r["ins_runtime"], g[f"{kind}_runtime"])                       # map insertion order
        assert np.array_equal(r["occurrences"][r["ins_runtime"]], g[f"{kind}_occurences"])
    # what the fixture must exercise
    assert len(set(np.diff(np.concatenate([[0], np.flatnonzero(np.diff(d["columns"]["traceid"])) + 1])))) > 1
    assert (np.diff(r["trace_id"]) > 1).any() and (np.diff(r["row_ptr"]) == 1).any()
    assert (d["columns"]["rt"] < 0).any() and {0, 30000} <= set(r["bucket"].tolist())
    assert 3 not in e2r and 4 in e2r                                                         # entry-id gap
    two = [k for k in range(len(r["ins_runtime"])) if sum(int(r["ins_runtime"][k]) in v for v in e2r.values()) > 1]
    assert two
    for k in two:                # representative = first trace in iteration order, not the smallest traceid
        rid = r["ins_runtime"][k]
        assert r["trace_id"][r["rep_trace"][k]] > r["trace_id"][np.flatnonzero(r["runtime"] == rid)].min()


def test_generators_are_deterministic():
    a, b = make_trace_table(5), make_trace_table(5)
    assert all(np.array_equal(a["columns"][k], b["columns"][k]) for k in a["columns"])
    assert a["resource_index"] == b["resource_index"] and np.array_equal(a["resource_values"], b["resource_values"])
    x, y = make_random_trace_table(3, 500, long_rows=50, n_long=2), make_random_trace_table(3, 500, long_rows=50, n_long=2)
    assert all(np.array_equal(x[k], y[k]) for k in x)
    c = x
    assert np.array_equal(np.sort(c["traceid"], kind="stable"), np.sort(c["traceid"]))
    assert (np.diff(c["traceid"]) < 0).any()                                                 # traces interleave


def test_oracle_rejects_a_trace_under_two_entries():
    c = dict(make_trace_table(5)["columns"])
    c["entryid"] = c["entryid"].copy()
    c["entryid"][np.flatnonzero(c["traceid"] == c["traceid"][0])[-1]] += 1
    with pytest.raises(ValueError):
        O.group_traces(c)


def test_trace_group_abi_rejects_bad_arguments_before_cuda():
    from pert_gnn_kdd23_b200 import _lib
    from pert_gnn_kdd23_b200.tracegroup import _Groups, _SpanTable

    L = _lib.lib()
    word = ctypes.c_int(0)
    status = ctypes.addressof(word)                       # never written: the calls must return before any CUDA call
    tab = _SpanTable(-1, *([None] * 9))
    assert L.pert_trace_group_range(None, status, status, None) == -1
    assert L.pert_trace_group_range(ctypes.byref(tab), status, status, None) == -1                 # R < 0
    tab = _SpanTable(10, *([None] * 9))
    assert L.pert_trace_group_range(ctypes.byref(tab), status, status, None) == -1                 # NULL columns
    ok = _SpanTable(0, *([None] * 9))
    assert L.pert_trace_group_range(ctypes.byref(ok), None, status, None) == -1
    assert L.pert_trace_group_keys(ctypes.byref(ok), -1, status, status, status, 1 << 20, None) == -1
    assert L.pert_trace_group_keys(ctypes.byref(ok), 4, None, status, status, 1 << 20, None) == -1
    assert L.pert_trace_group_workspace_bytes(-1, 0, 0, 0) == -1
    assert L.pert_trace_group_workspace_bytes(10, 5, 11, 1) == -1                                    # T > R
    assert L.pert_trace_group_workspace_bytes(10, 5, 4, 2) > 0
    out = _Groups(*([None] * len(_Groups._fields_)))
    rows = _SpanTable(10, *([status] * 9))                 # plausible pointers: only the tested argument is wrong

    def build(o=out, n_keys=5, T=4, n_ent=2, bits=64, ws=1 << 30):
        return L.pert_trace_group_build(ctypes.byref(rows), n_keys, T, n_ent, bits, status, status, ctypes.byref(o),
                                        status, ws, status, None)
    assert build() == -1                                                                             # NULL outputs
    full = _Groups(*([status] * len(_Groups._fields_)))
    assert build(full, T=-1) == -1 and build(full, n_ent=-1) == -1 and build(full, n_keys=-1) == -1
    assert build(full, bits=0) == -1 and build(full, bits=65) == -1 and build(full, ws=16) == -1
    assert L.pert_trace_group_gather(ctypes.byref(rows), status, status, status, status, -1, 0, status, None) == -1
    assert L.pert_trace_group_gather(ctypes.byref(rows), None, status, status, status, 1, 0, status, None) == -1
    assert word.value == 0
