"""The numpy restatement of rawtable.RawStream (tests/raw_stream_ref.py) against the oracle's whole-table
process_raw on one chunk, against a brute-force per-chunk form of its numbering rules, and the defect switches that
show the GPU comparisons of tests/test_gpu_raw_stream.py would catch each error."""
import numpy as np
import pytest

from oracle import raw_table_oracle as O
from pert_gnn_kdd23_b200.synthetic import make_random_raw_tables
from pert_gnn_kdd23_b200.tracegroup import COLUMNS
from tests.raw_stream_ref import DEFECTS, RefStream, time_chunks


def _same(a, b):
    for k in COLUMNS:
        if not np.array_equal(a["columns"][k], b["columns"][k]):
            return False
    return (np.array_equal(a["row"], b["row"]) and np.array_equal(a["resource_index"], b["resource_index"]) and
            np.array_equal(a["resource_values"], b["resource_values"], equal_nan=True))


@pytest.mark.parametrize("seed,min_occ", [(1, 100), (2, 3), (3, 0)])
def test_one_chunk_equals_oracle(seed, min_occ):
    raw = make_random_raw_tables(seed, 3000)
    r, s = O.process_raw(raw, min_occurence=min_occ), RefStream(min_occ).process(raw)
    assert _same(r, s)
    d = raw.dicts
    assert s["names"]["ms_names"] == [d["ms"][i] for i in r["ms_code"]] and s["n_ms"] == len(r["ms_code"])
    assert s["names"]["traceid_names"] == [d["traceid"][i] for i in r["tr_code"]]
    assert s["names"]["interface_names"] == [d["interface"][i] for i in r["if_code"]]
    assert s["names"]["rpcid_values"] == [d["rpcid"][i] for i in r["rpc_code"]]
    assert s["names"]["rpctype_names"] == [d["rpctype"][i] for i in r["rty_code"]]
    assert s["names"]["entry_names"] == [f"{d['ms'][a]}_{b}" for a, b in zip(r["ent_dm"], r["ent_if"])]


def _brute(chunks):
    """traceid and interface ids restated row by row: the first of every set of equal rows, the rows in (timestamp,
    row) order, and a Python dictionary per column handing out the next id to a value not seen in any chunk before."""
    ids = {"traceid": {}, "interface": {}}
    out = []
    for raw in chunks:
        d, c = raw.dicts, raw.calls
        seen, rows = set(), []
        for i in range(len(raw)):
            key = tuple(int(c[k][i]) for k in c)
            if key not in seen:
                seen.add(key)
                rows.append(i)
        rows.sort(key=lambda i: int(c["timestamp"][i]))
        chunk = {}
        for k in ids:
            for i in rows:
                ids[k].setdefault(d[k][c[k][i]], len(ids[k]))
            chunk[k] = {i: ids[k][d[k][c[k][i]]] for i in rows}
        out.append(chunk)
    return out, ids


def test_brute_force_numbering():
    """traceid and interface ids of every surviving row equal the brute-force numbering over the stream, and the
    name lists list the values in id order."""
    raw = make_random_raw_tables(4, 600)
    chunks = time_chunks(raw, 5, res_first=False, seed=1)
    ref = RefStream(2)
    got = [ref.process(c) for c in chunks]
    want, ids = _brute(chunks)
    for g, w in zip(got, want):
        for k, v in w.items():
            assert np.array_equal(g["columns"][k], [v[int(i)] for i in g["row"]]), k
    assert got[-1]["names"]["interface_names"] == list(ids["interface"])
    assert got[-1]["names"]["traceid_names"] == list(ids["traceid"])


def test_time_ordered_chunks_equal_whole_table():
    """Whole-trace chunks in time order, resources in chunk 1, min_occurence = 0: the concatenated outputs are the
    whole table's, with every id compared through its value."""
    raw = make_random_raw_tables(6, 2500)
    whole = O.process_raw(raw, min_occurence=0)
    d = raw.dicts
    val = {"traceid": [d["traceid"][i] for i in whole["tr_code"]], "interface": [d["interface"][i] for i in
                                                                                  whole["if_code"]],
           "rpcid": [d["rpcid"][i] for i in whole["rpc_code"]], "rpctype": [d["rpctype"][i] for i in whole["rty_code"]],
           "um": [d["ms"][i] for i in whole["ms_code"]]}
    val["dm"] = val["um"]
    ref = RefStream(0)
    parts = [ref.process(c) for c in time_chunks(raw, 4, res_first=True, seed=2)]
    names = parts[-1]["names"]
    mine = {"traceid": names["traceid_names"], "interface": names["interface_names"], "rpcid": names["rpcid_values"],
            "rpctype": names["rpctype_names"], "um": names["ms_names"], "dm": names["ms_names"]}
    cat = {k: np.concatenate([p["columns"][k] for p in parts]) for k in COLUMNS}
    # rows come in (chunk, timestamp) order; the whole table's in timestamp order: compare as multisets of rows
    assert len(cat["traceid"]) == len(whole["columns"]["traceid"])
    def rows(cols, v):
        return sorted(zip(*(([v[k][i] for i in cols[k]] if k in v else cols[k].tolist()) for k in COLUMNS
                            if k != "entryid")))
    assert rows(cat, mine) == rows(whole["columns"], val)
    for p in parts:
        assert np.all(np.diff(p["columns"]["timestamp"]) >= 0)


def _scenario():
    """Three chunks built to exercise every rule: each microservice's resources in one chunk, a low min_occurence."""
    raw = make_random_raw_tables(8, 1500, n_entries=16, n_ms=300, n_if=64)
    return time_chunks(raw, 3, res_first="by_ms", seed=3)


@pytest.mark.parametrize("defect", DEFECTS)
def test_each_defect_changes_a_compared_result(defect):
    chunks = _scenario()
    good, bad = RefStream(20), RefStream(20, defects=(defect,))
    differs = False
    for c in chunks:
        a, b = good.process(c), bad.process(c)
        differs |= not _same(a, b) or not np.array_equal(a["resource_ms"], b["resource_ms"])
    assert differs, defect
