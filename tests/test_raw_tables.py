"""CPU tests of the raw-table processing: the numpy restatement (oracle/raw_table_oracle.py) against the reference's own
get_df() run (tests/golden/ref_get_df.npz, written by oracle/gen_golden_get_df.py), read_raw against pandas' pyarrow
reader, and the host-side rejections."""
import os

import numpy as np
import pytest

from oracle import raw_table_oracle as O
from pert_gnn_kdd23_b200 import _lib
from pert_gnn_kdd23_b200.rawtable import CALL_COLUMNS, STATS, read_raw
from pert_gnn_kdd23_b200.synthetic import make_raw_tables

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "ref_get_df.npz")
FIXTURES = ("numeric", "dotted")
CODES = ("traceid", "rpcid", "rpctype", "interface", "entryid")


def write_fixture(tmp, gold, fx):
    """The fixture's CSV files under ``tmp`` -> (call-graph paths, resource paths) in the golden's listdir order."""
    d = make_raw_tables(int(gold[f"{fx}_seed"]), dotted_rpcid=bool(gold[f"{fx}_dotted"]))
    paths = {}
    for sub, files in (("callgraph", d["callgraph"]), ("resource", d["resource"])):
        os.makedirs(os.path.join(tmp, sub), exist_ok=True)
        for name, text in files.items():
            with open(os.path.join(tmp, sub, name), "w") as f:
                f.write(text)
        paths[sub] = [os.path.join(tmp, sub, str(n)) for n in gold[f"{fx}_{sub}_files"]]
    return paths["callgraph"], paths["resource"]


def ms_bijection(pairs):
    """{golden ms id: our ms id} from (golden, ours) id arrays; asserts it is one-to-one both ways."""
    fwd, back = {}, {}
    for a, b in zip(*(np.concatenate(x) for x in zip(*pairs))):
        assert fwd.setdefault(int(a), int(b)) == int(b), f"golden ms {a} maps to two ids"
        assert back.setdefault(int(b), int(a)) == int(a), f"ms {b} maps to two golden ids"
    return fwd


def same_float(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.array_equal(np.isnan(a), np.isnan(b)) and np.array_equal(a[~np.isnan(a)].view(np.int64),
                                                                       b[~np.isnan(b)].view(np.int64))


def assert_equals_golden(gold, fx, cols, row, res_index, res_values):
    """Processed rows (ours: columns, raw row index) against the golden frame.  Rows with equal timestamps are compared
    in raw-row order (the reference's sort is unstable; the fixture's ties differ only in um or the sign of rt)."""
    g = lambda k: gold[f"{fx}_{k}"]                                          # noqa: E731
    assert len(row) == len(g("df_index")) > 0
    mine = np.lexsort((row, cols["timestamp"]))
    ref = np.lexsort((g("df_index"), g("df_timestamp")))
    assert np.array_equal(np.asarray(row)[mine], g("df_index")[ref])
    for k in CODES + ("timestamp", "rt"):
        assert np.array_equal(np.asarray(cols[k])[mine], g(f"df_{k}")[ref].astype(np.int64)), k
    assert np.array_equal(np.asarray(cols["timestamp"] + np.abs(cols["rt"]))[mine], g("df_endTimestamp")[ref])
    bij = ms_bijection([(g("df_um")[ref], np.asarray(cols["um"])[mine]), (g("df_dm")[ref], np.asarray(cols["dm"])[mine]),
                        (g("res_msname"), res_index[:, 1])])
    assert len(bij) == len(set(g("res_msname")) | set(g("df_um")) | set(g("df_dm")))
    assert np.array_equal(res_index[:, 0], g("res_timestamp").astype(np.int64))
    for j, k in enumerate(STATS):
        assert same_float(res_values[:, j], g(f"res_{k}")), k


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLD)


@pytest.mark.parametrize("fx", FIXTURES)
def test_oracle_equals_reference_get_df(gold, fx, tmp_path):
    calls, res = write_fixture(str(tmp_path), gold, fx)
    r = O.process_raw(read_raw(calls, res))
    assert_equals_golden(gold, fx, r["columns"], r["row"], r["resource_index"], r["resource_values"])


def test_fixture_covers_the_branches(gold):
    """The golden keeps two entries of 101 traces (one through coverage exactly 0.6 and "(?)"-resolved entries), drops
    an entry of 100 traces, and holds the Kahan group (mean 0.5 where a plain sum gives 0) and an all-NaN group."""
    for fx in FIXTURES:
        ent, tr = gold[f"{fx}_df_entryid"], gold[f"{fx}_df_traceid"]
        counts = sorted(len(set(tr[ent == e])) for e in set(ent))
        assert counts == [101, 101], counts
        mean = gold[f"{fx}_res_instance_cpu_usage_mean"]
        assert np.any(mean == 0.5) and np.any(np.isnan(gold[f"{fx}_res_instance_cpu_usage_max"]))
    assert gold["numeric_df_rpcid"].dtype.kind == "f" and gold["dotted_df_rpcid"].dtype.kind in "fi"


@pytest.mark.parametrize("fx", FIXTURES)
def test_read_raw_values_are_pandas_pyarrow_values(gold, fx, tmp_path):
    import pandas as pd

    calls, res = write_fixture(str(tmp_path), gold, fx)
    raw = read_raw(calls, res)
    df = pd.concat([pd.read_csv(f, index_col=0, engine="pyarrow").replace(np.nan, "nan") for f in calls],
                   ignore_index=True)
    assert len(raw) == len(df)
    for k in CALL_COLUMNS:
        d = raw.dicts["ms" if k in ("um", "dm") else k] if k not in ("timestamp", "rt") else None
        got = raw.calls[k] if d is None else [d[i] for i in raw.calls[k]]
        assert list(got) == list(df[k]), k
    if fx == "numeric":                                  # "1" and "1.0" read as numbers and merged
        d = raw.dicts["rpcid"]
        assert all(isinstance(v, (int, float)) for v in d) and len({float(v) for v in d}) == len(d)
    else:
        assert "nan" in raw.dicts["rpcid"] and all(isinstance(v, str) for v in raw.dicts["rpcid"])
    assert raw.dicts["ms"] == sorted(raw.dicts["ms"]) and "nan" in raw.dicts["ms"]
    rdf = pd.concat([pd.read_csv(f, engine="pyarrow") for f in res], ignore_index=True)
    rdf = rdf[rdf.timestamp.notna() & rdf.msname.notna()]
    assert list(raw.resources["timestamp"]) == list(rdf.timestamp.astype(np.int64))
    assert [raw.dicts["ms"][i] for i in raw.resources["msname"]] == list(rdf.msname)
    for u in ("instance_cpu_usage", "instance_memory_usage"):
        assert same_float(raw.resources[u], rdf[u].to_numpy(dtype=np.float64))


def _write(path, text):
    with open(path, "w") as f:
        f.write(text)
    return str(path)


GOOD_CALL = ",traceid,timestamp,rpcid,um,rpctype,dm,interface,rt\n0,t0,10,0,(?),http,A,i,5\n1,t0,11,1,A,rpc,B,j,-2\n"
GOOD_RES = "timestamp,msname,instance_cpu_usage,instance_memory_usage\n0,A,0.5,1.0\n"


@pytest.mark.parametrize("text,match", [
    (",traceid,timestamp,rpcid,um,rpctype,dm,interface,rt\n0,t0,10,0,a,http,b,i,5\n1,t0,,1,a,rpc,b,j,3\n",
     r"bad\.csv: row 1: call-graph timestamp"),
    (",traceid,timestamp,rpcid,um,rpctype,dm,interface,rt\n0,t0,10,0,a,http,b,i,5\n1,t0,11,1,a,rpc,b,j,\n"
     "2,t0,12,1,a,rpc,b,j,4\n", r"bad\.csv: row 1: call-graph rt"),
    (",traceid,timestamp,rpcid,um,rpctype,dm,interface,rt\n0,t0,10,0,a,http,b,i,5\n1,t0,11,1,a,rpc,b,j,2.5\n",
     r"bad\.csv: row 1: call-graph rt"),
    (",traceid,timestamp,rpcid,um,rpctype,dm,interface\n0,t0,10,0,a,http,b,i\n", r"bad\.csv: no column 'rt'"),
])
def test_call_graph_rejections_name_file_and_row(tmp_path, text, match):
    bad = _write(tmp_path / "bad.csv", text)
    good = _write(tmp_path / "good.csv", GOOD_CALL)
    res = _write(tmp_path / "res.csv", GOOD_RES)
    with pytest.raises(_lib.PertGnnError, match=match):
        read_raw([good, bad], [res])


def test_resource_rejections_name_file_and_row(tmp_path):
    good = _write(tmp_path / "good.csv", GOOD_CALL)
    bad = _write(tmp_path / "res.csv", "timestamp,msname,instance_cpu_usage,instance_memory_usage\n0,A,0.5,1\n"
                                       ",A,0.5,1\n1.5,B,0.5,1\n")
    with pytest.raises(_lib.PertGnnError, match=r"res\.csv: row 2: resource timestamp"):
        read_raw([good], [bad])
    bad = _write(tmp_path / "res2.csv", "timestamp,msname,instance_cpu_usage\n0,A,0.5\n")
    with pytest.raises(_lib.PertGnnError, match=r"res2\.csv: no column 'instance_memory_usage'"):
        read_raw([good], [bad])
    bad = _write(tmp_path / "res3.csv", "timestamp,msname,instance_cpu_usage,instance_memory_usage\n0,7,0.5,1\n")
    with pytest.raises(_lib.PertGnnError, match="microservice name 7 is not a string"):
        read_raw([good], [bad])


def test_null_keys_dropped_and_ms_dictionary_recoded(tmp_path):
    from pert_gnn_kdd23_b200.rawtable import RawTables

    good = _write(tmp_path / "good.csv", GOOD_CALL)
    res = _write(tmp_path / "res.csv", "timestamp,msname,instance_cpu_usage,instance_memory_usage\n0,A,,1\n,A,1,1\n"
                                       "5,,1,1\n")
    raw = read_raw([good], [res])
    assert list(raw.resources["timestamp"]) == [0] and np.isnan(raw.resources["instance_cpu_usage"][0])
    # a caller's own encoding with an unsorted microservice dictionary is recoded to name order
    calls = {k: raw.calls[k] for k in CALL_COLUMNS}
    names = raw.dicts["ms"][::-1]
    calls["um"] = len(names) - 1 - calls["um"]
    calls["dm"] = len(names) - 1 - calls["dm"]
    resources = dict(raw.resources, msname=len(names) - 1 - raw.resources["msname"])
    again = RawTables(calls, resources, dict(raw.dicts, ms=names))
    assert again.dicts["ms"] == raw.dicts["ms"]
    for k in ("um", "dm"):
        assert np.array_equal(again.calls[k], raw.calls[k])
    assert np.array_equal(again.resources["msname"], raw.resources["msname"])
