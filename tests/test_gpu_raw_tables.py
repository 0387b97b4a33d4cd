"""Raw-table processing on the GPU (rawtable.process_raw, csrc/rawtable.cu) against the reference's own get_df() run
(tests/golden/ref_get_df.npz) and, at scale, against the numpy restatement (oracle/raw_table_oracle.py); forced hash
collisions, determinism, errors, a second device, and raw rows -> trace groups -> store -> train step against the same
chain fed the reference's processed table."""
import copy

import numpy as np
import pytest
import torch

from oracle import raw_table_oracle as O
from pert_gnn_kdd23_b200 import _lib
from pert_gnn_kdd23_b200.rawtable import STATS, process_raw, read_raw
from pert_gnn_kdd23_b200.synthetic import make_random_raw_tables
from pert_gnn_kdd23_b200.tracegroup import COLUMNS
from tests.test_raw_tables import FIXTURES, GOLD, assert_equals_golden, ms_bijection, write_fixture

pytestmark = pytest.mark.gpu


def _host(p):
    return ({k: v.cpu().numpy() for k, v in p.columns.items()}, p.row.cpu().numpy(), p.resource_index.cpu().numpy(),
            p.resource_values.cpu().numpy())


def _same_bits(a, b):
    """torch.equal that also matches NaN to NaN (floats compared bit for bit)."""
    if a.is_floating_point():
        a, b = (t.view(torch.int32 if t.element_size() == 4 else torch.int64) for t in (a, b))
    return torch.equal(a, b)


def _assert_equals_oracle(p, r):
    cols, row, idx, vals = _host(p)
    for k in COLUMNS:
        assert np.array_equal(cols[k], r["columns"][k]), k
    assert np.array_equal(row, r["row"])
    assert np.array_equal(idx, r["resource_index"])
    assert np.array_equal(np.isnan(vals), np.isnan(r["resource_values"]))
    ok = ~np.isnan(vals)
    assert np.array_equal(vals[ok].view(np.int64), r["resource_values"][ok].view(np.int64))


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLD)


@pytest.fixture(scope="module")
def big():
    raw = make_random_raw_tables(3, 200_000)
    return raw, O.process_raw(raw)


@pytest.mark.parametrize("fx", FIXTURES)
def test_fixture_equals_reference_get_df(gold, fx, tmp_path):
    calls, res = write_fixture(str(tmp_path), gold, fx)
    raw = read_raw(calls, res)
    p = process_raw(raw, "cuda").check()
    assert_equals_golden(gold, fx, *_host(p))
    _assert_equals_oracle(p, O.process_raw(raw))
    assert p.n_ms == len(p.ms_names) and len(p.entry_names) == int(p.columns["entryid"].max()) + 1


def test_scale_against_oracle(big):
    raw, r = big
    assert len(raw) > 5_000_000
    p = process_raw(raw, "cuda", min_occurence=100).check()
    assert len(p) > 1_000_000
    _assert_equals_oracle(p, r)
    assert p.ms_names == [raw.dicts["ms"][i] for i in r["ms_code"]]
    assert p.traceid_names == [raw.dicts["traceid"][i] for i in r["tr_code"]]
    assert p.interface_names == [raw.dicts["interface"][i] for i in r["if_code"]]
    assert p.rpcid_values == [raw.dicts["rpcid"][i] for i in r["rpc_code"]]
    assert p.rpctype_names == [raw.dicts["rpctype"][i] for i in r["rty_code"]]
    assert p.entry_names == [f"{raw.dicts['ms'][d]}_{i}" for d, i in zip(r["ent_dm"], r["ent_if"])]


def test_forced_hash_collisions_change_nothing():
    # 1500 traces (~5e4 rows), not the 2e5-trace table: 3-bit hashes send every row to one of 8 start slots, so linear
    # probing costs O(rows^2) comparisons -- the point is that collisions never merge distinct rows, not speed
    raw = make_random_raw_tables(5, 1500, dup=0.2)
    r = O.process_raw(raw, min_occurence=3)
    for bits in (64, 3):
        _assert_equals_oracle(process_raw(raw, "cuda", min_occurence=3, hash_bits=bits).check(), r)


def test_deterministic(big):
    raw, _ = big
    a, b = (process_raw(raw, "cuda").check() for _ in range(2))
    for k in COLUMNS:
        assert torch.equal(a.columns[k], b.columns[k]), k
    assert torch.equal(a.row, b.row) and torch.equal(a.resource_index, b.resource_index)
    assert torch.equal(a.resource_values.view(torch.int64), b.resource_values.view(torch.int64))


def _without(raw, calls=(), resources=()):
    """The table with the given call-graph / resource rows removed."""
    from pert_gnn_kdd23_b200.rawtable import RawTables

    kc = np.setdiff1d(np.arange(len(raw)), calls)
    kr = np.setdiff1d(np.arange(len(raw.resources["timestamp"])), resources)
    return RawTables({k: v[kc] for k, v in raw.calls.items()}, {k: v[kr] for k, v in raw.resources.items()},
                     raw.dicts)


@pytest.mark.parametrize("col,where,code", [("interface", "calls", "n"), ("um", "calls", "far"),
                                            ("dm", "calls", "neg"), ("msname", "resources", "neg"),
                                            ("msname", "resources", "far"), ("msname", "resources", "n")])
def test_out_of_range_codes_reported_and_left_out(col, where, code):
    """A code outside its dictionary (just past it, 10^9 past it, or negative) sets the status word, and the result
    is the one of the table without those rows."""
    raw = make_random_raw_tables(7, 300)
    n = len(raw.dicts["ms" if col in ("um", "dm", "msname") else col])
    rows = np.array([0, 5, 17])
    getattr(raw, where)[col][rows] = {"n": n, "far": n + 10 ** 9, "neg": -1}[code]
    p = process_raw(raw, "cuda", min_occurence=2)
    with pytest.raises(_lib.PertGnnError, match="out of range"):
        p.check()
    clean = _without(raw, **{where: rows})
    want = O.process_raw(clean, min_occurence=2)
    if where == "calls":                     # row indices of the clean table -> of the full table
        want["row"] = np.setdiff1d(np.arange(len(raw)), rows)[want["row"]]
    _assert_equals_oracle(p, want)
    process_raw(clean, "cuda", min_occurence=2).check()


def test_out_of_range_codes_reported():
    raw = make_random_raw_tables(7, 200)
    raw.calls["interface"][5] = len(raw.dicts["interface"])
    with pytest.raises(_lib.PertGnnError, match="out of range"):
        process_raw(raw, "cuda", min_occurence=0).check()
    for bad in (-1, len(raw.dicts["ms"]) + 10 ** 9):
        raw = make_random_raw_tables(7, 200)
        raw.resources["msname"][0] = bad
        with pytest.raises(_lib.PertGnnError, match="out of range"):
            process_raw(raw, "cuda", min_occurence=0).check()
    with pytest.raises(_lib.PertGnnError, match="CUDA device"):
        process_raw(raw, "cpu")
    torch.cuda.synchronize()


def test_to_frames_equal_get_df(gold, tmp_path):
    """to_frames() against the reference's frames: the same columns and values, microservice ids up to the one-to-one
    renumbering, rows with equal timestamps in raw-row order, code columns int64."""
    fx = "numeric"
    calls, res = write_fixture(str(tmp_path), gold, fx)
    df, rdf = process_raw(read_raw(calls, res), "cuda").check().to_frames()
    pre = f"{fx}_df_"
    assert list(df.columns) == [k[len(pre):] for k in gold.files if k.startswith(pre) and k != pre + "index"]
    assert list(rdf.columns) == [k[len(fx) + 5:] for k in gold.files if k.startswith(f"{fx}_res_")]
    assert all(df[k].dtype == np.int64 for k in df.columns) and rdf["msname"].dtype == np.int64
    assert str(gold[f"{fx}_dtype_df_rpcid"]) == "float64"        # the reference's codes in a float column
    cols = {k: df[k].to_numpy() for k in COLUMNS}
    assert_equals_golden(gold, fx, cols, df.index.to_numpy(), rdf[["timestamp", "msname"]].to_numpy(),
                         rdf[list(STATS)].to_numpy())
    mine = np.lexsort((df.index.to_numpy(), cols["timestamp"]))
    ref = np.lexsort((gold[f"{fx}_df_index"], gold[f"{fx}_df_timestamp"]))
    assert np.array_equal(df["endTimestamp"].to_numpy()[mine], gold[f"{fx}_df_endTimestamp"][ref])


def test_second_device():
    if torch.cuda.device_count() < 2:
        pytest.skip("one visible GPU")
    raw = make_random_raw_tables(9, 3000)
    p = process_raw(raw, "cuda:1", min_occurence=5).check()
    assert p.columns["traceid"].device == torch.device("cuda:1")
    _assert_equals_oracle(p, O.process_raw(raw, min_occurence=5))


@pytest.mark.parametrize("kind", ["span", "pert"])
def test_raw_rows_to_train_step(gold, kind, tmp_path):
    """raw CSV -> process_raw -> group_traces -> from_trace_groups -> GraphedTrainStep equals the same chain fed the
    reference's processed_df (rows with equal timestamps in raw-row order, microservice ids through the bijection)."""
    from pert_gnn_kdd23_b200.model import SAGEDeterministic
    from pert_gnn_kdd23_b200.store import PatternStore, StoreLoader
    from pert_gnn_kdd23_b200.tracegroup import group_traces
    from pert_gnn_kdd23_b200.train import FlatParams, FusedAdam, GraphedTrainStep

    fx = "numeric"
    calls, res = write_fixture(str(tmp_path), gold, fx)
    p = process_raw(read_raw(calls, res), "cuda").check()
    cols, row, idx, vals = _host(p)
    g = lambda k: gold[f"{fx}_{k}"]                                          # noqa: E731
    ref = np.lexsort((g("df_index"), g("df_timestamp")))
    mine = np.lexsort((row, cols["timestamp"]))
    assert np.array_equal(mine, np.arange(len(mine)))        # ours is already in that order
    bij = ms_bijection([(g("df_um")[ref], cols["um"]), (g("df_dm")[ref], cols["dm"]), (g("res_msname"), idx[:, 1])])
    ours_to_gold = {b: a for a, b in bij.items()}
    to_gold = np.vectorize(ours_to_gold.__getitem__, otypes=[np.int64])
    a_cols = dict(cols, um=to_gold(cols["um"]), dm=to_gold(cols["dm"]))
    b_cols = {k: g(f"df_{k}")[ref].astype(np.int64) for k in COLUMNS}
    a_idx = np.stack([idx[:, 0], to_gold(idx[:, 1])], axis=1)
    b_idx = np.stack([g("res_timestamp").astype(np.int64), g("res_msname")], axis=1)
    b_vals = np.stack([g(f"res_{k}") for k in STATS], axis=1)
    n_ms = int(max(a_idx[:, 1].max(), a_cols["um"].max(), a_cols["dm"].max())) + 1
    ga, gb = (group_traces(c, "cuda").check() for c in (a_cols, b_cols))
    assert ga.tr2data().keys() == gb.tr2data().keys()
    for k, v in gb.tr2data().items():
        w = ga.tr2data()[k]
        assert (w["entry_id"], w["runtime_id"], w["timestamp"], int(w["y"])) == \
            (v["entry_id"], v["runtime_id"], v["timestamp"], int(v["y"]))
    assert ga.entry2runtimes() == gb.entry2runtimes()
    # NaN statistics (groups without a value) become 0 on both sides, so the losses stay finite
    sa = PatternStore.from_trace_groups(ga, kind, a_idx, np.nan_to_num(vals), "cuda", n_ms=n_ms)
    sb = PatternStore.from_trace_groups(gb, kind, b_idx, np.nan_to_num(b_vals), "cuda", n_ms=n_ms)
    for k in sb.t:
        assert _same_bits(sa.t[k], sb.t[k]), k
    ids = list(range(len(sb)))
    la, lb = StoreLoader(sa, ids, 64), StoreLoader(sb, ids, 64)
    torch.manual_seed(0)
    ma = SAGEDeterministic(9, [n_ms], 8, 64, 8, 32, 2, 0.0).cuda()
    mb = copy.deepcopy(ma)
    sta = GraphedTrainStep(ma, FusedAdam(FlatParams(ma), lr=1e-3), 0.5)
    stb = GraphedTrainStep(mb, FusedAdam(FlatParams(mb), lr=1e-3), 0.5)
    n = 0
    for ba, bb in zip(la, lb):
        for key in ("x", "edge_index", "edge_attr", "cat_X", "rt_probs", "entry_id", "y"):
            assert _same_bits(ba[key], bb[key]), key
        lossa, lossb = sta(ba), stb(bb)
        assert torch.isfinite(lossa).all()
        torch.testing.assert_close(lossa, lossb, rtol=1e-5, atol=0)
        n += 1
    sa.check()
    sb.check()
    assert n == len(la) >= 3
