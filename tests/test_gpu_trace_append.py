"""PatternStore.append_traces (csrc/ingest.cu) on the GPU.  After every append the store must equal, bit for bit, the
constructor fed the chunk-ordered grouping (tests/trace_chunk_ref.py) -- and, where the chunk order is the plain order,
the store from_trace_groups builds from the whole table.  Also: forced hash collisions, rejected chunks leaving the
store as it was, assembly, predict and training after appends, and a 10^4-trace append to a 10^6-trace store."""
import copy

import numpy as np
import pytest
import torch

from oracle import trace_group_oracle as O
from pert_gnn_kdd23_b200.synthetic import make_random_trace_table, make_trace_table
from tests import trace_chunk_ref as R
from tests.helpers import assert_close

pytestmark = pytest.mark.gpu

KEYS = ("x", "edge_index", "edge_attr", "cat_X", "node_depth", "pattern_num_nodes", "rt_probs", "pattern_probs", "batch",
        "ptr", "entry_id", "y")
GOLD_SEED = int(np.load(__file__.rsplit("/", 1)[0] + "/golden/ref_preprocess.npz")["seed"])


def _group(cols, dev="cuda", **kw):
    from pert_gnn_kdd23_b200.tracegroup import group_traces

    return group_traces(cols, dev, **kw).check()


def _store(cols, kind, res, n_ms, dev="cuda", **kw):
    from pert_gnn_kdd23_b200.store import PatternStore

    return PatternStore.from_trace_groups(_group(cols, dev, **kw), kind, res[0], res[1], dev, n_ms=n_ms)


def _rows(cols, keep_trace):
    """The rows of the traces ``keep_trace(traceid array) -> bool array`` selects."""
    m = keep_trace(cols["traceid"])
    return {k: v[m] for k, v in cols.items()}


def _state(s):
    d = s.desc
    assert all((getattr(d, k) or 0) == v.data_ptr() for k, v in s.t.items())     # NULL reads back as None
    return {"t": {k: v.clone() for k, v in s.t.items()},
            "n": (d.n_pat, d.n_ent, d.n_res, d.n_ms, d.attr_cols, d.n_traces),
            "ids": (list(s.rt_ids), list(s.trace_keys)),
            "h": [np.array(a, dtype=np.int64) for a in (s._h_trace_entry, s._h_ent_nodes, s._h_ent_edges,
                                                         s._h_ent_pats)]}


def _assert_same(a, b):
    a, b = (x if isinstance(x, dict) else _state(x) for x in (a, b))
    assert list(a["t"]) == list(b["t"])
    for k in b["t"]:
        assert torch.equal(a["t"][k], b["t"][k]), k
    assert a["n"] == b["n"]
    assert a["ids"][0] == b["ids"][0], "rt_ids"
    assert a["ids"][1] == b["ids"][1], "trace_keys"
    for x, y in zip(a["h"], b["h"]):
        assert np.array_equal(x, y)


def _rebuilt(cols, chunk, kind, res, n_ms):
    """The constructor fed the chunk-ordered grouping of ``cols`` (rows) with ``chunk`` (per row)."""
    from pert_gnn_kdd23_b200.store import PatternStore

    r = R.group_traces(cols, chunk)
    r2g, e2r, tr = R.store_dicts(cols, r, kind)
    return PatternStore(r2g, e2r, res[0], res[1], tr, "cuda", n_ms=n_ms)


# ---- 1. chunk order = plain order: one append equals from_trace_groups of the whole table ---------------------------
@pytest.mark.parametrize("kind", ["span", "pert"])
def test_fixture_split_equals_whole_table(kind):
    d = make_trace_table(GOLD_SEED)
    cols, res = d["columns"], (d["resource_index"], d["resource_values"])
    first = cols["traceid"].min()
    assert set(cols["entryid"][cols["traceid"] == first]) == {0}
    s = _store(_rows(cols, lambda t: t == first), kind, res, d["n_ms"])
    got = s.append_traces(_rows(cols, lambda t: t != first))
    assert got == range(1, 300)
    assert (cols["entryid"][cols["traceid"] != first] == 0).any()             # entry 0 gains traces
    _assert_same(s, _store(cols, kind, res, d["n_ms"]))


@pytest.mark.parametrize("kind", ["span", "pert"])
def test_random_split_equals_whole_table(kind):
    cols = make_random_trace_table(31, 20_000, rows=(1, 12), n_patterns=400, n_entries=12, n_ms=256, n_if=64)
    res = ([(0, 1), (30000, 5)], np.random.default_rng(0).random((2, 8)))
    r = O.group_traces(cols)
    tid, ent = r["trace_id"], r["entry"]
    X, m = int(np.median(tid)), 6
    c1, c2 = tid[(tid <= X) & (ent <= m)], tid[(tid > X) & (ent >= m)]
    s = _store(_rows(cols, lambda t: np.isin(t, c1)), kind, res, 256)
    got = s.append_traces(_rows(cols, lambda t: np.isin(t, c2)))
    assert got == range(len(c1), len(c1) + len(c2))
    _assert_same(s, _store(_rows(cols, lambda t: np.isin(t, np.concatenate([c1, c2]))), kind, res, 256))


# ---- 2. general sequences against the chunk-ordered oracle ----------------------------------------------------------
def _chunks(cols, seed):
    """Chunk (0..4) of every trace: 0 a random 60 %; 1 only runtimes of chunk 0; 2 only runtimes new to the store; 3 a
    single trace; 4 the rest, with every trace of a new entry."""
    r = O.group_traces(cols)
    rng = np.random.default_rng(seed)
    tid, ent, rt = r["trace_id"], r["entry"], r["runtime"]
    new_entry = ent.max()
    ch = np.full(tid.shape[0], 4)
    free = ent != new_entry
    under_new = np.unique(rt[~free])
    cand = np.setdiff1d(np.unique(rt[free]), under_new)
    Z = rng.choice(cand, size=max(4, cand.shape[0] // 7), replace=False)
    in_z = np.isin(rt, Z)
    ch[in_z & np.isin(rt, Z[: Z.shape[0] // 2])] = 2
    pool = np.flatnonzero(free & ~in_z)
    c0 = pool[rng.random(pool.shape[0]) < 0.6]
    ch[c0] = 0
    known = np.flatnonzero((ch == 4) & free & ~in_z & np.isin(rt, rt[c0]))
    ch[rng.choice(known, size=min(300, known.shape[0] - 1), replace=False)] = 1
    ch[np.flatnonzero((ch == 4) & free)[0]] = 3
    return r, ch


@pytest.mark.parametrize("kind,bits", [("span", 64), ("pert", 64), ("span", 3)])
def test_sequences_equal_chunk_ordered_oracle(kind, bits):
    from pert_gnn_kdd23_b200._lib import PertGnnError

    cols = make_random_trace_table(29, 4000, rows=(1, 8), n_patterns=150, n_entries=10, n_ms=64, n_if=32)
    n_ms, res = 64, ([(0, 3)], np.ones((1, 8)))
    r, ch = _chunks(cols, 5)
    row_chunk = ch[np.searchsorted(r["trace_id"], cols["traceid"])]
    part = lambda c: {k: v[row_chunk == c] for k, v in cols.items()}       # noqa: E731
    plain = O.group_traces(cols)
    rt_of = lambda c: set(plain["runtime"][ch == c])                        # noqa: E731
    assert rt_of(1) <= rt_of(0) and not rt_of(2) & (rt_of(0) | rt_of(1)) and (ch == 3).sum() == 1
    assert set(plain["entry"][ch == 4]) - set(plain["entry"][ch < 4])
    s = _store(part(0), kind, res, n_ms, hash_bits=bits)
    for c in range(1, 5):
        if c == 2:                                                           # rejected chunks change nothing
            before = _state(s)
            c2 = part(2)
            dup = {k: np.concatenate([v, part(0)[k][:1]]) for k, v in c2.items()}
            dup["traceid"][-1] = part(0)["traceid"][0]
            ms_bad = {k: v.copy() for k, v in c2.items()}
            ms_bad["dm"][5] = n_ms
            lone = {k: np.concatenate([v, v[:1]]) for k, v in c2.items()}
            lone["traceid"][-1], lone["um"][-1], lone["dm"][-1] = cols["traceid"].max() + 11, 3, 3
            for bad, msg in ((dup, "already in the store"), (ms_bad, "span row 5: dm"), (lone, "runtime")):
                with pytest.raises(PertGnnError, match=msg):
                    s.append_traces(bad, hash_bits=bits)
                _assert_same(s, before)
        T0 = len(s)
        got = s.append_traces(part(c), hash_bits=bits)
        assert got == range(T0, T0 + int((ch == c).sum()))
        upto = row_chunk <= c
        want = _rebuilt({k: v[upto] for k, v in cols.items()}, row_chunk[upto], kind, res, n_ms)
        _assert_same(s, want)


# ---- 3. assembly, predict and training after an append --------------------------------------------------------------
def test_assembly_predict_and_training_after_append():
    from pert_gnn_kdd23_b200.model import SAGEDeterministic
    from pert_gnn_kdd23_b200.store import StoreLoader
    from pert_gnn_kdd23_b200.train import BucketedTrainStep, FlatParams, FusedAdam, predict

    d = make_trace_table(GOLD_SEED)
    cols, res, n_ms = d["columns"], (d["resource_index"], d["resource_values"]), d["n_ms"]
    r = O.group_traces(cols)
    tid, ent = r["trace_id"], r["entry"]
    late = tid[(ent == 6) | ((ent == 4) & (tid % 2 == 0))]                 # entry 4 grows, entry 6 is new
    c1 = _rows(cols, lambda t: ~np.isin(t, late))
    c2 = _rows(cols, lambda t: np.isin(t, late))
    s = _store(c1, "span", res, n_ms)
    untouched = [i for i in range(len(s)) if s._h_trace_entry[i] in (0, 1, 2)]
    before = s.assemble(untouched)
    torch.manual_seed(0)
    model = SAGEDeterministic(9, [n_ms], 7, 32, 6, 32, 2, 0.0).cuda()
    mb = copy.deepcopy(model)
    q_ent = np.array([0, 1, 2, 2, 1, 0] * 8)
    q_ts = np.arange(q_ent.shape[0]) * 7919 + 1000
    p0 = predict(model, s, q_ent, q_ts, batch_size=16, asof=True)
    r0 = s.assemble_requests(q_ent, q_ts, asof=True)
    new = s.append_traces(c2)
    chunk = np.where(np.isin(cols["traceid"], late), 1, 0)
    want = _rebuilt(cols, chunk, "span", res, n_ms)
    _assert_same(s, want)
    after = s.assemble(untouched)
    for k in KEYS:
        assert torch.equal(before[k], after[k]), k
    # the requests' batches are bit-identical; the eval forward itself repeats to within fp32 accumulation order
    r1 = s.assemble_requests(q_ent, q_ts, asof=True)
    for k in KEYS[:-1]:
        assert torch.equal(r0[k], r1[k]), k
    assert_close(predict(model, s, q_ent, q_ts, batch_size=16, asof=True), p0, what="predict after the append")
    a, b = s.assemble(list(new)), want.assemble(list(new))
    for k in KEYS:
        assert torch.equal(a[k], b[k]), k
    losses = []
    for st, m in ((s, model), (want, mb)):
        step = BucketedTrainStep(m, FusedAdam(FlatParams(m), lr=1e-3), 0.5)
        losses.append(torch.stack([step(batch).reshape(()) for batch in StoreLoader(st, list(new), 16)]))
    assert losses[0].numel() >= 4 and torch.isfinite(losses[0]).all()
    torch.testing.assert_close(losses[0], losses[1], rtol=1e-5, atol=0)
    s.check()


# ---- 4. scale, rejected calls, second device --------------------------------------------------------------------------
def test_scale_1e4_into_1e6():
    from pert_gnn_kdd23_b200._lib import PertGnnError

    cols = make_random_trace_table(41, 1_010_000, rows=(3, 10), n_patterns=20_000, n_entries=64)
    tid = np.unique(cols["traceid"])
    late = np.random.default_rng(1).choice(tid, 10_000, replace=False)
    in_late = np.isin(cols["traceid"], late)
    idx = np.flatnonzero(np.isin(cols["traceid"], late[::100]))          # 100 late traces get a runtime of their own
    first = idx[np.unique(cols["traceid"][idx], return_index=True)[1]]
    cols["interface"][first] = 1_000_000 + cols["traceid"][first]
    c1, c2 = ({k: v[m] for k, v in cols.items()} for m in (~in_late, in_late))
    s = _store(c1, "span", ([], np.zeros((0, 8))), 4096)
    before = _state(s)
    bad = {k: np.concatenate([v, c1[k][:1]]) for k, v in c2.items()}
    with pytest.raises(PertGnnError, match="already in the store"):
        s.append_traces(bad)
    _assert_same(s, before)
    n_pat0 = len(s.rt_ids)
    got = s.append_traces(c2)
    assert got == range(1_000_000, 1_010_000)
    r = R.group_traces(cols, in_late.astype(np.int64))
    o = r["order"]
    assert s.rt_ids == [int(x) for x in r["ins_runtime"]] and len(s.rt_ids) >= n_pat0 + 100
    assert s.trace_keys == r["trace_id"][o].tolist()
    for k, v in (("trace_entry", r["entry"]), ("trace_ts", r["bucket"]), ("trace_y", r["y"])):
        assert np.array_equal(s.t[k].cpu().numpy().astype(np.int64), v[o]), k
    pat = np.empty(len(s.rt_ids), dtype=np.int64)
    pat[r["ins_runtime"]] = np.arange(len(s.rt_ids))
    e2r = r["entry2runtimes"]
    n_ent = max(e2r) + 1
    ptr = np.cumsum([0] + [len(e2r.get(e, {})) for e in range(n_ent)])
    assert np.array_equal(s.t["ent_ptr"].cpu().numpy(), ptr)
    assert np.array_equal(s.t["ent_pat"].cpu().numpy(), pat[[rt for e in sorted(e2r) for rt in e2r[e]]])
    prob = np.array([p for e in sorted(e2r) for p in e2r[e].values()], dtype=np.float64).astype(np.float32)
    assert np.array_equal(s.t["ent_prob"].cpu().numpy().view(np.int32), prob.view(np.int32))
    assert int(s.t["pat_nptr"].shape[0]) == len(s.rt_ids) + 1


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="one visible device")
def test_second_device():
    d = make_trace_table(GOLD_SEED)
    cols, res = d["columns"], (d["resource_index"], d["resource_values"])
    first = cols["traceid"].min()
    s = _store(_rows(cols, lambda t: t == first), "pert", res, d["n_ms"], dev="cuda:1")
    with torch.cuda.device(0):
        s.append_traces(_rows(cols, lambda t: t != first))
    want = _store(cols, "pert", res, d["n_ms"], dev="cuda:1")
    _assert_same(s, want)
    assert all(v.device == torch.device("cuda:1") for v in s.t.values())
