"""PatternStore.evict_traces (csrc/ingest.cu) on the GPU.  After every eviction the store must equal, bit for bit, the
constructor fed the window restatement's dicts (tests/trace_window_ref.py), and its per-trace patterns, pair counts,
entry totals, sorted traceids and runtime keys must equal the restatement's.  Also: a representative evicted from a
surviving pattern, evicting every trace and appending again, interleaved append / evict sequences (also with 3-bit
hashes), assembly, requests, predict and training after an eviction, and the oldest bucket of a 10^6-trace store."""
import copy

import numpy as np
import pytest
import torch

from oracle import trace_group_oracle as O
from pert_gnn_kdd23_b200.synthetic import make_random_trace_table, make_trace_table
from tests.helpers import assert_close
from tests.trace_window_ref import TraceWindow

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


def _want(w, kind, res, n_ms, dev="cuda"):
    """The constructor fed the restatement's dicts."""
    from pert_gnn_kdd23_b200.store import PatternStore

    r2g, e2r, tr = w.store_dicts(kind, dev)
    return PatternStore(r2g, e2r, res[0], res[1], tr, dev, n_ms=n_ms)


def _assert_ingest(s, w):
    """What the store keeps beside ``t`` against the restatement."""
    ing = s._ingest
    cnt, tot = w.pair_counts()
    rows, ptr = w.key_rows()
    assert np.array_equal(ing.trace_pat.cpu().numpy(), w.trace_patterns())
    assert ing.trace_tid.cpu().tolist() == list(w.traces)
    assert np.array_equal(ing.cnt.cpu().numpy(), cnt) and np.array_equal(ing.tot.cpu().numpy(), tot)
    assert ing.tids.cpu().tolist() == sorted(w.traces)
    assert np.array_equal(ing.rows.cpu().numpy(), rows) and np.array_equal(ing.ptr.cpu().numpy(), ptr)
    assert ing.next_rt == w.next_rt and s.rt_ids == list(w.patterns)
    assert (ing.n_nodes, ing.n_edges) == (int(s.t["pat_nptr"][-1]), int(s.t["pat_eptr"][-1]))


def _fixture():
    d = make_trace_table(GOLD_SEED)
    return d["columns"], (d["resource_index"], d["resource_values"]), d["n_ms"]


# ---- 1. the fixture table, both graph kinds ---------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["span", "pert"])
def test_fixture_evictions_equal_the_restatement(kind):
    cols, res, n_ms = _fixture()
    s = _store(cols, kind, res, n_ms)
    w = TraceWindow()
    w.append(cols)
    _assert_same(s, _want(w, kind, res, n_ms))
    _assert_ingest(s, w)
    for cut in (30000, 60000):
        T0 = len(s)
        remap = s.evict_traces(cut)
        want_remap = w.evict(cut)
        assert remap.dtype == np.int64 and remap.shape == (T0,)
        assert np.array_equal(remap, want_remap) and len(s) < T0
        _assert_same(s, _want(w, kind, res, n_ms))
        _assert_ingest(s, w)
        assert (s.t["trace_ts"] >= cut).all()


def test_an_evicted_representative_leaves_its_pattern_graph():
    cols, res, n_ms = _fixture()
    r = O.group_traces(cols)
    b, rt = r["bucket"], r["runtime"]
    k = next(k for k, (g, t) in enumerate(zip(r["ins_runtime"], r["rep_trace"]))
             if b[t] < 30000 and (b[rt == g] >= 30000).any())
    s = _store(cols, "pert", res, n_ms)
    g = s.rt_ids[k]

    def pattern(j):
        """Graph arrays and key rows of pattern j."""
        n0, n1 = s.t["pat_nptr"][j:j + 2].tolist()
        e0, e1 = s.t["pat_eptr"][j:j + 2].tolist()
        k0, k1 = s._ingest.ptr[j:j + 2].tolist()
        out = {n: s.t[n][n0:n1].clone() for n in ("pat_ms", "pat_depth", "pat_last")}
        out.update({n: s.t[n][e0:e1].clone() for n in ("pat_src", "pat_dst", "pat_attr")})
        out["keys"] = s._ingest.rows[:, k0:k1].clone()
        return out

    before = pattern(k)
    s.evict_traces(30000)
    after = pattern(s.rt_ids.index(g))
    for n, v in before.items():
        assert torch.equal(after[n], v), n
    w = TraceWindow()
    w.append(cols)
    w.evict(30000)
    _assert_same(s, _want(w, "pert", res, n_ms))


def test_evict_every_trace_then_append():
    from pert_gnn_kdd23_b200._lib import PertGnnError

    cols, res, n_ms = _fixture()
    s = _store(cols, "span", res, n_ms)
    w = TraceWindow()
    w.append(cols)
    n_ent, next_rt, cols_attr = s.desc.n_ent, s._ingest.next_rt, s.attr_cols
    remap = s.evict_traces(1 << 62)
    w.evict(1 << 62)
    assert (remap == -1).all() and len(s) == 0 and s.rt_ids == [] and s.trace_keys == []
    assert (s.desc.n_pat, s.desc.n_traces, s.desc.n_ent) == (0, 0, n_ent)
    for name in ("pat_ms", "pat_src", "ent_pat", "ent_prob", "trace_entry", "trace_ts", "trace_y"):
        assert s.t[name].numel() == 0, name
    assert s.t["pat_attr"].shape == (0, cols_attr) and s.t["pat_nptr"].tolist() == [0]
    assert s.t["ent_ptr"].tolist() == [0] * (n_ent + 1) and (s._h_ent_pats == 0).all()
    for e in range(n_ent):
        with pytest.raises(PertGnnError, match=f"entry {e} has no patterns"):
            s.check_entries([e])
    _assert_ingest(s, w)
    assert np.array_equal(s.evict_traces(0), np.zeros(0, dtype=np.int64))
    # traces come back: their runtimes are new (new ids past every id issued), entries keep their slots
    r = O.group_traces(cols)
    pick = r["trace_id"][np.unique(r["runtime"], return_index=True)[1][:5]]
    chunk = {k: v[np.isin(cols["traceid"], pick)].copy() for k, v in cols.items()}
    chunk["traceid"] += int(cols["traceid"].max()) + 1
    got = s.append_traces(chunk)
    w.append(chunk)
    assert got == range(0, 5) and min(s.rt_ids) == next_rt
    _assert_same(s, _want(w, "span", res, n_ms))
    _assert_ingest(s, w)


# ---- 2. interleaved sequences ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,bits", [("span", 64), ("pert", 64), ("span", 3)])
def test_interleaved_append_evict_sequences(kind, bits):
    cols = make_random_trace_table(23, 6000, rows=(1, 8), n_patterns=220, n_entries=10, n_ms=64, n_if=16,
                                   span=300000)
    n_ms, res = 64, ([(0, 3)], np.ones((1, 8)))
    tid = np.unique(cols["traceid"])
    rng = np.random.default_rng(7)
    chunk_of = dict(zip(tid.tolist(), rng.integers(0, 4, tid.shape[0]).tolist()))
    row_chunk = np.array([chunk_of[t] for t in cols["traceid"].tolist()])
    part = lambda c: {k: v[row_chunk == c].copy() for k, v in cols.items()}   # noqa: E731
    late = part(3)
    late["entryid"][late["entryid"] == 3] = 10                               # entry 10 is new to the store
    first = part(0)
    s = _store(first, kind, res, n_ms, hash_bits=bits)
    w = TraceWindow()
    w.append(first)

    def returning():
        """Copies of the chunk-0 traces of runtimes the window has dropped, 6 buckets later, under new traceids."""
        r = O.group_traces(first)
        live = {w.patterns[g][0] for g in w.patterns}
        rp, perm = r["row_ptr"], r["perm"]
        key = lambda t: np.stack([first[k][perm[rp[t]:rp[t + 1]]] for k in ("um", "dm", "interface")], 1).tobytes()  # noqa: E731,E501
        gone = [int(r["trace_id"][t]) for t in range(len(r["trace_id"])) if key(t) not in live]
        c = {k: v[np.isin(first["traceid"], gone)].copy() for k, v in first.items()}
        c["traceid"] += 10_000_000
        c["timestamp"] += 180000
        assert len(gone) > 0
        return c

    steps = [("evict", 0), ("append", part(1)), ("evict", 30000), ("append", part(2)), ("evict", 120000),
             ("append", returning), ("evict", 135001), ("append", late), ("evict", 135001), ("evict", 210000)]
    for what, arg in steps:
        if what == "append":
            chunk = arg() if callable(arg) else arg
            n_rt = w.next_rt
            T0 = len(s)
            assert s.append_traces(chunk, hash_bits=bits) == w.append(chunk)
            if callable(arg):                                                  # returning runtimes are new
                assert len(s.rt_ids) > 0 and max(s.rt_ids) >= n_rt and len(s) > T0
        else:
            before = _state(s)
            remap = s.evict_traces(arg)
            assert np.array_equal(remap, w.evict(arg))
            if (remap == np.arange(remap.shape[0])).all():                    # nothing evicted: nothing changed
                _assert_same(s, before)
        _assert_same(s, _want(w, kind, res, n_ms))
        _assert_ingest(s, w)
    assert 10 in w.entries and w.n_ent == 11


# ---- 3. downstream of an eviction ------------------------------------------------------------------------------------
def test_assembly_requests_predict_and_training_after_eviction():
    from pert_gnn_kdd23_b200._lib import PertGnnError
    from pert_gnn_kdd23_b200.model import SAGEDeterministic
    from pert_gnn_kdd23_b200.store import StoreLoader
    from pert_gnn_kdd23_b200.train import BucketedTrainStep, FlatParams, FusedAdam, predict

    cols, res, n_ms = _fixture()
    s = _store(cols, "span", res, n_ms)
    w = TraceWindow()
    w.append(cols)
    mix0 = w.entry2runtimes()
    T0 = len(s)
    torch.manual_seed(0)
    model = SAGEDeterministic(9, [n_ms], 7, 32, 6, 32, 2, 0.0).cuda()
    mb = copy.deepcopy(model)
    live = [e for e in range(w.n_ent) if mix0[e]]
    q_ent = np.array(live * 8)
    q_ts = np.arange(q_ent.shape[0]) * 7919 + 1000
    p0 = predict(model, s, q_ent, q_ts, batch_size=16, asof=True)
    remap = s.evict_traces(30000)
    w.evict(30000)
    want = _want(w, "span", res, n_ms)
    _assert_same(s, want)
    # old ids, remapped
    held = [i for i in range(T0) if i % 3 != 1]
    ids = remap[held]
    ids = ids[ids >= 0]
    assert 0 < ids.shape[0] < len(held)
    a, b = s.assemble(ids), want.assemble(ids)
    for k in KEYS:
        assert torch.equal(a[k], b[k]), k
    # requests, exact and as-of, with the status word
    mix1 = w.entry2runtimes()
    alive = [e for e in range(w.n_ent) if mix1[e]]
    r_ent = np.array(alive * 4)
    r_ts = np.array([30000, 30000 + 17, 60000, 61000] * len(alive))[:r_ent.shape[0]]
    for asof in (False, True):
        a, b = (x.assemble_requests(r_ent, r_ts, asof=asof) for x in (s, want))
        for k in KEYS[:-1]:
            assert torch.equal(a[k], b[k]), (asof, k)
        assert torch.equal(s.status, want.status)
    s.check()
    for e in range(w.n_ent):
        if not mix1[e]:
            with pytest.raises(PertGnnError, match=f"entry {e} has no patterns"):
                s.check_entries([e])
    # predict: equal to the rebuilt store's; an entry whose mix did not change predicts as before
    q = np.isin(q_ent, alive)
    p1 = predict(model, s, q_ent[q], q_ts[q], batch_size=16, asof=True)
    assert_close(p1, predict(model, want, q_ent[q], q_ts[q], batch_size=16, asof=True), what="predict after evict")
    p0, p1 = p0.cpu()[torch.from_numpy(q)], p1.cpu()
    same = torch.from_numpy(np.array([list(mix0[e].items()) == list(mix1[e].items()) for e in q_ent[q]]))
    assert (~same).any()
    if same.any():
        assert_close(p1[same], p0[same], what="predict of entries whose mix did not change")
    assert not torch.equal(p1[~same], p0[~same])
    # a training pass over the remapped ids
    losses = []
    for st, m in ((s, model), (want, mb)):
        step = BucketedTrainStep(m, FusedAdam(FlatParams(m), lr=1e-3), 0.5)
        losses.append(torch.stack([step(batch).reshape(()) for batch in StoreLoader(st, ids.tolist(), 16)]))
    assert losses[0].numel() >= 4 and torch.isfinite(losses[0]).all()
    torch.testing.assert_close(losses[0], losses[1], rtol=1e-5, atol=0)


# ---- 4. scale, second device -----------------------------------------------------------------------------------------
def test_scale_evict_the_oldest_bucket_of_1e6():
    cols = make_random_trace_table(43, 1_000_000, rows=(3, 10), n_patterns=20_000, n_entries=64)
    # 100 traces of the oldest bucket get a runtime of their own (a unique first-row interface): their patterns go
    u, inv = np.unique(cols["traceid"], return_inverse=True)
    t_min = np.full(u.shape[0], np.iinfo(np.int64).max)
    np.minimum.at(t_min, inv, cols["timestamp"])
    lone = u[t_min < 30000][::97][:100]
    idx = np.flatnonzero(np.isin(cols["traceid"], lone))
    first = idx[np.unique(cols["traceid"][idx], return_index=True)[1]]
    cols["interface"][first] = 1_000_000 + cols["traceid"][first]
    s = _store(cols, "span", ([], np.zeros((0, 8))), 4096)
    ing = s._ingest
    T, n_pat, n_ent = len(s), len(s.rt_ids), s.desc.n_ent
    ts, ent, pat = (x.cpu().numpy().astype(np.int64) for x in (s.t["trace_ts"], s.t["trace_entry"], ing.trace_pat))
    tid = np.array(s.trace_keys, dtype=np.int64)
    ent_ptr, ent_pat = s.t["ent_ptr"].cpu().numpy(), s.t["ent_pat"].cpu().numpy().astype(np.int64)
    nlen, elen = s.t["pat_nptr"].diff().cpu().numpy(), s.t["pat_eptr"].diff().cpu().numpy()
    rt_ids = list(s.rt_ids)
    assert ts.min() == 0
    remap = s.evict_traces(30000)
    keep = ts >= 30000
    assert 0.05 * T < (~keep).sum() < 0.2 * T
    assert np.array_equal(remap, np.where(keep, np.cumsum(keep) - 1, -1))
    # recount of every (entry, pattern) pair from the surviving traces
    count = np.bincount(ent[keep] * n_pat + pat[keep], minlength=n_ent * n_pat)
    pair_ent = np.repeat(np.arange(n_ent), np.diff(ent_ptr))
    c = count[pair_ent * n_pat + ent_pat]
    alive_pair = c > 0
    alive_pat = np.zeros(n_pat, dtype=bool)
    alive_pat[ent_pat[alive_pair]] = True
    newpat = np.cumsum(alive_pat) - 1
    tot = np.bincount(ent[keep], minlength=n_ent)
    assert n_pat - alive_pat.sum() >= 100
    assert s.rt_ids == [g for g, a in zip(rt_ids, alive_pat) if a]
    assert s.trace_keys == tid[keep].tolist()
    for name, v in (("trace_ts", ts[keep]), ("trace_entry", ent[keep])):
        assert np.array_equal(s.t[name].cpu().numpy(), v), name
    assert np.array_equal(ing.trace_pat.cpu().numpy(), newpat[pat[keep]])
    assert np.array_equal(s.t["ent_ptr"].cpu().numpy(),
                          np.concatenate([[0], np.cumsum(np.bincount(pair_ent[alive_pair], minlength=n_ent))]))
    assert np.array_equal(s.t["ent_pat"].cpu().numpy(), newpat[ent_pat[alive_pair]])
    assert np.array_equal(ing.cnt.cpu().numpy(), c[alive_pair]) and np.array_equal(ing.tot.cpu().numpy(), tot)
    prob = (c[alive_pair] / tot[pair_ent[alive_pair]]).astype(np.float32)
    assert np.array_equal(s.t["ent_prob"].cpu().numpy().view(np.int32), prob.view(np.int32))
    assert np.array_equal(s.t["pat_nptr"].diff().cpu().numpy(), nlen[alive_pat])
    assert np.array_equal(s.t["pat_eptr"].diff().cpu().numpy(), elen[alive_pat])
    assert np.array_equal(ing.tids.cpu().numpy(), np.sort(tid[keep]))


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="one visible device")
def test_second_device():
    cols, res, n_ms = _fixture()
    s = _store(cols, "pert", res, n_ms, dev="cuda:1")
    with torch.cuda.device(0):
        s.evict_traces(30000)
    w = TraceWindow()
    w.append(cols)
    w.evict(30000)
    _assert_same(s, _want(w, "pert", res, n_ms, dev="cuda:1"))
    assert all(v.device == torch.device("cuda:1") for v in s.t.values())
