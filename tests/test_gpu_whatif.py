"""-m gpu: what-if request assembly (PatternStore.assemble_requests with mixes, overrides and scenario ids),
PatternStore.lookup_resources and what-if prediction (train.predict).

A request carrying its entry's own stored mix must assemble bit for bit as the plain request (and so as the reference's
Data objects, tests/golden/ref_loop.npz); a request carrying another mix as the plain request of a store built with
that mix as the entry's; a full batch as a numpy restatement from the store's host tables, with override rows and the
joins of oracle/asof_oracle.py; lookup_resources as the oracle's joins.  Prediction must follow assembly."""
import os

import numpy as np
import pytest
import torch

from oracle import asof_oracle as A
from tests.helpers import assert_close

pytestmark = pytest.mark.gpu

OUT_KEYS = ("x", "edge_index", "edge_attr", "cat_X", "node_depth", "pattern_num_nodes", "pattern_probs", "entry_id",
            "rt_probs", "batch", "ptr")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _equal(got, want, what=""):
    for k in OUT_KEYS:
        assert got[k].shape == want[k].shape and torch.equal(got[k], want[k]), (what, k)


def _csr(mixes):
    """[(runtime ids, probabilities)] per request -> (mix_ptr, mix_rt, mix_prob) host arrays."""
    ptr = np.concatenate([[0], np.cumsum([len(r) for r, _ in mixes])]).astype(np.int64)
    rt = np.concatenate([np.asarray(r, dtype=np.int64) for r, _ in mixes]) if mixes else np.zeros(0, np.int64)
    pr = np.concatenate([np.asarray(p, dtype=np.float64) for _, p in mixes]) if mixes else np.zeros(0)
    return ptr, rt, pr


def _own_mixes(store, ent):
    """Every request's entry's stored mix: runtime ids rt_ids[ent_pat], fp32 ent_prob passed as float64."""
    ptr, pat, prob = (store.t[k].cpu().numpy() for k in ("ent_ptr", "ent_pat", "ent_prob"))
    return [([store.rt_ids[p] for p in pat[ptr[e]:ptr[e + 1]]], prob[ptr[e]:ptr[e + 1]].astype(np.float64))
            for e in ent]


def _random_mixes(store, Q, rng):
    """Subsets and reorderings of all runtimes (so also runtimes never seen under the entry), a single runtime at 1.0,
    weights not summing to 1."""
    out = []
    for q in range(Q):
        k = 1 if q % 5 == 0 else int(rng.integers(1, 5))
        rts = [store.rt_ids[i] for i in rng.choice(len(store.rt_ids), k, replace=False)]
        p = np.ones(1) if q % 5 == 0 else rng.random(k) * 2
        out.append((rts, p))
    return out


def _restate(store, ent, ts, mixes, asof, res, overrides=None, scen=None):
    """The what-if batch from the store's host tables: patterns of every mix in order, the oracle's resource joins
    (``res`` = the store's (resource_index, resource_values) in arrival order) and the first override row of
    (scenario, ms).  -> dict of host arrays, and per node whether the exact join misses a row it needs."""
    h = {k: store.t[k].cpu().numpy() for k in ("pat_nptr", "pat_eptr", "pat_ms", "pat_depth", "pat_last", "pat_src",
                                                "pat_dst", "pat_attr", "ms_has_res")}
    rt_index = {r: i for i, r in enumerate(store.rt_ids)}
    f = {k: [] for k in ("g", "eg", "off", "pnn", "rtp", "batch", "pp")}
    ptr, nb = [0], 0
    for b, (rts, probs) in enumerate(mixes):
        for r, pr in zip(rts, np.asarray(probs, dtype=np.float64).astype(np.float32)):
            p = rt_index[r]
            g = np.arange(h["pat_nptr"][p], h["pat_nptr"][p + 1])
            eg = np.arange(h["pat_eptr"][p], h["pat_eptr"][p + 1])
            f["g"].append(g)
            f["eg"].append(eg)
            f["off"].append(np.full(eg.shape[0], nb, dtype=np.int64))
            f["pnn"].append(np.full(g.shape[0], g.shape[0], dtype=np.float32))
            f["rtp"].append(np.full(g.shape[0], pr, dtype=np.float32))
            f["batch"].append(np.full(g.shape[0], b, dtype=np.int64))
            f["pp"].append(pr)
            nb += g.shape[0]
        ptr.append(nb)
    g, eg, owner = np.concatenate(f["g"]), np.concatenate(f["eg"]), np.concatenate(f["batch"])
    off = np.concatenate(f["off"])
    ms = h["pat_ms"][g]
    last = h["pat_last"][g] == 1
    ov = np.full(g.shape[0], -1, dtype=np.int64)
    if overrides is not None:
        first = {}
        for i, key in enumerate(zip(*overrides[:2])):
            first.setdefault((int(key[0]), int(key[1])), i)
        s = np.asarray(scen)[owner]
        ov = np.array([first.get((int(a), int(m)), -1) if a >= 0 else -1 for a, m in zip(s, ms)], dtype=np.int64)
        ov[~last] = -1
    need = last & (h["ms_has_res"][ms] == 1) & (ov < 0)
    res_ts = np.array([t for t, _ in res[0]], dtype=np.int64)
    res_ms = np.array([m for _, m in res[0]], dtype=np.int64)
    rows = np.full(g.shape[0], -1, dtype=np.int64)
    rows[need] = (A.asof_rows if asof else A.exact_rows)(res_ts, res_ms, A.time_bucket(ts)[owner[need]], ms[need])
    x = A.features(rows, res[1])
    if overrides is not None:
        hit = ov >= 0
        x[hit, :8] = np.asarray(overrides[2], dtype=np.float64).astype(np.float32)[ov[hit]]
        x[hit, 8] = 0
    want = {"x": x, "cat_X": ms.reshape(-1, 1), "node_depth": h["pat_depth"][g].reshape(-1, 1),
            "pattern_num_nodes": np.concatenate(f["pnn"]).reshape(-1, 1),
            "rt_probs": np.concatenate(f["rtp"]).reshape(-1, 1), "batch": owner,
            "edge_index": np.stack([h["pat_src"][eg] + off, h["pat_dst"][eg] + off]).astype(np.int64),
            "edge_attr": h["pat_attr"][eg], "entry_id": np.asarray(ent, dtype=np.int64),
            "ptr": np.asarray(ptr, dtype=np.int64), "pattern_probs": np.asarray(f["pp"], np.float32).reshape(-1, 1)}
    return want, need & (rows < 0)


def _equal_restated(got, want):
    for k in OUT_KEYS:
        assert np.array_equal(got[k].cpu().numpy(), want[k]), k


def _sparse_art(seed=11):
    """Trace artefacts whose resource table covers buckets -60000 .. 180000 with ~30 % of the rows dropped (whole
    buckets included) and a few duplicate keys carrying other values."""
    from pert_gnn_kdd23_b200.synthetic import make_trace_artifacts

    art = make_trace_artifacts(seed, n_entries=10, n_traces=40)
    rng = np.random.default_rng(seed)
    res_ms = sorted({m for _, m in art["resource_index"]})
    buckets = [30000 * k for k in range(-2, 7)]
    index = [(b, m) for b in buckets if b not in (0, 120000) for m in res_ms]      # two whole buckets missing
    keep = rng.random(len(index)) < 0.85
    index = [ix for ix, k in zip(index, keep) if k]
    dup = rng.choice(len(index), 6, replace=False)
    index = index + [index[i] for i in dup]
    index = [index[i] for i in rng.permutation(len(index))]
    art["resource_index"] = index
    art["resource_values"] = rng.random((len(index), 8))
    return art


def _res(art):
    return art["resource_index"], art["resource_values"]


# ------------------------------------------------------------------------------------- 1. identity: the own mix
def test_own_mix_equals_plain_requests():
    from pert_gnn_kdd23_b200.store import PatternStore
    from pert_gnn_kdd23_b200.synthetic import make_trace_artifacts

    g = np.load(os.path.join(ROOT, "tests", "golden", "ref_loop.npz"))
    art = make_trace_artifacts(int(g["hyper"][0]))
    store = PatternStore.from_artifacts(art, "cuda")
    ent = store._h_trace_entry.astype(np.int64)
    ts = np.array([int(art["tr2data"][k]["timestamp"]) for k in store.trace_keys], dtype=np.int64)
    mixes = _csr(_own_mixes(store, ent))
    for r in (0, 1, 29999):
        for asof in (False, True):
            want = store.assemble_requests(ent, ts + r, asof=asof)
            got = store.assemble_requests(ent, ts + r, asof=asof, mixes=mixes)
            _equal(got, want, (r, asof))
            assert "y" not in got
            # no mixes, only an empty scenario: the entries' own mixes through the what-if kernels
            _equal(store.assemble_requests(ent, ts + r, asof=asof, scenario_ids=np.full(len(ent), -1)), want)
    store.check()
    # so every trace is also its own reference Data object
    for i in range(0, len(ent), 7):
        got = store.assemble_requests(ent[i:i + 1], ts[i:i + 1], mixes=_csr(_own_mixes(store, ent[i:i + 1])))
        for k in ("x", "edge_index", "edge_attr", "cat_X", "node_depth", "pattern_num_nodes", "pattern_probs"):
            assert np.array_equal(got[k].cpu().numpy(), g[f"d{i}_{k}"]), (i, k)


# ------------------------------------------------------------------------------- 2. mixes vs the constructor
def test_mixes_equal_a_store_built_with_them():
    from pert_gnn_kdd23_b200.store import PatternStore
    from pert_gnn_kdd23_b200.synthetic import make_trace_artifacts

    art = make_trace_artifacts(5)
    store = PatternStore.from_artifacts(art, "cuda")
    rng = np.random.default_rng(0)
    n_ent = len(art["entry2runtimes"])
    mixes = _random_mixes(store, 8, rng)
    ent = rng.integers(0, n_ent, 8)
    ts = 60000 * rng.integers(1, 6, 8) + rng.integers(0, 30000, 8)
    for q, (rts, p) in enumerate(mixes):
        e2r = dict(art["entry2runtimes"])
        e2r[int(ent[q])] = {int(r): float(v) for r, v in zip(rts, p)}               # an ordered dict: the mix order
        other = PatternStore.from_artifacts(dict(art, entry2runtimes=e2r), "cuda")
        assert other.rt_ids == store.rt_ids
        for asof in (False, True):
            want = other.assemble_requests(ent[q:q + 1], ts[q:q + 1], asof=asof)
            got = store.assemble_requests(ent[q:q + 1], ts[q:q + 1], asof=asof, mixes=_csr([mixes[q]]))
            _equal(got, want, (q, asof))
    # a full batch against the restatement
    Q = 300
    mixes = _random_mixes(store, Q, rng)
    ent = rng.integers(0, n_ent, Q)
    ts = 60000 * rng.integers(1, 6, Q) + rng.integers(0, 30000, Q)
    for asof in (False, True):
        got = store.assemble_requests(ent, ts, asof=asof, mixes=_csr(mixes))
        want, _ = _restate(store, ent, ts, mixes, asof, _res(art))
        _equal_restated(got, want)
    store.check()


def test_a_mix_may_use_an_entry_without_patterns():
    from pert_gnn_kdd23_b200 import _lib
    from pert_gnn_kdd23_b200.store import PatternStore
    from pert_gnn_kdd23_b200.synthetic import make_trace_artifacts

    art = make_trace_artifacts(7)
    n0 = len(art["entry2runtimes"])
    art["entry2runtimes"][n0 + 1] = dict(art["entry2runtimes"][1])     # entry n0 has no patterns
    store = PatternStore.from_artifacts(art, "cuda")
    mix = ([store.rt_ids[3], store.rt_ids[0]], [0.25, 0.5])
    got = store.assemble_requests([n0], [60000], mixes=_csr([mix]))
    want, _ = _restate(store, [n0], np.array([60000]), [mix], False, _res(art))
    _equal_restated(got, want)
    store.check()
    with pytest.raises(_lib.PertGnnError, match=f"request 0: entry {n0} has no patterns"):
        store.assemble_requests([n0], [60000], scenario_ids=[-1])


# ------------------------------------------------------------------ 3. identity: overrides equal to the joined row
def test_overrides_equal_to_the_joined_rows_change_nothing():
    from pert_gnn_kdd23_b200.store import PatternStore
    from pert_gnn_kdd23_b200.synthetic import make_trace_artifacts

    art = make_trace_artifacts(5)
    store = PatternStore.from_artifacts(art, "cuda")
    rng = np.random.default_rng(1)
    Q = 64
    ent = rng.choice(np.flatnonzero(store._h_ent_pats > 0), Q)
    ts = 60000 * rng.integers(1, 6, Q) + rng.integers(0, 30000, Q)
    pat_ms = store.t["pat_ms"].cpu().numpy()
    h = {k: store.t[k].cpu().numpy() for k in ("ent_ptr", "ent_pat", "pat_nptr")}
    for asof in (False, True):
        # one scenario per request, one row per microservice of its patterns: what lookup_resources reads for it
        sc, ms, q_ts = [], [], []
        for q, e in enumerate(ent):
            m = np.unique(np.concatenate([pat_ms[h["pat_nptr"][p]:h["pat_nptr"][p + 1]]
                                          for p in h["ent_pat"][h["ent_ptr"][e]:h["ent_ptr"][e + 1]]]))
            sc += [q] * len(m)
            ms += m.tolist()
            q_ts += [ts[q]] * len(m)
        vals, found = store.lookup_resources(np.array(q_ts), np.array(ms), asof=asof)
        keep = found.cpu().numpy()
        ov = (np.array(sc)[keep], np.array(ms)[keep], vals.cpu().numpy().astype(np.float64)[keep])
        want = store.assemble_requests(ent, ts, asof=asof)
        got = store.assemble_requests(ent, ts, asof=asof, overrides=ov, scenario_ids=np.arange(Q))
        _equal(got, want, asof)
    store.check()


# ------------------------------------------------------------------------------- 4. overrides vs the restatement
def test_overrides_match_the_restatement():
    from pert_gnn_kdd23_b200 import _lib
    from pert_gnn_kdd23_b200.store import PatternStore

    art = _sparse_art()
    store = PatternStore.from_artifacts(art, "cuda")
    rng = np.random.default_rng(2)
    Q = 400
    ent = rng.integers(0, 10, Q)
    ts = rng.integers(-4 * 30000, 9 * 30000, Q)
    ts[:8] = [-10 ** 9, -60001, -30001, -1, 0, 29999, 30000, 10 ** 12]
    has = store.t["ms_has_res"].cpu().numpy()
    no_res = np.flatnonzero(has == 0)
    with_res = np.flatnonzero(has == 1)
    assert no_res.size
    # 5 scenarios over 30 % of the resourced microservices and some without resources, with duplicate rows
    sc, ms = [], []
    for s in range(5):
        m = np.concatenate([rng.choice(with_res, int(0.3 * with_res.size), replace=False), no_res[:3]])
        sc += [s] * len(m)
        ms += m.tolist()
    dup = rng.choice(len(sc), 10, replace=False)
    sc, ms = np.array(sc + [sc[i] for i in dup]), np.array(ms + [ms[i] for i in dup])
    perm = rng.permutation(len(sc))
    ov = (sc[perm], ms[perm], rng.random((len(sc), 8)) * 10)
    scen = rng.integers(-1, 7, Q)                       # -1 and scenarios 5, 6 without rows mixed in
    mixes = _own_mixes(store, ent)
    for asof in (False, True):
        store.status.zero_()
        got = store.assemble_requests(ent, ts, asof=asof, overrides=ov, scenario_ids=scen)
        want, missing = _restate(store, ent, ts, mixes, asof, _res(art), overrides=ov, scen=scen)
        _equal_restated(got, want)
        if asof:
            store.check()
        else:
            assert missing.any()
            assert int(store.status.item()) == -3
        # requests whose only missing rows are overridden do not flag the exact join
        owner = want["batch"]
        clean = np.setdiff1d(np.arange(Q), owner[missing])
        store.status.zero_()
        store.assemble_requests(ent[clean], ts[clean], asof=asof, overrides=ov, scenario_ids=scen[clean])
        store.check()
        plain_missing = _restate(store, ent[clean], ts[clean], [mixes[i] for i in clean], asof, _res(art))[1]
        if not asof and plain_missing.any():            # ... where the plain requests do
            with pytest.raises(_lib.PertGnnError):
                store.assemble_requests(ent[clean], ts[clean])
                store.check()
        store.status.zero_()
    # overrides together with random mixes
    rm = _random_mixes(store, Q, rng)
    got = store.assemble_requests(ent, ts, asof=True, mixes=_csr(rm), overrides=ov, scenario_ids=scen)
    _equal_restated(got, _restate(store, ent, ts, rm, True, _res(art), overrides=ov, scen=scen)[0])


# -------------------------------------------------------------------------------------------- 5. lookup_resources
def test_lookup_resources_matches_the_oracle():
    from pert_gnn_kdd23_b200.store import PatternStore

    art = _sparse_art(12)
    store = PatternStore.from_artifacts(art, "cuda")
    rng = np.random.default_rng(3)
    k = 2000
    ts = rng.integers(-5 * 30000, 10 * 30000, k)
    ts[:6] = [-10 ** 12, -60001, -1, 0, 180000 + 29999, 10 ** 12]      # before the first, after the last bucket
    ms = rng.integers(-2, store.n_ms + 2, k)
    res_ts = np.array([t for t, _ in art["resource_index"]], dtype=np.int64)
    res_ms = np.array([m for _, m in art["resource_index"]], dtype=np.int64)
    inside = (ms >= 0) & (ms < store.n_ms)
    for asof in (False, True):
        rows = np.full(k, -1, dtype=np.int64)
        rows[inside] = (A.asof_rows if asof else A.exact_rows)(res_ts, res_ms, A.time_bucket(ts)[inside], ms[inside])
        vals, found = store.lookup_resources(ts, torch.from_numpy(ms).cuda(), asof=asof)
        assert vals.dtype == torch.float32 and found.dtype == torch.bool and vals.shape == (k, 8)
        assert np.array_equal(found.cpu().numpy(), rows >= 0)
        assert np.array_equal(vals.cpu().numpy(), A.features(rows, art["resource_values"])[:, :8])
        assert (rows >= 0).any() and (rows < 0).any()
    v, f = store.lookup_resources([], [])
    assert v.shape == (0, 8) and f.shape == (0,)


# ------------------------------------------------------------------------------------------------ 6. live updates
def test_mixes_across_appends_and_evictions():
    from pert_gnn_kdd23_b200 import _lib
    from pert_gnn_kdd23_b200.store import PatternStore
    from pert_gnn_kdd23_b200.synthetic import make_trace_table
    from pert_gnn_kdd23_b200.tracegroup import group_traces
    from tests.trace_window_ref import TraceWindow

    d = make_trace_table(5)
    cols, res, n_ms = d["columns"], (d["resource_index"], d["resource_values"]), d["n_ms"]
    tids = np.unique(cols["traceid"])
    part = lambda m: {k: v[m] for k, v in cols.items()}          # noqa: E731
    chunks = [part(np.isin(cols["traceid"], c)) for c in np.array_split(tids, 3)]
    store = PatternStore.from_trace_groups(group_traces(chunks[0], "cuda").check(), "span", *res, "cuda", n_ms=n_ms)
    w = TraceWindow()
    w.append(chunks[0])
    rng = np.random.default_rng(4)

    def check(s):
        assert np.array_equal(s._h_pat_nodes, s.t["pat_nptr"].diff().cpu().numpy())
        assert np.array_equal(s._h_pat_edges, s.t["pat_eptr"].diff().cpu().numpy())
        r2g, e2r, tr = w.store_dicts("span", "cuda")
        rebuilt = PatternStore(r2g, e2r, *res, tr, "cuda", n_ms=n_ms)
        assert rebuilt.rt_ids == s.rt_ids
        Q = 60
        mixes = _random_mixes(s, Q, rng)
        ent = rng.integers(0, int(s.desc.n_ent), Q)
        ts = 30000 * rng.integers(0, 12, Q) + rng.integers(0, 30000, Q)
        got = s.assemble_requests(ent, ts, asof=True, mixes=_csr(mixes))
        _equal(got, rebuilt.assemble_requests(ent, ts, asof=True, mixes=_csr(mixes)))
        _equal_restated(got, _restate(s, ent, ts, mixes, True, res)[0])
        return mixes

    mixes = check(store)
    for c in chunks[1:]:
        store.append_traces(c)
        w.append(c)
        check(store)
    cut = int(store.t["trace_ts"].min()) + 30000
    before = list(store.rt_ids)
    store.evict_traces(cut)
    w.evict(cut)
    gone = sorted(set(before) - set(store.rt_ids))
    check(store)
    if gone:
        mix = ([store.rt_ids[0], gone[0]], [0.5, 0.5])
        with pytest.raises(_lib.PertGnnError, match=f"request 1: runtime {gone[0]} is not in the store"):
            store.assemble_requests([0, 0], [0, 0], mixes=_csr([_random_mixes(store, 1, rng)[0], mix]))
    store.evict_traces(1 << 62)                           # every trace: no pattern is left, every runtime is evicted
    assert store._h_pat_nodes.shape == (0,) and store._h_pat_edges.shape == (0,)
    with pytest.raises(_lib.PertGnnError, match="is not in the store"):
        store.assemble_requests([0], [0], mixes=_csr([mixes[0]]))


# ----------------------------------------------------------------------------------------------- 7.-9. predict
@pytest.fixture(scope="module")
def pert_store():
    from pert_gnn_kdd23_b200.store import PatternStore
    from pert_gnn_kdd23_b200.synthetic import make_pert_artifacts

    art, _ = make_pert_artifacts(seed=3, n_patterns=64, n_entries=24, n_traces=400, device="cuda")
    return art, PatternStore.from_artifacts(art, "cuda")


def _trained_model(store, hidden=64, p=0.0, steps=4):
    from pert_gnn_kdd23_b200.model import SAGEDeterministic
    from pert_gnn_kdd23_b200.store import StoreLoader
    from pert_gnn_kdd23_b200.synthetic import model_args
    from pert_gnn_kdd23_b200.train import FlatParams, FusedAdam, fused_train_step

    torch.manual_seed(0)
    args = list(model_args(2))
    args[5] = hidden
    m = SAGEDeterministic(*args).cuda()
    m.dropout = p
    m.seed_dropout(77)
    opt = FusedAdam(FlatParams(m), lr=1e-3)
    for i, d in enumerate(StoreLoader(store, list(range(len(store))), 64)):
        if i >= steps:
            break
        fused_train_step(m, opt, d, 0.5)
    return m, opt


def _requests(store, Q, seed):
    rng = np.random.default_rng(seed)
    ok = np.flatnonzero(store._h_ent_pats > 0)
    return rng.choice(ok, Q), 60000 * rng.integers(1, 6, Q) + rng.integers(0, 30000, Q)


def _same_or_close(got, want, what):
    same = torch.equal(got, want)
    print(f"{what}: {'bitwise equal' if same else 'not bitwise equal'}")
    if not same:
        assert_close(got, want, what=what)


@pytest.mark.parametrize("asof", [False, True])
def test_predict_own_mixes_equal_plain_predict(pert_store, asof):
    from pert_gnn_kdd23_b200.train import predict

    art, store = pert_store
    model, _ = _trained_model(store)
    ent, ts = _requests(store, 500, 1)
    want = predict(model, store, ent, ts, batch_size=96, asof=asof)
    got = predict(model, store, ent, ts, batch_size=96, asof=asof, mixes=_csr(_own_mixes(store, ent)))
    _same_or_close(got, want, f"own-mix predict vs plain predict (asof={asof})")
    store.check()


def test_predict_under_a_scenario_and_mixes_equals_the_rebuilt_store(pert_store):
    from pert_gnn_kdd23_b200.store import PatternStore
    from pert_gnn_kdd23_b200.train import predict

    art, store = pert_store
    model, _ = _trained_model(store)
    rng = np.random.default_rng(5)
    Q = 400
    ent, ts = _requests(store, Q, 2)
    # one mix per entry, the same for all its requests, so a store built with those mixes answers the plain requests
    per_ent = dict(zip(np.unique(ent).tolist(), _random_mixes(store, len(np.unique(ent)), rng)))
    mixes = [per_ent[int(e)] for e in ent]
    e2r = dict(art["entry2runtimes"])
    for e, (rts, p) in per_ent.items():
        e2r[e] = {int(r): float(v) for r, v in zip(rts, p)}
    # scenario 0 overrides 10 % of the resourced microservices at every bucket; the rebuilt store's rows of those
    # microservices are the override values, at the buckets the requests read
    res_ms = np.unique([m for _, m in art["resource_index"]])
    o_ms = rng.choice(res_ms, max(1, res_ms.size // 10), replace=False)
    o_vals = rng.random((o_ms.size, 8))
    buckets = np.unique(A.time_bucket(ts)).tolist()
    o_set = set(o_ms.tolist())
    keep = [i for i, (_, m) in enumerate(art["resource_index"]) if int(m) not in o_set]
    index = [art["resource_index"][i] for i in keep] + [(b, int(m)) for b in buckets for m in o_ms]
    values = np.concatenate([np.asarray(art["resource_values"])[keep], np.tile(o_vals, (len(buckets), 1))])
    rebuilt = PatternStore.from_artifacts(dict(art, entry2runtimes=e2r, resource_index=index,
                                               resource_values=values), "cuda")
    ov = (np.zeros(o_ms.size, dtype=np.int64), o_ms, o_vals)
    for asof in (False, True):
        got = predict(model, store, ent, ts, batch_size=128, asof=asof, mixes=_csr(mixes), overrides=ov,
                      scenario_ids=np.zeros(Q, dtype=np.int64))
        want = predict(model, rebuilt, ent, ts, batch_size=128, asof=asof)
        _same_or_close(got, want, f"what-if predict vs the rebuilt store (asof={asof})")
        rebuilt.check()
        store.check()


def test_what_if_predict_replays_sets_node_ptr_and_has_no_side_effects(pert_store):
    from pert_gnn_kdd23_b200.train import predict

    art, store = pert_store
    model, opt = _trained_model(store, p=0.2)
    ent, ts = _requests(store, 640, 6)
    rng = np.random.default_rng(7)
    mixes = _random_mixes(store, 640, rng)
    scen = rng.integers(-1, 2, 640)
    res_ms = np.unique([m for _, m in art["resource_index"]])
    ov = (np.repeat([0, 1], 5), rng.choice(res_ms, 10), rng.random((10, 8)))
    kw = dict(batch_size=64, asof=True, mixes=_csr(mixes), overrides=ov, scenario_ids=scen)
    eng = model.engine()
    before = [opt.fp.flat.clone(), eng.bn_running.clone(), eng.bn_nbt.clone(), model.dropout_state().clone(),
              opt.m.clone(), opt.v.clone(), opt.fp.grad.clone()]
    first = predict(model, store, ent, ts, **kw)
    predict(model, store, ent, ts, **kw)
    st = model.__dict__["_bucketed_predict"]
    c0, r0 = st.captures, st.replays
    third, loc, node_ptr = predict(model, store, ent, ts, local=True, **kw)
    assert st.capture_error is None, st.capture_error
    assert st.captures == c0 and st.replays - r0 == 10                # every batch replayed, nothing captured again
    assert_close(third, first, what="repeated what-if predict")
    sizes = [sum(int(store._h_pat_nodes[store.rt_ids.index(r)]) for r in rts) for rts, _ in mixes]
    assert node_ptr.tolist() == np.concatenate([[0], np.cumsum(sizes)]).tolist()
    assert loc.shape == (sum(sizes),)
    torch.cuda.synchronize()
    after = [opt.fp.flat, eng.bn_running, eng.bn_nbt, model.dropout_state(), opt.m, opt.v, opt.fp.grad]
    for k, (b, a) in enumerate(zip(before, after)):
        assert torch.equal(b, a), k
    assert model.training and model._engine is eng
    # a plain call whose batches land in the what-if call's buckets replays those graphs too
    own = predict(model, store, ent, ts, batch_size=64, asof=True, mixes=_csr(_own_mixes(store, ent)))
    _same_or_close(own, predict(model, store, ent, ts, batch_size=64, asof=True), "own mixes after what-if calls")


# --------------------------------------------------------------------------------------------- 10. second device
@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs a second CUDA device")
def test_second_device():
    from pert_gnn_kdd23_b200.store import PatternStore

    art = _sparse_art()
    s0, s1 = (PatternStore.from_artifacts(art, f"cuda:{i}") for i in (0, 1))
    rng = np.random.default_rng(8)
    ent, ts = rng.integers(0, 10, 50), rng.integers(0, 6 * 30000, 50)
    mixes = _csr(_random_mixes(s0, 50, rng))
    ov = (np.array([0, 0, 1]), np.array([1, 2, 3]), rng.random((3, 8)))
    scen = rng.integers(-1, 2, 50)
    a, b = (s.assemble_requests(ent, ts, asof=True, mixes=mixes, overrides=ov, scenario_ids=scen) for s in (s0, s1))
    assert b.x.device == torch.device("cuda:1")
    for k in OUT_KEYS:
        assert torch.equal(a[k].cpu(), b[k].cpu()), k
    v0, f0 = s0.lookup_resources(ts, np.full(50, 2))
    v1, f1 = s1.lookup_resources(ts, np.full(50, 2))
    assert v1.device == torch.device("cuda:1") and torch.equal(v0.cpu(), v1.cpu()) and torch.equal(f0.cpu(), f1.cpu())
