"""CPU tests of what-if request assembly (PatternStore.assemble_requests / train.predict with mixes, overrides and
scenario ids; PatternStore.lookup_resources): the host-side resolution of runtime ids against a brute-force loop, every
host check with the first bad request, row or runtime named (no launch, the store untouched), and the argument checks
of pert_store_assemble_whatif and pert_store_lookup_resources (no CUDA call is made for a rejected call)."""
import copy
import ctypes as C

import numpy as np
import pytest

RT_IDS = [7, 3, 11, 40, 5, 22]                      # the store's runtime ids, not sorted
N_MS = 9


def _host_store(rng=None):
    from pert_gnn_kdd23_b200.store import PatternStore

    rng = rng or np.random.default_rng(0)
    store = PatternStore.__new__(PatternStore)
    store.rt_ids = list(RT_IDS)
    store.n_ms = N_MS
    store._h_pat_nodes = rng.integers(1, 30, len(RT_IDS)).astype(np.int64)
    store._h_pat_edges = rng.integers(0, 60, len(RT_IDS)).astype(np.int64)
    n_ent = 6
    store._h_ent_nodes = rng.integers(3, 90, n_ent).astype(np.int64)
    store._h_ent_edges = rng.integers(0, 90, n_ent).astype(np.int64)
    store._h_ent_pats = rng.integers(1, 4, n_ent).astype(np.int64)
    for a in (store._h_ent_nodes, store._h_ent_edges, store._h_ent_pats):
        a[4] = 0                                    # entry 4 has no patterns (e.g. all its traces were evicted)
    return store


def _state(store):
    return copy.deepcopy({k: v for k, v in store.__dict__.items()})


def _same(a, b):
    assert a.keys() == b.keys()
    for k in a:
        if isinstance(a[k], np.ndarray):
            assert np.array_equal(a[k], b[k]), k
        else:
            assert a[k] == b[k], k


@pytest.mark.parametrize("ids", [RT_IDS, [3 << 40, -7, 11, 1 << 50, 5, 22]])    # compact ids and sparse ones
def test_mixes_resolve_to_pattern_indices_and_sizes(ids):
    from pert_gnn_kdd23_b200.store import _resolve_mixes

    rng = np.random.default_rng(1)
    store = _host_store(rng)
    store.rt_ids = list(ids)
    for _ in range(20):
        Q = int(rng.integers(1, 12))
        lens = rng.integers(1, len(ids) + 1, Q)
        rts = [rng.choice(ids, n, replace=False) for n in lens]
        ptr = np.concatenate([[0], np.cumsum(lens)])
        rt = np.concatenate(rts)
        prob = rng.random(rt.shape[0]) * 3           # not normalised
        p, pat, pr, nodes, edges, pats = _resolve_mixes((ptr, rt, prob), Q, store.rt_ids, store._h_pat_nodes,
                                                        store._h_pat_edges)
        assert p.dtype == np.int64 and pat.dtype == np.int32 and pr.dtype == np.float32
        assert np.array_equal(p, ptr)
        assert [ids[i] for i in pat] == rt.tolist()
        assert np.array_equal(pr, prob.astype(np.float32))
        for q in range(Q):
            sl = [ids.index(r) for r in rts[q]]
            assert nodes[q] == store._h_pat_nodes[sl].sum() and edges[q] == store._h_pat_edges[sl].sum()
            assert pats[q] == lens[q]
    # float32 probabilities pass through unchanged, tensors are accepted
    import torch

    p32 = np.array([0.1, 0.7], dtype=np.float32)
    out = _resolve_mixes((torch.tensor([0, 1, 2]), torch.tensor([ids[3], ids[1]]), p32), 2, store.rt_ids,
                         store._h_pat_nodes, store._h_pat_edges)
    assert np.array_equal(out[2], p32) and out[1].tolist() == [3, 1]
    # ids the store does not hold, inside and outside the range of its ids
    for bad in (min(ids) - 1, max(ids) + 1, 6):
        with pytest.raises(Exception, match=f"runtime {bad} is not in the store"):
            _resolve_mixes((np.array([0, 1]), np.array([bad]), np.ones(1)), 1, store.rt_ids, store._h_pat_nodes,
                           store._h_pat_edges)


GOOD_MIX = (np.array([0, 2, 3, 5]), np.array([7, 3, 11, 40, 5]), np.array([0.5, 0.5, 1.0, 0.2, 0.9]))


@pytest.mark.parametrize("mixes, match", [
    ("nope", "triple expected"),
    ((np.array([0, 2, 3]), GOOD_MIX[1], GOOD_MIX[2]), "mix_ptr: 3 offsets, expected 4 for 3 requests"),
    ((np.array([1, 2, 3, 5]), GOOD_MIX[1], GOOD_MIX[2]), r"mix_ptr\[0\] = 1"),
    ((np.array([0, 3, 2, 5]), GOOD_MIX[1], GOOD_MIX[2]), "request 1: mix_ptr is not monotone"),
    ((np.array([0, 2, 3, 4]), GOOD_MIX[1], GOOD_MIX[2]), r"mix_ptr\[3\] = 4, but mix_rt holds 5"),
    ((np.array([0, 2, 2, 5]), GOOD_MIX[1], GOOD_MIX[2]), "request 1: empty mix"),
    ((np.array([0., 2, 3, 5]), GOOD_MIX[1], GOOD_MIX[2]), "mix_ptr: a 1-d array of int64"),
    ((GOOD_MIX[0], GOOD_MIX[1].astype(float), GOOD_MIX[2]), "mix_rt: a 1-d array of int64"),
    ((GOOD_MIX[0], GOOD_MIX[1], GOOD_MIX[2][:4]), r"mix_prob: shape \(4,\), expected \(5,\)"),
    ((GOOD_MIX[0], GOOD_MIX[1], ["a"] * 5), "mix_prob: numbers expected"),
    ((GOOD_MIX[0], np.array([7, 3, 11, 41, 5]), GOOD_MIX[2]), "request 2: runtime 41 is not in the store"),
    ((GOOD_MIX[0], np.array([7, 3, 11, 40, 40]), GOOD_MIX[2]), "request 2: runtime 40 occurs twice"),
    ((GOOD_MIX[0], np.array([7, 7, 11, 40, 5]), GOOD_MIX[2]), "request 0: runtime 7 occurs twice"),
    ((GOOD_MIX[0], GOOD_MIX[1], np.array([0.5, 0.5, 1.0, -0.2, 0.9])), "request 2: probability -0.2 of runtime 40"),
    ((GOOD_MIX[0], GOOD_MIX[1], np.array([0.5, 0.5, np.nan, 0.2, 0.9])), "request 1: probability nan"),
    ((GOOD_MIX[0], GOOD_MIX[1], np.array([0.5, np.inf, 1.0, 0.2, 0.9])), "request 0: probability inf"),
    # the first bad request is named, whichever check it fails
    ((GOOD_MIX[0], np.array([7, 3, 99, 40, 40]), np.array([0.5, -1, 1.0, 0.2, 0.9])), "request 0: probability -1"),
])
def test_bad_mixes_are_refused(mixes, match):
    from pert_gnn_kdd23_b200._lib import PertGnnError

    store = _host_store()
    before = _state(store)
    with pytest.raises(PertGnnError, match=match):
        store._what_if_arrays([0, 1, 2], [0, 0, 0], mixes=mixes)
    _same(before, _state(store))


def test_entries_with_and_without_mixes():
    from pert_gnn_kdd23_b200._lib import PertGnnError

    store = _host_store()
    for ent, q in (([0, 6, 2], 1), ([0, 1, -1], 2)):
        with pytest.raises(PertGnnError, match=f"request {q}: entry {ent[q]} is outside"):
            store._what_if_arrays(ent, [0, 0, 0], mixes=GOOD_MIX)
    # without a mix the entry's own mix is read, so an entry without patterns is refused as in plain assembly
    with pytest.raises(PertGnnError, match="request 1: entry 4 has no patterns"):
        store._what_if_arrays([0, 4, 1], [0, 0, 0], scenario_ids=[0, 0, 0])
    with pytest.raises(PertGnnError, match="3 entry ids but 2 timestamps"):
        store._what_if_arrays([0, 4, 1], [0, 0], mixes=GOOD_MIX)


@pytest.mark.parametrize("overrides, match", [
    ("x", "triple expected"),
    (([0, 1], [2, 9], np.zeros((2, 8))), "override row 1: microservice 9 is outside"),
    (([0, 1, 2], [2, 3, -1], np.zeros((3, 8))), "override row 2: microservice -1 is outside"),
    (([0, -2], [2, 3], np.zeros((2, 8))), "override row 1: scenario -2 is negative"),
    (([0, (1 << 63) // N_MS], [2, 8], np.zeros((2, 8))), "override row 1: scenario .* overflows"),
    (([0, 1], [2, 3], np.zeros((2, 7))), r"shape \(2, 7\), expected \(2, 8\)"),
    (([0, 1], [2, 3], [["a"] * 8] * 2), "overrides values: .* numbers expected"),
    (([0, 1], [2], np.zeros((2, 8))), "2 scenario ids but 1 microservices"),
    (([0.0, 1], [2, 3], np.zeros((2, 8))), "overrides scenario: a 1-d array of int64"),
])
def test_bad_overrides_are_refused(overrides, match):
    from pert_gnn_kdd23_b200._lib import PertGnnError

    store = _host_store()
    before = _state(store)
    with pytest.raises(PertGnnError, match=match):
        store._what_if_arrays([0, 1, 2], [0, 0, 0], mixes=GOOD_MIX, overrides=overrides, scenario_ids=[0, -1, 1])
    _same(before, _state(store))


def test_override_keys_and_the_largest_scenario():
    from pert_gnn_kdd23_b200.store import _override_rows

    s_max = ((1 << 63) - 1 - (N_MS - 1)) // N_MS          # every ms of this scenario fits
    keys, vals = _override_rows(([3, 0, s_max], [1, 8, 8], np.arange(24.).reshape(3, 8) / 7), N_MS)
    assert keys.tolist() == [3 * N_MS + 1, 8, s_max * N_MS + 8] and vals.dtype == np.float32
    assert np.array_equal(vals, (np.arange(24.).reshape(3, 8) / 7).astype(np.float32))
    keys, vals = _override_rows(((), (), ()), N_MS)
    assert keys.shape == (0,) and vals.shape == (0, 8)


@pytest.mark.parametrize("scen, match", [([0, -2, 1], "request 1: scenario id -2 is below -1"),
                                         ([0, 1], "3 requests but 2 scenario ids"),
                                         ([0, 1.5, 1], "scenario_ids: a 1-d array of int64")])
def test_bad_scenario_ids_are_refused(scen, match):
    from pert_gnn_kdd23_b200._lib import PertGnnError

    store = _host_store()
    with pytest.raises(PertGnnError, match=match):
        store._what_if_arrays([0, 1, 2], [0, 0, 0], mixes=GOOD_MIX, scenario_ids=scen)


def test_totals_above_int32_are_refused():
    from pert_gnn_kdd23_b200._lib import PertGnnError
    from pert_gnn_kdd23_b200.store import _WhatIfArrays

    store = _host_store()
    big = np.array([1 << 30, 1 << 30], dtype=np.int64)
    one = np.ones(2, dtype=np.int64)
    for nodes, edges, pats, what in ((big, one, one, "nodes"), (one, big, one, "edges"), (one, one, big, "patterns")):
        w = _WhatIfArrays(np.zeros(2, dtype=np.int64), nodes, edges, pats, None, None, None, None, None, None, None,
                          None)
        with pytest.raises(PertGnnError, match=f"{1 << 31} {what}"):
            store._assemble_what_if(w, False)


def test_device_arrays_of_a_plain_call_are_refused_with_what_if_inputs():
    from pert_gnn_kdd23_b200._lib import PertGnnError

    store = _host_store()
    store.device = None
    with pytest.raises(PertGnnError, match="what-if call takes its inputs on the host"):
        store.assemble_requests([0], [0], device_arrays=(None, None), scenario_ids=[0])


# ------------------------------------------------------------------------------------------------ C-ABI checks
def _store_desc():
    from pert_gnn_kdd23_b200._lib import PertStore

    d = PertStore()
    d.n_pat, d.n_ent, d.n_res, d.n_ms, d.attr_cols, d.n_traces = 2, 2, 3, 4, 2, 0
    for name, _ in PertStore._fields_[6:]:
        setattr(d, name, 16)                                  # non-NULL, never dereferenced on the host
    return d


def _whatif(**over):
    from pert_gnn_kdd23_b200._lib import PertWhatIf

    f = dict(mix_ptr=16, mix_pat=16, mix_prob=16, scenario=16, n_ov=3, ov_keys=16, ov_vals=32)
    f.update(over)
    return PertWhatIf(**f)


def _args(**over):
    from pert_gnn_kdd23_b200._lib import PertResourceAsOf
    from pert_gnn_kdd23_b200._lib import PertBatchOut

    a = dict(store=C.byref(_store_desc()), asof=None, w=C.byref(_whatif()), entry_ids=16, timestamps=16, B=2, N=10,
             E=20, offsets=16, out=C.byref(PertBatchOut()), status=None, stream=None)
    if over.pop("with_asof", False):
        a["asof"] = C.byref(PertResourceAsOf(16, 16, 16))
    a.update(over)
    return list(a.values())


@pytest.mark.parametrize("over", [
    {"store": None}, {"out": None}, {"w": None}, {"B": -1}, {"N": -1}, {"E": -1}, {"entry_ids": None},
    {"timestamps": None}, {"offsets": None}, {"entry_ids": None, "with_asof": True},
    {"w": "mix_pat"}, {"w": "mix_prob"}, {"w": "ov_keys"}, {"w": "ov_vals"}, {"w": "neg_ov"}, {"w": "misaligned"},
])
def test_assemble_whatif_rejects_bad_arguments(over):
    from pert_gnn_kdd23_b200 import _lib

    w = over.get("w", "")
    if isinstance(w, str) and w:
        over = dict(w=C.byref({"mix_pat": _whatif(mix_pat=None), "mix_prob": _whatif(mix_prob=None),
                               "ov_keys": _whatif(ov_keys=None), "ov_vals": _whatif(ov_vals=None),
                               "neg_ov": _whatif(n_ov=-1), "misaligned": _whatif(ov_vals=36)}[w]))
    assert _lib.lib().pert_store_assemble_whatif(*_args(**over)) == -1


def test_assemble_whatif_accepts_what_it_does_not_read():
    from pert_gnn_kdd23_b200 import _lib

    L = _lib.lib()
    # B = 0 returns before any CUDA call; without a mix, mix_pat / mix_prob are not read; without rows, no table
    for w in (_whatif(mix_ptr=None, mix_pat=None, mix_prob=None), _whatif(n_ov=0, ov_keys=None, ov_vals=None),
              _whatif(scenario=None), _whatif(mix_ptr=None, mix_pat=None, mix_prob=None, scenario=None, n_ov=0,
                                              ov_keys=None, ov_vals=None)):
        assert L.pert_store_assemble_whatif(*_args(w=C.byref(w), B=0, N=0, E=0)) == 0
    assert L.pert_store_assemble_whatif(*_args(B=0, N=0, E=0, entry_ids=None, timestamps=None, offsets=None)) == 0
    d = _store_desc()
    d.ent_prob = None
    assert L.pert_store_assemble_whatif(*_args(store=C.byref(d), B=0, N=0, E=0)) == -1


def _lookup_args(**over):
    from pert_gnn_kdd23_b200._lib import PertResourceAsOf

    a = dict(store=C.byref(_store_desc()), asof=None, timestamps=16, ms=16, k=5, values=16, found=16, stream=None)
    if over.pop("with_asof", False):
        a["asof"] = C.byref(PertResourceAsOf(16, 16, 16))
    a.update(over)
    return list(a.values())


@pytest.mark.parametrize("over", [
    {"store": None}, {"k": -1}, {"k": 1 << 31}, {"timestamps": None}, {"ms": None}, {"values": None},
    {"found": None}, {"asof": "no_ms_ptr"}, {"asof": "no_ts"},
])
def test_lookup_resources_rejects_bad_arguments(over):
    from pert_gnn_kdd23_b200 import _lib
    from pert_gnn_kdd23_b200._lib import PertResourceAsOf

    if over.get("asof") == "no_ms_ptr":
        over = {"asof": C.byref(PertResourceAsOf(None, 16, 16))}
    elif over.get("asof") == "no_ts":
        over = {"asof": C.byref(PertResourceAsOf(16, None, 16))}
    assert _lib.lib().pert_store_lookup_resources(*_lookup_args(**over)) == -1


def test_lookup_resources_with_no_queries_launches_nothing():
    from pert_gnn_kdd23_b200 import _lib

    L = _lib.lib()
    assert L.pert_store_lookup_resources(*_lookup_args(k=0, timestamps=None, ms=None, values=None, found=None)) == 0
    assert L.pert_store_lookup_resources(*_lookup_args(k=0, with_asof=True)) == 0
    d = _store_desc()
    d.res_vals = None
    assert L.pert_store_lookup_resources(*_lookup_args(store=C.byref(d), k=0)) == -1
