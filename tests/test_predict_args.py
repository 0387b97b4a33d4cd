"""CPU tests of request assembly (PatternStore.assemble_requests, train.predict): the time-bucket rule, the numpy
restatement of the exact and as-of resource joins (oracle/asof_oracle.py) against a brute-force scan, the layout of
the store's as-of index, the host-side entry-id check and the host-side argument checks of
pert_store_assemble_requests (no CUDA call is made for a rejected call)."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import asof_oracle as A


def test_time_bucket_is_floor_division():
    ts = [-60001, -60000, -30001, -30000, -29999, -1, 0, 1, 29999, 30000, 30001, 59999, 60000]
    want = [-90000, -60000, -60000, -30000, -30000, -30000, 0, 0, 0, 30000, 30000, 30000, 60000]
    assert A.time_bucket(ts).tolist() == want
    # the trace grouping's rule (get_tr2ts_map) is the same one
    from oracle.trace_group_oracle import BUCKET

    assert BUCKET == A.BUCKET


def _brute(res_ts, res_ms, b, m, asof):
    best = -1
    for i in range(len(res_ts)):
        if res_ms[i] != m:
            continue
        if asof:
            if res_ts[i] <= b and (best < 0 or res_ts[i] > res_ts[best]):
                best = i                                  # strictly later only: ties keep the first row
        elif res_ts[i] == b and best < 0:
            best = i
    return best


@pytest.mark.parametrize("seed", range(6))
def test_joins_match_a_brute_force_scan(seed):
    rng = np.random.default_rng(seed)
    n_ms, n_b = 7, 9
    buckets = 30000 * np.arange(-3, n_b - 3)                  # negative, zero and positive buckets
    n = int(rng.integers(0, 60)) if seed else 0               # seed 0: an empty resource table
    res_ts = rng.choice(buckets, n)
    res_ms = rng.integers(0, n_ms, n)
    if n > 4:                                                 # duplicate keys: the first row must win
        dup = rng.choice(n, 4, replace=False)
        res_ts = np.concatenate([res_ts, res_ts[dup]])
        res_ms = np.concatenate([res_ms, res_ms[dup]])
    # requests before the first bucket, between and on buckets, after the last one
    q_t = rng.integers(-5 * 30000, (n_b + 2) * 30000, 300)
    q_t[:4] = [-10 ** 9, int(buckets[0]) - 1, int(buckets[-1]), 10 ** 12]
    q_b = A.time_bucket(q_t)
    q_ms = rng.integers(0, n_ms + 1, 300)                     # ms n_ms has no rows at all
    got_a, got_e = A.asof_rows(res_ts, res_ms, q_b, q_ms), A.exact_rows(res_ts, res_ms, q_b, q_ms)
    for i in range(300):
        assert got_a[i] == _brute(res_ts, res_ms, q_b[i], q_ms[i], True), i
        assert got_e[i] == _brute(res_ts, res_ms, q_b[i], q_ms[i], False), i
    hit = got_e >= 0
    assert np.array_equal(got_a[hit], got_e[hit])             # an exact hit reads the same row in both modes
    assert (got_a[q_t < buckets[0]] == -1).all()
    vals = rng.random((len(res_ts), 8))
    x = A.features(got_a, vals)
    assert x.dtype == np.float32 and np.array_equal(x[:, 8], (got_a < 0).astype(np.float32))


@pytest.mark.parametrize("seed", range(4))
def test_asof_index_layout(seed):
    from pert_gnn_kdd23_b200.store import asof_index

    rng = np.random.default_rng(seed)
    n_ms = 11
    n = int(rng.integers(0, 80)) if seed else 0
    ts = rng.integers(-4, 5, n) * 30000
    ms = rng.integers(0, n_ms - 1, n)                         # the last microservice has no rows
    keys = np.sort(np.concatenate([ts * n_ms + ms, (ts * n_ms + ms)[:3]]))    # sorted, with duplicate keys
    ms_ptr, a_ts, row = (t.numpy() for t in asof_index(torch.from_numpy(keys), n_ms))
    assert ms_ptr.dtype == np.int32 and a_ts.dtype == np.int64 and row.dtype == np.int32
    assert ms_ptr.shape == (n_ms + 1,) and a_ts.shape == row.shape == keys.shape
    assert ms_ptr[0] == 0 and ms_ptr[-1] == keys.shape[0] and (np.diff(ms_ptr) >= 0).all()
    assert ms_ptr[-1] == ms_ptr[-2]
    assert sorted(row.tolist()) == list(range(keys.shape[0]))       # a permutation of the sorted rows
    for m in range(n_ms):
        seg = slice(ms_ptr[m], ms_ptr[m + 1])
        r = row[seg]
        assert (keys[r] % n_ms == m).all()
        assert np.array_equal(a_ts[seg], keys[r] // n_ms)
        assert (np.diff(r) > 0).all()                       # ascending rows: ascending ts, equal ts in sorted order
        assert r.shape[0] == int(((keys % n_ms) == m).sum())


def _host_store(rng, n_ent=30):
    from pert_gnn_kdd23_b200.store import PatternStore

    store = PatternStore.__new__(PatternStore)
    store._h_ent_nodes = rng.integers(3, 400, n_ent).astype(np.int64)
    store._h_ent_edges = rng.integers(0, 900, n_ent).astype(np.int64)
    store._h_ent_pats = rng.integers(1, 4, n_ent).astype(np.int64)
    store._h_ent_pats[[4, 17]] = 0                            # two entries without patterns
    store._h_ent_nodes[[4, 17]] = 0
    store._h_ent_edges[[4, 17]] = 0
    return store


def test_bad_entry_ids_are_rejected_on_the_host():
    from pert_gnn_kdd23_b200._lib import PertGnnError

    store = _host_store(np.random.default_rng(1))
    assert store.check_entries([0, 29, 3]).tolist() == [0, 29, 3]
    for ids, first, what in (([0, 1, -1, 30], 2, "outside"), ([2, 30], 1, "outside"), ([5, 17, 4], 1, "no patterns"),
                             ([4], 0, "no patterns")):
        with pytest.raises(PertGnnError, match=f"request {first}: entry {ids[first]} .*{what}"):
            store.check_entries(ids)


def _store_desc():
    from pert_gnn_kdd23_b200.store import _PertStore

    d = _PertStore()
    d.n_pat, d.n_ent, d.n_res, d.n_ms, d.attr_cols, d.n_traces = 2, 2, 3, 4, 2, 0
    for name, _ in _PertStore._fields_[6:]:
        setattr(d, name, 1)                                   # non-NULL, never dereferenced on the host
    return d


def _req_args(**over):
    from pert_gnn_kdd23_b200._lib import PertResourceAsOf
    from pert_gnn_kdd23_b200.store import _PertBatchOut

    a = dict(store=C.byref(_store_desc()), asof=None, entry_ids=1, timestamps=1, B=2, N=10, E=20, offsets=1,
             out=C.byref(_PertBatchOut()), status=None, stream=None)
    if over.pop("with_asof", False):
        a["asof"] = C.byref(PertResourceAsOf(1, 1, 1))
    a.update(over)
    return list(a.values())


@pytest.mark.parametrize("over", [
    {"store": None}, {"out": None}, {"B": -1}, {"N": -1}, {"E": -1}, {"entry_ids": None}, {"timestamps": None},
    {"offsets": None}, {"entry_ids": None, "with_asof": True},
])
def test_assemble_requests_rejects_bad_arguments(over):
    from pert_gnn_kdd23_b200 import _lib

    assert _lib.lib().pert_store_assemble_requests(*_req_args(**over)) == -1


def test_assemble_requests_rejects_incomplete_descriptors():
    from pert_gnn_kdd23_b200 import _lib
    from pert_gnn_kdd23_b200._lib import PertResourceAsOf

    L = _lib.lib()
    for field in ("ent_ptr", "ent_pat", "ent_prob", "pat_nptr", "pat_eptr"):
        d = _store_desc()
        setattr(d, field, None)
        assert L.pert_store_assemble_requests(*_req_args(store=C.byref(d))) == -1, field
    for field in ("ms_ptr", "ts", "row"):
        a = PertResourceAsOf(1, 1, 1)
        setattr(a, field, None)
        assert L.pert_store_assemble_requests(*_req_args(asof=C.byref(a))) == -1, field
    # the trace table is not read: a store without traces is fine; with no resource rows the as-of index is just ms_ptr
    d = _store_desc()
    d.trace_entry = d.trace_ts = d.trace_y = None
    d.n_res = 0
    assert L.pert_store_assemble_requests(*_req_args(store=C.byref(d), asof=C.byref(PertResourceAsOf(1, None, None)),
                                                     B=0, N=0, E=0)) == 0


def test_assemble_requests_with_no_requests_launches_nothing():
    from pert_gnn_kdd23_b200 import _lib

    L = _lib.lib()
    # B = 0 returns before any CUDA call, so NULL request arrays and offsets are fine (this machine may have no GPU)
    assert L.pert_store_assemble_requests(*_req_args(B=0, N=0, E=0, entry_ids=None, timestamps=None,
                                                     offsets=None)) == 0
    assert L.pert_store_assemble_requests(*_req_args(B=0, N=0, E=0, with_asof=True)) == 0
