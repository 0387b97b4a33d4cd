"""CPU tests of resource updates of a live store (PatternStore.append_resources / evict_resources): the host-side row
checks name the first bad row, a rejected update leaves the store exactly as it was, and both C entry points
(pert_store_resources_count / _merge) reject NULL pointers and bad sizes before any CUDA call."""
import ctypes as C

import numpy as np
import pytest
import torch

I64_MAX = (1 << 63) - 1


def test_key_bounds_are_the_int64_limits():
    from pert_gnn_kdd23_b200.store import _key_bounds

    for n_ms in (1, 2, 7, 48, 4096, 1 << 31):
        lo, hi = _key_bounds(n_ms)
        assert lo * n_ms >= -(1 << 63) and (lo - 1) * n_ms < -(1 << 63)
        assert hi * n_ms + n_ms - 1 <= I64_MAX and (hi + 1) * n_ms + n_ms - 1 > I64_MAX


def test_rows_are_checked_and_the_first_bad_one_named():
    from pert_gnn_kdd23_b200._lib import PertGnnError
    from pert_gnn_kdd23_b200.store import _check_resource_rows

    n_ms = 48
    ts = np.arange(10, dtype=np.int64) * 30000
    ms = np.arange(10, dtype=np.int64)
    _check_resource_rows(ts, ms, n_ms)
    # ms 0 at the largest timestamp whose key fits: fine; the same timestamp overflows for ms n_ms - 1 only if the
    # timestamp is past the per-ms limit
    top = (I64_MAX - 0) // n_ms
    _check_resource_rows(np.array([top]), np.array([0]), n_ms)
    _check_resource_rows(np.array([-((1 << 63) // n_ms)]), np.array([0]), n_ms)
    cases = [
        (3, -1, None, "resource row 3: microservice -1 is outside \\[0, 48\\).*ms < store.n_ms.*larger n_ms"),
        (5, n_ms, None, "resource row 5: microservice 48 is outside"),
        (2, 47, top, "resource row 2: timestamp .* overflows the int64 key"),
        (7, 0, top + 1, "resource row 7: timestamp .* overflows"),
        (0, 0, -((1 << 63) // n_ms) - 1, "resource row 0: timestamp .* overflows"),
    ]
    for row, bad_ms, bad_ts, msg in cases:
        t, m = ts.copy(), ms.copy()
        m[row] = bad_ms
        if bad_ts is not None:
            t[row] = bad_ts
        t[row + 1:] = I64_MAX if row < 9 else t[row + 1:]          # later rows are bad too: the first one is named
        with pytest.raises(PertGnnError, match=msg):
            _check_resource_rows(t, m, n_ms)


def test_integer_index_forms_are_accepted():
    from pert_gnn_kdd23_b200.store import _index_rows

    want = np.array([[-30000, 1], [I64_MAX, 0]], dtype=np.int64)
    for idx in ([(-30000, 1), (I64_MAX, 0)], want, want.astype(object), [(np.int32(-30000), np.uint8(1)),
                                                                           (I64_MAX, 0)]):
        got = _index_rows(idx)
        assert got.dtype == np.int64 and np.array_equal(got, want)
    got = _index_rows(np.array([[30000, 1], [60000, 2]], dtype=np.uint64))
    assert got.dtype == np.int64 and got.tolist() == [[30000, 1], [60000, 2]]
    assert _index_rows([]).shape == (0, 2)


class _FakeLib:
    """Stands in for libpertgnn on a host-only store: the count writes the sizes a device would, the merge must not be
    reached."""

    def __init__(self, sizes):
        self.sizes, self.merged = sizes, False

    def pert_store_resources_count(self, *args):
        C.memmove(args[8], np.array(self.sizes, dtype=np.int64).ctypes.data, 24)
        return 0

    def pert_store_resources_merge(self, *args):
        self.merged = True
        return 0


def _host_store(n_ms=48, n_res=6):
    """A store whose arrays live in host memory: enough for every check that runs before a launch."""
    from pert_gnn_kdd23_b200 import _lib
    from pert_gnn_kdd23_b200._lib import PertStore
    from pert_gnn_kdd23_b200.store import PatternStore

    s = PatternStore.__new__(PatternStore)
    s.device, s.n_ms = torch.device("cpu"), n_ms
    keys = torch.arange(n_res, dtype=torch.int64) * n_ms
    s.t = {"res_keys": keys, "res_vals": torch.rand(n_res, 8), "ms_has_res": torch.zeros(n_ms, dtype=torch.uint8)}
    s.desc = PertStore()
    s.desc.n_res, s.desc.n_ms = n_res, n_ms
    for k, v in s.t.items():
        setattr(s.desc, k, v.data_ptr())
    s.asof_t = {"ms_ptr": torch.zeros(n_ms + 1, dtype=torch.int32), "ts": keys // n_ms,
                "row": torch.arange(n_res, dtype=torch.int32)}
    s.asof_desc = _lib.PertResourceAsOf()
    return s


def _snapshot(s):
    return ({k: (v, v.clone()) for k, v in {**s.t, **s.asof_t}.items()}, bytes(s.desc), s.asof_desc)


def _unchanged(s, snap):
    arrays, desc, asof_desc = snap
    assert bytes(s.desc) == desc and s.asof_desc is asof_desc
    for k, (obj, copy) in arrays.items():
        now = s.t.get(k, s.asof_t.get(k))
        assert now is obj and torch.equal(now, copy), k


@pytest.mark.parametrize("case", ["values_shape", "values_cols", "index_shape", "ms_negative", "ms_too_large",
                                  "ts_overflow", "evict_outside_int64", "ts_above_int64", "ts_above_int64_signed",
                                  "ts_string", "index_float", "index_bool", "index_ragged", "values_string"])
def test_rejected_updates_change_nothing(case):
    from pert_gnn_kdd23_b200._lib import PertGnnError

    s = _host_store()
    snap = _snapshot(s)
    idx = [(30000 * i, i) for i in range(5)]
    vals = np.random.default_rng(0).random((5, 8))
    kw = {}
    if case == "values_shape":
        vals, msg = vals[:4], "resource_values: shape \\(4, 8\\), expected \\(5, 8\\)"
    elif case == "values_cols":
        vals, msg = vals[:, :7], "expected \\(5, 8\\)"
    elif case == "index_shape":
        idx, msg = np.zeros((5, 3), dtype=np.int64), "resource_index: \\[k, 2\\]"
    elif case == "ms_negative":
        idx[3], msg = (0, -2), "resource row 3: microservice -2"
    elif case == "ms_too_large":
        idx[1], msg = (0, 48), "resource row 1: microservice 48 is outside \\[0, 48\\)"
    elif case == "ts_overflow":
        idx[4], msg = (I64_MAX // 10, 1), "resource row 4: timestamp"
    elif case == "ts_above_int64":                  # every entry >= 0: numpy makes it uint64
        idx[2], msg = (1 << 63, 1), "resource row 2: .* not a pair of int64 integers"
    elif case == "ts_above_int64_signed":           # with a negative entry: an object array
        idx[0], idx[3], msg = (-30000, 0), (1 << 64, 1), "resource row 3: .* not a pair of int64 integers"
    elif case == "ts_string":
        idx[1], msg = ("30000", 1), "resource row 1: .* not a pair of int64 integers"
    elif case == "index_float":                     # refused, not truncated
        idx, msg = np.array(idx, dtype=np.float64), "resource row 0: .* not a pair of int64 integers"
    elif case == "index_bool":
        idx, msg = np.ones((5, 2), dtype=bool), "resource row 0: .* not a pair of int64 integers"
    elif case == "index_ragged":
        idx[2], msg = (0, 1, 2), "resource_index: \\(timestamp, ms\\) pairs expected"
    elif case == "values_string":
        vals, msg = [["a"] * 8] * 5, "resource_values: \\[k, 8\\] numbers expected"
    else:
        kw, msg = {"evict_before": 1 << 63}, "evict_before"
    with pytest.raises(PertGnnError, match=msg):
        s.append_resources(idx, vals, **kw)
    _unchanged(s, snap)


def test_too_many_rows_are_rejected_after_the_count(monkeypatch):
    """The row limit depends on what the eviction drops, so it is checked on the count's sizes, before the merge."""
    from pert_gnn_kdd23_b200 import _lib
    from pert_gnn_kdd23_b200._lib import PertGnnError

    s = _host_store()
    snap = _snapshot(s)
    fake = _FakeLib([0, 0, 1 << 31])
    monkeypatch.setattr(_lib, "lib", lambda: fake)
    monkeypatch.setattr(_lib, "stream", lambda: None)
    with pytest.raises(PertGnnError, match=f"would leave {1 << 31} resource rows"):
        s.append_resources(np.array([[0, 1], [30000, 2]]), np.zeros((2, 8)))
    assert not fake.merged
    _unchanged(s, snap)
    fake.sizes = [0, 0, 6]                             # nothing evicted, nothing appended: no merge, no change
    s.evict_resources(-10 ** 12)
    assert not fake.merged
    _unchanged(s, snap)
    s.append_resources([], [])                          # no rows and no cut: returns before the count
    _unchanged(s, snap)


# --------------------------------------------------------------------------------------------- C-ABI argument checks
def _descs(n_res=3, n_ms=4):
    from pert_gnn_kdd23_b200._lib import PertResourceAsOf
    from pert_gnn_kdd23_b200._lib import PertStore

    d = PertStore()
    d.n_res, d.n_ms = n_res, n_ms
    for name, _ in PertStore._fields_[6:]:
        setattr(d, name, 16)                           # non-NULL and aligned, never dereferenced on the host
    return d, PertResourceAsOf(16, 16, 16)


def _count_args(**over):
    d, a = _descs(over.pop("n_res", 3), over.pop("n_ms", 4))
    for f in ("res_keys", "res_vals"):
        if over.pop(f"no_{f}", False):
            setattr(d, f, None)
    for f in ("ms_ptr", "ts", "row"):
        if over.pop(f"no_{f}", False):
            setattr(a, f, None)
    args = dict(store=C.byref(d), asof=C.byref(a), new_keys=16, new_group=16, k=5, evict_before=0, ms_ptr_out=16,
                seg=16, sizes=16, stream=None)
    args.update(over)
    return list(args.values())


def _merge_args(**over):
    d, a = _descs(over.pop("n_res", 3), over.pop("n_ms", 4))
    if "res_vals" in over:
        d.res_vals = over.pop("res_vals")
    args = dict(store=C.byref(d), asof=C.byref(a), new_keys=16, new_perm=16, new_vals=16, new_group=16, k=5,
                ms_ptr_out=16, seg=16, p=1, q=2, n_out=5, keys_out=16, vals_out=16, has_out=16, ts_out=16, row_out=16,
                stream=None)
    args.update(over)
    return list(args.values())


@pytest.mark.parametrize("over", [
    {"store": None}, {"asof": None}, {"no_ms_ptr": True}, {"no_ts": True}, {"no_row": True}, {"no_res_keys": True},
    {"no_res_vals": True}, {"n_ms": 0}, {"n_res": -1}, {"k": -1}, {"k": 1 << 31}, {"new_keys": None},
    {"new_group": None}, {"ms_ptr_out": None}, {"seg": None}, {"sizes": None},
])
def test_count_rejects_bad_arguments(over):
    from pert_gnn_kdd23_b200 import _lib

    assert _lib.lib().pert_store_resources_count(*_count_args(**over)) == -1


@pytest.mark.parametrize("over", [
    {"store": None}, {"asof": None}, {"n_ms": 0}, {"k": -1}, {"p": -1}, {"q": -1}, {"n_out": -1}, {"p": 4, "n_out": 4},
    {"q": 6, "n_out": 4}, {"n_out": 6}, {"new_keys": None}, {"new_perm": None}, {"new_vals": None},
    {"new_group": None}, {"ms_ptr_out": None}, {"seg": None}, {"has_out": None}, {"keys_out": None},
    {"vals_out": None}, {"ts_out": None}, {"row_out": None},
    {"new_vals": 20}, {"vals_out": 24}, {"res_vals": 4},                 # value rows not 16-byte aligned
])
def test_merge_rejects_bad_arguments(over):
    from pert_gnn_kdd23_b200 import _lib

    assert _lib.lib().pert_store_resources_merge(*_merge_args(**over)) == -1
