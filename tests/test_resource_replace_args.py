"""CPU tests of replacing and deleting resource rows of a live store (PatternStore.append_resources(replace=True),
delete_resources): the host checks name the first bad row and leave the store as it was, the two C entry points
(pert_store_resources_update_count / _update_merge) reject bad arguments before any CUDA call, and the host mirror of
the store's rows equals a brute-force dict-of-lists statement of the same updates."""
import ctypes as C

import numpy as np
import pytest

from tests.resource_rows_ref import ResourceRows
from tests.test_resource_update_args import _descs, _host_store, _snapshot, _unchanged

I64_MAX = (1 << 63) - 1


def _bad_index(case):
    """(index, message) of five rows with one bad row, the cases shared by delete and replace."""
    idx = [(30000 * i, i) for i in range(5)]
    if case == "index_shape":
        return np.zeros((5, 3), dtype=np.int64), "resource_index: \\[k, 2\\]"
    if case == "ms_negative":
        idx[3] = (0, -2)
        return idx, "resource row 3: microservice -2"
    if case == "ms_too_large":
        idx[1] = (0, 48)
        return idx, "resource row 1: microservice 48 is outside \\[0, 48\\)"
    if case == "ts_overflow":
        idx[4] = (I64_MAX // 10, 1)
        return idx, "resource row 4: timestamp"
    if case == "ts_above_int64":
        idx[2] = (1 << 63, 1)
        return idx, "resource row 2: .* not a pair of int64 integers"
    if case == "ts_string":
        idx[1] = ("30000", 1)
        return idx, "resource row 1: .* not a pair of int64 integers"
    if case == "index_float":
        return np.array(idx, dtype=np.float64), "resource row 0: .* not a pair of int64 integers"
    if case == "index_bool":
        return np.ones((5, 2), dtype=bool), "resource row 0: .* not a pair of int64 integers"
    if case == "index_ragged":
        idx[2] = (0, 1, 2)
        return idx, "resource_index: \\(timestamp, ms\\) pairs expected"
    assert case == "evict_outside_int64"
    return idx, "evict_before"


INDEX_CASES = ["index_shape", "ms_negative", "ms_too_large", "ts_overflow", "ts_above_int64", "ts_string",
               "index_float", "index_bool", "index_ragged", "evict_outside_int64"]


@pytest.mark.parametrize("case", INDEX_CASES)
def test_rejected_deletes_change_nothing(case):
    from pert_gnn_kdd23_b200._lib import PertGnnError

    s = _host_store()
    snap = _snapshot(s)
    idx, msg = _bad_index(case)
    kw = {"evict_before": 1 << 63} if case == "evict_outside_int64" else {}
    with pytest.raises(PertGnnError, match=msg):
        s.delete_resources(idx, **kw)
    _unchanged(s, snap)


@pytest.mark.parametrize("case", INDEX_CASES + ["values_shape", "values_cols", "values_string"])
def test_rejected_replaces_change_nothing(case):
    from pert_gnn_kdd23_b200._lib import PertGnnError

    s = _host_store()
    snap = _snapshot(s)
    vals = np.random.default_rng(0).random((5, 8))
    if case.startswith("values"):
        idx = [(30000 * i, i) for i in range(5)]
        vals, msg = {"values_shape": (vals[:4], "resource_values: shape \\(4, 8\\), expected \\(5, 8\\)"),
                     "values_cols": (vals[:, :7], "expected \\(5, 8\\)"),
                     "values_string": ([["a"] * 8] * 5, "resource_values: \\[k, 8\\] numbers expected")}[case]
    else:
        idx, msg = _bad_index(case)
    kw = {"evict_before": 1 << 63} if case == "evict_outside_int64" else {}
    with pytest.raises(PertGnnError, match=msg):
        s.append_resources(idx, vals, replace=True, **kw)
    _unchanged(s, snap)


class _FakeLib:
    """Stands in for libpertgnn on a host-only store: the update count writes the sizes a device would and records the
    drop set and batch it was given; the merge must not be reached."""

    def __init__(self, sizes):
        self.sizes, self.merged, self.calls = sizes, False, []

    def pert_store_resources_update_count(self, *args):
        n_drop, k = args[4], args[7]
        drop = np.ctypeslib.as_array(C.cast(args[2], C.POINTER(C.c_int64)), (n_drop,)).copy() if n_drop else []
        self.calls.append((list(drop), k))
        C.memmove(args[12], np.array(self.sizes, dtype=np.int64).ctypes.data, 32)
        return 0

    def pert_store_resources_update_merge(self, *args):
        self.merged = True
        return 0


def test_update_sizes_are_checked_before_the_merge(monkeypatch):
    """The row limit is checked on the count's sizes, and an update that changes nothing stops there too.  The drop set
    handed to the count is the batch's sorted unique keys, and a replace inserts one row per key."""
    from pert_gnn_kdd23_b200 import _lib
    from pert_gnn_kdd23_b200._lib import PertGnnError

    s = _host_store()
    snap = _snapshot(s)
    fake = _FakeLib([0, 0, 1 << 31, 0])
    monkeypatch.setattr(_lib, "lib", lambda: fake)
    monkeypatch.setattr(_lib, "stream", lambda: None)
    rows = np.array([[30000, 2], [0, 1], [30000, 2], [0, 3]])
    with pytest.raises(PertGnnError, match=f"would leave {1 << 31} resource rows"):
        s.append_resources(rows, np.zeros((4, 8)), replace=True)
    assert not fake.merged and fake.calls[-1] == ([1, 3, 30000 * 48 + 2], 3)
    _unchanged(s, snap)
    fake.sizes = [0, 0, 6, 0]                          # nothing evicted, nothing dropped: no merge, no change
    assert s.delete_resources(rows) == 0
    assert not fake.merged and fake.calls[-1] == ([1, 3, 30000 * 48 + 2], 0)
    _unchanged(s, snap)
    fake.sizes = [0, 3, 6, 0]                          # every replacement row below the cut, nothing old evicted
    s.append_resources(rows, np.zeros((4, 8)), replace=True, evict_before=-1)
    assert not fake.merged
    _unchanged(s, snap)
    n = len(fake.calls)
    assert s.delete_resources([]) == 0                 # no keys and no cut: returns before the count
    s.append_resources([], [], replace=True)
    assert len(fake.calls) == n
    _unchanged(s, snap)


# --------------------------------------------------------------------------------------------- C-ABI argument checks
def _count_args(**over):
    d, a = _descs(over.pop("n_res", 3), over.pop("n_ms", 4))
    for f in ("res_keys", "res_vals"):
        if over.pop(f"no_{f}", False):
            setattr(d, f, None)
    args = dict(store=C.byref(d), asof=C.byref(a), drop_keys=16, drop_group=16, n_drop=2, new_keys=16, new_group=16,
                k=5, evict_before=0, drop_cnt=16, ms_ptr_out=16, seg=16, sizes=16, stream=None)
    args.update(over)
    return list(args.values())


def _merge_args(**over):
    d, a = _descs(over.pop("n_res", 3), over.pop("n_ms", 4))
    if "res_vals" in over:
        d.res_vals = over.pop("res_vals")
    args = dict(store=C.byref(d), asof=C.byref(a), drop_keys=16, drop_group=16, drop_cnt=16, n_drop=2, new_keys=16,
                new_perm=16, new_vals=16, new_group=16, k=5, ms_ptr_out=16, seg=16, p=1, q=2, n_dropped=1, n_out=4,
                keys_out=16, vals_out=16, has_out=16, ts_out=16, row_out=16, stream=None)
    args.update(over)
    return list(args.values())


@pytest.mark.parametrize("over", [
    {"store": None}, {"asof": None}, {"no_res_keys": True}, {"no_res_vals": True}, {"n_ms": 0}, {"n_res": -1},
    {"k": -1}, {"k": 1 << 31}, {"n_drop": -1}, {"n_drop": (1 << 31) - 1}, {"new_keys": None}, {"new_group": None},
    {"drop_keys": None}, {"drop_group": None}, {"drop_cnt": None}, {"ms_ptr_out": None}, {"seg": None},
    {"sizes": None},
])
def test_update_count_rejects_bad_arguments(over):
    from pert_gnn_kdd23_b200 import _lib

    assert _lib.lib().pert_store_resources_update_count(*_count_args(**over)) == -1


@pytest.mark.parametrize("over", [
    {"store": None}, {"asof": None}, {"n_ms": 0}, {"k": -1}, {"k": 1 << 31}, {"n_drop": -1},
    {"n_drop": (1 << 31) - 1}, {"p": -1}, {"q": -1}, {"n_dropped": -1}, {"n_out": -1},
    {"p": 4, "n_out": 2}, {"q": 6, "n_out": 3}, {"n_out": 5}, {"n_dropped": 3, "n_out": 2},
    {"n_drop": 0, "drop_keys": None, "drop_group": None},           # n_dropped = 1 with no drop set
    {"new_keys": None}, {"new_perm": None}, {"new_vals": None}, {"new_group": None}, {"drop_keys": None},
    {"drop_group": None}, {"drop_cnt": None}, {"ms_ptr_out": None}, {"seg": None}, {"has_out": None},
    {"keys_out": None}, {"vals_out": None}, {"ts_out": None}, {"row_out": None},
    {"new_vals": 20}, {"vals_out": 24}, {"res_vals": 4},                 # value rows not 16-byte aligned
])
def test_update_merge_rejects_bad_arguments(over):
    from pert_gnn_kdd23_b200 import _lib

    assert _lib.lib().pert_store_resources_update_merge(*_merge_args(**over)) == -1


# ------------------------------------------------------------------------------- the mirror against a brute force
def _brute(rows):
    """dict key -> list of values in arrival order: what the constructor's stable sort makes of L."""
    d = {}
    for key, v in rows:
        d.setdefault(key, []).append(v)
    return d


@pytest.mark.parametrize("seed", range(6))
def test_mirror_equals_a_dict_of_lists(seed):
    rng = np.random.default_rng(seed)
    n_ms, B = 5, 30000
    art = {"n_ms": n_ms, "resource_index": [(int(B * rng.integers(0, 6)), int(rng.integers(0, n_ms)))
                                            for _ in range(30)]}
    art["resource_values"] = rng.random((30, 8))
    m = ResourceRows(art)
    d = _brute([(t * n_ms + ms, tuple(v)) for (t, ms), v in zip(art["resource_index"], art["resource_values"])])
    for _ in range(40):
        k = int(rng.integers(0, 9))
        ts, ms = B * rng.integers(0, 8, k), rng.integers(0, n_ms, k)
        vals = rng.random((k, 8))
        cut = int(B * rng.integers(0, 3)) if rng.random() < 0.2 else None
        op = rng.choice(["append", "replace", "delete"])
        keys = (ts * n_ms + ms).tolist()
        before = sum(len(v) for v in d.values())
        if op == "append":
            m.append(ts, ms, vals, cut)
            for key, v in zip(keys, vals):
                d.setdefault(key, []).append(tuple(v))
        elif op == "replace":
            m.replace(ts, ms, vals, cut)
            for key, v in zip(keys, vals):                # dict update: the last row of a key wins
                d[key] = [tuple(v)]
        else:
            removed = m.delete(ts, ms, cut)
            for key in keys:
                d.pop(key, None)
        if cut is not None:
            d = {key: v for key, v in d.items() if key >= cut * n_ms}     # ts >= cut, as 0 <= ms < n_ms
        if op == "delete":
            assert removed == before - sum(len(v) for v in d.values())
        order = np.argsort(m.keys(), kind="stable")
        got = [(int(key), tuple(v)) for key, v in zip(m.keys()[order], m.vals[order])]
        want = [(key, v) for key in sorted(d) for v in d[key]]
        assert got == want
