"""CPU tests of the open-bucket sample window (rawtable.ResourceSampleWindow): the host checks name the first bad sample
and leave the window as it was, the C entry points (pert_raw_window_*) reject bad arguments before any CUDA call, and
the host mirror (tests/resource_samples_ref.py) equals pandas' groupby(["timestamp", "msname"]).agg([max, min, mean,
median])."""
import numpy as np
import pytest
import torch

from tests.resource_samples_ref import SampleWindowRef

I64_MAX, I64_MIN = (1 << 63) - 1, -(1 << 63)
N_MS = 48


def _host_window():
    """A window whose state lives on the CPU: every check runs, and nothing reaches the library."""
    from pert_gnn_kdd23_b200.rawtable import ResourceSampleWindow

    w = ResourceSampleWindow.__new__(ResourceSampleWindow)
    w.device, w.n_ms, w.sealed, w.n_samples = torch.device("cpu"), N_MS, I64_MIN, 3
    w._set(torch.tensor([5 * N_MS + 1, 6 * N_MS]), torch.tensor([0, 2, 3], dtype=torch.int32),
           torch.arange(20, dtype=torch.float64).reshape(2, 10), torch.tensor([1.0, 2.0, 3.0]),
           torch.tensor([4.0, 5.0, 6.0]))
    return w


def _snapshot(w):
    return {k: v.clone() for k, v in w.t.items()}, (w.sealed, w.n_samples)


def _assert_unchanged(w, snap):
    t, h = snap
    assert (w.sealed, w.n_samples) == h
    for k, v in t.items():
        assert torch.equal(w.t[k], v), k


def _bad(case):
    """(timestamps, ms, cpu, mem, message) of five samples with one bad sample or column."""
    ts, ms = [30000 * i for i in range(5)], [i for i in range(5)]
    cpu, mem = [0.5] * 5, [1.5] * 5
    if case == "lengths":
        return ts, ms[:4], cpu, mem, "different lengths"
    if case == "ms_negative":
        ms[3] = -1
        return ts, ms, cpu, mem, "resource row 3: microservice -1"
    if case == "ms_too_large":
        ms[2] = N_MS
        return ts, ms, cpu, mem, f"resource row 2: microservice {N_MS} is outside \\[0, {N_MS}\\)"
    if case == "ts_overflow":
        ts[4] = I64_MAX // 10
        return ts, ms, cpu, mem, "resource row 4: timestamp .* overflows"
    if case == "ts_underflow":
        ts[1] = I64_MIN // 2
        return ts, ms, cpu, mem, "resource row 1: timestamp .* overflows"
    if case == "ts_float":
        return np.array(ts, dtype=np.float64), ms, cpu, mem, "resource row 0: .* not a pair of int64 integers"
    if case == "ts_float_in_list":
        ts[2] = 60000.0
        return ts, ms, cpu, mem, "resource row 2: .* not a pair of int64 integers"
    if case == "ts_string":
        ts[1] = "30000"
        return ts, ms, cpu, mem, "resource row 1: .* not a pair of int64 integers"
    if case == "ts_above_int64":
        ts[3] = 1 << 63
        return ts, ms, cpu, mem, "resource row 3: .* not a pair of int64 integers"
    if case == "cpu_string":
        cpu[2] = "0.5"
        return ts, ms, cpu, mem, "sample 2: instance_cpu_usage '0.5' is not a number"
    if case == "mem_none":
        mem[4] = None
        return ts, ms, cpu, mem, "sample 4: instance_memory_usage None is not a number"
    if case == "cpu_bool":
        return ts, ms, np.ones(5, dtype=bool), mem, "sample 0: instance_cpu_usage True is not a number"
    assert case == "mem_2d"
    return ts, ms, cpu, np.ones((5, 2)), "instance_memory_usage: shape"


CASES = ["lengths", "ms_negative", "ms_too_large", "ts_overflow", "ts_underflow", "ts_float", "ts_float_in_list",
         "ts_string", "ts_above_int64", "cpu_string", "mem_none", "cpu_bool", "mem_2d"]


@pytest.mark.parametrize("case", CASES)
def test_rejected_adds_change_nothing(case):
    from pert_gnn_kdd23_b200._lib import PertGnnError

    w = _host_window()
    snap = _snapshot(w)
    ts, ms, cpu, mem, msg = _bad(case)
    with pytest.raises(PertGnnError, match=msg):
        w.add(ts, ms, cpu, mem)
    _assert_unchanged(w, snap)


def test_host_checks_accept_what_pandas_accepts():
    """NaN and +-inf usages, integer usages, numpy integer timestamps of any width: checked and converted."""
    w = _host_window()
    ts, ms, cpu, mem = w._batch(np.array([1, 2, 3], dtype=np.int32), [0, 1, N_MS - 1],
                                [np.nan, np.inf, -np.inf], np.array([1, 2, 3], dtype=np.int16))
    assert ts.dtype == ms.dtype == torch.int64 and cpu.dtype == mem.dtype == torch.float64
    assert torch.equal(ts, torch.tensor([1, 2, 3])) and torch.equal(ms, torch.tensor([0, 1, N_MS - 1]))
    assert bool(torch.isnan(cpu[0])) and cpu[1] == np.inf and cpu[2] == -np.inf
    assert torch.equal(mem, torch.tensor([1.0, 2.0, 3.0], dtype=torch.float64))
    lo, hi = -((1 << 63) // N_MS), (I64_MAX - (N_MS - 1)) // N_MS    # the extreme keys that fit
    ts, ms, _, _ = w._batch([lo, hi], [0, N_MS - 1], [0.0, 0.0], [0.0, 0.0])
    assert int(ts[0]) * N_MS >= I64_MIN and int(ts[1]) * N_MS + N_MS - 1 <= I64_MAX
    ts, _, _, _ = w._batch([], [], [], [])
    assert ts.shape == (0,)


def test_seal_checks():
    from pert_gnn_kdd23_b200._lib import PertGnnError

    w = _host_window()
    snap = _snapshot(w)
    with pytest.raises(PertGnnError, match="seal: before"):
        w.seal(1 << 63)
    _assert_unchanged(w, snap)
    w.sealed = 100
    w.seal(50)                                           # a lower cut is a no-op: no device work at all
    assert w.sealed == 100
    _assert_unchanged(w, (snap[0], (100, 3)))


def test_window_needs_cuda():
    from pert_gnn_kdd23_b200._lib import PertGnnError
    from pert_gnn_kdd23_b200.rawtable import ResourceSampleWindow

    with pytest.raises(PertGnnError, match="CUDA"):
        ResourceSampleWindow(4, device="cpu")


def test_entry_points_reject_bad_arguments():
    from pert_gnn_kdd23_b200 import _lib

    L = _lib.lib()
    BAD, X = -1, 16                                       # PERT_ERR_BADARG; a non-NULL dummy pointer
    big = 0x7ffffff0 + 1
    assert L.pert_raw_window_workspace_bytes(0, 0, 0) > 0
    for args in ((-1, 0, 0), (0, -1, 0), (0, 0, -1), (big, 0, 0), (0, big, 0), (0, 0, big)):
        assert L.pert_raw_window_workspace_bytes(*args) == BAD, args
    ws = 1 << 20

    def count(k=4, bkeys=X, n_ms=8, U=2, keys=X, flags=X, sizes=X, w=X, wb=ws):
        return L.pert_raw_window_count(k, bkeys, n_ms, I64_MIN, U, keys, flags, sizes, w, wb, None)

    for kw in ({"k": -1}, {"k": big}, {"U": -1}, {"n_ms": 0}, {"bkeys": None}, {"flags": None}, {"keys": None},
               {"sizes": None}, {"w": None}, {"wb": 0}):
        assert count(**kw) == BAD, kw

    def merge(U=2, S=5, keys=X, off=X, state=X, k=4, bkeys=X, cpu=X, flags=X, n_late=0, u=2, U2=3, keys2=X, off2=X,
              run2=X, ustart=X, upos=X, w=X, wb=ws):
        return L.pert_raw_window_merge(U, S, keys, off, state, X, X, k, bkeys, X, cpu, X, X, X, flags, n_late, u, U2,
                                       keys2, off2, X, run2, X, ustart, upos, w, wb, None)

    for kw in ({"U": -1}, {"S": -1}, {"S": 1}, {"U": 0}, {"k": -1}, {"k": big}, {"S": big}, {"n_late": -1},
               {"n_late": 5}, {"u": 5}, {"u": -1}, {"U2": 1}, {"U2": 6}, {"keys": None}, {"off": None},
               {"state": None}, {"bkeys": None}, {"cpu": None}, {"flags": None}, {"keys2": None}, {"off2": None},
               {"run2": None}, {"ustart": None}, {"upos": None}, {"w": None}, {"wb": 0}):
        assert merge(**kw) == BAD, kw

    def emit(n=2, slot=X, U=2, keys=X, off=X, state=X, n_ms=8, index=X, vals=X):
        return L.pert_raw_window_emit(n, slot, U, keys, off, state, X, X, n_ms, index, vals, None)

    for kw in ({"n": -1}, {"n": big}, {"U": -1}, {"slot": None, "n": 3}, {"n_ms": 0}, {"keys": None}, {"off": None},
               {"state": None}, {"index": None}, {"vals": None}):
        assert emit(**kw) == BAD, kw
    assert emit(n=0, keys=None, off=None, state=None, index=None, vals=None) == 0   # nothing to emit: no launch


def _pandas_stats(ts, ms, cpu, mem):
    import pandas as pd

    df = pd.DataFrame({"timestamp": ts, "msname": ms, "instance_cpu_usage": cpu, "instance_memory_usage": mem})
    g = df.groupby(["timestamp", "msname"]).agg(["max", "min", "mean", "median"])
    idx = np.array([list(k) for k in g.index], dtype=np.int64).reshape(-1, 2)
    return idx, g.to_numpy(dtype=np.float64)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_mirror_matches_pandas(seed):
    pytest.importorskip("pandas")
    rng = np.random.default_rng(seed)
    n_ms = 7
    ref = SampleWindowRef(n_ms)
    all_ts, all_ms, all_c, all_m = [], [], [], []
    for step in range(12):
        k = int(rng.integers(0, 40))
        ts = 30000 * rng.integers(0, 4, k) + rng.integers(0, 2, k)
        ms = rng.integers(0, n_ms, k)
        cpu = rng.integers(-3, 4, k) * 0.25                # equal values and +-0 ties
        cpu[rng.random(k) < 0.2] = np.nan
        mem = rng.random(k) * 1e3
        mem[rng.random(k) < 0.05] = np.inf
        cpu[(ts == 30000) & (ms == 3)] = np.nan           # an all-NaN key
        touched, late = ref.add(ts, ms, cpu, mem)
        assert late == 0 and touched == sorted(set((ts * n_ms + ms).tolist()))
        for a, b in zip((all_ts, all_ms, all_c, all_m), (ts, ms, cpu, mem)):
            a.append(b)
        cat = [np.concatenate(a) for a in (all_ts, all_ms, all_c, all_m)]
        if not cat[0].size:
            continue
        want_idx, want = _pandas_stats(*cat)
        got_idx, got = ref.stats(ref.keys())
        assert np.array_equal(got_idx, want_idx), step
        np.testing.assert_array_equal(got, want)          # NaN equal to NaN, -0.0 equal to 0.0
    ref.seal(30000 * 2)
    assert all(k // n_ms >= 60000 for k in ref.keys())
    touched, late = ref.add([0, 60000], [1, 1], [1.0, 2.0], [3.0, 4.0])
    assert late == 1 and touched == [60000 * n_ms + 1]
