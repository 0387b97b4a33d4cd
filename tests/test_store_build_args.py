"""CPU tests of the store constructors' host logic: the last-node flags (pat_last) against a numpy restatement, and the
resource rows, which go through the checks and conversion of ``append_resources``.  The constructors run here on host
tensors: the CUDA-device check is lifted for the test, which is enough for every array the constructor builds."""
import contextlib

import numpy as np
import pytest
import torch

I64_MAX = (1 << 63) - 1


def _last_occurrence_flags(all_ms, nptr):
    """flags[i] = 1 iff node i is the LAST node of its microservice inside its pattern (patterns = nptr slices): the
    first occurrence of (pattern, ms) in the reversed node list."""
    n_all = int(all_ms.shape[0])
    flags = np.zeros(n_all, dtype=np.uint8)
    if n_all:
        pid = np.repeat(np.arange(len(nptr) - 1, dtype=np.int64), np.diff(nptr))
        lo = int(all_ms.min())
        key = pid * (int(all_ms.max()) - lo + 1) + (all_ms - lo)
        _, first_rev = np.unique(key[::-1], return_index=True)
        flags[n_all - 1 - first_rev] = 1
    return flags


def _random_patterns(rng, n_pat, lo, hi):
    sizes = rng.integers(0, 12, n_pat)
    sizes[rng.random(n_pat) < 0.2] = 0                                   # patterns without nodes
    nptr = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    return nptr, rng.integers(lo, hi, int(nptr[-1]), dtype=np.int64)


CASES = {
    "empty": ([0], []),
    "zero_nodes": ([0, 0, 3, 3, 5, 5], [4, 4, 7, 7, 2]),
    "repeated": ([0, 6, 9], [1, 2, 1, 1, 3, 2, 5, 5, 5]),
    "negative": ([0, 4, 7], [-3, 0, -3, -(1 << 40), -3, -3, 0]),
    # pattern * 2^32 + ms collides for these: two different (pattern, ms) pairs share one key
    "split_at_2^31": ([0, 1, 2], [1 << 31, -(1 << 31)]),
    "above_2^32": ([0, 2, 4], [(1 << 32) + 5, 7, 5, (1 << 32) + 7]),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_last_flags(case):
    from pert_gnn_kdd23_b200.store import _last_flags

    nptr, ms = (np.asarray(a, dtype=np.int64) for a in CASES[case])
    got = _last_flags(torch.from_numpy(nptr), torch.from_numpy(ms))
    assert got.dtype == torch.uint8
    assert np.array_equal(got.numpy(), _last_occurrence_flags(ms, nptr))


# spans the restatement's key pattern * (max - min + 1) + ms holds without overflow
@pytest.mark.parametrize("span", [(0, 6), (-(1 << 33), 1 << 33), (-(1 << 52), 1 << 52)])
def test_last_flags_random(span):
    from pert_gnn_kdd23_b200.store import _last_flags

    rng = np.random.default_rng(span[1] % 1000)
    for n_pat in (1, 5, 300):
        nptr, ms = _random_patterns(rng, n_pat, *span)
        got = _last_flags(torch.from_numpy(nptr), torch.from_numpy(ms)).numpy()
        assert np.array_equal(got, _last_occurrence_flags(ms, nptr))


# ------------------------------------------------------------------------------------------------ resource rows
@pytest.fixture
def host_store(monkeypatch):
    """store.PatternStore with the CUDA-device check lifted: the constructors build their arrays in host memory."""
    from pert_gnn_kdd23_b200 import store

    monkeypatch.setattr(store, "_cuda_device", torch.device)
    monkeypatch.setattr(torch.cuda, "device", lambda dev: contextlib.nullcontext())
    return store.PatternStore


def _art(n_rows=20, seed=0):
    from pert_gnn_kdd23_b200.synthetic import make_trace_artifacts

    art = make_trace_artifacts(seed=seed)
    rng = np.random.default_rng(seed)
    idx = [(int(30000 * rng.integers(-3, 4)), int(rng.integers(0, 48))) for _ in range(n_rows)]
    idx += idx[:4]                                                        # equal keys keep their input order
    art.update(resource_index=idx, resource_values=rng.normal(size=(len(idx), 8)))
    return art


@pytest.mark.parametrize("n_ms", [None, 48, 1000])
def test_valid_rows_build_the_sorted_table(host_store, n_ms):
    art = _art()
    s = host_store.from_artifacts(dict(art, n_ms=n_ms), "cpu")
    idx = np.array(art["resource_index"], dtype=np.int64)
    pat_ms = np.concatenate([g["ms_id"].reshape(-1).numpy() for g in art["runtime2graph"].values()])
    want_ms = n_ms if n_ms is not None else max(int(pat_ms.max()), int(idx[:, 1].max())) + 1
    keys = idx[:, 0] * want_ms + idx[:, 1]
    order = np.argsort(keys, kind="stable")
    has = np.zeros(want_ms, dtype=np.uint8)
    has[idx[:, 1]] = 1
    assert s.n_ms == want_ms and s.desc.n_ms == want_ms and s.desc.n_res == len(idx)
    assert np.array_equal(s.t["res_keys"].numpy(), keys[order])
    assert np.array_equal(s.t["res_vals"].numpy(), np.asarray(art["resource_values"])[order].astype(np.float32))
    assert np.array_equal(s.t["ms_has_res"].numpy(), has)
    assert all((getattr(s.desc, k) or 0) == v.data_ptr() for k, v in s.t.items())


def test_no_rows(host_store):
    s = host_store.from_artifacts(dict(_art(), resource_index=[], resource_values=np.zeros((0, 8)), n_ms=48), "cpu")
    assert s.desc.n_res == 0 and tuple(s.t["res_vals"].shape) == (0, 8) and int(s.t["ms_has_res"].sum()) == 0


@pytest.mark.parametrize("case", ["width", "ms_too_large", "ms_negative", "key_overflow", "index_float"])
def test_bad_rows_are_refused(host_store, case):
    from pert_gnn_kdd23_b200._lib import PertGnnError

    art = _art()
    idx, vals, n_ms = list(art["resource_index"]), art["resource_values"], 48
    if case == "width":                          # the assembly kernels read 8 values per row
        vals, msg = vals[:, :7], r"resource_values: shape \(24, 7\), expected \(24, 8\)"
    elif case == "ms_too_large":
        idx[5], msg = (0, 48), r"resource row 5: microservice 48 is outside \[0, 48\)"
    elif case == "ms_negative":                  # also with the default n_ms
        idx[2], msg, n_ms = (0, -1), r"resource row 2: microservice -1 is outside \[0, ", None
    elif case == "key_overflow":
        idx[7], msg = (I64_MAX // 10, 3), r"resource row 7: timestamp .* overflows"
    else:                                        # refused, not truncated
        idx, msg = np.array(idx, dtype=np.float64), r"resource row 0: .* not a pair of int64 integers"
    with pytest.raises(PertGnnError, match=msg):
        host_store.from_artifacts(dict(art, resource_index=idx, resource_values=vals, n_ms=n_ms), "cpu")
