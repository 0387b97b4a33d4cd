"""CPU tests of rawtable.RawStream's refusals and of the C entry points pert_raw_stream_*: every PERT_ERR_BADARG case
before any CUDA call, and the host refusals (a traceid of an earlier chunk, named; a dictionary repeating a value or
holding an unhashable one; something that is not a RawTables), each leaving the stream as it was.  The refusal read
on the device (new microservice ids reaching max_ms) and the next chunk after each refusal are checked on the GPU at
the end of the file."""
import ctypes as C

import numpy as np
import pytest
import torch

from pert_gnn_kdd23_b200 import _lib
from pert_gnn_kdd23_b200.rawtable import RawStream, RawTables
from pert_gnn_kdd23_b200.synthetic import make_random_raw_tables
from tests.raw_stream_ref import chunk_of


def _host_stream():
    """A stream whose state lives on the CPU: the host checks run, and nothing reaches the library."""
    s = RawStream.__new__(RawStream)
    s._reset(torch.device("cpu"), 5, None, 64)
    return s


def _snapshot(s):
    return ({k: v.clone() for k, v in s.t.items()}, {k: dict(v) for k, v in s._codes.items()}, set(s._traceids),
            {k: list(v) for k, v in s._names.items()}, dict(s._n))


def _assert_unchanged(s, snap):
    t, codes, trs, names, n = snap
    for k, v in t.items():
        assert torch.equal(s.t[k], v), k
    assert s._codes == codes and s._traceids == trs and s._names == names and s._n == n


def _tiny(traceids=("a", "b"), interface=("i0", "i1"), rpcid=(0, 1)):
    calls = dict(traceid=[0, 1], timestamp=[1, 2], rpcid=[0, 1], um=[0, 1], rpctype=[0, 0], dm=[1, 0],
                 interface=[0, 1], rt=[5, 6])
    res = dict(timestamp=[0], msname=[0], instance_cpu_usage=[0.5], instance_memory_usage=[1.0])
    return RawTables(calls, res, dict(traceid=list(traceids), interface=list(interface), rpcid=list(rpcid),
                                      rpctype=["http"], ms=["m0", "m1"]))


@pytest.mark.parametrize("case", ["repeated_traceid", "traceid_dict_repeats", "interface_dict_repeats",
                                  "unhashable_rpcid", "unhashable_traceid", "not_raw_tables", "hash_bits"])
def test_host_refusals_leave_the_stream_unchanged(case):
    s = _host_stream()
    s._traceids = {"b"}                                 # as if an earlier chunk held trace "b"
    s._codes["interface"]["i0"] = 0
    snap = _snapshot(s)
    err, match, raw = _lib.PertGnnError, None, _tiny()
    if case == "repeated_traceid":
        match = "traceid 'b' was in an earlier chunk"
    elif case == "traceid_dict_repeats":
        raw, match = _tiny(traceids=("c", "c")), "traceid dictionary repeats"
    elif case == "interface_dict_repeats":
        raw, match = _tiny(traceids=("c", "d"), interface=("i0", "i0")), "interface dictionary repeats"
    elif case == "unhashable_rpcid":
        raw, match = _tiny(traceids=("c", "d"), rpcid=([0], 1)), "rpcid dictionary value is not hashable"
    elif case == "unhashable_traceid":
        raw, match = _tiny(traceids=(["c"], "d")), "traceid is not hashable"
    elif case == "not_raw_tables":
        raw, err, match = {"calls": {}}, TypeError, "a RawTables expected"
    else:
        s.hash_bits, match = 0, "hash_bits"
    with pytest.raises(err, match=match):
        s.process(raw)
    _assert_unchanged(s, snap)


def test_constructor_refusals():
    with pytest.raises(_lib.PertGnnError, match="CUDA device"):
        RawStream("cpu")
    with pytest.raises(_lib.PertGnnError, match="hash_bits"):
        RawStream("cuda:0", hash_bits=65)


def test_entry_points_reject_bad_arguments():
    L = _lib.lib()
    BAD, X = -1, 16                                       # PERT_ERR_BADARG; a non-NULL dummy pointer
    calls = _lib.PertRawCalls(4, 2, 2, 2, 2, 3, 0, -1, *([X] * 8))
    assert L.pert_raw_stream_workspace_bytes(C.byref(calls), 4) > L.pert_raw_process_workspace_bytes(C.byref(calls), 4)
    assert L.pert_raw_stream_workspace_bytes(None, 0) == BAD
    assert L.pert_raw_stream_workspace_bytes(C.byref(calls), 5) == BAD
    assert L.pert_raw_stream_workspace_bytes(C.byref(calls), -1) == BAD
    ws = 1 << 24

    def state(**kw):
        f = dict(ms_map=X, if_map=X, rpc_map=X, rty_map=X, ms_id=X, if_id=X, rpc_id=X, rty_id=X, n_ms_codes=3,
                 n_if_codes=2, n_rpc_codes=2, n_rty_codes=2, has_res=X, ent_key=X, ent_id=X, ent_cnt=X, ent_cap=64,
                 n_tr=0, n_if=2, n_rpc=2, n_rty=2, n_ent=1, n_ms=3)
        f.update(kw)
        return _lib.PertRawState(**f)

    state_cases = [{k: None} for k in ("ms_map", "if_map", "rpc_map", "rty_map", "ms_id", "if_id", "rpc_id",
                                       "rty_id", "has_res", "ent_key", "ent_id", "ent_cnt")] + \
        [{"ent_cap": 63}, {"ent_cap": 96}, {"ent_cap": 32}, {"n_ent": 33}, {"n_tr": -1}, {"n_ms": 0x7ffffff1},
         {"n_ms_codes": -1}, {"n_if_codes": 0x7ffffff1}]

    def process(N=4, order=X, has_res=X, st=None, sizes=X, w=X, wb=ws, tab=calls):
        st = state() if st is None else st
        return L.pert_raw_stream_process(C.byref(tab) if tab is not None else None, N, order, has_res, 5,
                                         C.byref(st) if st is not False else None, sizes, w, wb, None)

    for kw in ({"N": -1}, {"N": 5}, {"order": None}, {"has_res": None}, {"sizes": None}, {"w": None}, {"wb": 0},
               {"tab": None}, {"st": False}) + tuple({"st": state(**c)} for c in state_cases):
        assert process(**kw) == BAD, kw

    def sout(**kw):
        f = dict(ms_id=X, if_id=X, rpc_id=X, rty_id=X, has_res=X, ent_key=X, ent_id=X, ent_cnt=X, ent_cap2=64,
                 resource_ms=X)
        f.update(kw)
        return _lib.PertRawStateOut(**f)

    out = _lib.PertRawOut(*([X] * len(_lib.RAW_OUT)))

    def emit(N=4, order=X, G=2, g=X, K=3, r_ms=X, has_res=X, st=None, o=out, so=None, w=X, wb=ws):
        st = state() if st is None else st
        so = sout() if so is None else so
        return L.pert_raw_stream_emit(C.byref(calls), N, order, G, g, g, K, r_ms, has_res, C.byref(st),
                                      C.byref(o) if o is not None else None, C.byref(so) if so is not False else None,
                                      w, wb, None)

    so_cases = [{k: None} for k in ("ms_id", "if_id", "rpc_id", "rty_id", "has_res", "ent_key", "ent_id", "ent_cnt",
                                    "resource_ms")] + [{"ent_cap2": 32}, {"ent_cap2": 96}, {"ent_cap2": 1 << 41}]
    bad_out = _lib.PertRawOut(*([X] * (len(_lib.RAW_OUT) - 1) + [0]))
    for kw in ({"N": -1}, {"N": 5}, {"order": None}, {"G": -1}, {"g": None}, {"K": -1}, {"K": 0x7ffffff1},
               {"r_ms": None}, {"has_res": None}, {"o": None}, {"o": bad_out}, {"so": False}, {"w": None}, {"wb": 0}) + \
            tuple({"st": state(**c)} for c in state_cases) + tuple({"so": sout(**c)} for c in so_cases):
        assert emit(**kw) == BAD, kw


# ---- on the GPU: the max_ms refusal, and the chunk after any refusal -------------------------------------------------
def _parts():
    raw = make_random_raw_tables(41, 600, n_entries=6, n_ms=120, n_if=16)
    tr, ms = raw.calls["traceid"], raw.resources["msname"]
    cut = int(np.median(tr))
    a = chunk_of(raw, np.flatnonzero(tr <= cut), np.flatnonzero(ms < 60))
    b = chunk_of(raw, np.flatnonzero(tr > cut), np.flatnonzero(ms >= 60))
    again = chunk_of(raw, np.flatnonzero(tr == cut), np.zeros(0, np.int64))     # a trace of chunk a
    return a, b, again


@pytest.mark.gpu
def test_refused_chunks_change_nothing_on_the_gpu():
    a, b, again = _parts()
    clean = RawStream("cuda", min_occurence=2)
    clean.process(a).check()
    want = clean.process(b).check()
    s = RawStream("cuda", min_occurence=2)
    s.process(a).check()
    s.max_ms = s.n_ms + 1                                 # chunk b brings more than one new microservice
    snap = _snapshot(s)
    with pytest.raises(_lib.PertGnnError, match="would reach max_ms"):
        s.process(b)
    _assert_unchanged(s, snap)
    with pytest.raises(_lib.PertGnnError, match="was in an earlier chunk"):
        s.process(again)
    _assert_unchanged(s, snap)
    s.max_ms = None
    got = s.process(b).check()
    for k in want.columns:
        assert torch.equal(got.columns[k], want.columns[k]), k
    assert torch.equal(got.resource_ms, want.resource_ms) and torch.equal(got.resource_index, want.resource_index)
    assert got.ms_names == want.ms_names and got.entry_names == want.entry_names
