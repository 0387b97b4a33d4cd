"""Raw call-graph and resource rows -> the processed span and resource tables, on the GPU.

The reference's preprocess.py get_df() (:191-266) reads the Alibaba ``MSCallGraph`` / ``MSResource`` CSV files with
pandas and turns them into ``processed_df`` and ``processed_resource_df``: drop duplicates, sort by timestamp,
factorise five columns, find every trace's entry in a Python loop over traces, filter traces by resource coverage and
per-entry occurrence, renumber the microservices and aggregate the resource rows per (timestamp, msname).

Here the host only parses the files and dictionary-encodes their values (``read_raw``); everything after that runs
over the whole table in csrc/rawtable.cu (``process_raw``).  ``ResourceSampleWindow`` keeps the same resource
statistics of the still-open (timestamp, msname) keys up to date as raw samples arrive.  The result's ``columns`` are the nine
``tracegroup.COLUMNS`` that ``group_traces`` takes, and ``resource_index`` / ``resource_values`` are the rows the
``PatternStore`` constructors take.  There is no CPU fallback: without the CUDA library the calls raise.

Two orders the reference leaves unspecified are fixed here: rows with equal timestamps keep their concatenation order
(pandas' sort_values is an unstable quicksort), and microservice ids follow the lexicographic order of the names (the
reference numbers a Python ``set``, whose order is hash-randomised).
"""
from __future__ import annotations

import ctypes as C
import os
from typing import NamedTuple

import numpy as np
import torch

from . import _lib
from .store import _I64_MAX, _I64_MIN, _check_resource_rows, _index_rows, _key_bounds
from .tracegroup import COLUMNS

CALL_COLUMNS = ("traceid", "timestamp", "rpcid", "um", "rpctype", "dm", "interface", "rt")   # MSCallGraph order
RESOURCE_COLUMNS = ("timestamp", "msname", "instance_cpu_usage", "instance_memory_usage")
USAGE = ("instance_cpu_usage", "instance_memory_usage")
STATS = tuple(f"{u}_{s}" for u in USAGE for s in ("max", "min", "mean", "median"))   # processed_resource_df columns
CODED = ("traceid", "interface", "rpcid", "rpctype")                                # own dictionaries; ms shared


class RawTables:
    """Dictionary-encoded raw rows.
      calls: the eight CALL_COLUMNS as int64 arrays in concatenation order; timestamp and rt hold values, traceid /
        interface / rpcid / rpctype hold codes into ``dicts[column]`` and um / dm codes into ``dicts["ms"]``.
      resources: timestamp int64, msname codes into ``dicts["ms"]``, instance_cpu_usage / instance_memory_usage float64.
      dicts: code -> value, one list per coded column; "ms" is shared by um, dm and msname.
    Equal codes must mean equal values (the duplicate drop, the factorisations and the entry key compare codes).  A
    caller with its own reader (Parquet, say) builds this directly and skips ``read_raw``."""

    def __init__(self, calls, resources, dicts):
        self.calls = {k: np.ascontiguousarray(calls[k], dtype=np.int64) for k in CALL_COLUMNS}
        self.resources = {k: np.ascontiguousarray(resources[k], dtype=np.float64 if k in USAGE else np.int64)
                          for k in RESOURCE_COLUMNS}
        self.dicts = {k: list(dicts[k]) for k in CODED + ("ms",)}
        R, K = len(self.calls["traceid"]), len(self.resources["timestamp"])
        if any(len(v) != R for v in self.calls.values()) or any(len(v) != K for v in self.resources.values()):
            raise ValueError("RawTables: columns of different lengths")
        names = self.dicts["ms"]
        if any(not isinstance(m, str) for m in names):
            raise _lib.PertGnnError("RawTables: microservice names must be strings")
        rank = np.argsort(np.array(names, dtype=object), kind="stable") if names else np.zeros(0, np.int64)
        if len(set(names)) != len(names):
            raise _lib.PertGnnError("RawTables: the microservice dictionary repeats a name")
        if np.any(rank != np.arange(len(names))):             # codes must follow the names' order: recode
            new = np.empty(len(names), dtype=np.int64)
            new[rank] = np.arange(len(names))
            self.dicts["ms"] = [names[i] for i in rank]
            for col, tab in (("um", self.calls), ("dm", self.calls), ("msname", self.resources)):
                c = tab[col]
                ok = (c >= 0) & (c < len(names))
                tab[col] = np.where(ok, new[np.where(ok, c, 0)], c)   # out-of-range codes stay out of range

    def __len__(self):
        return len(self.calls["traceid"])


def _encode(parts, merged):
    """Global codes of one column from per-file (codes, uniques) pairs: ``merged`` maps value -> code with Python
    equality (so 1 == 1.0, as pandas' object factorize), new values appended in concatenation order."""
    out = []
    for codes, uniq in parts:
        lut = np.empty(len(uniq), dtype=np.int64)
        for i, v in enumerate(uniq):
            v = v.item() if isinstance(v, np.generic) else v
            lut[i] = merged.setdefault(v, len(merged))
        out.append(lut[codes])
    return np.concatenate(out) if out else np.zeros(0, np.int64)


def _int_column(s, rows, path, what):
    """int64 values of a timestamp / rt column (``rows``: the file's data row of every value); PertGnnError naming the
    file and data row of the first null or non-integer (the reference fails on it later, at rt.abs())."""
    import pandas as pd

    if pd.api.types.is_integer_dtype(s.dtype) and not s.isna().any():
        return s.to_numpy(dtype=np.int64)
    v = pd.to_numeric(s, errors="coerce").to_numpy(dtype=np.float64, na_value=np.nan)
    bad = np.isnan(v) | (v % 1 != 0)
    if bad.any():
        i = int(np.flatnonzero(bad)[0])
        raise _lib.PertGnnError(f"{path}: row {int(rows[i])}: {what} {s.name} {s.iloc[i]!r} is not an integer")
    return v.astype(np.int64)


def read_raw(callgraph_csvs, resource_csvs):
    """Parse and dictionary-encode the raw CSV files, concatenated in the order given (the reference concatenates in
    os.listdir order).  Files are read by ``pd.read_csv(engine="pyarrow")`` as in the reference, call-graph files with
    their leading index column (``index_col=0``), and null cells of the call graph become the string "nan"
    (``.replace(np.nan, "nan")``); rpcid is encoded by value, so a numeric-looking column merges "0" and "0.0".
    Resource rows with a null timestamp or msname are dropped (groupby drops NaN keys); NaN usages are kept.
    A null or non-integer call-graph timestamp or rt raises PertGnnError naming the file and row."""
    import pandas as pd

    merged = {k: {} for k in CODED + ("ms",)}
    parts = {k: [] for k in CALL_COLUMNS}
    for path in callgraph_csvs:
        df = pd.read_csv(path, index_col=0, engine="pyarrow").replace(np.nan, "nan")
        missing = [c for c in CALL_COLUMNS if c not in df.columns]
        if missing:
            raise _lib.PertGnnError(f"{path}: no column {missing[0]!r}")
        for col in ("timestamp", "rt"):
            parts[col].append(_int_column(df[col], np.arange(len(df)), path, "call-graph"))
        for col in ("traceid", "interface", "rpcid", "rpctype", "um", "dm"):
            parts[col].append(pd.factorize(df[col].to_numpy(dtype=object)))
    calls = {}
    for col in CALL_COLUMNS:
        if col in ("timestamp", "rt"):
            calls[col] = np.concatenate(parts[col]) if parts[col] else np.zeros(0, np.int64)
        else:
            calls[col] = _encode(parts[col], merged["ms" if col in ("um", "dm") else col])
    res = {k: [] for k in RESOURCE_COLUMNS}
    for path in resource_csvs:
        df = pd.read_csv(path, engine="pyarrow")
        missing = [c for c in RESOURCE_COLUMNS if c not in df.columns]
        if missing:
            raise _lib.PertGnnError(f"{path}: no column {missing[0]!r}")
        keep = (df["timestamp"].notna() & df["msname"].notna()).to_numpy()
        df = df.loc[keep, list(RESOURCE_COLUMNS)]
        res["timestamp"].append(_int_column(df["timestamp"], np.flatnonzero(keep), path, "resource"))
        res["msname"].append(pd.factorize(df["msname"].to_numpy(dtype=object)))
        for u in USAGE:
            res[u].append(pd.to_numeric(df[u], errors="raise").to_numpy(dtype=np.float64))
    resources = {k: (np.concatenate(v) if v else np.zeros(0, np.float64 if k in USAGE else np.int64))
                 for k, v in res.items() if k != "msname"}
    resources["msname"] = _encode(res["msname"], merged["ms"])
    for name in merged["ms"]:
        if not isinstance(name, str):
            raise _lib.PertGnnError(f"microservice name {name!r} is not a string (um, dm and msname must be strings)")
    dicts = {k: list(v) for k, v in merged.items()}
    return RawTables(calls, resources, dicts)


_NAME_CODES_OF = {"ms_names": ("ms_code", "ms"), "traceid_names": ("tr_code", "traceid"),
                  "interface_names": ("if_code", "interface"), "rpcid_values": ("rpc_code", "rpcid"),
                  "rpctype_names": ("rty_code", "rpctype")}
_NAME_CODES = ("ms_code", "tr_code", "if_code", "rpc_code", "rty_code", "ent_dm", "ent_if")


class ProcessedTables:
    """Device result of ``process_raw``.
      columns: the nine tracegroup.COLUMNS, int64 [M], processed row order (get_df()'s processed_df); row [M]: each
        processed row's index in the concatenated raw table (processed_df's index).
      resource_index int64 [G, 2] (timestamp, ms id), resource_values float64 [G, 8] (STATS order), ascending by
        timestamp then microservice name (processed_resource_df).
      n_ms and the id -> value lists ms_names, traceid_names, interface_names, rpcid_values, rpctype_names and
        entry_names (the reference's entry string dm + "_" + interface id), each built on first access.
    Call ``check()`` before trusting the result."""

    def __init__(self, t, dicts, status, views=None, n_ms=None):
        self.status = status
        self.columns = {k: t[k] for k in COLUMNS}
        self.row = t["row"]
        self.resource_index, self.resource_values = t["res_index"], t["res_vals"]
        self._codes, self._dicts, self._names = {k: t[k] for k in _NAME_CODES}, dicts, {}
        self._views = views                  # RawStream results: name -> (the stream's list, its length then)
        self.n_ms = int(t["ms_code"].shape[0]) if n_ms is None else n_ms

    def _lookup(self, name):
        """An id -> value list, built on first use (one device-to-host copy of its code array and a Python list as
        long as the ids: a million traces make a million-element traceid_names)."""
        if name not in self._names and self._views is not None:
            lst, n = self._views[name]
            self._names[name] = lst[:n]
        if name not in self._names:
            code = lambda k: self._codes[k].cpu().numpy()    # noqa: E731
            d = self._dicts
            if name == "entry_names":
                v = [f"{d['ms'][m]}_{i}" for m, i in zip(code("ent_dm"), code("ent_if"))]
            else:
                k, col = _NAME_CODES_OF[name]
                v = [d[col][i] for i in code(k)]
            self._names[name] = v
        return self._names[name]

    ms_names = property(lambda self: self._lookup("ms_names"))
    traceid_names = property(lambda self: self._lookup("traceid_names"))
    interface_names = property(lambda self: self._lookup("interface_names"))
    rpcid_values = property(lambda self: self._lookup("rpcid_values"))
    rpctype_names = property(lambda self: self._lookup("rpctype_names"))
    entry_names = property(lambda self: self._lookup("entry_names"))

    def __len__(self):
        return int(self.columns["traceid"].shape[0])

    def check(self):
        """Synchronising check of the status word: a code outside its dictionary (or a resource msname outside the
        microservice dictionary) raises PertGnnError."""
        code = int(self.status.item())
        if code != 0:
            _lib.check(code, "raw tables (a dictionary code out of range)")
        return self

    def to_frames(self):
        """(processed_df, processed_resource_df) as pandas frames with the columns of get_df()'s result: the call-graph
        columns, entryid and endTimestamp (= timestamp + |rt|, :263) indexed by the raw row, and timestamp, msname and
        the eight statistics.  The values are get_df()'s, with three differences: every code column is int64 (the
        reference keeps the dtype of the column its codes were written into, e.g. float64 for a numeric rpcid, object
        for strings); microservice ids are in name order (the reference's are in Python set order, so the two agree up
        to a one-to-one renumbering); rows with equal timestamps are in raw-row order (the reference's sort is
        unstable)."""
        import pandas as pd

        c = {k: v.cpu().numpy() for k, v in self.columns.items()}
        df = pd.DataFrame({k: c[k] for k in CALL_COLUMNS}, index=pd.Index(self.row.cpu().numpy()))
        df["entryid"] = c["entryid"]
        df["endTimestamp"] = c["timestamp"] + np.abs(c["rt"])
        idx, vals = self.resource_index.cpu().numpy(), self.resource_values.cpu().numpy()
        res = pd.DataFrame({"timestamp": idx[:, 0], "msname": idx[:, 1]})
        for j, k in enumerate(STATS):
            res[k] = vals[:, j]
        return df, res


def _code_of(values, v):
    try:
        return values.index(v)
    except ValueError:
        return -1


def _check_raw(raw, what, hash_bits):
    if not isinstance(raw, RawTables):
        raise TypeError(f"{what}: a RawTables expected (read_raw builds one)")
    if not 1 <= int(hash_bits) <= 64:
        raise _lib.PertGnnError(f"{what}: hash_bits must lie in 1..64")
    R, K = len(raw), len(raw.resources["timestamp"])
    if R > 1 << 30 or len(raw.dicts["traceid"]) > 1 << 30:
        raise _lib.PertGnnError(f"{what}: {max(R, len(raw.dicts['traceid']))} call-graph rows or traceids exceed "
                                "2^30")
    if K > 0x7ffffff0:
        raise _lib.PertGnnError(f"{what}: {K} resource rows exceed 2^31 - 16")


class _Front(NamedTuple):
    """What the resource groups, the statistics, the duplicate drop and the timestamp sort leave for the call-graph
    passes (process_raw's steps 9, 1 and 2); cols keeps the device columns ``tab`` points into alive."""
    status: torch.Tensor
    G: int
    g_ts: torch.Tensor
    g_ms: torch.Tensor
    res_vals: torch.Tensor
    has_res: torch.Tensor
    r_ms: torch.Tensor
    tab: object
    cols: dict
    N: int
    order: torch.Tensor


def _front(raw, dev, hash_bits):
    """Steps 9, 1 and 2 on the current device and stream: host synchronisations (1) G and (2) the distinct rows."""
    L, st = _lib.lib(), _lib.stream()
    R, K = len(raw), len(raw.resources["timestamp"])
    i32, i64, f64 = (dict(dtype=d, device=dev) for d in (torch.int32, torch.int64, torch.float64))
    status = torch.zeros(1, **i32)
    n_ms = len(raw.dicts["ms"])
    # ---- resources: stable sort by (timestamp, ms), groups, statistics (:227-242)
    r_ts, r_ms = (torch.from_numpy(raw.resources[k]).to(dev) for k in ("timestamp", "msname"))
    usage = [torch.from_numpy(raw.resources[u]).to(dev) for u in USAGE]
    p1 = torch.sort(r_ms, stable=True).indices
    perm = p1[torch.sort(r_ts[p1], stable=True).indices]
    bad = ((r_ms < 0) | (r_ms >= n_ms))[perm]           # rows with an ms outside the dictionary go last
    keep = torch.sort(bad.to(torch.uint8), stable=True).indices
    perm, bad = perm[keep].contiguous(), bad[keep]
    gflag, gptr = torch.empty(K + 1, **i32), torch.empty(K + 1, **i32)
    has_res = torch.empty(max(n_ms, 1), **i32)
    g_ts, g_ms, ng = torch.empty(max(K, 1), **i64), torch.empty(max(K, 1), **i64), torch.empty(1, **i64)
    ws = torch.empty(int(L.pert_raw_resource_workspace_bytes(K)), dtype=torch.uint8, device=dev)
    _lib.check(L.pert_raw_resource_groups(K, _lib.ptr(r_ts), _lib.ptr(r_ms), _lib.ptr(perm), n_ms,
                                          gflag.data_ptr(), has_res.data_ptr(), gptr.data_ptr(), g_ts.data_ptr(),
                                          g_ms.data_ptr(), ng.data_ptr(), ws.data_ptr(), ws.numel(),
                                          status.data_ptr(), st), "pert_raw_resource_groups")
    G = int(ng.item())                                                           # sync 1
    gid = torch.where(bad, G, gflag[1:] - 1)           # the left-out rows sort after every group
    sorted_usage = []
    for u in usage:                      # every group's values ascending (NaN last) at the group's positions
        s = torch.sort(u[perm], stable=True)
        sorted_usage.append(s.values[torch.sort(gid[s.indices], stable=True).indices].contiguous())
    res_vals = torch.empty(G, 8, **f64)
    _lib.check(L.pert_raw_resource_stats(G, _lib.ptr(perm), gptr.data_ptr(), _lib.ptr(usage[0]),
                                         _lib.ptr(usage[1]), _lib.ptr(sorted_usage[0]), _lib.ptr(sorted_usage[1]),
                                         res_vals.data_ptr(), st), "pert_raw_resource_stats")
    # ---- call graph: duplicates, stable sort by timestamp (:212-213)
    cols = {k: torch.from_numpy(raw.calls[k]).to(dev) for k in CALL_COLUMNS}
    n = {k: len(raw.dicts[k]) for k in CODED}
    tab = _lib.PertRawCalls(R, n["traceid"], n["interface"], n["rpcid"], n["rpctype"], n_ms,
                            _code_of(raw.dicts["rpctype"], "http"), _code_of(raw.dicts["ms"], "(?)"),
                            *(cols[k].data_ptr() for k in CALL_COLUMNS))
    rows, keys, nk = torch.empty(max(R, 1), **i32), torch.empty(max(R, 1), **i64), torch.empty(1, **i64)
    ws = torch.empty(int(L.pert_raw_dedup_workspace_bytes(R)), dtype=torch.uint8, device=dev)
    _lib.check(L.pert_raw_dedup(C.byref(tab), int(hash_bits), rows.data_ptr(), keys.data_ptr(), nk.data_ptr(),
                                ws.data_ptr(), ws.numel(), status.data_ptr(), st), "pert_raw_dedup")
    N = int(nk.item())                                                           # sync 2
    order = rows[:N].long()[torch.sort(keys[:N], stable=True).indices].contiguous()
    return _Front(status, G, g_ts, g_ms, res_vals, has_res, r_ms, tab, cols, N, order)


def _alloc_out(dev, M, G, n_ids, n_tr, n_if, n_ent, n_rpc, n_rty):
    """Output tensors of pert_raw_emit: every one at least one element, so no pointer is NULL; sliced to its size.
    The id -> code arrays share one buffer (one device -> host copy reads them all)."""
    alloc = lambda n, *w: torch.empty(max(n, 1), *w, dtype=torch.int64, device=dev)[:n]   # noqa: E731
    t = {k: alloc(M) for k in COLUMNS + ("row",)}
    t["res_index"] = alloc(G, 2)
    sizes = {"ms_code": n_ids, "tr_code": n_tr, "if_code": n_if, "rpc_code": n_rpc, "rty_code": n_rty,
             "ent_dm": n_ent, "ent_if": n_ent}
    buf = torch.empty(max(sum(sizes.values()), 1), dtype=torch.int64, device=dev)
    o = 0
    for k, n in sizes.items():
        t[k] = buf[o:o + n]
        o += n
    t["_codes"] = buf[:o]
    return t


def _raw_out(t, spare=None):
    """PertRawOut of ``t``; with ``spare`` (a one-element tensor) an empty output points there instead of NULL."""
    return _lib.PertRawOut(*(t[k].data_ptr() or (spare.data_ptr() if spare is not None else 0) for k in _lib.RAW_OUT))


def process_raw(raw, device="cuda", min_occurence=100, hash_bits=64):
    """get_df()'s processing (:212-254) of a RawTables on the GPU -> ProcessedTables.  ``min_occurence``: an entry is
    kept with strictly more traces than this (:185).  ``hash_bits`` narrows the duplicate-row hash (1..64); only tests
    lower it, to force collisions.
    Host synchronisations: (1) the number of resource groups G, (2) the number of distinct call-graph rows, (3) the
    seven output sizes -- each a read of a few integers that sizes the next outputs.  The id -> value lists of the
    result are copied to the host only when first read.  Errors found on the device go to the status word
    (``check()``): a code outside its dictionary sets it and its row is left out.  At most 2^30 call-graph rows and
    traceid codes (every hash-table slot is an int32)."""
    dev = torch.device(device)
    if dev.type != "cuda":
        raise _lib.PertGnnError("process_raw needs a CUDA device (no CPU fallback)")
    _check_raw(raw, "process_raw", hash_bits)
    with torch.cuda.device(dev):
        L, st = _lib.lib(), _lib.stream()
        f = _front(raw, dev, hash_bits)
        tab, N = f.tab, f.N
        nbytes = int(L.pert_raw_process_workspace_bytes(C.byref(tab), N))
        if nbytes < 0:
            raise _lib.PertGnnError("process_raw: table sizes out of range")
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        sizes = torch.empty(7, dtype=torch.int64, device=dev)
        _lib.check(L.pert_raw_process(C.byref(tab), N, _lib.ptr(f.order), f.has_res.data_ptr(), int(min_occurence),
                                      sizes.data_ptr(), ws.data_ptr(), ws.numel(), st), "pert_raw_process")
        M, n_ids, n_tr, n_if, n_ent, n_rpc, n_rty = (int(v) for v in sizes.cpu())   # sync 3
        t = _alloc_out(dev, M, f.G, n_ids, n_tr, n_if, n_ent, n_rpc, n_rty)
        out = _raw_out(t)
        _lib.check(L.pert_raw_emit(C.byref(tab), N, _lib.ptr(f.order), f.G, f.g_ts.data_ptr(), f.g_ms.data_ptr(),
                                   C.byref(out), ws.data_ptr(), ws.numel(), st), "pert_raw_emit")
        t["res_vals"] = f.res_vals
    return ProcessedTables(t, raw.dicts, f.status)


_STREAM_CODED = (("ms", "ms"), ("interface", "if"), ("rpcid", "rpc"), ("rpctype", "rty"))   # (dictionary, id array)
_STREAM_NAMES = ("ms_names", "traceid_names", "interface_names", "rpcid_values", "rpctype_names", "entry_names")


class RawStream:
    """``process_raw`` a chunk at a time, with ids that stay fixed for the life of the stream: what a serving loop
    needs to turn the raw ``MSCallGraph`` / ``MSResource`` rows a cluster keeps emitting into ``append_traces`` /
    ``ResourceSampleWindow.add`` input that agrees with a live ``PatternStore``.

    ``process(raw)`` takes a ``RawTables`` with its own dictionaries (what ``read_raw`` returns) and runs
    ``process_raw``'s steps over that chunk alone, continued from the stream's state (DESIGN.md §8p):
      - deduplication and the timestamp sort are chunk-local; traceid ids continue a counter (next + rank of the
        trace's first sorted position); a traceid an earlier chunk held is refused, so chunks hold whole traces;
      - interface (all rows), rpcid and rpctype (rows of traces with an entry) values keep the id they have; a value
        without one gets next + its rank by first sorted position among the chunk's new values;
      - entries are keyed by (dm, interface); a known key keeps its id, new keys are numbered next + rank by first
        position over the traces with an entry, before the filters (so gaps stay, as in process_raw);
      - coverage reads every microservice with a resource row in this chunk or an earlier one;
      - occurrence: a chunk's covered traces of entry e are kept iff e's covered traces over the stream so far,
        this chunk included, are more than ``min_occurence``.  Traces dropped before their entry was admitted are
        never revisited: the one departure from a whole-table run;
      - a microservice gets an id the first time it appears in a surviving row's um / dm or in a chunk's resource
        rows: next + its rank in name order among the chunk's new names.
    The result is a ``ProcessedTables`` whose ids index the stream's name lists (each covering every id issued up to
    that chunk), plus ``resource_ms`` (int64 CUDA [K]): each raw resource row's microservice id, -1 for a row
    process_raw leaves out.  A fresh stream's first chunk gives process_raw's result bit for bit.

    Refused with ``PertGnnError``, the stream left bit for bit as it was: a traceid of an earlier chunk (named), a
    chunk whose new microservice ids would reach ``max_ms`` (the store's fixed ``n_ms``; None = no limit), a
    dictionary that repeats a value or holds an unhashable one, and the sizes process_raw refuses (``TypeError`` for
    something that is not a RawTables).  Codes outside a chunk's dictionary set the status word, as in process_raw.

    Device state, O(dictionary sizes): an int64 id per stream code of the microservice, interface, rpcid and rpctype
    dictionaries, an int32 has_res per microservice, and the entry table (two int64 per slot, load <= 1/2) with an
    int64 count per entry.  Host state: the value -> stream code dictionaries, the id -> value lists, and a set of
    every traceid seen -- the one part that grows with traces (about 150 bytes per trace for short string ids)."""

    def __init__(self, device="cuda", min_occurence=100, max_ms=None, hash_bits=64):
        dev = torch.device(device)
        if dev.type != "cuda":
            raise _lib.PertGnnError("RawStream needs a CUDA device (no CPU fallback)")
        if dev.index is None:
            dev = torch.device("cuda", torch.cuda.current_device())
        if not 1 <= int(hash_bits) <= 64:
            raise _lib.PertGnnError("RawStream: hash_bits must lie in 1..64")
        self._reset(dev, min_occurence, max_ms, hash_bits)

    def _reset(self, dev, min_occurence, max_ms, hash_bits):
        self.device, self.min_occurence, self.max_ms, self.hash_bits = dev, int(min_occurence), max_ms, int(hash_bits)
        self._codes = {k: {} for k, _ in _STREAM_CODED}          # value -> stream code
        self._traceids = set()
        self._names = {k: [] for k in _STREAM_NAMES}
        self._n = dict(tr=0, **{a: 0 for _, a in _STREAM_CODED}, ent=0)   # ids issued
        i32, i64 = (dict(dtype=d, device=dev) for d in (torch.int32, torch.int64))
        self.t = {f"{a}_id": torch.zeros(0, **i64) for _, a in _STREAM_CODED}
        self.t.update(has_res=torch.zeros(0, **i32), ent_key=torch.full((64,), -1, **i64),
                      ent_id=torch.zeros(64, **i64), ent_cnt=torch.zeros(0, **i64))

    n_ms = property(lambda self: self._n["ms"], doc="microservice ids issued so far")
    ms_names = property(lambda self: list(self._names["ms_names"]))
    traceid_names = property(lambda self: list(self._names["traceid_names"]))
    interface_names = property(lambda self: list(self._names["interface_names"]))
    rpcid_values = property(lambda self: list(self._names["rpcid_values"]))
    rpctype_names = property(lambda self: list(self._names["rpctype_names"]))
    entry_names = property(lambda self: list(self._names["entry_names"]))

    def _map(self, raw):
        """Chunk code -> stream code of every coded dictionary (new values numbered after the known ones, not yet
        added), and the chunk's traceids; refuses repeated or unhashable values and traceids of earlier chunks."""
        maps, new = {}, {}
        for col, _ in _STREAM_CODED:
            known, add = self._codes[col], {}
            vals, n = raw.dicts[col], len(self._codes[col])
            try:
                m = np.fromiter((known[v] if v in known else add.setdefault(v, n + len(add)) for v in vals),
                                np.int64, len(vals))
            except TypeError:
                raise _lib.PertGnnError(f"RawStream.process: a {col} dictionary value is not hashable") from None
            if len(np.unique(m)) != len(m):
                raise _lib.PertGnnError(f"RawStream.process: the {col} dictionary repeats a value")
            maps[col], new[col] = m, add
        trs = raw.dicts["traceid"]
        try:
            tset = set(trs)
        except TypeError:
            raise _lib.PertGnnError("RawStream.process: a traceid is not hashable") from None
        if len(tset) != len(trs):
            raise _lib.PertGnnError("RawStream.process: the traceid dictionary repeats a value")
        if not self._traceids.isdisjoint(tset):
            v = next(v for v in trs if v in self._traceids)
            raise _lib.PertGnnError(f"RawStream.process: traceid {v!r} was in an earlier chunk (a chunk holds whole "
                                    "traces)")
        return maps, new, tset

    def _state(self, maps):
        t, n = self.t, self._n
        p = lambda x: x.data_ptr() if x.numel() else None     # noqa: E731
        return _lib.PertRawState(*(p(maps[c]) for c, _ in _STREAM_CODED), *(p(t[f"{a}_id"]) for _, a in _STREAM_CODED),
                                 *(len(self._codes[c]) for c, _ in _STREAM_CODED), p(t["has_res"]),
                                 p(t["ent_key"]), p(t["ent_id"]), p(t["ent_cnt"]), int(t["ent_key"].shape[0]),
                                 n["tr"], n["if"], n["rpc"], n["rty"], n["ent"], n["ms"])

    def process(self, raw):
        """The next chunk -> ProcessedTables with the stream's ids (and ``resource_ms``); see the class.  Host
        synchronisations: process_raw's three, then one copy of the new ids' codes, which extends the name lists.
        Call ``check()`` on the result before trusting it."""
        _check_raw(raw, "RawStream.process", self.hash_bits)
        maps, new, tset = self._map(raw)
        dev = self.device
        with torch.cuda.device(dev):
            L, st = _lib.lib(), _lib.stream()
            i64 = dict(dtype=torch.int64, device=dev)
            dmaps = {c: torch.from_numpy(m).to(dev) for c, m in maps.items()}
            f = _front(raw, dev, self.hash_bits)
            tab, N = f.tab, f.N
            state = self._state(dmaps)
            ws = torch.empty(int(L.pert_raw_stream_workspace_bytes(C.byref(tab), N)), dtype=torch.uint8,
                             device=dev)
            sizes = torch.empty(7, **i64)
            _lib.check(L.pert_raw_stream_process(C.byref(tab), N, _lib.ptr(f.order), f.has_res.data_ptr(),
                                                 self.min_occurence, C.byref(state), sizes.data_ptr(), ws.data_ptr(),
                                                 ws.numel(), st), "pert_raw_stream_process")
            M, n_ids, n_tr, n_if, n_ent, n_rpc, n_rty = (int(v) for v in sizes.cpu())   # sync 3
            n = self._n
            if self.max_ms is not None and n["ms"] + n_ids > int(self.max_ms):
                raise _lib.PertGnnError(f"RawStream.process: the chunk brings {n_ids} new microservices; "
                                        f"{n['ms']} + {n_ids} ids would reach max_ms = {int(self.max_ms)}")
            # fresh state: the old contents, then room for the chunk's new stream codes and entries
            old = self.t
            fresh = {f"{a}_id": torch.cat([old[f"{a}_id"], torch.full((len(new[c]),), -1, **i64)])
                     for c, a in _STREAM_CODED}
            fresh["has_res"] = torch.cat([old["has_res"], torch.zeros(len(new["ms"]), dtype=torch.int32,
                                                                      device=dev)])
            n_ent2, cap = n["ent"] + n_ent, int(old["ent_key"].shape[0])
            while 2 * n_ent2 > cap:
                cap *= 2
            fresh["ent_key"], fresh["ent_id"] = torch.empty(cap, **i64), torch.empty(cap, **i64)
            fresh["ent_cnt"] = torch.zeros(max(n_ent2, 1), **i64)[:n_ent2]
            fresh["ent_cnt"][:n["ent"]] = old["ent_cnt"]
            K = len(raw.resources["timestamp"])
            resource_ms = torch.empty(max(K, 1), **i64)[:K]
            t = _alloc_out(dev, M, f.G, n_ids, n_tr, n_if, n_ent, n_rpc, n_rty)
            spare = torch.empty(1, **i64)                        # an empty chunk's outputs point here
            out = _raw_out(t, spare)
            p = lambda x: x.data_ptr() if x.numel() else None     # noqa: E731
            so = _lib.PertRawStateOut(*(p(fresh[k]) for k in ("ms_id", "if_id", "rpc_id", "rty_id", "has_res",
                                                              "ent_key", "ent_id")),
                                      fresh["ent_cnt"].data_ptr(), cap, p(resource_ms))
            _lib.check(L.pert_raw_stream_emit(C.byref(tab), N, _lib.ptr(f.order), f.G, f.g_ts.data_ptr(),
                                              f.g_ms.data_ptr(), K, p(f.r_ms), f.has_res.data_ptr(), C.byref(state),
                                              C.byref(out), C.byref(so), ws.data_ptr(), ws.numel(), st),
                       "pert_raw_stream_emit")
            # accepted: swap the state in, then name the new ids
            self.t = fresh
            for c, _ in _STREAM_CODED:
                self._codes[c].update(new[c])
            self._traceids |= tset
            for k, v in (("tr", n_tr), ("ms", n_ids), ("if", n_if), ("rpc", n_rpc), ("rty", n_rty), ("ent", n_ent)):
                n[k] += v
            h = {k: v.tolist() for k, v in zip(("ms_code", "tr_code", "if_code", "rpc_code", "rty_code", "ent_dm",
                                                "ent_if"),
                                               t["_codes"].cpu().split([n_ids, n_tr, n_if, n_rpc, n_rty, n_ent,
                                                                        n_ent]))}   # sync 4
            d, nm = raw.dicts, self._names
            nm["ms_names"] += [d["ms"][i] for i in h["ms_code"]]
            nm["traceid_names"] += [d["traceid"][i] for i in h["tr_code"]]
            nm["interface_names"] += [d["interface"][i] for i in h["if_code"]]
            nm["rpcid_values"] += [d["rpcid"][i] for i in h["rpc_code"]]
            nm["rpctype_names"] += [d["rpctype"][i] for i in h["rty_code"]]
            nm["entry_names"] += [f"{d['ms'][m]}_{i}" for m, i in zip(h["ent_dm"], h["ent_if"])]
            t["res_vals"] = f.res_vals
        views = {k: (v, len(v)) for k, v in nm.items()}
        res = ProcessedTables(t, raw.dicts, f.status, views=views, n_ms=n["ms"])
        res.resource_ms = resource_ms
        return res


def list_csvs(directory):
    """The .csv files of a directory in os.listdir order, the order get_df() concatenates them in."""
    return [os.path.join(directory, f) for f in os.listdir(directory) if f.endswith(".csv")]


_WIN_MAX = 0x7ffffff0                                    # keys, samples and batch samples of a window (int32 offsets)


class WindowRows(NamedTuple):
    """Statistics rows of a ``ResourceSampleWindow``: ``index`` int64 CUDA [u, 2] (timestamp, ms) ascending by key,
    ``values`` float64 CUDA [u, 8] in STATS order, ``late`` the samples an ``add`` skipped because their key is sealed
    (0 for ``rows()``).  ``index`` / ``values`` are what ``PatternStore.append_resources`` takes."""
    index: torch.Tensor
    values: torch.Tensor
    late: int


def _usage_column(a, what, k, dev):
    """float64 [k] on ``dev`` of a usage column: any real numbers (NaN and +-inf allowed, as pandas); ``PertGnnError``
    naming the first sample that is not one."""
    if torch.is_tensor(a) and a.is_cuda:
        if a.dtype == torch.bool or a.dtype.is_complex:
            raise _lib.PertGnnError(f"{what}: numbers expected, got {a.dtype}")
        if a.dim() != 1 or int(a.shape[0]) != k:
            raise _lib.PertGnnError(f"{what}: shape {tuple(a.shape)}, expected ({k},): one value per sample")
        return a.to(dev, torch.float64).contiguous()
    a = a.numpy() if torch.is_tensor(a) else a
    try:
        v = np.asarray(a)
    except (TypeError, ValueError) as e:
        raise _lib.PertGnnError(f"{what}: numbers expected ({e})") from None
    if v.ndim != 1 or v.shape[0] != k:
        raise _lib.PertGnnError(f"{what}: shape {v.shape}, expected ({k},): one value per sample")
    if v.dtype.kind not in "iuf":
        v = np.asarray(a, dtype=object)
        for i, x in enumerate(v):
            if isinstance(x, (bool, np.bool_)) or not isinstance(x, (int, float, np.integer, np.floating)):
                raise _lib.PertGnnError(f"sample {i}: {what} {x!r} is not a number")
    return torch.from_numpy(v.astype(np.float64)).to(dev)


class ResourceSampleWindow:
    """The open buckets of a live resource table, fed raw samples: the statistics preprocess.py:237-242 computes with
    ``groupby(["timestamp", "msname"]).agg(["max", "min", "mean", "median"])``, kept on the GPU and continued sample by
    sample, so a server can publish its open buckets without a host pass or a rebuild over every open sample.

    ``n_ms``: the store's microservice count; samples carry the store's ids (``process_raw``'s name-order ids:
    ``{name: i for i, name in enumerate(proc.ms_names)}``).  A sample's key is its exact (timestamp, ms), as in
    get_df()'s groupby; a caller who wants 30 s buckets floors the timestamps first.

    ``add(timestamps, ms, cpu, mem)`` -> ``WindowRows`` of the keys the call touched, each with the statistics of ALL
    its samples so far: after any sequence of ``add`` and ``seal`` calls they are bit for bit ``process_raw``'s for the
    concatenation of the key's samples in arrival order (calls in order, input order within a call): max / min with a
    strict compare (the first of tied values, so -0.0 vs 0.0, is kept), the Kahan mean, NaN skipped (an all-NaN key
    has NaN statistics), and the median of the key's values in a stable ascending sort, NaN last and +-0 tied.
    ``seal(before)`` makes every key with timestamp < before final and frees its samples; later samples of such keys
    are counted in ``late`` and change nothing.  ``rows()``: the same pair for every open key.

    Device state (csrc/rawtable.cu, pert_raw_window_*): the sorted unique open keys, their run offsets, the resumable
    fold of both columns per key (80 bytes) and each key's values of both columns kept sorted (NaN last, so the runs
    of both columns share the offsets): 16 bytes per open sample and 92 per open key.  An ``add`` sorts the batch
    (torch), merges the keys, continues the folds of the touched keys and merges each touched key's sorted run with
    the batch's, O(S + k log k) for S open and k new samples."""

    STATE_BYTES = 80                                      # per key: GroupStats of cpu and memory (5 doubles each)

    def __init__(self, n_ms, device="cuda"):
        dev = torch.device(device)
        if dev.type != "cuda":
            raise _lib.PertGnnError("ResourceSampleWindow needs a CUDA device (no CPU fallback)")
        if dev.index is None:
            dev = torch.device("cuda", torch.cuda.current_device())
        n_ms = int(n_ms)
        if not 1 <= n_ms <= _I64_MAX:
            raise _lib.PertGnnError(f"ResourceSampleWindow: n_ms = {n_ms} must be at least 1")
        self.device, self.n_ms = dev, n_ms
        self.sealed = _I64_MIN                           # samples with timestamp < sealed are late
        self.n_samples = 0                               # S, known on the host: no read needed to size an add
        self._set(torch.zeros(0, dtype=torch.int64, device=dev), torch.zeros(1, dtype=torch.int32, device=dev),
                  torch.zeros(0, self.STATE_BYTES // 8, dtype=torch.float64, device=dev),
                  torch.zeros(0, dtype=torch.float64, device=dev), torch.zeros(0, dtype=torch.float64, device=dev))

    def _set(self, keys, off, state, cpu_run, mem_run):
        self.t = {"keys": keys, "off": off, "state": state, "cpu_run": cpu_run, "mem_run": mem_run}

    @property
    def n_keys(self):
        return int(self.t["keys"].shape[0])

    def _batch(self, timestamps, ms, cpu, mem):
        """Checked (ts, ms, cpu, mem) on the window's device: int64, int64, float64, float64 [k].  ``PertGnnError``
        naming the first bad sample, before anything changes."""
        dev, n_ms = self.device, self.n_ms
        cols = [timestamps, ms, cpu, mem]
        lens = []
        for c in cols:
            try:
                lens.append(int(c.shape[0]) if hasattr(c, "shape") and len(c.shape) else len(c))
            except TypeError:
                raise _lib.PertGnnError("add: the four columns must be 1-d sequences") from None
        if len(set(lens)) != 1:
            raise _lib.PertGnnError(f"add: columns of different lengths {lens} (timestamps, ms, cpu, mem)")
        k = lens[0]
        if k > _WIN_MAX:
            raise _lib.PertGnnError(f"add: {k} samples exceed 2^31 - 16 per call")
        if all(torch.is_tensor(c) and c.is_cuda for c in cols[:2]):
            for c, what in ((timestamps, "timestamps"), (ms, "ms")):
                if c.dtype.is_floating_point or c.dtype.is_complex or c.dtype == torch.bool:
                    raise _lib.PertGnnError(f"{what}: integers expected, got {c.dtype}")
                if c.dim() != 1:
                    raise _lib.PertGnnError(f"{what}: a 1-d column expected, got shape {tuple(c.shape)}")
            ts, m = (c.to(dev, torch.int64).contiguous() for c in cols[:2])
            if k:
                lo, hi = _key_bounds(n_ms)
                mm = torch.stack([m.min(), m.max(), ts.min(), ts.max()]).tolist()   # one device -> host read
                if mm[0] < 0 or mm[1] >= n_ms or mm[2] < lo or mm[3] > hi:
                    _check_resource_rows(ts.cpu().numpy(), m.cpu().numpy(), n_ms)
        else:
            h = [c.cpu().numpy() if torch.is_tensor(c) else c for c in cols[:2]]
            pairs = np.stack([np.asarray(h[0]), np.asarray(h[1])], 1) if all(
                isinstance(x, np.ndarray) for x in h) else list(zip(h[0], h[1]))
            idx = _index_rows(pairs)                      # floats refused, not truncated; names the first bad sample
            if idx.ndim != 2 or idx.shape[1] != 2:
                raise _lib.PertGnnError("add: timestamps and ms must be 1-d integer columns")
            _check_resource_rows(idx[:, 0], idx[:, 1], n_ms)
            ts, m = (torch.from_numpy(np.ascontiguousarray(idx[:, j])).to(dev) for j in (0, 1))
        return ts, m, _usage_column(cpu, "instance_cpu_usage", k, dev), _usage_column(mem, "instance_memory_usage",
                                                                                       k, dev)

    @_lib.on_device_of
    def add(self, timestamps, ms, cpu, mem):
        """Adds raw samples, one per element of the four columns (host arrays / lists or CUDA tensors): integer
        timestamps (floats are refused), ms in [0, n_ms), cpu and memory usage (numbers; NaN and +-inf allowed).
        Returns ``WindowRows`` of the distinct keys this call touched, ascending by key, with the statistics of all
        their samples so far.  k = 0 is allowed.  Checked on the host before anything changes (``PertGnnError`` naming
        the first bad sample, the window left as it was): equal column lengths, integer timestamps, ms in [0, n_ms),
        keys timestamp * n_ms + ms within int64, numeric usages; CUDA index columns cost one read of their minima and
        maxima.  Beyond that the call makes one device -> host read: the sizes of the merged key table.  Ordered on the
        current stream."""
        ts, m, cpu, mem = self._batch(timestamps, ms, cpu, mem)
        k = int(ts.shape[0])
        dev, n_ms = self.device, self.n_ms
        i32, i64, f64 = (dict(dtype=d, device=dev) for d in (torch.int32, torch.int64, torch.float64))
        if k == 0:
            return WindowRows(torch.zeros(0, 2, **i64), torch.zeros(0, 8, **f64), 0)
        L, st = _lib.lib(), _lib.stream()
        t, U, S = self.t, self.n_keys, self.n_samples
        key = ts * n_ms + m
        bkeys, perm = torch.sort(key, stable=True)        # arrival order within a key
        flags, sizes = torch.empty(2 * (k + 1), **i32), torch.empty(3, **i64)
        ws = torch.empty(int(L.pert_raw_window_workspace_bytes(U, k, min(U + k, _WIN_MAX))), dtype=torch.uint8,
                         device=dev)
        _lib.check(L.pert_raw_window_count(k, bkeys.data_ptr(), n_ms, self.sealed, U, t["keys"].data_ptr(),
                                           flags.data_ptr(), sizes.data_ptr(), ws.data_ptr(), ws.numel(), st),
                   "pert_raw_window_count")
        # every key's batch values ascending (NaN last, ties in arrival order) at the key's positions of bkeys
        srt = []
        for c in (cpu, mem):
            s = torch.sort(c, stable=True)
            srt.append(s.values[torch.sort(key[s.indices], stable=True).indices].contiguous())
        n_late, u, U2 = sizes.tolist()                    # the one device -> host read
        if u == 0:
            return WindowRows(torch.zeros(0, 2, **i64), torch.zeros(0, 8, **f64), n_late)
        S2 = S + k - n_late
        if U2 > _WIN_MAX or S2 > _WIN_MAX:
            raise _lib.PertGnnError(f"add: the window would hold {U2} keys and {S2} samples; at most 2^31 - 16 each")
        new = (torch.empty(U2, **i64), torch.empty(U2 + 1, **i32), torch.empty(U2, self.STATE_BYTES // 8, **f64),
               torch.empty(S2, **f64), torch.empty(S2, **f64))
        ustart, upos = torch.empty(u + 1, **i32), torch.empty(u, **i32)
        p = lambda x: x.data_ptr() if x.numel() else None      # noqa: E731
        _lib.check(L.pert_raw_window_merge(
            U, S, p(t["keys"]), t["off"].data_ptr(), p(t["state"]), p(t["cpu_run"]), p(t["mem_run"]), k,
            bkeys.data_ptr(), perm.data_ptr(), cpu.data_ptr(), mem.data_ptr(), srt[0].data_ptr(), srt[1].data_ptr(),
            flags.data_ptr(), n_late, u, U2, *(p(x) for x in new), ustart.data_ptr(), upos.data_ptr(), ws.data_ptr(),
            ws.numel(), st), "pert_raw_window_merge")
        self._set(*new)
        self.n_samples = S2
        index, values = self._emit(u, upos)
        return WindowRows(index, values, n_late)

    def _emit(self, n, slot):
        t, dev = self.t, self.device
        index = torch.empty(n, 2, dtype=torch.int64, device=dev)
        values = torch.empty(n, 8, dtype=torch.float64, device=dev)
        p = lambda x: x.data_ptr() if x.numel() else None      # noqa: E731
        _lib.check(_lib.lib().pert_raw_window_emit(
            n, None if slot is None else slot.data_ptr(), self.n_keys, p(t["keys"]), t["off"].data_ptr(),
            p(t["state"]), p(t["cpu_run"]), p(t["mem_run"]), self.n_ms, p(index), p(values), _lib.stream()),
            "pert_raw_window_emit")
        return index, values

    @_lib.on_device_of
    def rows(self):
        """``WindowRows`` of every open key (late = 0): what a restarted server republishes."""
        index, values = self._emit(self.n_keys, None)
        return WindowRows(index, values, 0)

    @_lib.on_device_of
    def seal(self, before):
        """Makes every key with timestamp < ``before`` final: its samples are freed now, and later samples of such keys
        are late.  Monotone: a cut at or below the current one does nothing.  One device -> host read (the sealed
        prefix's key and sample counts) when the window holds keys."""
        cut = int(before)
        if not _I64_MIN <= cut <= _I64_MAX:
            raise _lib.PertGnnError(f"seal: before = {cut} is outside int64")
        if cut <= self.sealed:
            return self
        self.sealed = cut
        t, U = self.t, self.n_keys
        if U == 0:
            return self
        ck = cut * self.n_ms                               # ts < cut  <=>  key < cut * n_ms (every ms < n_ms)
        if ck > _I64_MAX:
            j = torch.full((), U, dtype=torch.int64, device=self.device)
        else:
            j = torch.searchsorted(t["keys"], torch.tensor([max(ck, _I64_MIN)], device=self.device))[0]
        j, s0 = torch.stack([j, t["off"][j].long()]).tolist()
        if j == 0:
            return self
        off = t["off"][j:] - s0
        self._set(t["keys"][j:].clone(), off, t["state"][j:].clone(), t["cpu_run"][s0:].clone(),
                  t["mem_run"][s0:].clone())
        self.n_samples -= s0
        return self
