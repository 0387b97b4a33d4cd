"""Raw call-graph and resource rows -> the processed span and resource tables, on the GPU.

The reference's preprocess.py get_df() (:191-266) reads the Alibaba ``MSCallGraph`` / ``MSResource`` CSV files with
pandas and turns them into ``processed_df`` and ``processed_resource_df``: drop duplicates, sort by timestamp,
factorise five columns, find every trace's entry in a Python loop over traces, filter traces by resource coverage and
per-entry occurrence, renumber the microservices and aggregate the resource rows per (timestamp, msname).

Here the host only parses the files and dictionary-encodes their values (``read_raw``); everything after that runs
over the whole table in csrc/rawtable.cu (``process_raw``).  The result's ``columns`` are the nine
``tracegroup.COLUMNS`` that ``group_traces`` takes, and ``resource_index`` / ``resource_values`` are the rows the
``PatternStore`` constructors take.  There is no CPU fallback: without the CUDA library the calls raise.

Two orders the reference leaves unspecified are fixed here: rows with equal timestamps keep their concatenation order
(pandas' sort_values is an unstable quicksort), and microservice ids follow the lexicographic order of the names (the
reference numbers a Python ``set``, whose order is hash-randomised).
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np
import torch

from . import _lib
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

    def __init__(self, t, dicts, status):
        self.status = status
        self.columns = {k: t[k] for k in COLUMNS}
        self.row = t["row"]
        self.resource_index, self.resource_values = t["res_index"], t["res_vals"]
        self._codes, self._dicts, self._names = {k: t[k] for k in _NAME_CODES}, dicts, {}
        self.n_ms = int(t["ms_code"].shape[0])

    def _lookup(self, name):
        """An id -> value list, built on first use (one device-to-host copy of its code array and a Python list as
        long as the ids: a million traces make a million-element traceid_names)."""
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
    if not isinstance(raw, RawTables):
        raise TypeError("process_raw: a RawTables expected (read_raw builds one)")
    if not 1 <= int(hash_bits) <= 64:
        raise _lib.PertGnnError("process_raw: hash_bits must lie in 1..64")
    R, K = len(raw), len(raw.resources["timestamp"])
    if R > 1 << 30 or len(raw.dicts["traceid"]) > 1 << 30:
        raise _lib.PertGnnError(f"process_raw: {max(R, len(raw.dicts['traceid']))} call-graph rows or traceids exceed "
                                "2^30")
    if K > 0x7ffffff0:
        raise _lib.PertGnnError(f"process_raw: {K} resource rows exceed 2^31 - 16")
    with torch.cuda.device(dev):
        L, st = _lib.lib(), _lib.stream()
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
        # ---- call graph: duplicates, stable sort by timestamp, the filters, the processed columns (:212-254)
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
        nbytes = int(L.pert_raw_process_workspace_bytes(C.byref(tab), N))
        if nbytes < 0:
            raise _lib.PertGnnError("process_raw: table sizes out of range")
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        sizes = torch.empty(7, **i64)
        _lib.check(L.pert_raw_process(C.byref(tab), N, _lib.ptr(order), has_res.data_ptr(), int(min_occurence),
                                      sizes.data_ptr(), ws.data_ptr(), ws.numel(), st), "pert_raw_process")
        M, n_ids, n_tr, n_if, n_ent, n_rpc, n_rty = (int(v) for v in sizes.cpu())   # sync 3
        # every output at least one element, so no pointer is NULL; sliced to its size
        alloc = lambda n, *w: torch.empty(max(n, 1), *w, **i64)[:n]           # noqa: E731
        t = {k: alloc(M) for k in COLUMNS + ("row",)}
        t.update(res_index=alloc(G, 2), ms_code=alloc(n_ids), tr_code=alloc(n_tr), if_code=alloc(n_if),
                 rpc_code=alloc(n_rpc), rty_code=alloc(n_rty), ent_dm=alloc(n_ent), ent_if=alloc(n_ent))
        out = _lib.PertRawOut(*(t[k].data_ptr() for k in _lib.RAW_OUT))
        _lib.check(L.pert_raw_emit(C.byref(tab), N, _lib.ptr(order), G, g_ts.data_ptr(), g_ms.data_ptr(),
                                   C.byref(out), ws.data_ptr(), ws.numel(), st), "pert_raw_emit")
        t["res_vals"] = res_vals
    return ProcessedTables(t, raw.dicts, status)


def list_csvs(directory):
    """The .csv files of a directory in os.listdir order, the order get_df() concatenates them in."""
    return [os.path.join(directory, f) for f in os.listdir(directory) if f.endswith(".csv")]
