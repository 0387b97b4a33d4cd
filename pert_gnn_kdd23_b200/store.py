"""Device-resident pattern store + on-device batch assembly (SURVEY.md section 8f rows N1 and N4).

The reference assembles every sample on the host (``get_entry_data``, pert_gnn.py:134-173: pandas feature join
``get_x`` :40-67, cached per-pattern tensor builders :77-131), caches the resulting 100k-element ``data_list``
("10+hrs", README.md:12), collates batches with PyG's DataLoader (:201-209) and rebuilds the per-node pattern
probability on the host every step with B tiny H2D copies (:220-230).

``PatternStore`` keeps the reference's artefacts (``runtime2graph``, ``entry2runtimes``, ``resource_df``, ``tr2data`` --
what pert_gnn.py:297-305 loads) resident in HBM in concatenated int32/int64/float32 arrays; ``assemble(trace_ids)``
turns a list of trace ids (8 bytes per graph of H2D traffic instead of ~33 KB) into the collated device ``Batch`` with
4 kernel launches (csrc/store.cu) -- the tensors are bit-identical to ``Batch.from_data_list([get_entry_data(...)])`` +
``transform_pattern_probs`` (tests/test_store.py checks them against the reference's own outputs,
tests/golden/ref_loop.npz).  No CPU fallback: the store lives on a CUDA device.
"""
from __future__ import annotations

import ctypes as C
import itertools

import numpy as np
import torch

from . import _lib, pertgraph
from .data import Batch

# the C structs under the names this module has always exported (the mirrors themselves live in _lib)
_PertStore, _PertBatchOut, _RuntimeKeys, _RuntimeTable = (_lib.PertStore, _lib.PertBatchOut, _lib.PertRuntimeKeys,
                                                          _lib.PertRuntimeTable)
_ChunkMix, _MixOut, _IngestState, _EvictOut = (_lib.PertChunkMix, _lib.PertMixOut, _lib.PertIngestState,
                                                _lib.PertEvictOut)
_EVICT_ARRAYS = _lib.EVICT_ARRAYS


def _last_flags(nptr, ms):
    """pat_last: 1 for the LAST node of every microservice of a pattern, else 0 (get_x's dict ms2nid keeps the last
    one, pert_gnn.py:54-65).  ``nptr``: int64 [n_pat+1] node offsets, ``ms``: int64 [n_all], on one device.  A stable
    sort by ms, then a stable sort by pattern, orders the nodes by (pattern, ms, node index): the last node of every
    run of equal (pattern, ms) is flagged.  Exact for every int64 ms, and no host synchronisation."""
    dev, n_all = ms.device, int(ms.shape[0])
    pid = torch.repeat_interleave(torch.arange(int(nptr.shape[0]) - 1, device=dev), nptr.diff(), output_size=n_all)
    by_ms = torch.sort(ms, stable=True)[1]
    idx = by_ms[torch.sort(pid[by_ms], stable=True)[1]]
    p, m = pid[idx], ms[idx]
    run_end = torch.ones(n_all, dtype=torch.bool, device=dev)
    run_end[:-1] = (p[1:] != p[:-1]) | (m[1:] != m[:-1])
    last = torch.zeros(n_all, dtype=torch.uint8, device=dev)
    last[idx[run_end]] = 1
    return last


def _pattern_arrays(graphs, dev):
    """The pat_* entries of a store's ``t`` on ``dev`` from concatenated patterns (``pertgraph.PertGraphs``: host node /
    edge offsets, ms_id, node_depth, pattern-local edge_index and edge_attr, host or device tensors)."""
    i32, i64 = torch.int32, torch.int64
    nptr, eptr = (torch.from_numpy(np.asarray(p, dtype=np.int64)).to(dev) for p in (graphs.node_ptr, graphs.edge_ptr))
    ms = graphs.ms_id.reshape(-1).to(dev, i64).contiguous()
    ei = graphs.edge_index.to(dev)
    return {"pat_nptr": nptr.to(i32), "pat_eptr": eptr.to(i32), "pat_ms": ms,
            "pat_depth": graphs.node_depth.reshape(-1).to(dev, i64).contiguous(), "pat_last": _last_flags(nptr, ms),
            "pat_src": ei[0].to(i32).contiguous(), "pat_dst": ei[1].to(i32).contiguous(),
            "pat_attr": graphs.edge_attr.to(dev, i64).contiguous()}


def _mix_out(n_ent, n_pairs, dev):
    """The arrays of a rewritten entry mix of n_ent entries with room for n_pairs pairs, and their ``PertMixOut``."""
    i32 = torch.int32
    o = {"ent_ptr": torch.empty(n_ent + 1, dtype=i32, device=dev),
         "ent_pat": torch.empty(n_pairs, dtype=i32, device=dev),
         "ent_prob": torch.empty(n_pairs, dtype=torch.float32, device=dev),
         "cnt": torch.empty(n_pairs, dtype=i32, device=dev), "ent_nodes": torch.empty(n_ent, dtype=i32, device=dev),
         "ent_edges": torch.empty(n_ent, dtype=i32, device=dev), "tot": torch.empty(n_ent, dtype=i32, device=dev)}
    return o, _lib.PertMixOut(*(o[name].data_ptr() for name, _ in _lib.PertMixOut._fields_))


def _cuda_device(device):
    dev = torch.device(device)
    if dev.type != "cuda":
        raise _lib.PertGnnError("PatternStore lives on a CUDA device (no CPU fallback for the hot path)")
    return dev


def asof_index(res_keys, n_ms):
    """As-of index of a store's sorted resource keys (``timestamp * n_ms + ms``, ascending), on their device:
    (ms_ptr [n_ms+1] int32, ts [n_res] int64, row [n_res] int32) -- the rows of microservice m are
    ms_ptr[m] .. ms_ptr[m+1]-1, with ascending timestamps ``ts`` and ``row`` their index into the sorted keys (ascending
    among equal timestamps: a stable regrouping by ms of an order that is already timestamp-major)."""
    ms = torch.remainder(res_keys, n_ms)
    ts = torch.div(res_keys - ms, n_ms, rounding_mode="floor")
    _, row = torch.sort(ms, stable=True)
    ms_ptr = torch.zeros(n_ms + 1, dtype=torch.int64, device=res_keys.device)
    ms_ptr[1:] = torch.cumsum(torch.bincount(ms, minlength=n_ms), 0)
    return ms_ptr.to(torch.int32), ts[row].contiguous(), row.to(torch.int32)


_I64_MIN, _I64_MAX, _I32_MAX = -(1 << 63), (1 << 63) - 1, (1 << 31) - 1


def _key_bounds(n_ms):
    """(lo, hi): the timestamps whose key timestamp * n_ms + ms fits in int64 for every ms in [0, n_ms)."""
    return -((1 << 63) // n_ms), (_I64_MAX - (n_ms - 1)) // n_ms


def _index_rows(idx):
    """int64 [k, 2] host array of (timestamp, ms) pairs (shape checked by the caller); ``PertGnnError`` naming the first
    row that is not a pair of integers within int64 (floats are refused, not truncated)."""
    rows = idx if isinstance(idx, np.ndarray) else list(idx)
    if rows is not idx:
        try:                                             # pairs of integers: one pass per column, no per-row arrays
            ts, ms = np.array([t for t, _ in rows]), np.array([m for _, m in rows])
            if ts.ndim == ms.ndim == 1 and ts.dtype.kind == ms.dtype.kind == "i":
                return np.stack([ts, ms], 1).astype(np.int64)
        except (TypeError, ValueError, OverflowError):
            pass                                         # the general path below names the bad row
    try:
        a = np.asarray(rows)
        if a.dtype.kind != "i" and not isinstance(idx, np.ndarray):
            a = np.array(rows, dtype=object)             # keep every entry's own type, to find the first bad row
    except (TypeError, ValueError, OverflowError) as e:
        raise _lib.PertGnnError(f"resource_index: (timestamp, ms) pairs expected ({e})") from None
    if a.size == 0:
        return np.zeros((0, 2), dtype=np.int64)
    if a.ndim != 2 or a.shape[1] != 2 or a.dtype.kind == "i":
        return a.astype(np.int64) if a.dtype.kind == "i" else a
    if a.dtype.kind == "u":
        bad = (a > _I64_MAX).any(1)
    else:                                                # object, float, bool, str: row by row
        bad = np.array([not all(isinstance(v, (int, np.integer)) and not isinstance(v, (bool, np.bool_)) and
                                _I64_MIN <= int(v) <= _I64_MAX for v in row) for row in a])
    if bad.any():
        i = int(np.argmax(bad))
        raise _lib.PertGnnError(f"resource row {i}: {tuple(a[i].tolist())} is not a pair of int64 integers")
    return a.astype(np.int64)


def _check_resource_rows(ts, ms, n_ms):
    """Raises ``PertGnnError`` naming the first row (int64 host columns) whose microservice is outside [0, n_ms) or
    whose key timestamp * n_ms + ms overflows int64."""
    bad_ms = (ms < 0) | (ms >= n_ms)
    hi = (_I64_MAX - np.where(bad_ms, 0, ms)) // n_ms
    bad = bad_ms | (ts < _key_bounds(n_ms)[0]) | (ts > hi)
    if bad.any():
        i = int(np.argmax(bad))
        if bad_ms[i]:
            raise _lib.PertGnnError(
                f"resource row {i}: microservice {int(ms[i])} is outside [0, {n_ms}), so no pattern can read it: "
                f"keep the rows with ms < store.n_ms, or build the store with a larger n_ms")
        raise _lib.PertGnnError(f"resource row {i}: timestamp {int(ts[i])} overflows the int64 key timestamp * n_ms + "
                                f"ms (n_ms = {n_ms})")


def _int_column(a, what):
    """1-d int64 host copy of an integer array, list or tensor; ``PertGnnError`` for anything else (floats and bools
    are refused, not truncated)."""
    a = a.cpu().numpy() if torch.is_tensor(a) else a
    try:
        a = np.asarray(a)
    except (TypeError, ValueError) as e:
        raise _lib.PertGnnError(f"{what}: integers expected ({e})") from None
    if a.size == 0:
        return np.zeros(0, dtype=np.int64)
    if a.ndim != 1 or a.dtype.kind not in "iu" or (a.dtype.kind == "u" and (a > _I64_MAX).any()):
        raise _lib.PertGnnError(f"{what}: a 1-d array of int64 integers expected, got {a.dtype} of shape {a.shape}")
    return a.astype(np.int64)


def _resolve_mixes(mixes, Q, rt_ids, pat_nodes, pat_edges):
    """Checks the what-if mixes of Q requests and resolves their runtime ids to pattern indices (a dense table for
    compact ids, else a sorted copy of ``rt_ids`` and ``np.searchsorted``): -> (ptr int64 [Q+1], pat int32, prob
    float32 -- float64 rounded as the
    constructor rounds it --, and the requests' node, edge and pattern counts, int64 [Q]).  ``PertGnnError`` naming the
    first bad request."""
    try:
        mix_ptr, mix_rt, mix_prob = mixes
    except (TypeError, ValueError):
        raise _lib.PertGnnError("mixes: a (mix_ptr, mix_rt, mix_prob) triple expected") from None
    ptr, rt = _int_column(mix_ptr, "mix_ptr"), _int_column(mix_rt, "mix_rt")
    try:
        prob = np.asarray(mix_prob.cpu().numpy() if torch.is_tensor(mix_prob) else mix_prob, dtype=np.float64)
    except (TypeError, ValueError) as e:
        raise _lib.PertGnnError(f"mix_prob: numbers expected ({e})") from None
    prob = prob.reshape(-1) if prob.size == 0 else prob
    if prob.ndim != 1 or prob.shape[0] != rt.shape[0]:
        raise _lib.PertGnnError(f"mix_prob: shape {prob.shape}, expected ({rt.shape[0]},): one per runtime of mix_rt")
    if ptr.shape[0] != Q + 1:
        raise _lib.PertGnnError(f"mix_ptr: {ptr.shape[0]} offsets, expected {Q + 1} for {Q} requests")
    if ptr[0] != 0:
        raise _lib.PertGnnError(f"mix_ptr[0] = {int(ptr[0])}, expected 0")
    n = np.diff(ptr)
    if (n < 0).any():
        i = int(np.argmax(n < 0))
        raise _lib.PertGnnError(f"request {i}: mix_ptr is not monotone ({int(ptr[i])} > {int(ptr[i + 1])})")
    if ptr[-1] != rt.shape[0]:
        raise _lib.PertGnnError(f"mix_ptr[{Q}] = {int(ptr[-1])}, but mix_rt holds {rt.shape[0]} runtimes")
    if (n == 0).any():
        raise _lib.PertGnnError(f"request {int(np.argmax(n == 0))}: empty mix")
    # per slot, in request order: unknown runtime, a runtime repeated within its mix, a bad probability
    ids = np.asarray(rt_ids, dtype=np.int64)
    if ids.shape[0] and int(ids.max()) - int(ids.min()) < 4 * ids.shape[0] + (1 << 16):
        # compact ids (the stores' runtime numbering): a dense table, one gather per slot instead of a binary search
        lo, hi = int(ids.min()), int(ids.max())
        lut = np.full(hi - lo + 1, -1, dtype=np.int64)
        lut[ids - lo] = np.arange(ids.shape[0])
        inside = (rt >= lo) & (rt <= hi)
        pidx = np.where(inside, lut[np.where(inside, rt - lo, 0)], -1)
        known = pidx >= 0
        pidx = np.maximum(pidx, 0)
    else:
        order = np.argsort(ids, kind="stable")
        pos = np.minimum(np.searchsorted(ids[order], rt), max(ids.shape[0] - 1, 0))
        known = ids[order][pos] == rt if ids.shape[0] else np.zeros(rt.shape[0], dtype=bool)
        pidx = order[pos] if ids.shape[0] else np.zeros(rt.shape[0], dtype=np.int64)
    owner = np.repeat(np.arange(Q, dtype=np.int64), n)
    again = np.zeros(rt.shape[0], dtype=bool)
    n_ids = max(ids.shape[0], 1)
    if Q * n_ids < (1 << 62):                                   # one int64 sort finds whether any mix repeats a runtime
        key = np.where(known, owner * n_ids + pidx, -1 - np.arange(rt.shape[0]))
        srt = np.sort(key)
        maybe = bool((srt[1:] == srt[:-1]).any())
    else:
        maybe = True
    if maybe:                                                   # which slot: (request, runtime, slot) order
        by = np.lexsort((np.arange(rt.shape[0]), rt, owner))
        again[by[1:]] = (owner[by[1:]] == owner[by[:-1]]) & (rt[by[1:]] == rt[by[:-1]])
    bad_p = ~np.isfinite(prob) | (prob < 0)
    bad = ~known | again | bad_p
    if bad.any():
        k = int(np.argmax(bad))
        q = int(owner[k])
        if not known[k]:
            raise _lib.PertGnnError(f"request {q}: runtime {int(rt[k])} is not in the store (never seen, or evicted)")
        if again[k]:
            raise _lib.PertGnnError(f"request {q}: runtime {int(rt[k])} occurs twice in its mix")
        raise _lib.PertGnnError(f"request {q}: probability {float(prob[k])} of runtime {int(rt[k])} is negative, NaN "
                                "or infinite")
    pat = pidx.astype(np.int64)
    sizes = []
    for per_pat in (pat_nodes, pat_edges):
        cs = np.zeros(rt.shape[0] + 1, dtype=np.int64)
        np.cumsum(per_pat[pat], out=cs[1:])
        sizes.append(cs[ptr[1:]] - cs[ptr[:-1]])
    return ptr, pat.astype(np.int32), prob.astype(np.float32), sizes[0], sizes[1], n


def _override_rows(overrides, n_ms):
    """Checks an override table ``(scenario [k], ms [k], values [k, 8])``: -> (keys scenario * n_ms + ms int64 [k],
    values float32 [k, 8], in input order).  ``PertGnnError`` naming the first bad row."""
    try:
        sc, ms, vals = overrides
    except (TypeError, ValueError):
        raise _lib.PertGnnError("overrides: a (scenario, ms, values) triple expected") from None
    sc, ms = _int_column(sc, "overrides scenario"), _int_column(ms, "overrides ms")
    k = sc.shape[0]
    if ms.shape[0] != k:
        raise _lib.PertGnnError(f"overrides: {k} scenario ids but {ms.shape[0]} microservices")
    try:
        vals = np.asarray(vals.cpu().numpy() if torch.is_tensor(vals) else vals, dtype=np.float64)
    except (TypeError, ValueError) as e:
        raise _lib.PertGnnError(f"overrides values: [k, 8] numbers expected ({e})") from None
    if vals.size == 0 and k == 0:
        vals = vals.reshape(0, 8)
    if vals.shape != (k, 8):
        raise _lib.PertGnnError(f"overrides values: shape {vals.shape}, expected ({k}, 8) for {k} rows")
    bad_m = (ms < 0) | (ms >= n_ms)
    bad_s = sc < 0
    over = ~bad_m & ~bad_s & (sc > (_I64_MAX - np.where(bad_m, 0, ms)) // n_ms)
    bad = bad_m | bad_s | over
    if bad.any():
        i = int(np.argmax(bad))
        if bad_m[i]:
            raise _lib.PertGnnError(f"override row {i}: microservice {int(ms[i])} is outside [0, {n_ms})")
        if bad_s[i]:
            raise _lib.PertGnnError(f"override row {i}: scenario {int(sc[i])} is negative")
        raise _lib.PertGnnError(f"override row {i}: scenario {int(sc[i])} overflows the int64 key scenario * n_ms + "
                                f"ms (n_ms = {n_ms})")
    return sc * n_ms + ms, vals.astype(np.float32)


class _WhatIfArrays:
    """The checked inputs of one what-if call on the device (``PatternStore._what_if_arrays``), or a slice of them:
    host entry ids and the requests' node / edge / pattern counts (sizing), device entry ids, timestamps, the mixes'
    CSR (mix_ptr absolute into mix_pat / mix_prob; None: the entries' own mixes), the scenario ids (None: none) and
    the sorted override table.  Pattern indices are resolved for the store as it is: valid until it changes."""

    def __init__(self, ent, nodes, edges, pats, ent_d, ts_d, ptr_d, pat_d, prob_d, scen_d, ov_keys, ov_vals):
        self.ent, self.nodes, self.edges, self.pats = ent, nodes, edges, pats
        self.ent_d, self.ts_d, self.ptr_d, self.pat_d, self.prob_d = ent_d, ts_d, ptr_d, pat_d, prob_d
        self.scen_d, self.ov_keys, self.ov_vals = scen_d, ov_keys, ov_vals

    def slice(self, i, j):
        return _WhatIfArrays(self.ent[i:j], self.nodes[i:j], self.edges[i:j], self.pats[i:j], self.ent_d[i:j],
                             self.ts_d[i:j], None if self.ptr_d is None else self.ptr_d[i:j + 1], self.pat_d,
                             self.prob_d, None if self.scen_d is None else self.scen_d[i:j], self.ov_keys,
                             self.ov_vals)

    def desc(self):
        p = lambda t: None if t is None else t.data_ptr()            # noqa: E731
        return _lib.PertWhatIf(p(self.ptr_d), p(self.pat_d), p(self.prob_d), p(self.scen_d),
                               int(self.ov_keys.shape[0]), p(self.ov_keys), p(self.ov_vals))


class _TraceIngest:
    """What ``append_traces`` keeps beside a store built by ``from_trace_groups`` (outside ``t``): the graph kind, the
    runtime keys -- rows [3, R'] int64 (um, dm, interface of every pattern's representative, pattern order) and ptr
    [n_pat+1] int32 --, cnt [n_pairs] int32 (traces of every (entry, pattern) pair, in ent_pat order), tot [n_ent] int32
    (traces per entry), tids [n_traces] int64 (every traceid, ascending), the node / edge totals of the patterns, and
    the runtime table (csrc/ingest.cu), built at the first append.  For ``evict_traces``: trace_pat [n_traces] int32
    and trace_tid [n_traces] int64 (the pattern and traceid of every trace, trace-table order), and next_rt, the
    number of runtime ids ever issued (ids are never reused: a runtime seen again after its pattern was evicted is
    new)."""

    def __init__(self, kind, rows, ptr, cnt, tot, tids, n_nodes, n_edges, trace_pat, trace_tid, next_rt):
        self.kind, self.rows, self.ptr, self.cnt, self.tot, self.tids = kind, rows, ptr, cnt, tot, tids
        self.n_nodes, self.n_edges = n_nodes, n_edges
        self.trace_pat, self.trace_tid, self.next_rt = trace_pat, trace_tid, next_rt
        self.table = None                                # dict(slot, h1, h2, S, bits)

    def state(self):
        return _lib.PertIngestState(self.keys(), self.trace_pat.data_ptr(), self.trace_tid.data_ptr(),
                                    self.cnt.data_ptr(), self.tot.data_ptr(), int(self.cnt.shape[0]), self.n_nodes,
                                    self.n_edges, int(self.rows.shape[1]))

    def keys(self):
        return _lib.PertRuntimeKeys(int(self.ptr.shape[0]) - 1, int(self.rows.shape[1]), self.ptr.data_ptr(),
                                    self.rows.data_ptr())

    def table_desc(self):
        t = self.table
        return _lib.PertRuntimeTable(t["S"], t["bits"], t["slot"].data_ptr(), t["h1"].data_ptr(), t["h2"].data_ptr())

    def insert(self, first, hash_bits):
        """Inserts runtimes first.. into the table; rebuilds it (larger) first when the load would pass 1/2 or the hash
        width changes."""
        n = int(self.ptr.shape[0]) - 1
        t = self.table
        if t is None or t["bits"] != hash_bits or 2 * n > t["S"]:
            S = 64
            while S < 4 * n:                             # room to grow to twice the runtimes before the next rebuild
                S <<= 1
            dev = self.rows.device
            self.table = t = {"S": S, "bits": int(hash_bits), "slot": torch.empty(S, dtype=torch.int32, device=dev),
                              "h1": torch.empty(S // 2, dtype=torch.int64, device=dev),
                              "h2": torch.empty(S // 2, dtype=torch.int64, device=dev)}
            first = 0
        keys, tab = self.keys(), self.table_desc()
        _lib.check(_lib.lib().pert_ingest_table_insert(C.byref(keys), first, C.byref(tab), _lib.stream()),
                   "pert_ingest_table_insert")


def _check_span_ms(columns, n_ms):
    """Raises ``PertGnnError`` naming the first span row whose um or dm lies outside [0, n_ms).  Host columns are
    checked on the host; CUDA columns cost one device -> host read of their minima and maxima (and the rows
    themselves only when one is out of range)."""
    host = {}
    dev = [k for k in ("um", "dm") if torch.is_tensor(columns[k]) and columns[k].is_cuda]
    if dev:
        mm = torch.stack([f(columns[k].reshape(-1).long()) for k in dev for f in (torch.min, torch.max)]).tolist()
        if min(mm[0::2]) >= 0 and max(mm[1::2]) < n_ms:
            dev = []
    for k in ("um", "dm"):
        v = columns[k]
        if k in dev:
            host[k] = v.reshape(-1).cpu().numpy()
        elif not (torch.is_tensor(v) and v.is_cuda):
            host[k] = np.asarray(v.numpy() if torch.is_tensor(v) else v).reshape(-1)
    bad = None
    for k, v in host.items():
        b = np.flatnonzero((v < 0) | (v >= n_ms))
        if b.size and (bad is None or b[0] < bad[0]):
            bad = (int(b[0]), k, int(v[b[0]]))
    if bad is not None:
        i, k, v = bad
        raise _lib.PertGnnError(f"span row {i}: {k} = {v} is outside [0, {n_ms}); the store's microservice ids are "
                                f"fixed by its n_ms")


class PatternStore:
    """Patterns, entries, resource table and traces on one CUDA device."""

    def __init__(self, runtime2graph, entry2runtimes, resource_index, resource_values, tr2data, device, n_ms=None):
        # ---- patterns, in the dict order of runtime2graph, concatenated on the host.  Patterns may be CUDA tensors
        # (pertgraph.PertGraphs.pattern), copied one by one; for many patterns use PatternStore.from_graphs
        rt_ids = list(runtime2graph.keys())
        gs = [runtime2graph[rt] for rt in rt_ids]
        ms = [g["ms_id"].reshape(-1).to(torch.int64).cpu() for g in gs]
        ei, ea = [g["edge_index"].cpu() for g in gs], [g["edge_attr"].cpu() for g in gs]
        for g, m, a in zip(gs, ms, ea):
            assert m.shape[0] == int(g["num_nodes"]) and a.shape[1] == ea[0].shape[1]
        ptr = lambda sizes: np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)      # noqa: E731
        graphs = pertgraph.PertGraphs(ptr([m.shape[0] for m in ms]), ptr([e.shape[1] for e in ei]), torch.cat(ms),
                                      torch.cat(ei, 1), torch.cat(ea),
                                      torch.cat([g["node_depth"].reshape(-1).to(torch.int64).cpu() for g in gs]),
                                      None, None)
        self._init_dicts(graphs, rt_ids, entry2runtimes, resource_index, resource_values, tr2data, device, n_ms)

    @classmethod
    def from_graphs(cls, graphs, runtime_ids, entry2runtimes, resource_index, resource_values, tr2data, device=None,
                    n_ms=None):
        """Patterns straight from ``pertgraph.build_pert_graphs`` / ``build_span_graphs`` (``graphs``: PertGraphs;
        ``runtime_ids[i]`` names pattern i): no per-pattern copy or Python work."""
        self = cls.__new__(cls)
        self._init_dicts(graphs, runtime_ids, entry2runtimes, resource_index, resource_values, tr2data,
                         device if device is not None else graphs.ms_id.device, n_ms)
        return self

    def _init_dicts(self, graphs, rt_ids, entry2runtimes, resource_index, resource_values, tr2data, device, n_ms):
        """The constructor's store from concatenated patterns (``graphs``: PertGraphs, host or device tensors; pattern i
        is runtime ``rt_ids[i]``) and the reference's dicts entry2runtimes and tr2data."""
        dev = _cuda_device(device)
        self.rt_ids = list(rt_ids)
        assert len(self.rt_ids) == len(graphs.node_ptr) - 1
        t = _pattern_arrays(graphs, dev)
        pat_nodes, pat_edges = (np.diff(np.asarray(p, dtype=np.int64)) for p in (graphs.node_ptr, graphs.edge_ptr))
        # ---- entries, in the dict order of entry2runtimes[entry] (get_all_runtimes_id_probs, pert_gnn.py:70-74)
        rt_index = {rt: i for i, rt in enumerate(self.rt_ids)}
        n_ent = max(entry2runtimes.keys()) + 1
        ent_ptr, ent_pat, ent_prob = [0], [], []
        ent_nodes, ent_edges = np.zeros(n_ent, dtype=np.int32), np.zeros(n_ent, dtype=np.int32)
        for e in range(n_ent):
            for rt, pr in entry2runtimes.get(e, {}).items():
                k = rt_index[rt]
                ent_pat.append(k)
                ent_prob.append(pr)
                ent_nodes[e] += pat_nodes[k]
                ent_edges[e] += pat_edges[k]
            ent_ptr.append(len(ent_pat))
        # ---- traces, in the dict order of tr2data (get_data_list, pert_gnn.py:176-188)
        self.trace_keys = list(tr2data.keys())
        t_ent = np.array([int(tr2data[k]["entry_id"]) for k in self.trace_keys], dtype=np.int32)
        t_ts = np.array([int(tr2data[k]["timestamp"]) for k in self.trace_keys], dtype=np.int64)
        t_y = np.array([int(tr2data[k]["y"]) for k in self.trace_keys], dtype=np.int64)
        # host copies used to size the outputs without a device sync
        self._h_ent_nodes, self._h_ent_edges = ent_nodes.astype(np.int64), ent_edges.astype(np.int64)
        self._h_ent_pats = np.diff(np.array(ent_ptr)).astype(np.int64)
        self._h_trace_entry = t_ent.astype(np.int64)
        self._h_pat_nodes, self._h_pat_edges = pat_nodes, pat_edges

        def up(a, dtype):
            return torch.from_numpy(np.ascontiguousarray(a, dtype=dtype)).to(dev)

        t.update({
            "ent_ptr": up(ent_ptr, np.int32), "ent_pat": up(ent_pat, np.int32),
            # torch.tensor(python floats, dtype=torch.float) of the reference == float64 -> float32 rounding
            "ent_prob": up(np.array(ent_prob, dtype=np.float64).astype(np.float32), np.float32),
            "ent_nodes": up(ent_nodes, np.int32), "ent_edges": up(ent_edges, np.int32),
            "trace_entry": up(t_ent, np.int32), "trace_ts": up(t_ts, np.int64), "trace_y": up(t_y, np.int64),
        })
        ms_max = int(graphs.ms_id.max()) if n_ms is None and graphs.ms_id.numel() else 0
        self._finish(dev, t, ms_max, resource_index, resource_values, n_ms)

    @classmethod
    def from_artifacts(cls, art, device):
        """``art``: dict with the reference's artefacts (synthetic.make_trace_artifacts schema; with ``graphs`` +
        ``runtime_ids`` -- synthetic.make_pert_artifacts -- the patterns are taken from the device-resident PertGraphs)."""
        if art.get("graphs") is not None:
            return cls.from_graphs(art["graphs"], art["runtime_ids"], art["entry2runtimes"], art["resource_index"],
                                   art["resource_values"], art["tr2data"], device, n_ms=art.get("n_ms"))
        return cls(art["runtime2graph"], art["entry2runtimes"], art["resource_index"], art["resource_values"],
                   art["tr2data"], device, n_ms=art.get("n_ms"))

    @classmethod
    def from_trace_groups(cls, groups, kind, resource_index, resource_values, device=None, n_ms=None):
        """The store of ``PatternStore(runtime2graph, groups.entry2runtimes(), resource_index, resource_values,
        groups.tr2data(), ...)`` with runtime2graph the ``kind`` ("pert" / "span") graph map, built from the device
        arrays of a ``tracegroup.TraceGroups`` without a Python loop over entries, patterns or traces.  Patterns in the
        reference's insertion order, traces in tr2data's key order; the one device->host copy besides the graph build
        is the host sizing arrays the store keeps (per-trace entry and id, per-entry node / edge / pattern totals)."""
        graphs, rt_ids = groups.graphs(kind)
        dev = _cuda_device(device if device is not None else graphs.ms_id.device)
        self = cls.__new__(cls)
        self.rt_ids = list(rt_ids)
        i32, i64 = torch.int32, torch.int64
        with torch.cuda.device(dev):
            t = _pattern_arrays(graphs, dev)
            n_pat, n_all = len(self.rt_ids), int(graphs.node_ptr[-1])
            # entries: entry2runtimes[e] in key order = the (entry, runtime) pairs of the groups
            ent_ptr = groups.ent_pair_ptr
            n_ent, n_pairs = int(ent_ptr.shape[0]) - 1, int(groups.pair_runtime.shape[0])
            ent_pat = groups.runtime_ins[groups.pair_runtime.long()]
            pair_entry = torch.repeat_interleave(torch.arange(n_ent, device=dev), ent_ptr.diff(), output_size=n_pairs)
            sums = []
            for per_pat in (t["pat_nptr"].diff().long(), t["pat_eptr"].diff().long(),
                            torch.ones(n_pat, dtype=i64, device=dev)):
                sums.append(torch.zeros(n_ent, dtype=i64, device=dev).index_add_(0, pair_entry,
                                                                                  per_pat[ent_pat.long()]))
            ent_nodes, ent_edges, ent_pats = sums
            # what append_traces needs besides self.t: the runtime keys and the pair counts.  pair_prob = count / total
            # correctly rounded with count <= total < 2^31, so prob * total rounds back to the count exactly
            tot = groups.ent_trace_ptr.diff().to(i32)
            cnt = torch.round(groups.pair_prob * tot[pair_entry].double()).to(i32)
            order = groups.order.long()
            self._ingest = _TraceIngest(kind, groups._rows[:3].contiguous(), groups.rep_ptr.clone(), cnt, tot,
                                        groups.trace_id, int(graphs.node_ptr[-1]), int(graphs.edge_ptr[-1]),
                                        groups.runtime_ins[groups.runtime[order].long()].to(i32),
                                        groups.trace_id[order], n_pat)
            t_ent = groups.entry[order]
            host = torch.cat([t_ent.long(), groups.trace_id[order], ent_nodes, ent_edges, ent_pats,
                              t["pat_ms"].max().reshape(1) if n_all else torch.zeros(1, dtype=i64, device=dev)]
                             ).cpu().numpy()
            t.update({
                "ent_ptr": ent_ptr.to(dev, i32).contiguous(), "ent_pat": ent_pat.to(i32).contiguous(),
                "ent_prob": groups.pair_prob.to(dev, torch.float32).contiguous(),      # float64 -> float32 rounding
                "ent_nodes": ent_nodes.to(i32), "ent_edges": ent_edges.to(i32),
                "trace_entry": t_ent.to(i32).contiguous(), "trace_ts": groups.bucket[order].contiguous(),
                "trace_y": groups.y[order].contiguous(),
            })
        T = int(order.shape[0])
        self._h_trace_entry, self.trace_keys = host[:T], host[T:2 * T].tolist()
        self._h_ent_nodes, self._h_ent_edges, self._h_ent_pats = (host[2 * T + k * n_ent:2 * T + (k + 1) * n_ent]
                                                                 for k in range(3))
        self._h_pat_nodes, self._h_pat_edges = (np.diff(np.asarray(p, dtype=np.int64))
                                                for p in (graphs.node_ptr, graphs.edge_ptr))
        self._finish(dev, t, int(host[-1]), resource_index, resource_values, n_ms)
        return self

    def _finish(self, dev, t, ms_max, resource_index, resource_values, n_ms):
        """Completes a constructor.  ``t``: the pattern, entry and trace arrays on ``dev``; ``ms_max``: the largest
        microservice id of the patterns (0 without nodes; not read when ``n_ms`` is given).  Adds the resource table:
        the rows go through ``append_resources``' conversion and checks (``PertGnnError`` naming the first bad row),
        are sorted stably by key timestamp * n_ms + ms (equal keys keep their input order), and n_ms defaults to the
        largest microservice id of the patterns and the rows, plus one.  Then the descriptor, the status word and the
        as-of index of the rows (12 bytes per row, kept beside the descriptor; ``append_resources`` keeps it
        current)."""
        idx = _index_rows(resource_index.cpu().numpy() if torch.is_tensor(resource_index) else resource_index)
        if n_ms is None:
            res_max = int(idx[:, 1].max(initial=0)) if idx.ndim == 2 and idx.shape[1] == 2 else 0   # else refused below
            n_ms = max(ms_max, res_max, 0) + 1
        self.device, self.n_ms, self.attr_cols = dev, int(n_ms), int(t["pat_attr"].shape[1])
        with torch.cuda.device(dev):
            ts, ms, vals = self._resource_batch(idx, resource_values)
            keys, order = torch.sort(ts * self.n_ms + ms, stable=True)
            has = torch.zeros(self.n_ms, dtype=torch.uint8, device=dev)
            has[ms] = 1                                          # ms_with_resources (pert_gnn.py:138)
            t.update({"res_keys": keys, "res_vals": vals[order], "ms_has_res": has})
            self.t, self.desc = {}, _lib.PertStore()
            self.status = torch.zeros(1, dtype=torch.int32, device=dev)
            self._commit({name: t[name] for name, _ in _lib.PertStore._fields_[6:]}, asof=asof_index(keys, self.n_ms))

    def _commit(self, t, asof=None, ingest=None):
        """The one place where the store's arrays change: installs ``t`` (entries of ``self.t``), ``asof`` (the as-of
        index, (ms_ptr, ts, row)) and ``ingest`` (fields of ``self._ingest``), then rewrites the descriptor, its counts
        taken from the arrays.  Every tensor replaced is first recorded on the current stream: the kernels that made the
        new arrays and the assembly issued earlier on that stream still read it, so torch's allocator reuses its memory
        only after them."""
        old = [self.t[name] for name in t if name in self.t]
        if asof is not None and hasattr(self, "asof_t"):
            old += list(self.asof_t.values())
        if ingest is not None:
            old += [v for v in (getattr(self._ingest, name) for name in ingest) if torch.is_tensor(v)]
        st = torch.cuda.current_stream() if old else None
        for v in old:
            v.record_stream(st)
        self.t.update(t)
        if asof is not None:
            self._set_asof(*asof)
        for name, v in (ingest or {}).items():
            setattr(self._ingest, name, v)
        d = self.desc
        d.n_pat, d.n_ent = int(self.t["pat_nptr"].shape[0]) - 1, int(self.t["ent_ptr"].shape[0]) - 1
        d.n_res, d.n_ms, d.attr_cols = int(self.t["res_keys"].shape[0]), self.n_ms, self.attr_cols
        d.n_traces = int(self.t["trace_entry"].shape[0])
        for name, v in self.t.items():
            setattr(d, name, v.data_ptr())

    def _set_asof(self, ms_ptr, ts, row):
        self.asof_t = {"ms_ptr": ms_ptr, "ts": ts, "row": row}
        a = _lib.PertResourceAsOf()
        for k, v in self.asof_t.items():
            setattr(a, k, v.data_ptr())
        self.asof_desc = a

    def _resource_batch(self, resource_index, resource_values):
        """Checked (ts, ms, values) of an update on the store's device: int64 [k], int64 [k], float32 [k, 8]."""
        idx = self._index_array(resource_index)
        k = int(idx.shape[0])
        vals = resource_values
        if not (torch.is_tensor(vals) and vals.is_cuda):
            try:
                vals = np.asarray(vals.numpy() if torch.is_tensor(vals) else vals, dtype=np.float64)
            except (TypeError, ValueError) as e:
                raise _lib.PertGnnError(f"resource_values: [k, 8] numbers expected ({e})") from None
            if vals.size == 0 and k == 0:
                vals = vals.reshape(0, 8)
        if tuple(vals.shape) != (k, 8):
            raise _lib.PertGnnError(f"resource_values: shape {tuple(vals.shape)}, expected ({k}, 8) for {k} rows")
        ts, ms = self._index_columns(idx)
        if torch.is_tensor(vals):
            vals = vals.to(self.device)
            vals = (vals if vals.dtype == torch.float32 else vals.double().float()).contiguous()
            if vals.data_ptr() % 16:                     # the merge reads rows with 16-byte vector loads
                vals = vals.clone()
        else:
            vals = torch.from_numpy(vals.astype(np.float32)).to(self.device)  # the constructor's float64 -> float32
        return ts, ms, vals

    def _index_array(self, resource_index):
        """[k, 2] integer (timestamp, ms) pairs of an update: an int64 tensor on the store's device for CUDA input, else
        an int64 host array (``PertGnnError`` naming the first row that is not a pair of int64 integers)."""
        if torch.is_tensor(resource_index) and resource_index.is_cuda:
            if resource_index.dtype.is_floating_point or resource_index.dtype.is_complex or \
                    resource_index.dtype == torch.bool:
                raise _lib.PertGnnError(f"resource_index: integer (timestamp, ms) pairs expected, got "
                                        f"{resource_index.dtype}")
            idx = resource_index.to(self.device, torch.int64)
        else:
            idx = _index_rows(resource_index.numpy() if torch.is_tensor(resource_index) else resource_index)
        if idx.ndim != 2 or idx.shape[1] != 2:
            raise _lib.PertGnnError(f"resource_index: [k, 2] (timestamp, ms) pairs expected, got shape "
                                    f"{tuple(idx.shape)}")
        return idx

    def _index_columns(self, idx):
        """Checked (ts, ms) int64 [k] on the store's device of ``_index_array``'s pairs: ``PertGnnError`` naming the first
        row whose microservice is outside [0, n_ms) or whose key overflows int64."""
        n_ms = self.n_ms
        if torch.is_tensor(idx):
            ts, ms = idx[:, 0].contiguous(), idx[:, 1].contiguous()
            if int(idx.shape[0]):
                lo, hi = _key_bounds(n_ms)
                mm = torch.stack([ms.min(), ms.max(), ts.min(), ts.max()]).tolist()   # one device -> host read
                if mm[0] < 0 or mm[1] >= n_ms or mm[2] < lo or mm[3] > hi:
                    _check_resource_rows(ts.cpu().numpy(), ms.cpu().numpy(), n_ms)
            return ts, ms
        ts, ms = idx[:, 0], idx[:, 1]
        _check_resource_rows(ts, ms, n_ms)
        return tuple(torch.from_numpy(np.ascontiguousarray(c)).to(self.device) for c in (ts, ms))

    @_lib.on_device_of
    def append_resources(self, resource_index, resource_values, evict_before=None, replace=False):
        """Appends resource rows to the live store and, with ``evict_before``, drops every row whose timestamp is
        < ``evict_before`` (old rows and the appended ones alike), on the device: the sorted table and the as-of index
        are merged, not rebuilt (csrc/resources.cu, O(n + k log k) for n rows and k new ones).

        ``replace=True`` gives the table dict-update semantics: every (timestamp, ms) key of the batch first removes all
        the store's rows with that key (duplicates left by plain appends included), then the batch's last row of that
        key, in input order, goes in.  A key the store does not hold is simply inserted.  The result is the constructor's
        store of the old rows without the batch's keys, followed by those last rows in input order; the cut applies as
        for a plain append.  It costs one more device -> host read (the number of distinct keys) and one binary search
        per old row into the batch's keys.  ``replace=False`` (the default) keeps every row, as described below.

        ``resource_index``: the constructor's (timestamp, ms) pairs, or an integer array / CUDA tensor [k, 2] (floats
        are refused, not truncated); ``resource_values``: [k, 8], a host array (float64, rounded to float32 as the
        constructor rounds it) or a CUDA tensor (copied if its data is not 16-byte aligned).  k = 0 is allowed.  Afterwards the resource state (``desc.n_res``, ``t["res_keys"]``,
        ``t["res_vals"]``, ``t["ms_has_res"]``, ``asof_t``) is bit for bit that of a store built by the constructor,
        with the same ``n_ms``, from the surviving rows in arrival order: the constructor's rows, then every append's in
        order.  Rows with equal (timestamp, ms) are all kept and the joins read the first to arrive: a later row does
        not replace an earlier one unless the call has ``replace=True``.  A microservice gains ``ms_has_res`` with its
        first row and loses it with its last.

        Checked on the host before anything changes (``PertGnnError`` naming the first bad row; the store is left as it
        was): the shape of ``resource_values``, microservice ids in [0, n_ms), keys timestamp * n_ms + ms within int64
        and at most 2^31 - 1 rows after the update.  CUDA-tensor input costs one device -> host read of the columns'
        minima and maxima, and every update one read of the resulting sizes.

        Ordered on the current stream: a batch assembled earlier on that stream sees the old table, one assembled later
        the new one; ``desc``, ``t``, ``asof_t`` and ``asof_desc`` point at the new arrays and the old ones return to
        torch's caching allocator on that stream.  Other streams that read the store need the caller's
        synchronisation, as for any tensor, and a CUDA graph the caller captured around ``pert_store_assemble*`` holds
        the old pointers and has to be captured again (``train.predict`` assembles eagerly and needs nothing)."""
        cut = self._cut(evict_before)
        ts, ms, vals = self._resource_batch(resource_index, resource_values)
        k = int(ts.shape[0])
        if k == 0 and evict_before is None:
            return self
        if replace:
            self._update_resources(ts * self.n_ms + ms, vals, cut, insert=True)
            return self
        dev, n_ms, i32 = self.device, self.n_ms, torch.int32
        L = _lib.lib()
        nk, perm = torch.sort(ts * n_ms + ms, stable=True)
        grp = torch.sort(torch.remainder(nk, n_ms), stable=True)[1].to(i32)     # (ms, ts)-grouped, stable
        ms_ptr = torch.empty(n_ms + 1, dtype=i32, device=dev)
        seg = torch.empty(2 * n_ms, dtype=i32, device=dev)
        sizes = torch.empty(3, dtype=torch.int64, device=dev)
        _lib.check(L.pert_store_resources_count(C.byref(self.desc), C.byref(self.asof_desc), nk.data_ptr(),
                                                grp.data_ptr(), k, cut, ms_ptr.data_ptr(), seg.data_ptr(),
                                                sizes.data_ptr(), _lib.stream()), "pert_store_resources_count")
        p, q, n_out = sizes.tolist()
        if n_out > _I32_MAX:
            raise _lib.PertGnnError(f"the update would leave {n_out} resource rows; a store holds at most 2^31 - 1")
        if p == 0 and q == k:
            return self                                  # nothing evicted, nothing appended
        out = {"res_keys": torch.empty(n_out, dtype=torch.int64, device=dev),
               "res_vals": torch.empty(n_out, 8, dtype=torch.float32, device=dev),
               "ms_has_res": torch.empty(n_ms, dtype=torch.uint8, device=dev)}
        a_ts, a_row = torch.empty(n_out, dtype=torch.int64, device=dev), torch.empty(n_out, dtype=i32, device=dev)
        _lib.check(L.pert_store_resources_merge(
            C.byref(self.desc), C.byref(self.asof_desc), nk.data_ptr(), perm.data_ptr(), vals.data_ptr(),
            grp.data_ptr(), k, ms_ptr.data_ptr(), seg.data_ptr(), p, q, n_out, out["res_keys"].data_ptr(),
            out["res_vals"].data_ptr(), out["ms_has_res"].data_ptr(), a_ts.data_ptr(), a_row.data_ptr(),
            _lib.stream()), "pert_store_resources_merge")
        self._commit(out, asof=(ms_ptr, a_ts, a_row))
        return self

    @_lib.on_device_of
    def delete_resources(self, resource_index, evict_before=None):
        """Removes every resource row whose (timestamp, ms) key is in ``resource_index`` and, with ``evict_before``,
        every row whose timestamp is < ``evict_before``; returns the number of rows removed, by key and by the cut
        together.  Keys the store does not hold and repeated keys are allowed and remove nothing more.  The result is
        the constructor's store of the surviving rows in arrival order: the exact join then reports a deleted
        ``(bucket, ms)`` row as missing (``PERT_ERR_RANGE``) while ``ms`` keeps other rows, the as-of join reads the
        newest earlier row, and ``ms`` loses ``ms_has_res`` with its last row.

        ``resource_index`` takes the formats of ``append_resources`` and the same host checks (microservice ids in
        [0, n_ms), keys within int64; ``PertGnnError`` naming the first bad row, the store left as it was).  The count
        comes from the sizes the update reads back anyway.  Ordered on the current stream, fresh arrays swapped in, as
        ``append_resources``."""
        cut = self._cut(evict_before)
        ts, ms = self._index_columns(self._index_array(resource_index))
        if int(ts.shape[0]) == 0 and evict_before is None:
            return 0
        return self._update_resources(ts * self.n_ms + ms, None, cut, insert=False)

    def _cut(self, evict_before):
        if evict_before is None:
            return _I64_MIN
        cut = int(evict_before)
        if not _I64_MIN <= cut <= _I64_MAX:
            raise _lib.PertGnnError(f"evict_before = {cut} is outside int64")
        return cut

    def _update_resources(self, keys, vals, cut, insert):
        """The drop-set update of ``append_resources(replace=True)`` (``insert``: the last row of each key goes back in)
        and ``delete_resources``: ``keys`` int64 [k] checked batch keys on the device, ``vals`` float32 [k, 8] or None.
        Returns the number of rows removed."""
        dev, n_ms, i32 = self.device, self.n_ms, torch.int32
        L = _lib.lib()
        nk, perm = torch.sort(keys, stable=True)
        last = torch.ones_like(nk, dtype=torch.bool)
        last[:-1] = nk[1:] != nk[:-1]                    # the last of each run of a stable sort: the last in input order
        dk = nk[last]                                    # the drop set: sorted unique keys (one device -> host read)
        dgrp = torch.sort(torch.remainder(dk, n_ms), stable=True)[1].to(i32)
        n_drop = int(dk.shape[0])
        # a replace inserts the drop set's keys (grouped alike), with the values of each key's last row
        ik, iperm, igrp, k = (dk, perm[last], dgrp, n_drop) if insert else (dk[:0], perm[:0], dgrp[:0], 0)
        cnt = torch.empty(2 * (n_drop + 1), dtype=i32, device=dev)
        ms_ptr = torch.empty(n_ms + 1, dtype=i32, device=dev)
        seg = torch.empty(3 * n_ms + 1, dtype=i32, device=dev)
        sizes = torch.empty(4, dtype=torch.int64, device=dev)
        _lib.check(L.pert_store_resources_update_count(
            C.byref(self.desc), C.byref(self.asof_desc), dk.data_ptr(), dgrp.data_ptr(), n_drop, ik.data_ptr(),
            igrp.data_ptr(), k, cut, cnt.data_ptr(), ms_ptr.data_ptr(), seg.data_ptr(), sizes.data_ptr(),
            _lib.stream()), "pert_store_resources_update_count")
        p, q, n_out, n_dropped = sizes.tolist()
        if n_out > _I32_MAX:
            raise _lib.PertGnnError(f"the update would leave {n_out} resource rows; a store holds at most 2^31 - 1")
        if p == 0 and q == k and n_dropped == 0:
            return 0                                     # nothing evicted, inserted or dropped
        out = {"res_keys": torch.empty(n_out, dtype=torch.int64, device=dev),
               "res_vals": torch.empty(n_out, 8, dtype=torch.float32, device=dev),
               "ms_has_res": torch.empty(n_ms, dtype=torch.uint8, device=dev)}
        a_ts, a_row = torch.empty(n_out, dtype=torch.int64, device=dev), torch.empty(n_out, dtype=i32, device=dev)
        _lib.check(L.pert_store_resources_update_merge(
            C.byref(self.desc), C.byref(self.asof_desc), dk.data_ptr(), dgrp.data_ptr(), cnt.data_ptr(), n_drop,
            ik.data_ptr(), iperm.data_ptr(), vals.data_ptr() if insert else 0, igrp.data_ptr(), k, ms_ptr.data_ptr(),
            seg.data_ptr(), p, q, n_dropped, n_out, out["res_keys"].data_ptr(), out["res_vals"].data_ptr(),
            out["ms_has_res"].data_ptr(), a_ts.data_ptr(), a_row.data_ptr(), _lib.stream()),
            "pert_store_resources_update_merge")
        self._commit(out, asof=(ms_ptr, a_ts, a_row))
        return p + n_dropped

    def evict_resources(self, before):
        """Drops every resource row whose timestamp is < ``before``: ``append_resources`` with no rows."""
        return self.append_resources(np.zeros((0, 2), dtype=np.int64), np.zeros((0, 8)), evict_before=before)

    @_lib.on_device_of
    def append_traces(self, columns, hash_bits=64):
        """Takes a chunk of processed span rows (``columns``: the nine ``tracegroup.COLUMNS``, int64 host arrays or CUDA
        tensors, whole traces) into the live store and returns the store indices of its traces, a ``range`` at the
        end of the trace table: existing trace indices, pattern indices and entry key orders stay valid.  Only stores
        built by ``from_trace_groups`` keep the runtime keys this needs.

        Afterwards the store equals, bit for bit (``t``, the descriptor's counts, ``rt_ids``, ``trace_keys`` and the
        host sizing arrays), the constructor fed the grouping of all chunks so far in which the chunk is the leading
        key of every order: runtime ids by (chunk, smallest traceid), so a new runtime gets id next_rt + j (next_rt:
        the number of runtime ids the store has issued, n_rt unless ``evict_traces`` dropped patterns); iteration
        order (chunk, entry, traceid); a runtime the store has keeps its representative and graph, a new one's
        representative is its first trace in the chunk's iteration order and its pattern goes after the existing ones;
        entry e keeps its old keys in order, then the runtimes new to it in order of first appearance in the chunk;
        probabilities (old count + chunk count) / (old total + chunk total) in fp64, rounded to fp32.  The graphs of
        the new runtimes are built as ``TraceGroups.graphs`` builds them, with the store's graph kind.  The resource
        rows and the as-of index are untouched.  ``hash_bits`` narrows the runtime hashes (tests force collisions
        with it); a collision costs a row comparison and never merges two runtimes.

        Checked before anything changes (``PertGnnError``, the store is left as it was): the chunk's grouping errors
        (``TraceGroups.check``), a traceid the store already has, um / dm outside [0, n_ms) (naming the first row),
        a new representative emptied by the row filters (naming the runtime), an ``edge_attr`` width other than the
        store's, and node, edge, pair or trace counts above 2^31 - 1.

        Host synchronisations: those of ``group_traces`` and its ``check()``; for CUDA um / dm columns one read of their
        minima and maxima; one read of the chunk's traceids and entries; one of the match result (new runtimes and the
        representatives' row offsets), followed, when there are new runtimes, by the copy of their rows for the host
        row filters and the graph build's own read; one of the merged entry sizes.  Ordered on the current stream,
        like ``append_resources``: the old arrays return to torch's allocator on that stream."""
        from . import tracegroup

        ing = self._ingest_of("append_traces")
        missing = [k for k in tracegroup.COLUMNS if k not in columns]
        if missing:
            raise _lib.PertGnnError(f"append_traces: columns {missing} are missing")
        dev, L = self.device, _lib.lib()
        i32, i64 = torch.int32, torch.int64
        _check_span_ms(columns, self.n_ms)
        g = tracegroup.group_traces(columns, dev, hash_bits).check()
        T_old, Tc = len(self.trace_keys), len(g)
        order = g.order.long()
        c_tid, c_ent = g.trace_id[order], g.entry[order]
        tids = ing.tids
        if tids.numel():
            pos = torch.searchsorted(tids, g.trace_id).clamp_(max=int(tids.shape[0]) - 1)
            dup = tids[pos] == g.trace_id
        else:                                            # every trace was evicted
            dup = torch.zeros_like(g.trace_id, dtype=torch.bool)
        host = torch.cat([c_tid, c_ent.long(), g.trace_id, dup.long()]).cpu().numpy()
        h_tid, h_ent = host[:Tc], host[Tc:2 * Tc]
        if host[3 * Tc:].any():
            raise _lib.PertGnnError(f"append_traces: traceid {int(host[2 * Tc + np.argmax(host[3 * Tc:])])} is "
                                    "already in the store (a chunk holds whole traces, each traceid once)")
        if T_old + Tc > _I32_MAX:
            raise _lib.PertGnnError(f"append_traces: {T_old + Tc} traces exceed the store's 2^31 - 1")
        # ---- match the chunk's runtimes against the store's (runtime table, csrc/ingest.cu)
        n_pat, n_c = len(self.rt_ids), g.n_runtimes
        if ing.table is None or ing.table["bits"] != hash_bits:
            ing.insert(0, hash_bits)
        keys, tab = ing.keys(), ing.table_desc()
        ck = _lib.PertRuntimeKeys(n_c, int(g._rows.shape[1]), g.rep_ptr.data_ptr(), g._rows.data_ptr())
        pat_of, new_rep, new_rt = (torch.empty(n_c, dtype=i32, device=dev) for _ in range(3))
        n_new_d = torch.empty(1, dtype=i64, device=dev)
        ws = torch.empty(int(L.pert_ingest_match_workspace_bytes(n_c)), dtype=torch.uint8, device=dev)
        _lib.check(L.pert_ingest_match(C.byref(keys), C.byref(tab), C.byref(ck), g.runtime_ins.data_ptr(),
                                       pat_of.data_ptr(), new_rep.data_ptr(), new_rt.data_ptr(), n_new_d.data_ptr(),
                                       ws.data_ptr(), ws.numel(), _lib.stream()), "pert_ingest_match")
        h = torch.cat([n_new_d, new_rep.long(), new_rt.long(), g.rep_ptr.long()]).cpu().numpy()
        k = int(h[0])
        reps, new_ids, rep_ptr = h[1:1 + k], h[1 + n_c:1 + n_c + k], h[1 + 2 * n_c:]
        new_ids = new_ids + (ing.next_rt - n_pat)        # ids n_pat + j -> next_rt + j: evicted ids are not reused
        # ---- graphs of the new runtimes, built as TraceGroups.graphs builds them
        lens = rep_ptr[reps + 1] - rep_ptr[reps]
        new_ptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
        sel = torch.from_numpy(np.repeat(rep_ptr[reps] - new_ptr[:-1], lens) + np.arange(int(new_ptr[-1]))).to(dev)
        new_rows = g._rows[:, sel]
        g_nptr = g_eptr = np.zeros(1, dtype=np.int64)
        if k:
            graphs = tracegroup.representative_graphs(new_rows.cpu().numpy(), new_ptr, new_ids, dev, ing.kind,
                                                      "append_traces: ")
            if int(graphs.edge_attr.shape[1]) != self.attr_cols:
                raise _lib.PertGnnError(f"append_traces: edge_attr has {int(graphs.edge_attr.shape[1])} columns, the "
                                        f"store {self.attr_cols}")
            g_nptr, g_eptr = (np.asarray(p, dtype=np.int64) for p in (graphs.node_ptr, graphs.edge_ptr))
        n_nodes, n_edges = ing.n_nodes + int(g_nptr[-1]), ing.n_edges + int(g_eptr[-1])
        n_pairs, n_pc = int(ing.cnt.shape[0]), int(g.pair_runtime.shape[0])
        for what, v in (("pattern nodes", n_nodes), ("pattern edges", n_edges), ("(entry, runtime) pairs",
                                                                                  n_pairs + n_pc)):
            if v > _I32_MAX:
                raise _lib.PertGnnError(f"append_traces: {v} {what} exceed the store's 2^31 - 1")
        t = {}
        if k:                                            # the new patterns go after the old ones
            new = _pattern_arrays(graphs, dev)
            new["pat_nptr"], new["pat_eptr"] = new["pat_nptr"][1:] + ing.n_nodes, new["pat_eptr"][1:] + ing.n_edges
            t = {name: torch.cat([self.t[name], v]) for name, v in new.items()}
        # ---- entry mixes (csrc/ingest.cu)
        n_ent_c = int(g.ent_pair_ptr.shape[0]) - 1
        n_ent = max(int(self.desc.n_ent), n_ent_c)
        mix = _lib.PertChunkMix(n_ent_c, n_pc, g.ent_pair_ptr.data_ptr(), g.ent_trace_ptr.data_ptr(),
                                g.pair_runtime.data_ptr(), g.pair_prob.data_ptr(), g.runtime_ins.data_ptr(),
                                pat_of.data_ptr())
        o, out = _mix_out(n_ent, n_pairs + n_pc, dev)
        ws = torch.empty(int(L.pert_ingest_merge_workspace_bytes(n_pairs, n_pc, n_ent)), dtype=torch.uint8, device=dev)
        nptr, eptr = (t.get(name, self.t[name]) for name in ("pat_nptr", "pat_eptr"))
        _lib.check(L.pert_ingest_merge(C.byref(self.desc), ing.cnt.data_ptr(), ing.tot.data_ptr(), n_pairs,
                                       C.byref(mix), nptr.data_ptr(), eptr.data_ptr(), n_ent, C.byref(out),
                                       ws.data_ptr(), ws.numel(), _lib.stream()), "pert_ingest_merge")
        sizes = torch.cat([o["ent_ptr"], o["ent_nodes"], o["ent_edges"]]).long().cpu().numpy()
        ent_ptr_h = sizes[:n_ent + 1]
        n_pairs_out = int(ent_ptr_h[-1])
        t.update({"ent_ptr": o["ent_ptr"], "ent_pat": o["ent_pat"][:n_pairs_out],
                  "ent_prob": o["ent_prob"][:n_pairs_out], "ent_nodes": o["ent_nodes"], "ent_edges": o["ent_edges"],
                  "trace_entry": torch.cat([self.t["trace_entry"], c_ent]),
                  "trace_ts": torch.cat([self.t["trace_ts"], g.bucket[order]]),
                  "trace_y": torch.cat([self.t["trace_y"], g.y[order]])})
        key_rows_old = int(ing.rows.shape[1])
        self._commit(t, ingest={
            "rows": torch.cat([ing.rows, new_rows[:3]], dim=1),
            "ptr": torch.cat([ing.ptr, torch.from_numpy(new_ptr[1:] + key_rows_old).to(dev, i32)]),
            "cnt": o["cnt"][:n_pairs_out], "tot": o["tot"],
            "tids": torch.sort(torch.cat([ing.tids, g.trace_id])).values,
            "trace_pat": torch.cat([ing.trace_pat, pat_of[g.runtime_ins[g.runtime[order].long()].long()]]),
            "trace_tid": torch.cat([ing.trace_tid, c_tid]), "n_nodes": n_nodes, "n_edges": n_edges,
            "next_rt": ing.next_rt + k})
        self.rt_ids.extend(int(r) for r in new_ids)
        self.trace_keys.extend(h_tid.tolist())
        self._h_trace_entry = np.concatenate([self._h_trace_entry, h_ent])
        self._h_ent_nodes, self._h_ent_edges = sizes[n_ent + 1:2 * n_ent + 1], sizes[2 * n_ent + 1:]
        self._h_ent_pats = np.diff(ent_ptr_h)
        self._h_pat_nodes = np.concatenate([self._h_pat_nodes, np.diff(g_nptr)])
        self._h_pat_edges = np.concatenate([self._h_pat_edges, np.diff(g_eptr)])
        if k:
            ing.insert(n_pat, hash_bits)
        return range(T_old, T_old + Tc)

    @_lib.on_device_of
    def evict_traces(self, before):
        """Drops every trace whose bucket (``t["trace_ts"]``) is < ``before`` from the live store, with what only those
        traces held, and returns ``remap``: a numpy int64 array over the old trace indices, the new index of every
        surviving trace and -1 for an evicted one.  Survivors keep their order (``remap`` is monotone on them), so a
        held ``StoreLoader`` dataset or index list stays valid after ``remap[ids]`` and dropping the -1s.  Only stores
        built by ``from_trace_groups`` keep the per-trace patterns this needs.

        Afterwards the store equals, bit for bit (``t``, the descriptor's counts, ``rt_ids``, ``trace_keys`` and the
        host sizing arrays), ``PatternStore(runtime2graph', entry2runtimes', resources, tr2data', n_ms=store.n_ms)``:
        tr2data' the old one without the evicted traces, in order; entry2runtimes'[e] for every e < n_ent (n_ent never
        shrinks) e's old keys in order without those left with no trace, probabilities surviving count / surviving
        total in fp64, rounded to fp32, and ``{}`` for an entry with no trace left (``check_entries`` refuses it);
        runtime2graph' the old map restricted to the runtimes that keep a trace, in order, with the same graphs -- a
        pattern whose representative was evicted keeps that representative's graph and key rows.  A pattern with no
        trace left goes with its nodes, edges and runtime key; its runtime id is not reused: the runtime, seen again by
        ``append_traces``, is new (a new id, representative and graph).  The resource rows and the as-of index are
        untouched; every new array has its exact new size (the kernels of csrc/ingest.cu count, then compact).

        ``before`` outside int64 raises ``PertGnnError``.  When no trace is evicted the store is left as it is and the
        identity is returned.  Host synchronisations: one read of the surviving sizes, one read of the host copies
        (remap, the surviving traces' entries, the surviving patterns, the entry sizing arrays).  Ordered on the
        current stream, like ``append_resources``: the old arrays return to torch's allocator on that stream."""
        cut = int(before)
        if not _I64_MIN <= cut <= _I64_MAX:
            raise _lib.PertGnnError(f"evict_traces: before = {cut} is outside int64")
        ing = self._ingest_of("evict_traces")
        dev, L = self.device, _lib.lib()
        i32, i64 = torch.int32, torch.int64
        T, n_pat, n_ent = int(self.desc.n_traces), int(self.desc.n_pat), int(self.desc.n_ent)
        if T == 0:
            return np.zeros(0, dtype=np.int64)
        state = ing.state()
        ws = torch.empty(int(L.pert_ingest_evict_workspace_bytes(T, int(ing.cnt.shape[0]), n_pat, n_ent)),
                         dtype=torch.uint8, device=dev)
        sizes_d = torch.empty(6, dtype=i64, device=dev)
        _lib.check(L.pert_ingest_evict_count(C.byref(self.desc), C.byref(state), cut, ws.data_ptr(), ws.numel(),
                                             sizes_d.data_ptr(), _lib.stream()), "pert_ingest_evict_count")
        sizes = [int(x) for x in sizes_d.tolist()]
        T2, P2, n_pat2, N2, E2, K2 = sizes
        if T2 == T:
            return np.arange(T, dtype=np.int64)
        empty = lambda n, dt: torch.empty(n, dtype=dt, device=dev)            # noqa: E731
        mix, mix_out = _mix_out(n_ent, P2, dev)
        o = {"remap": empty(T, i64), "trace_entry": empty(T2, i32), "trace_ts": empty(T2, i64),
             "trace_y": empty(T2, i64), "trace_pat": empty(T2, i32), "trace_tid": empty(T2, i64),
             "pat_new": empty(n_pat, i32), "pat_nptr": empty(n_pat2 + 1, i32), "pat_eptr": empty(n_pat2 + 1, i32),
             "pat_ms": empty(N2, i64), "pat_depth": empty(N2, i64), "pat_last": empty(N2, torch.uint8),
             "pat_src": empty(E2, i32), "pat_dst": empty(E2, i32), "pat_attr": empty((E2, self.attr_cols), i64),
             "key_ptr": empty(n_pat2 + 1, i32), "key_rows": empty((3, K2), i64)}
        out = _lib.PertEvictOut(mix_out, *(o[name].data_ptr() for name in _lib.EVICT_ARRAYS), K2)
        _lib.check(L.pert_ingest_evict_apply(C.byref(self.desc), C.byref(state), (C.c_longlong * 6)(*sizes),
                                             ws.data_ptr(), ws.numel(), C.byref(out), _lib.stream()),
                   "pert_ingest_evict_apply")
        host = torch.cat([o["remap"], o["trace_entry"].long(), o["pat_new"].long(), mix["ent_ptr"].long(),
                          mix["ent_nodes"].long(), mix["ent_edges"].long()]).cpu().numpy()
        remap, h_ent, pat_new, ent_ptr_h, h_nodes, h_edges = np.split(host, np.cumsum([T, T2, n_pat, n_ent + 1, n_ent]))
        tids = torch.sort(o["trace_tid"]).values
        t = {"pat_nptr": o["pat_nptr"], "pat_eptr": o["pat_eptr"], "pat_ms": o["pat_ms"], "pat_depth": o["pat_depth"],
             "pat_last": o["pat_last"], "pat_src": o["pat_src"], "pat_dst": o["pat_dst"], "pat_attr": o["pat_attr"],
             "ent_ptr": mix["ent_ptr"], "ent_pat": mix["ent_pat"], "ent_prob": mix["ent_prob"],
             "ent_nodes": mix["ent_nodes"], "ent_edges": mix["ent_edges"], "trace_entry": o["trace_entry"],
             "trace_ts": o["trace_ts"], "trace_y": o["trace_y"]}
        self._commit(t, ingest={"rows": o["key_rows"], "ptr": o["key_ptr"], "cnt": mix["cnt"], "tot": mix["tot"],
                                "tids": tids, "trace_pat": o["trace_pat"], "trace_tid": o["trace_tid"], "n_nodes": N2,
                                "n_edges": E2})
        ing.table = None                                 # it holds pattern indices: the next append rebuilds it
        self.rt_ids = [r for r, p in zip(self.rt_ids, pat_new) if p >= 0]
        # the surviving keys in order: a C-level filter of the list, several times faster than a list of the device
        # traceids (no new int objects)
        self.trace_keys = list(itertools.compress(self.trace_keys, (remap >= 0).view(np.uint8).tobytes()))
        self._h_trace_entry, self._h_ent_nodes, self._h_ent_edges = h_ent, h_nodes, h_edges
        self._h_ent_pats = np.diff(ent_ptr_h)
        self._h_pat_nodes, self._h_pat_edges = self._h_pat_nodes[pat_new >= 0], self._h_pat_edges[pat_new >= 0]
        return remap

    def _ingest_of(self, fn):
        """``_ingest``, or ``PertGnnError`` for ``fn`` when the store keeps no runtime keys."""
        ing = getattr(self, "_ingest", None)
        if ing is None:
            raise _lib.PertGnnError(f"{fn}: this store keeps no runtime keys (it was built from dicts or by "
                                    "from_graphs); build it with PatternStore.from_trace_groups to "
                                    f"{fn.replace('_', ' ')}")
        return ing

    def __len__(self):
        return len(self.trace_keys)

    @property
    def resident_bytes(self):
        return sum(v.numel() * v.element_size() for v in self.t.values())

    def sizes(self, trace_ids):
        """(N, E, P) of a batch from the host copies -- no device sync."""
        ent = self._h_trace_entry[np.asarray(trace_ids, dtype=np.int64)]
        return int(self._h_ent_nodes[ent].sum()), int(self._h_ent_edges[ent].sum()), int(self._h_ent_pats[ent].sum())

    def _outputs(self, B, N, E, Pn, launch, keepalive, label=True):
        """Allocates the Batch tensors, runs ``launch(offsets_ptr, out_ptr)`` (one of the assembly entry points) and
        wraps the outputs into a device ``Batch``; without ``label`` there is no ``y`` (its pointer stays NULL)."""
        dev = self.device
        f32, i64 = torch.float32, torch.int64
        out = {
            "x": torch.empty(N, 9, dtype=f32, device=dev), "edge_index": torch.empty(2, E, dtype=i64, device=dev),
            "edge_attr": torch.empty(E, self.attr_cols, dtype=i64, device=dev),
            "cat_X": torch.empty(N, 1, dtype=i64, device=dev), "node_depth": torch.empty(N, 1, dtype=i64, device=dev),
            "pattern_num_nodes": torch.empty(N, 1, dtype=f32, device=dev),
            "pattern_probs": torch.empty(Pn, 1, dtype=f32, device=dev),
            "entry_id": torch.empty(B, dtype=i64, device=dev), "y": torch.empty(B, dtype=i64, device=dev),
            "rt_probs": torch.empty(N, 1, dtype=f32, device=dev), "batch": torch.empty(N, dtype=i64, device=dev),
            "ptr": torch.empty(B + 1, dtype=i64, device=dev) if B else torch.zeros(1, dtype=i64, device=dev),
        }
        if not label:
            del out["y"]
        offsets = torch.empty(3 * (B + 1), dtype=torch.int32, device=dev)
        o = _lib.PertBatchOut()
        for k, v in out.items():
            setattr(o, k, v.data_ptr())
        launch(offsets.data_ptr(), C.byref(o))
        from . import ops

        if B:
            ops.LAUNCHES["n"] += 4
        b = Batch()
        b._store.update(out)
        object.__setattr__(b, "_num_graphs", B)
        object.__setattr__(b, "_keepalive", keepalive + (offsets,))
        return b

    @_lib.on_device_of
    def assemble(self, trace_ids, ids_device=None):
        """-> device ``Batch`` of the traces ``trace_ids`` (sequence of ints into the store's trace table).
        ``ids_device``: the same ids already on the device (int64) -- e.g. a slice of a resident epoch permutation --
        to skip even the 8-byte-per-graph H2D copy."""
        ids = np.asarray(trace_ids, dtype=np.int64)
        B = int(ids.shape[0])
        N, E, Pn = self.sizes(ids)
        if ids_device is None:
            ids_device = torch.from_numpy(ids).to(self.device, non_blocking=True)

        def launch(offsets, out):
            rc = _lib.lib().pert_store_assemble(C.byref(self.desc), ids_device.data_ptr(), B, N, E, offsets, out,
                                                self.status.data_ptr(), _lib.stream())
            _lib.check(rc, "pert_store_assemble")

        return self._outputs(B, N, E, Pn, launch, (ids_device,))

    def check_entries(self, entry_ids):
        """Raises ``PertGnnError`` naming the first request whose entry id is out of range or has no patterns."""
        ent = np.asarray(entry_ids, dtype=np.int64).reshape(-1)
        n_ent = int(self._h_ent_nodes.shape[0])
        inside = (ent >= 0) & (ent < n_ent)
        bad = ~inside
        bad[inside] = self._h_ent_pats[ent[inside]] == 0
        if bad.any():
            i = int(np.argmax(bad))
            why = "has no patterns" if inside[i] else f"is outside [0, {n_ent})"
            raise _lib.PertGnnError(f"request {i}: entry {int(ent[i])} {why}")
        return ent

    @_lib.on_device_of
    def assemble_requests(self, entry_ids, timestamps, asof=False, device_arrays=None, mixes=None, overrides=None,
                          scenario_ids=None):
        """-> device ``Batch`` of the requests (entry ``entry_ids[b]`` at time ``timestamps[b]``, in ms): every field of
        ``assemble`` but ``y``.  The resources are those of the time bucket floor(t / 30000) * 30000, joined exactly
        (a missing row of a resourced microservice sets the status word, see ``check``) or, with ``asof``, from the
        newest row at or before the bucket (none: the missing indicator, no error).  The entry ids are checked and the
        outputs sized on the host (``PertGnnError`` before any launch); ``device_arrays``: the same two columns already
        on the device (int64), e.g. slices of a request list uploaded once -- ``timestamps`` may then be None.

        What-if requests (``mixes``, ``overrides``, ``scenario_ids``; with all three None the call above):

        - ``mixes = (mix_ptr [Q+1], mix_rt, mix_prob)``: request q's own pattern mix, runtime ids ``mix_rt[k]`` (the
          store's numbering, ``rt_ids``) with probabilities ``mix_prob[k]`` (float64 or float32, rounded to float32 as
          the constructor rounds them) for k = mix_ptr[q] .. mix_ptr[q+1]-1.  The graph is the concatenation of those
          patterns in mix order, with these probabilities as ``pattern_probs`` / ``rt_probs``, in place of the entry's
          stored mix; the entry id still selects the entry embedding and is written to ``entry_id``.  Probabilities
          need not sum to 1 (the model is defined for any weights, so a mix may be scaled).  Runtime ids are resolved on
          every call, so a mix stays valid across ``append_traces`` and ``evict_traces`` unless one of its runtimes was
          evicted.
        - ``overrides = (scenario [k], ms [k], values [k, 8])`` and ``scenario_ids [Q]`` (-1: none): at the node that
          receives statistics for microservice m (its last node in the pattern), a request with scenario s reads the
          override row (s, m) if there is one -- its values, indicator 0, no store join, even for an m without resource
          rows -- and the store's exact or as-of join otherwise.  Among several rows of one (s, m) the first given
          wins.  A scenario without rows means no override.

        Checked on the host before any launch (``PertGnnError`` naming the first bad request, row or runtime): a
        malformed ``mix_ptr`` (length, ``mix_ptr[0] != 0``, not monotone, last offset != ``len(mix_rt)``), an empty
        mix, a runtime the store does not hold or repeated within a mix, a negative, NaN or infinite probability, an
        entry outside [0, n_ent) (with ``mixes`` an entry whose own mix is empty is fine: it is not read; without, as
        above), override rows with ms outside [0, n_ms), a negative scenario or an int64-overflowing key, override
        values that are not [k, 8] numbers, scenario ids below -1, and node, edge or pattern totals above 2^31 - 1.
        The override table is sorted stably on the device once per call."""
        if isinstance(device_arrays, _WhatIfArrays):
            return self._assemble_what_if(device_arrays, asof)
        if mixes is not None or overrides is not None or scenario_ids is not None:
            if device_arrays is not None:
                raise _lib.PertGnnError("device_arrays: a what-if call takes its inputs on the host")
            return self._assemble_what_if(self._what_if_arrays(entry_ids, timestamps, mixes, overrides, scenario_ids),
                                          asof)
        ent = self.check_entries(entry_ids)
        B = int(ent.shape[0])
        N, E, Pn = (int(self._h_ent_nodes[ent].sum()), int(self._h_ent_edges[ent].sum()),
                    int(self._h_ent_pats[ent].sum()))
        if device_arrays is None:
            ts = np.asarray(timestamps, dtype=np.int64).reshape(-1)
            if ts.shape[0] != B:
                raise _lib.PertGnnError(f"{B} entry ids but {ts.shape[0]} timestamps")
            device_arrays = (torch.from_numpy(ent).to(self.device, non_blocking=True),
                             torch.from_numpy(ts).to(self.device, non_blocking=True))
        ent_d, ts_d = device_arrays
        if ent_d.numel() != B or ts_d.numel() != B or ent_d.dtype != torch.int64 or ts_d.dtype != torch.int64:
            raise _lib.PertGnnError("device_arrays: two int64 device tensors of one element per request")
        ent_d, ts_d = ent_d.contiguous(), ts_d.contiguous()

        def launch(offsets, out):
            rc = _lib.lib().pert_store_assemble_requests(
                C.byref(self.desc), C.byref(self.asof_desc) if asof else None, ent_d.data_ptr(), ts_d.data_ptr(), B,
                N, E, offsets, out, self.status.data_ptr(), _lib.stream())
            _lib.check(rc, "pert_store_assemble_requests")

        return self._outputs(B, N, E, Pn, launch, (ent_d, ts_d), label=False)

    @_lib.on_device_of
    def _what_if_arrays(self, entry_ids, timestamps, mixes=None, overrides=None, scenario_ids=None):
        """Checks a what-if call's inputs (``assemble_requests``) and uploads them once: -> ``_WhatIfArrays``."""
        ent = _int_column(entry_ids, "entry_ids")
        Q = int(ent.shape[0])
        ts = _int_column(timestamps, "timestamps")
        if ts.shape[0] != Q:
            raise _lib.PertGnnError(f"{Q} entry ids but {ts.shape[0]} timestamps")
        mix = None
        if mixes is None:
            self.check_entries(ent)
            nodes, edges, pats = self._h_ent_nodes[ent], self._h_ent_edges[ent], self._h_ent_pats[ent]
        else:
            n_ent = int(self._h_ent_nodes.shape[0])
            out = (ent < 0) | (ent >= n_ent)
            if out.any():
                i = int(np.argmax(out))
                raise _lib.PertGnnError(f"request {i}: entry {int(ent[i])} is outside [0, {n_ent})")
            *mix, nodes, edges, pats = _resolve_mixes(mixes, Q, self.rt_ids, self._h_pat_nodes, self._h_pat_edges)
        sc = None
        if scenario_ids is not None:
            sc = _int_column(scenario_ids, "scenario_ids")
            if sc.shape[0] != Q:
                raise _lib.PertGnnError(f"{Q} requests but {sc.shape[0]} scenario ids")
            if (sc < -1).any():
                i = int(np.argmax(sc < -1))
                raise _lib.PertGnnError(f"request {i}: scenario id {int(sc[i])} is below -1 (-1: no scenario)")
        keys, vals = _override_rows(overrides if overrides is not None else ((), (), ()), self.n_ms)
        # ---- every check passed: one upload of each array
        dev = self.device
        up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev, non_blocking=True)    # noqa: E731
        ptr_d, pat_d, prob_d = (None,) * 3 if mix is None else (up(a) for a in mix)
        scen_d = None if sc is None else up(sc)
        if keys.shape[0]:
            ov_keys, perm = torch.sort(up(keys), stable=True)    # the first of equal keys stays first
            ov_vals = up(vals)[perm].contiguous()                # a fresh allocation: 16-byte aligned
        else:
            ov_keys = torch.zeros(0, dtype=torch.int64, device=dev)
            ov_vals = torch.zeros(0, 8, dtype=torch.float32, device=dev)
        return _WhatIfArrays(ent, nodes, edges, pats, up(ent), up(ts), ptr_d, pat_d, prob_d, scen_d, ov_keys, ov_vals)

    def _assemble_what_if(self, w, asof):
        B = int(w.ent.shape[0])
        N, E, Pn = int(w.nodes.sum()), int(w.edges.sum()), int(w.pats.sum())
        for what, v in (("nodes", N), ("edges", E), ("patterns", Pn)):
            if v > _I32_MAX:
                raise _lib.PertGnnError(f"the requests hold {v} {what}; a batch holds at most 2^31 - 1")
        d = w.desc()

        def launch(offsets, out):
            rc = _lib.lib().pert_store_assemble_whatif(
                C.byref(self.desc), C.byref(self.asof_desc) if asof else None, C.byref(d), w.ent_d.data_ptr(),
                w.ts_d.data_ptr(), B, N, E, offsets, out, self.status.data_ptr(), _lib.stream())
            _lib.check(rc, "pert_store_assemble_whatif")

        keep = tuple(t for t in (w.ent_d, w.ts_d, w.ptr_d, w.pat_d, w.prob_d, w.scen_d, w.ov_keys, w.ov_vals)
                     if t is not None)
        return self._outputs(B, N, E, Pn, launch, keep, label=False)

    @_lib.on_device_of
    def lookup_resources(self, timestamps, ms, asof=False):
        """The resource row request assembly joins for each (timestamp, ms) query: -> (values [k, 8] float32, found [k]
        bool), device tensors.  The row of (floor(t / 30000) * 30000, ms) under the exact join, or with ``asof`` the
        newest row of ms at or before that bucket (the first of equal keys, as assembly reads it); no row, or ms
        outside [0, n_ms): zeros and False.  E.g. the scenario "the current row x 1.2" is ``values * 1.2`` as override
        values.  ``timestamps`` / ``ms``: int64 host arrays or CUDA tensors of one length."""
        dev = self.device
        cols = []
        for a, what in ((timestamps, "timestamps"), (ms, "ms")):
            if torch.is_tensor(a) and a.is_cuda:
                if a.dtype.is_floating_point or a.dtype.is_complex or a.dtype == torch.bool:
                    raise _lib.PertGnnError(f"{what}: integers expected, got {a.dtype}")
                cols.append(a.reshape(-1).to(dev, torch.int64).contiguous())
            else:
                cols.append(torch.from_numpy(_int_column(a, what)).to(dev, non_blocking=True))
        ts_d, ms_d = cols
        k = int(ts_d.shape[0])
        if ms_d.shape[0] != k:
            raise _lib.PertGnnError(f"{k} timestamps but {ms_d.shape[0]} microservices")
        values = torch.empty(k, 8, dtype=torch.float32, device=dev)
        found = torch.empty(k, dtype=torch.bool, device=dev)
        _lib.check(_lib.lib().pert_store_lookup_resources(
            C.byref(self.desc), C.byref(self.asof_desc) if asof else None, ts_d.data_ptr(), ms_d.data_ptr(), k,
            values.data_ptr(), found.data_ptr(), _lib.stream()), "pert_store_lookup_resources")
        return values, found

    def id_bounds(self):
        """The embedding rows the store's live data needs, {"entry", "cat", "interface", "rpctype"}: n_ent entries,
        the largest microservice id of the patterns (``pat_ms``) + 1, and the largest interface and rpctype ids of
        the pattern edges (``pat_attr`` columns 0 and 1) + 1; 0 where there is none.  Reduced on the device, one
        device-to-host read (``train.grow_embeddings`` grows a model to these counts)."""
        t = self.t
        with torch.cuda.device(self.device):
            cols = [t["pat_ms"].reshape(-1)] + [t["pat_attr"][:, c] if self.attr_cols > c else t["pat_ms"][:0]
                                                for c in (0, 1)]
            top = torch.stack([torch.cat([c, c.new_full((1,), -1)]).amax() for c in cols]).cpu().tolist()
        return {"entry": int(self.desc.n_ent), "cat": top[0] + 1, "interface": top[1] + 1, "rpctype": top[2] + 1}

    def check(self):
        """Synchronising check of the status word (trace id or entry id out of range / missing (timestamp, ms) row of
        the exact join)."""
        code = int(self.status.item())
        if code != 0:
            _lib.check(code, "pert_store_assemble")


class StoreLoader:
    """DataLoader-shaped iterator over a PatternStore: yields device batches assembled on the GPU.
    ``torch_geometric.loader.DataLoader(data_list, batch_size, shuffle)`` look-alike (``len(loader.dataset)``, iteration)
    for the part of the reference loop that consumes batches (pert_gnn.py:219, :260)."""

    def __init__(self, store: PatternStore, trace_ids, batch_size, shuffle=False, generator=None):
        self.store, self.batch_size, self.shuffle, self.generator = store, int(batch_size), shuffle, generator
        self.dataset = list(trace_ids)

    def __len__(self):
        return -(-len(self.dataset) // self.batch_size)

    def max_sizes(self):
        """Host-only upper bound (N, E, B) of any batch of any shuffle: the sums of the ``batch_size`` largest
        per-trace node and edge counts, and ``batch_size`` graphs (``train.BucketedTrainStep.reserve``)."""
        ids = np.asarray(self.dataset, dtype=np.int64)
        b = min(self.batch_size, len(ids))
        ent = self.store._h_trace_entry[ids]
        n = np.sort(np.asarray(self.store._h_ent_nodes, dtype=np.int64)[ent])[::-1]
        e = np.sort(np.asarray(self.store._h_ent_edges, dtype=np.int64)[ent])[::-1]
        return int(n[:b].sum()), int(e[:b].sum()), int(b)

    def __iter__(self):
        ids = np.asarray(self.dataset, dtype=np.int64)
        if self.shuffle:
            perm = torch.randperm(len(ids), generator=self.generator).numpy()
            ids = ids[perm]
        for i in range(0, len(ids), self.batch_size):
            yield self.store.assemble(ids[i:i + self.batch_size])
