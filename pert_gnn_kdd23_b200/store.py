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

import numpy as np
import torch

from . import _lib
from .data import Batch

I32, I64, P = C.c_int32, C.c_longlong, C.c_void_p


class _PertStore(C.Structure):
    _fields_ = [("n_pat", I32), ("n_ent", I32), ("n_res", I32), ("n_ms", I32), ("attr_cols", I32),
                ("n_traces", I64),
                ("pat_nptr", P), ("pat_eptr", P), ("pat_ms", P), ("pat_depth", P), ("pat_last", P), ("pat_src", P),
                ("pat_dst", P), ("pat_attr", P), ("ent_ptr", P), ("ent_pat", P), ("ent_prob", P), ("ent_nodes", P),
                ("ent_edges", P), ("res_keys", P), ("res_vals", P), ("ms_has_res", P), ("trace_entry", P),
                ("trace_ts", P), ("trace_y", P)]


class _PertBatchOut(C.Structure):
    _fields_ = [(k, P) for k in ("x", "cat_X", "node_depth", "pattern_num_nodes", "rt_probs", "batch", "edge_index",
                                 "edge_attr", "entry_id", "y", "ptr", "pattern_probs")]


def _last_occurrence_flags(all_ms, nptr):
    """flags[i] = 1 iff node i is the LAST node of its microservice inside its pattern (patterns = nptr slices)."""
    n_all = int(all_ms.shape[0])
    flags = np.zeros(n_all, dtype=np.uint8)
    if n_all:
        pid = np.repeat(np.arange(len(nptr) - 1, dtype=np.int64), np.diff(nptr))
        lo = int(all_ms.min())
        key = pid * (int(all_ms.max()) - lo + 1) + (all_ms - lo)
        _, first_rev = np.unique(key[::-1], return_index=True)
        flags[n_all - 1 - first_rev] = 1
    return flags


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


class _BulkPatterns:
    """Concatenated host arrays of many patterns (PatternStore.from_graphs)."""

    def __init__(self, rt_ids, node_ptr, edge_ptr, ms_id, node_depth, edge_index, edge_attr):
        self.rt_ids, self.node_ptr, self.edge_ptr = rt_ids, node_ptr, edge_ptr
        self.ms_id, self.node_depth, self.edge_index, self.edge_attr = ms_id, node_depth, edge_index, edge_attr


class PatternStore:
    """Patterns, entries, resource table and traces on one CUDA device."""

    def __init__(self, runtime2graph, entry2runtimes, resource_index, resource_values, tr2data, device, n_ms=None):
        dev = torch.device(device)
        if dev.type != "cuda":
            raise _lib.PertGnnError("PatternStore lives on a CUDA device (no CPU fallback for the hot path)")
        self.device = dev
        # ---- patterns, in the dict order of runtime2graph (or the bulk arrays of pertgraph.PertGraphs, see from_graphs)
        if isinstance(runtime2graph, _BulkPatterns):
            bp = runtime2graph
            self.rt_ids = list(bp.rt_ids)
            nptr, eptr = bp.node_ptr.astype(np.int64), bp.edge_ptr.astype(np.int64)
            ms = [bp.ms_id.astype(np.int64)]
            depth = [bp.node_depth.astype(np.int64)]
            src, dst = [bp.edge_index[0].astype(np.int32)], [bp.edge_index[1].astype(np.int32)]
            attr = [bp.edge_attr.astype(np.int64)]
            cols = bp.edge_attr.shape[1]
        else:
            self.rt_ids = list(runtime2graph.keys())
            nptr, eptr = [0], [0]
            ms, depth, src, dst, attr = [], [], [], [], []
            cols = None
            for rt in self.rt_ids:
                g = runtime2graph[rt]
                n = int(g["num_nodes"])
                # patterns may be CUDA tensors (pertgraph.PertGraphs.pattern): the host copy sizes batches and finds the
                # last occurrence of every microservice; for many patterns use PatternStore.from_graphs (one bulk copy)
                m = g["ms_id"].reshape(-1).to(torch.int64).cpu().numpy()
                assert m.shape[0] == n
                ei = g["edge_index"].cpu().numpy()
                ea = g["edge_attr"].cpu().numpy()
                cols = ea.shape[1] if cols is None else cols
                assert ea.shape[1] == cols
                nptr.append(nptr[-1] + n)
                eptr.append(eptr[-1] + ei.shape[1])
                ms.append(m)
                depth.append(g["node_depth"].reshape(-1).to(torch.int64).cpu().numpy())
                src.append(ei[0].astype(np.int32))
                dst.append(ei[1].astype(np.int32))
                attr.append(ea.astype(np.int64))
        rt_index = {rt: i for i, rt in enumerate(self.rt_ids)}
        nptr, eptr = np.asarray(nptr, dtype=np.int64), np.asarray(eptr, dtype=np.int64)
        # get_x's dict ms2nid keeps the LAST node of every microservice of a pattern (pert_gnn.py:54-65): vectorised as
        # the first occurrence of (pattern, ms) in the reversed node list
        all_ms = np.concatenate(ms) if ms else np.zeros(0, dtype=np.int64)
        last_flags = _last_occurrence_flags(all_ms, nptr)
        last = [last_flags]
        self.attr_cols = int(cols)
        pat_nodes = np.diff(nptr)
        pat_edges = np.diff(eptr)
        # ---- entries, in the dict order of entry2runtimes[entry] (get_all_runtimes_id_probs, pert_gnn.py:70-74)
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
        res_ms = np.array([m for _, m in resource_index], dtype=np.int64)
        res_ts = np.array([t for t, _ in resource_index], dtype=np.int64)
        self.n_ms = int(n_ms if n_ms is not None else max(int(all_ms.max(initial=0)), int(res_ms.max(initial=0))) + 1)
        keys = res_ts * self.n_ms + res_ms
        order = np.argsort(keys, kind="stable")
        has = np.zeros(self.n_ms, dtype=np.uint8)
        has[res_ms] = 1                                          # ms_with_resources (pert_gnn.py:138)
        # ---- traces, in the dict order of tr2data (get_data_list, pert_gnn.py:176-188)
        self.trace_keys = list(tr2data.keys())
        t_ent = np.array([int(tr2data[k]["entry_id"]) for k in self.trace_keys], dtype=np.int32)
        t_ts = np.array([int(tr2data[k]["timestamp"]) for k in self.trace_keys], dtype=np.int64)
        t_y = np.array([int(tr2data[k]["y"]) for k in self.trace_keys], dtype=np.int64)
        # host copies used to size the outputs without a device sync
        self._h_ent_nodes, self._h_ent_edges = ent_nodes.astype(np.int64), ent_edges.astype(np.int64)
        self._h_ent_pats = np.diff(np.array(ent_ptr)).astype(np.int64)
        self._h_trace_entry = t_ent.astype(np.int64)

        def up(a, dtype):
            return torch.from_numpy(np.ascontiguousarray(a, dtype=dtype)).to(dev)

        cat = lambda xs, dt: np.concatenate(xs).astype(dt) if xs else np.zeros(0, dtype=dt)   # noqa: E731
        self.t = {
            "pat_nptr": up(nptr, np.int32), "pat_eptr": up(eptr, np.int32), "pat_ms": up(cat(ms, np.int64), np.int64),
            "pat_depth": up(cat(depth, np.int64), np.int64), "pat_last": up(cat(last, np.uint8), np.uint8),
            "pat_src": up(cat(src, np.int32), np.int32), "pat_dst": up(cat(dst, np.int32), np.int32),
            "pat_attr": up(np.concatenate(attr, axis=0) if attr else np.zeros((0, 2)), np.int64),
            "ent_ptr": up(ent_ptr, np.int32), "ent_pat": up(ent_pat, np.int32),
            # torch.tensor(python floats, dtype=torch.float) of the reference == float64 -> float32 rounding
            "ent_prob": up(np.array(ent_prob, dtype=np.float64).astype(np.float32), np.float32),
            "ent_nodes": up(ent_nodes, np.int32), "ent_edges": up(ent_edges, np.int32),
            "res_keys": up(keys[order], np.int64),
            "res_vals": up(np.asarray(resource_values, dtype=np.float64)[order].astype(np.float32), np.float32),
            "ms_has_res": up(has, np.uint8), "trace_entry": up(t_ent, np.int32), "trace_ts": up(t_ts, np.int64),
            "trace_y": up(t_y, np.int64),
        }
        d = _PertStore()
        d.n_pat, d.n_ent, d.n_res, d.n_ms, d.attr_cols = len(self.rt_ids), n_ent, int(keys.shape[0]), self.n_ms, \
            self.attr_cols
        d.n_traces = len(self.trace_keys)
        for k, v in self.t.items():
            setattr(d, k, v.data_ptr())
        self.desc = d
        self.status = torch.zeros(1, dtype=torch.int32, device=dev)
        self._build_asof()

    @classmethod
    def from_graphs(cls, graphs, runtime_ids, entry2runtimes, resource_index, resource_values, tr2data, device=None,
                    n_ms=None):
        """Patterns straight from ``pertgraph.build_pert_graphs`` / ``build_span_graphs`` (``graphs``: PertGraphs;
        ``runtime_ids[i]`` names pattern i): ONE device->host copy of the concatenated tensors instead of one per
        pattern, no per-pattern Python work."""
        dev = torch.device(device) if device is not None else graphs.ms_id.device
        bp = _BulkPatterns(list(runtime_ids), np.asarray(graphs.node_ptr), np.asarray(graphs.edge_ptr),
                           graphs.ms_id.cpu().numpy().reshape(-1), graphs.node_depth.cpu().numpy().reshape(-1),
                           graphs.edge_index.cpu().numpy(), graphs.edge_attr.cpu().numpy())
        assert len(bp.rt_ids) == len(bp.node_ptr) - 1
        return cls(bp, entry2runtimes, resource_index, resource_values, tr2data, dev, n_ms=n_ms)

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
        is the host sizing arrays the store keeps (per-trace entry and id, per-entry node / edge / pattern totals).
        Microservice ids must lie in [0, 2^31)."""
        graphs, rt_ids = groups.graphs(kind)
        dev = torch.device(device) if device is not None else graphs.ms_id.device
        if dev.type != "cuda":
            raise _lib.PertGnnError("PatternStore lives on a CUDA device (no CPU fallback for the hot path)")
        self = cls.__new__(cls)
        self.device, self.rt_ids = dev, list(rt_ids)
        i32, i64 = torch.int32, torch.int64
        with torch.cuda.device(dev):
            nptr = torch.from_numpy(np.asarray(graphs.node_ptr, dtype=np.int64)).to(dev)
            eptr = torch.from_numpy(np.asarray(graphs.edge_ptr, dtype=np.int64)).to(dev)
            n_pat, n_all = len(self.rt_ids), int(graphs.node_ptr[-1])
            ms = graphs.ms_id.reshape(-1).to(dev, i64)
            # get_x keeps the LAST node of every microservice of a pattern (pert_gnn.py:54-65): stable sort by
            # (pattern, ms); the last of every run of equal keys is the largest node index
            pid = torch.repeat_interleave(torch.arange(n_pat, device=dev), nptr.diff(), output_size=n_all)
            key, idx = torch.sort(pid * (1 << 32) + ms, stable=True)
            run_end = torch.ones(n_all, dtype=torch.bool, device=dev)
            run_end[:-1] = key[1:] != key[:-1]
            last = torch.zeros(n_all, dtype=torch.uint8, device=dev)
            last[idx[run_end]] = 1
            # entries: entry2runtimes[e] in key order = the (entry, runtime) pairs of the groups
            ent_ptr = groups.ent_pair_ptr
            n_ent, n_pairs = int(ent_ptr.shape[0]) - 1, int(groups.pair_runtime.shape[0])
            ent_pat = groups.runtime_ins[groups.pair_runtime.long()]
            pair_entry = torch.repeat_interleave(torch.arange(n_ent, device=dev), ent_ptr.diff(), output_size=n_pairs)
            sums = []
            for per_pat in (nptr.diff(), eptr.diff(), torch.ones(n_pat, dtype=i64, device=dev)):
                sums.append(torch.zeros(n_ent, dtype=i64, device=dev).index_add_(0, pair_entry,
                                                                                  per_pat[ent_pat.long()]))
            ent_nodes, ent_edges, ent_pats = sums
            order = groups.order.long()
            t_ent = groups.entry[order]
            host = torch.cat([t_ent.long(), groups.trace_id[order], ent_nodes, ent_edges, ent_pats,
                              ms.max().reshape(1) if n_all else torch.zeros(1, dtype=i64, device=dev)]).cpu().numpy()
        T = int(order.shape[0])
        self._h_trace_entry, self.trace_keys = host[:T], host[T:2 * T].tolist()
        self._h_ent_nodes, self._h_ent_edges, self._h_ent_pats = (host[2 * T + k * n_ent:2 * T + (k + 1) * n_ent]
                                                                 for k in range(3))
        res_ms = np.array([m for _, m in resource_index], dtype=np.int64)
        res_ts = np.array([t for t, _ in resource_index], dtype=np.int64)
        self.n_ms = int(n_ms if n_ms is not None else max(int(host[-1]), int(res_ms.max(initial=0))) + 1)
        keys = res_ts * self.n_ms + res_ms
        korder = np.argsort(keys, kind="stable")
        has = np.zeros(self.n_ms, dtype=np.uint8)
        has[res_ms] = 1                                          # ms_with_resources (pert_gnn.py:138)
        self.attr_cols = int(graphs.edge_attr.shape[1])

        def up(a, dtype):
            return torch.from_numpy(np.ascontiguousarray(a, dtype=dtype)).to(dev)

        ei = graphs.edge_index.to(dev)
        self.t = {
            "pat_nptr": nptr.to(i32), "pat_eptr": eptr.to(i32), "pat_ms": ms.contiguous(),
            "pat_depth": graphs.node_depth.reshape(-1).to(dev, i64).contiguous(), "pat_last": last,
            "pat_src": ei[0].to(i32).contiguous(), "pat_dst": ei[1].to(i32).contiguous(),
            "pat_attr": graphs.edge_attr.to(dev, i64).contiguous(),
            "ent_ptr": ent_ptr.to(dev, i32).contiguous(), "ent_pat": ent_pat.to(i32).contiguous(),
            "ent_prob": groups.pair_prob.to(dev, torch.float32).contiguous(),      # float64 -> float32 rounding
            "ent_nodes": ent_nodes.to(i32), "ent_edges": ent_edges.to(i32),
            "res_keys": up(keys[korder], np.int64),
            "res_vals": up(np.asarray(resource_values, dtype=np.float64)[korder].astype(np.float32), np.float32),
            "ms_has_res": up(has, np.uint8), "trace_entry": t_ent.to(i32).contiguous(),
            "trace_ts": groups.bucket[order].contiguous(), "trace_y": groups.y[order].contiguous(),
        }
        d = _PertStore()
        d.n_pat, d.n_ent, d.n_res, d.n_ms, d.attr_cols = n_pat, n_ent, int(keys.shape[0]), self.n_ms, self.attr_cols
        d.n_traces = T
        for k, v in self.t.items():
            setattr(d, k, v.data_ptr())
        self.desc = d
        self.status = torch.zeros(1, dtype=torch.int32, device=dev)
        self._build_asof()
        return self

    def _build_asof(self):
        """The as-of index of the resource rows (``asof_index``), 12 bytes per row, kept beside the descriptor: the
        resource table is fixed once the store is built."""
        with torch.cuda.device(self.device):
            ms_ptr, ts, row = asof_index(self.t["res_keys"], self.n_ms)
        self.asof_t = {"ms_ptr": ms_ptr, "ts": ts, "row": row}
        a = _lib.PertResourceAsOf()
        for k, v in self.asof_t.items():
            setattr(a, k, v.data_ptr())
        self.asof_desc = a

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
        o = _PertBatchOut()
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
    def assemble_requests(self, entry_ids, timestamps, asof=False, device_arrays=None):
        """-> device ``Batch`` of the requests (entry ``entry_ids[b]`` at time ``timestamps[b]``, in ms): every field of
        ``assemble`` but ``y``.  The resources are those of the time bucket floor(t / 30000) * 30000, joined exactly
        (a missing row of a resourced microservice sets the status word, see ``check``) or, with ``asof``, from the
        newest row at or before the bucket (none: the missing indicator, no error).  The entry ids are checked and the
        outputs sized on the host (``PertGnnError`` before any launch); ``device_arrays``: the same two columns already
        on the device (int64), e.g. slices of a request list uploaded once -- ``timestamps`` may then be None."""
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
