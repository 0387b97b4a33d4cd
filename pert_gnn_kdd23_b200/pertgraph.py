"""PERT-graph construction (SURVEY.md section 8f row N2): span rows of many traces -> the per-pattern graph tensors
the reference stores in ``runtime2pertgraph_map`` (preprocess.py:350-371), built on the GPU.

Reference: misc.py ``GraphConstruct``
  ``get_root_ms`` / ``drop_wrong_edges``  (misc.py:138-142 / :87-105)  row filters; host numpy, as in the reference
  ``build_span_graphs``                   (misc.py:190-219 + :113-175) CUDA: sorted unique ids + one edge per row
  ``build_pert_graphs``                   (misc.py:221-319 + :113-175) CUDA: csrc/pertgraph.cu builds the stage chains
      and the call / return edges of every trace (one CTA each); the level index (csrc/index.cu pert_min_depth /
      pert_node_depth) gives ``node_depth``.
Node numbering is canonical (callers by (calls desc, id asc), then leaves by id asc) where the reference's depends on
pandas / set iteration order; everything else (edge order, attributes, depth) is the reference's.  There is no CPU
fallback: without the CUDA library the calls raise.
"""
from __future__ import annotations

import numpy as np
import torch

from . import _lib
from . import index as _index

COLUMNS = ("um", "dm", "interface", "rpctype", "timestamp", "endTimestamp")
MAX_ROWS = 2048          # PERT_PERT_GRAPH_MAX_ROWS (include/pertgnn.h)


def get_root_ms(table):
    """misc.py:138-142 get_root_spanID: ``um`` of the first row with the largest |rt| AND the smallest timestamp."""
    a = np.abs(np.asarray(table["rt"]))
    ts = np.asarray(table["timestamp"])
    hit = np.flatnonzero((a == a.max()) & (ts == ts.min()))
    if hit.size == 0:
        raise IndexError("trace has no root row (largest |rt| at the smallest timestamp)")
    return int(np.asarray(table["um"])[hit[0]])


def _keep_first(keys, idx):
    """rows of ``idx`` (ascending) whose key appears for the first time."""
    _, first = np.unique(keys, return_index=True)
    return idx[np.sort(first)]


def drop_wrong_edges(table, root):
    """misc.py:87-105 -> indices of the surviving rows (table order): no self loops, first row per rpcid, no calls
    into the root, last row per (um, dm), first row per unordered {um, dm} pair."""
    um, dm = np.asarray(table["um"], dtype=np.int64), np.asarray(table["dm"], dtype=np.int64)
    idx = np.flatnonzero(um != dm)
    idx = _keep_first(np.asarray(table["rpcid"])[idx], idx)
    idx = idx[dm[idx] != root]
    if idx.size:
        pair = np.stack([um[idx], dm[idx]], axis=1)
        rev = idx[::-1]
        _, first = np.unique(pair[::-1], axis=0, return_index=True)        # keep="last" = first of the reversed table
        idx = np.sort(rev[first])
        lo, hi = np.minimum(um[idx], dm[idx]), np.maximum(um[idx], dm[idx])
        _, first = np.unique(np.stack([lo, hi], axis=1), axis=0, return_index=True)
        idx = idx[np.sort(first)]
    return idx.astype(np.int64)


def _group_pick(cols, last=False):
    """Boolean mask over rows: the first (or last) row, in table order, of every distinct tuple of ``cols``."""
    n = cols[0].shape[0]
    mask = np.zeros(n, dtype=bool)
    if n == 0:
        return mask
    order = np.lexsort(tuple(reversed(cols)))              # stable: equal tuples keep table order
    new = np.ones(n, dtype=bool)
    diff = np.zeros(n - 1, dtype=bool)
    for c in cols:
        cs = c[order]
        diff |= cs[1:] != cs[:-1]
    new[1:] = diff
    if last:
        pick = np.ones(n, dtype=bool)
        pick[:-1] = new[1:]
    else:
        pick = new
    mask[order[pick]] = True
    return mask


def clean_span_tables_flat(columns, row_ptr):
    """``get_root_ms`` + ``drop_wrong_edges`` for MANY traces at once, without a Python loop over traces.
    ``columns``: dict of int64 arrays over all rows (um, dm, rpcid, rt, timestamp [, ...]) grouped by trace;
    ``row_ptr`` [T+1].  -> (keep: surviving row indices in table order, new_row_ptr [T+1], roots [T]).
    Same result as the per-trace functions (misc.py:138-142, :87-105), tests/test_pert_graph.py."""
    row_ptr = np.asarray(row_ptr, dtype=np.int64)
    T = len(row_ptr) - 1
    lens = np.diff(row_ptr)
    if T <= 0 or (lens <= 0).any():
        raise ValueError("every trace needs at least one span row")
    um, dm = np.asarray(columns["um"], dtype=np.int64), np.asarray(columns["dm"], dtype=np.int64)
    rpcid = np.asarray(columns["rpcid"], dtype=np.int64)
    a, ts = np.abs(np.asarray(columns["rt"], dtype=np.int64)), np.asarray(columns["timestamp"], dtype=np.int64)
    tid = np.repeat(np.arange(T, dtype=np.int64), lens)
    starts = row_ptr[:-1]
    amax, tmin = np.maximum.reduceat(a, starts), np.minimum.reduceat(ts, starts)
    cand = np.flatnonzero((a == amax[tid]) & (ts == tmin[tid]))
    tr, first = np.unique(tid[cand], return_index=True)            # cand ascending -> first candidate row per trace
    if tr.shape[0] != T:
        raise IndexError("a trace has no root row (largest |rt| at the smallest timestamp)")
    roots = um[cand[first]]
    idx = np.flatnonzero(um != dm)                                                          # :89
    idx = idx[_group_pick([tid[idx], rpcid[idx]])]                                          # :92 keep first
    idx = idx[dm[idx] != roots[tid[idx]]]                                                   # :95
    idx = idx[_group_pick([tid[idx], um[idx], dm[idx]], last=True)]                         # :97 keep last
    lo, hi = np.minimum(um[idx], dm[idx]), np.maximum(um[idx], dm[idx])
    idx = idx[_group_pick([tid[idx], lo, hi])]                                              # :100-103 keep first
    new_ptr = np.concatenate([[0], np.cumsum(np.bincount(tid[idx], minlength=T))]).astype(np.int64)
    return idx.astype(np.int64), new_ptr, roots.astype(np.int64)


class PertGraphs:
    """T PERT graphs, concatenated on the device.  ``edge_index`` holds trace-LOCAL node ids (the per-pattern tensors
    of runtime2pertgraph_map); trace t owns nodes ``node_ptr[t]:node_ptr[t+1]`` and edges ``edge_ptr[t]:edge_ptr[t+1]``."""

    def __init__(self, node_ptr, edge_ptr, ms_id, edge_index, edge_attr, node_depth, root_nid, status):
        self.node_ptr, self.edge_ptr = node_ptr, edge_ptr            # host int64 arrays [T+1]
        self.ms_id, self.edge_index, self.edge_attr = ms_id, edge_index, edge_attr
        self.node_depth, self.root_nid, self.status = node_depth, root_nid, status

    def __len__(self):
        return len(self.node_ptr) - 1

    def check(self):
        code = int(self.status.item())
        if code != 0:
            _lib.check(code, "PERT graph construction")
        return self

    def pattern(self, t):
        """The dict preprocess.py:363-370 stores for one runtime pattern."""
        n0, n1, e0, e1 = (int(v) for v in (self.node_ptr[t], self.node_ptr[t + 1], self.edge_ptr[t],
                                           self.edge_ptr[t + 1]))
        return {"edge_index": self.edge_index[:, e0:e1], "edge_attr": self.edge_attr[e0:e1],
                "ms_id": self.ms_id[n0:n1].reshape(-1, 1), "num_nodes": n1 - n0,
                "node_depth": self.node_depth[n0:n1]}


def build_span_graphs(tables, roots, device="cuda"):
    """Span graphs (misc.py:190-219; ``--graph_type span``): like ``build_pert_graphs``; ``pattern(t)`` is the dict
    preprocess.py:333-340 stores (edge_attr has the two columns [interface, rpctype]).  Bit-identical to the
    reference's tensors."""
    return build_pert_graphs(tables, roots, device, kind="span")


def build_pert_graphs(tables, roots, device="cuda", kind="pert"):
    """``tables``: per trace a dict of the CLEANED span rows (COLUMNS, int64 array-likes); ``roots``: root
    microservice per trace.  Concatenates on the host and calls ``build_pert_graphs_flat``."""
    T = len(tables)
    rows = np.array([len(t["um"]) for t in tables], dtype=np.int64)
    row_ptr = np.concatenate([[0], np.cumsum(rows)]).astype(np.int64)
    R = int(row_ptr[-1])
    if T == 0 or R == 0:
        raise ValueError("no span rows")
    host = np.empty((len(COLUMNS), R), dtype=np.int64)
    for c, name in enumerate(COLUMNS):
        host[c] = np.concatenate([np.asarray(t[name], dtype=np.int64).reshape(-1) for t in tables])
    return build_pert_graphs_flat(host, row_ptr, roots, device, kind)


def build_pert_graphs_flat(columns, row_ptr, roots, device="cuda", kind="pert"):
    """``columns``: int64 [6, R] (rows of COLUMNS, all traces concatenated -- a span table grouped by trace id, host
    array or CUDA tensor); ``row_ptr``: int64 [T+1] host array; ``roots``: [T].  One H2D copy of the rows, two kernel
    launches for the graphs, the level index for ``node_depth``; the only synchronisation is reading the node total
    to size the outputs.  ``kind``: "pert" (misc.py:221-319) or "span" (misc.py:190-219)."""
    assert kind in ("pert", "span")
    span = kind == "span"
    dev = torch.device(device)
    if dev.type != "cuda":
        raise _lib.PertGnnError("build_pert_graphs needs a CUDA device (no CPU fallback)")
    row_ptr = np.asarray(row_ptr, dtype=np.int64)
    T, R = len(row_ptr) - 1, int(row_ptr[-1])
    rows = np.diff(row_ptr)
    if T <= 0 or R <= 0:
        raise ValueError("no span rows")
    max_rows = int(rows.max())
    if max_rows > MAX_ROWS:
        raise _lib.PertGnnError(f"a trace has {max_rows} rows; the kernel handles at most {MAX_ROWS}")
    with torch.cuda.device(dev):
        cols = columns if torch.is_tensor(columns) else torch.from_numpy(np.ascontiguousarray(columns, dtype=np.int64))
        cols = cols.to(dev).contiguous()
        assert cols.dtype == torch.int64 and tuple(cols.shape) == (len(COLUMNS), R)
        rp = torch.from_numpy(row_ptr).to(dev)
        rm = torch.as_tensor(np.asarray(roots, dtype=np.int64)).to(dev)
        status = torch.zeros(1, dtype=torch.int32, device=dev)
        cnt = torch.empty(T, dtype=torch.int64, device=dev)
        st = _lib.stream()
        _lib.call("pert_span_graph_count" if span else "pert_pert_graph_count", _lib.ptr(rp), T, _lib.ptr(cols[0]),
                  _lib.ptr(cols[1]), max_rows, _lib.ptr(cnt), _lib.ptr(status), st)
        node_ptr = torch.zeros(T + 1, dtype=torch.int64, device=dev)
        torch.cumsum(cnt, 0, out=node_ptr[1:])
        node_ptr_h = node_ptr.cpu().numpy()                       # sizes the outputs (the one sync)
        epr = 1 if span else 4                                    # edges per span row
        N, E = int(node_ptr_h[-1]), epr * R
        ms_id = torch.empty(N, dtype=torch.int64, device=dev)
        ei = torch.empty(2, E, dtype=torch.int64, device=dev)
        ea = torch.empty(E, 2 if span else 4, dtype=torch.int64, device=dev)
        root_nid = torch.empty(T, dtype=torch.int64, device=dev)
        if span:
            _lib.call("pert_span_graph_build", _lib.ptr(rp), T, R, *(_lib.ptr(cols[c]) for c in range(4)),
                      _lib.ptr(rm), _lib.ptr(node_ptr), max_rows, 1, _lib.ptr(ms_id), _lib.ptr(ei), _lib.ptr(ea),
                      _lib.ptr(root_nid), _lib.ptr(status), st)
        else:
            _lib.call("pert_pert_graph_build", _lib.ptr(rp), T, R, *(_lib.ptr(cols[c]) for c in range(6)),
                      _lib.ptr(rm), _lib.ptr(node_ptr), max_rows, 1, _lib.ptr(ms_id), _lib.ptr(ei), _lib.ptr(ea),
                      _lib.ptr(root_nid), _lib.ptr(status), st)
        # level index over the whole batch of graphs (global ids), then back to trace-local ids
        gi = _index.build_index(ei, N)
        gptr = node_ptr.to(torch.int32)
        depth = _index.min_depth(gptr, gi, root_nid.clamp_min(0).to(torch.int32))
        node_depth = _index.node_depth(gptr, depth)
        off = torch.repeat_interleave(node_ptr[:-1], torch.from_numpy(epr * rows).to(dev), output_size=E)
        ei -= off
    return PertGraphs(node_ptr_h, epr * row_ptr, ms_id, ei, ea, node_depth, root_nid, status)
