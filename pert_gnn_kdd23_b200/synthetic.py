"""Seeded synthetic call-graph generator for the BASELINE.json configurations.

The reference trains on the Alibaba 2021 micro-service traces (200 GB, not
available); its per-sample tensor schema is reference pert_gnn.py:163-173.
This module emits ``Data`` objects of exactly that schema with the shapes
SURVEY.md section 8d defines:

  x [n,9] f32 (8 resource stats + missing indicator, stats zeroed where the
  indicator is 1 -- mirrors pert_gnn.py:44-66), edge_index [2,e] i64,
  edge_attr [e,2|4] i64 (interface id, rpctype id[, call_ind, same_ms]),
  cat_X [n,1] i64 (micro-service id), node_depth [n,1] i64,
  pattern_num_nodes [n,1] f32, pattern_probs [P,1] f32, entry_id [1] i64,
  y 0-dim i64, plus ``rt_probs`` [n,1] f32 = the per-node pattern probability the
  reference's train loop rebuilds on the host every step (pert_gnn.py:220-230).

DAG law: n nodes on L levels, node 0 the sole root (level 0); every other node
gets one parent drawn uniformly from the previous level (so every node is reachable);
the remaining m-(n-1) edges are uniform (lower level -> strictly higher level)
pairs, no duplicates; node ids (except the root) and the edge order are
shuffled -- sorting is part of the measured collation.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from .data import Data

N_MS, N_IF, N_RPC, N_ENTRY, N_FEAT = 4096, 1024, 8, 64, 9

# id -> (graphs, nodes, edges, hidden, num_layers, levels);  nodes=None => power law
CONFIGS = {
    1: dict(graphs=64, nodes=50, edges=150, hidden=32, num_layers=1, levels=5),
    2: dict(graphs=256, nodes=200, edges=600, hidden=64, num_layers=3, levels=8),
    3: dict(graphs=1024, nodes=None, edges=None, hidden=128, num_layers=3, levels=None),
    4: dict(graphs=4096, nodes=200, edges=600, hidden=128, num_layers=3, levels=8),
    5: dict(graphs=256, nodes=1000, edges=3000, hidden=128, num_layers=5, levels=12),
}


def model_args(cfg_id):
    """Positional ctor args of SAGEDeterministic for a config (SURVEY.md 8d)."""
    c = CONFIGS[cfg_id]
    return (N_FEAT, [N_MS], N_ENTRY - 1, N_IF - 1, N_RPC - 1, c["hidden"], c["num_layers"], 0.0)


def _level_sizes(rng, n, L):
    L = max(1, min(L, n))
    if L == 1:
        return np.array([n], dtype=np.int64)
    sizes = np.ones(L, dtype=np.int64)
    extra = n - L
    if extra > 0:
        sizes[1:] += np.bincount(rng.integers(1, L, size=extra), minlength=L)[1:] if L > 1 else 0
    return sizes


def random_dag(rng, n, m, L):
    """Returns (edge_index int64 [2,m'], level int64 [n]); m' = min(m, max possible)."""
    sizes = _level_sizes(rng, n, L)
    L = len(sizes)
    level_sorted = np.repeat(np.arange(L), sizes)               # level of position p (sorted)
    ids = np.concatenate([[0], 1 + rng.permutation(n - 1)]) if n > 1 else np.array([0])
    level = np.empty(n, dtype=np.int64)
    level[ids] = level_sorted
    starts = np.concatenate([[0], np.cumsum(sizes)])
    # spanning tree: parent uniform in previous level
    pos = np.arange(sizes[0], n)
    lv = level_sorted[pos]
    par_pos = starts[lv - 1] + (rng.random(pos.shape[0]) * sizes[lv - 1]).astype(np.int64)
    src = ids[par_pos]
    dst = ids[pos]
    have = set((src * n + dst).tolist())
    # cap by the number of admissible (lower -> strictly higher level) pairs
    cum = np.cumsum(sizes)
    max_pairs = int(sum(int(sizes[l]) * int(n - cum[l]) for l in range(L)))
    m = min(m, max_pairs)
    extra_s, extra_d = [], []
    need = m - (n - 1)
    while need > 0:
        k = max(64, 3 * need)
        u = rng.integers(0, n, size=k)
        v = rng.integers(0, n, size=k)
        ok = level[u] < level[v]
        for a, b in zip(u[ok].tolist(), v[ok].tolist()):
            key = a * n + b
            if key not in have:
                have.add(key)
                extra_s.append(a)
                extra_d.append(b)
                need -= 1
                if need == 0:
                    break
    src = np.concatenate([src, np.array(extra_s, dtype=np.int64)])
    dst = np.concatenate([dst, np.array(extra_d, dtype=np.int64)])
    order = rng.permutation(src.shape[0])
    return np.stack([src[order], dst[order]]).astype(np.int64), level


def bfs_min_depth(edge_index, n, root=0):
    """Min hop depth from ``root`` over out-edges (what misc.py:59-63 computes); -1 if unreachable."""
    depth = np.full(n, -1, dtype=np.int64)
    depth[root] = 0
    src, dst = edge_index
    frontier = np.zeros(n, dtype=bool)
    frontier[root] = True
    d = 0
    while frontier.any():
        nxt = np.zeros(n, dtype=bool)
        nxt[dst[frontier[src]]] = True
        nxt &= depth < 0
        d += 1
        depth[nxt] = d
        frontier = nxt
    return depth


def _node_depth(depth):
    # reference quirk (misc.py:159-175,215): unreachable -> 0, depth/max truncated to long -> {0,1}
    d = np.where(depth < 0, 0, depth).astype(np.float64)
    mx = d.max() if d.max() > 0 else 1.0
    return (d / mx).astype(np.int64).reshape(-1, 1)


def make_graph(rng, n, m, L, patterns=1, edge_attr_cols=2):
    """One reference-schema ``Data``: disjoint union of ``patterns`` runtime-pattern
    DAGs (pert_gnn.py:134-173)."""
    eis, levels, depths, pnn, rtp = [], [], [], [], []
    probs = rng.random(patterns) + 0.1
    probs = probs / probs.sum()
    off = 0
    for p in range(patterns):
        np_ = n if patterns == 1 else max(2, int(n // patterns))
        mp_ = m if patterns == 1 else max(np_ - 1, int(m // patterns))
        ei, lv = random_dag(rng, np_, mp_, L)
        eis.append(ei + off)
        levels.append(lv)
        depths.append(bfs_min_depth(ei, np_, 0))
        pnn.append(np.full((np_, 1), float(np_), dtype=np.float32))
        rtp.append(np.full((np_, 1), float(probs[p]), dtype=np.float32))
        off += np_
    edge_index = np.concatenate(eis, axis=1)
    level = np.concatenate(levels)
    nn_, ne = off, edge_index.shape[1]
    x = rng.random((nn_, N_FEAT), dtype=np.float32)
    miss = rng.random(nn_) < 0.2
    x[:, 8] = miss.astype(np.float32)
    x[miss, :8] = 0.0
    ea = np.zeros((ne, edge_attr_cols), dtype=np.int64)
    ea[:, 0] = rng.integers(0, N_IF, size=ne)
    ea[:, 1] = rng.integers(0, N_RPC, size=ne)
    if edge_attr_cols == 4:
        ea[:, 2] = rng.integers(0, 2, size=ne)
        ea[:, 3] = rng.integers(0, 2, size=ne)
    return Data(
        x=torch.from_numpy(x),
        edge_index=torch.from_numpy(edge_index),
        edge_attr=torch.from_numpy(ea),
        cat_X=torch.from_numpy(rng.integers(0, N_MS, size=(nn_, 1))),
        node_depth=torch.from_numpy(np.concatenate([_node_depth(d) for d in depths])),
        pattern_num_nodes=torch.from_numpy(np.concatenate(pnn)),
        pattern_probs=torch.from_numpy(probs.astype(np.float32).reshape(-1, 1)),
        entry_id=torch.from_numpy(rng.integers(0, N_ENTRY, size=1)),
        y=torch.tensor(int(rng.integers(1, 5000)), dtype=torch.long),
        rt_probs=torch.from_numpy(np.concatenate(rtp)),
        level=torch.from_numpy(level),
        min_depth=torch.from_numpy(np.concatenate(depths)),
    )


def _powerlaw_nodes(rng, lo=20, hi=500, alpha=1.5):
    # truncated Pareto(alpha) on [lo, hi] by inverse CDF
    u = rng.random()
    a = lo ** (-alpha)
    b = hi ** (-alpha)
    return int((a - u * (a - b)) ** (-1.0 / alpha))


def make_data_list(cfg_id, num_graphs=None, seed=None, patterns=1, edge_attr_cols=2, jitter=0.0):
    """List of ``Data`` for one BASELINE config; seed defaults to 1000+cfg_id.  ``jitter`` j draws every graph's node
    count uniformly from nodes*(1 +- j) (edges scale with it): BASELINE says "~200 nodes / ~600 edges"."""
    c = CONFIGS[cfg_id]
    rng = np.random.default_rng(1000 + cfg_id if seed is None else seed)
    out = []
    for _ in range(c["graphs"] if num_graphs is None else num_graphs):
        if c["nodes"] is None:
            n = _powerlaw_nodes(rng)
            m = 3 * n
            L = int(min(10, max(3, round(math.log2(n)))))
        else:
            n, m, L = c["nodes"], c["edges"], c["levels"]
            if jitter > 0:
                n = max(2, int(round(n * (1.0 + jitter * (2.0 * rng.random() - 1.0)))))
                m = int(round(n * c["edges"] / c["nodes"]))
        out.append(make_graph(rng, n, m, L, patterns=patterns, edge_attr_cols=edge_attr_cols))
    return out


# ------------------------------------------------------------------------------------------------------------------
# Synthetic "processed/" artefacts in the reference's own schema (what preprocess.py:378-381 writes and pert_gnn.py:
# 297-305 loads): the inputs of get_entry_data / get_data_list (pert_gnn.py:134-188).  Used to run the reference's
# own sample assembly + train/test loop (oracle/gen_golden_loop.py -> tests/golden/ref_loop.npz) and, with the same
# seed, the device-side pattern store (store.py).
def make_trace_artifacts(seed=7, n_ms=48, n_patterns=14, n_entries=6, n_traces=72, n_timestamps=5, n_if=32, n_rpc=6,
                         nodes=(5, 40), resource_frac=0.7, y_max=10, runtime2graph=None, patterns_per_entry=(1, 3)):
    """-> dict(runtime2graph, entry2runtimes, tr2data, resource_index [(timestamp, msname)], resource_values [R,8],
    n_ms, n_if, n_rpc).
      runtime2graph[rt] = {edge_index [2,e] i64, edge_attr [e,4] i64, ms_id [n,1] i64, num_nodes int, node_depth [n,1] i64}
      entry2runtimes[entry] = {rt: prob}        (probabilities of an entry's runtime patterns sum to 1)
      tr2data[trace] = {entry_id int, timestamp int, y 0-dim i64 tensor}
    Microservice ids repeat inside a pattern (PERT graphs have several stage nodes per microservice), which exercises
    the last-occurrence rule of the reference's feature join (pert_gnn.py:54-65)."""
    rng = np.random.default_rng(seed)
    given = runtime2graph is not None          # patterns built elsewhere (e.g. pertgraph.build_pert_graphs)
    runtime2graph = dict(runtime2graph) if given else {}
    for rt in range(0 if given else n_patterns):
        n = int(rng.integers(nodes[0], nodes[1] + 1))
        m = min(3 * n, n * (n - 1) // 2)
        L = int(min(6, max(2, round(math.log2(n)))))
        ei, _ = random_dag(rng, n, m, L)
        e = ei.shape[1]
        ea = np.stack([rng.integers(0, n_if, e), rng.integers(0, n_rpc, e), rng.integers(0, 2, e),
                       rng.integers(0, 2, e)], axis=1).astype(np.int64)
        ms = rng.integers(0, n_ms, size=(n, 1)).astype(np.int64)
        if n >= 4:
            ms[n - 1, 0] = ms[0, 0]                     # guaranteed duplicate microservice inside the pattern
        runtime2graph[100 + rt] = {
            "edge_index": torch.from_numpy(ei), "edge_attr": torch.from_numpy(ea), "ms_id": torch.from_numpy(ms),
            "num_nodes": n, "node_depth": torch.from_numpy(_node_depth(bfs_min_depth(ei, n, 0))),
        }
    rts = list(runtime2graph.keys())
    entry2runtimes = {}
    for entry in range(n_entries):
        k = int(rng.integers(patterns_per_entry[0], patterns_per_entry[1] + 1))
        chosen = [int(x) for x in rng.choice(rts, size=k, replace=False)]
        p = rng.random(k) + 0.2
        p = p / p.sum()
        entry2runtimes[entry] = {rt: float(pp) for rt, pp in zip(chosen, p)}
    timestamps = [int(60000 * (t + 1)) for t in range(n_timestamps)]
    tr2data = {}
    for tr in range(n_traces):
        tr2data[f"trace{tr:04d}"] = {"entry_id": int(rng.integers(0, n_entries)),
                                     "timestamp": int(timestamps[int(rng.integers(0, n_timestamps))]),
                                     "y": torch.tensor(int(rng.integers(1, y_max)))}
    with_res = np.sort(rng.choice(n_ms, size=max(1, int(resource_frac * n_ms)), replace=False))
    index = [(t, int(ms)) for t in timestamps for ms in with_res]       # every resourced ms has every timestamp
    values = rng.random((len(index), N_FEAT - 1)).astype(np.float64)     # read back from CSV as float64
    return {"runtime2graph": runtime2graph, "entry2runtimes": entry2runtimes, "tr2data": tr2data,
            "resource_index": index, "resource_values": values, "n_ms": n_ms, "n_if": n_if, "n_rpc": n_rpc}


def make_span_tables(seed=11, n_traces=24, n_ms=40, calls=(1, 30), n_if=32, n_rpc=6, anomalies=True):
    """Raw per-trace span tables with the columns the reference's preprocessing hands to GraphConstruct
    (preprocess.py:296-318: timestamp, rpcid, um, rpctype, dm, interface, rt, endTimestamp = timestamp + |rt|, :263),
    all int64.  -> list of dicts.  The first generated call (root -> entry service) has the strictly largest |rt| and
    the smallest timestamp, which is how misc.py:138-142 identifies the root.  Timestamps are coarse on purpose
    (many ties, zero-length calls) and, with ``anomalies``, the rows include what misc.py:87-105 drop_wrong_edges
    removes: self loops, repeated rpcids, calls back to the root, repeated (um, dm) pairs and reversed pairs."""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n_traces):
        m = int(rng.integers(calls[0], calls[1] + 1))
        root, entry = (int(v) for v in rng.choice(n_ms, size=2, replace=False))
        t0 = int(rng.integers(1000, 5000))
        rows = [[t0, root, entry, 200 + int(rng.integers(0, 50))]]     # timestamp, um, dm, rt
        called = [entry]
        for _k in range(m - 1):
            um = called[int(rng.integers(0, len(called)))] if rng.random() < 0.8 else int(rng.integers(0, n_ms))
            dm = int(rng.integers(0, n_ms))
            if anomalies and rng.random() < 0.06:
                dm = um                                              # self loop
            elif anomalies and rng.random() < 0.06:
                dm = root                                            # call back to the root
            elif anomalies and rng.random() < 0.08 and len(rows) > 1:
                o = rows[int(rng.integers(1, len(rows)))]
                um, dm = (o[1], o[2]) if rng.random() < 0.5 else (o[2], o[1])   # repeated / reversed pair
            rt = int(rng.integers(0, 6)) * (1 if rng.random() < 0.5 else -1)
            rows.append([t0 + int(rng.integers(0, 8)), um, dm, rt])
            called.append(dm)
        rows = np.array(rows, dtype=np.int64)
        rows = rows[rng.permutation(len(rows))]
        n = len(rows)
        rpcid = np.arange(n, dtype=np.int64)
        if anomalies and n > 3:
            for _d in range(int(rng.integers(0, 3))):
                a, b = rng.integers(0, n, size=2)
                rpcid[a] = rpcid[b]                                  # repeated rpcid
        out.append({"timestamp": rows[:, 0].copy(), "um": rows[:, 1].copy(), "dm": rows[:, 2].copy(),
                    "rt": rows[:, 3].copy(), "rpcid": rpcid, "interface": rng.integers(0, n_if, n).astype(np.int64),
                    "rpctype": rng.integers(0, n_rpc, n).astype(np.int64),
                    "endTimestamp": rows[:, 0] + np.abs(rows[:, 3])})
    return out


def make_pert_artifacts(seed=3, n_patterns=256, n_entries=64, n_traces=4096, calls=(60, 72), device="cuda", n_ms=4096,
                        n_if=1024, n_rpc=8, kind="pert"):
    """PERT-exact synthetic artefacts (SURVEY N2): span tables -> host row filters (misc.py:87-105,138-142) -> PERT (or
    span) graphs built ON THE GPU (pertgraph.build_pert_graphs) -> the processed/ artefact schema of
    make_trace_artifacts with ONE pattern per entry, so a trace's sample is one PERT graph (nodes = 2 calls + distinct
    microservices, edges = 4 calls).  -> (artifacts, info) with info = rows / nodes / edges / seconds of the build."""
    import time

    from . import pertgraph

    tabs = make_span_tables(seed, n_patterns, n_ms=n_ms, calls=calls, n_if=n_if, n_rpc=n_rpc, anomalies=False)
    tables, roots = [], []
    for tab in tabs:
        root = pertgraph.get_root_ms(tab)
        keep = pertgraph.drop_wrong_edges(tab, root)
        tables.append({k: v[keep] for k, v in tab.items()})
        roots.append(root)
    torch.cuda.synchronize(device)
    t0 = time.perf_counter()
    pg = pertgraph.build_pert_graphs(tables, roots, device, kind=kind).check()
    torch.cuda.synchronize(device)
    secs = time.perf_counter() - t0
    # entries / traces / resources around the patterns; the pattern dict only carries the ids here (the graphs stay on the
    # device: art["graphs"] + art["runtime_ids"] go to PatternStore.from_graphs)
    ids = [100 + i for i in range(len(pg))]
    art = make_trace_artifacts(seed, n_ms=n_ms, n_entries=n_entries, n_traces=n_traces, n_if=n_if, n_rpc=n_rpc,
                               y_max=5000, runtime2graph={i: None for i in ids}, patterns_per_entry=(1, 1))
    art["graphs"], art["runtime_ids"] = pg, ids
    info = {"patterns": len(pg), "span_rows": int(sum(len(t["um"]) for t in tables)), "nodes": int(pg.node_ptr[-1]),
            "edges": int(pg.edge_ptr[-1]), "build_s": secs}
    return art, info


# ------------------------------------------------------------------------------------------------------------------
# Processed span tables (what preprocess.py get_df() returns, :191-266): one row per span in file order, the traces
# interleaved, every column an integer.  Input of tracegroup.group_traces (the body of preprocess.py main()).
TRACE_COLUMNS = ("traceid", "timestamp", "rpcid", "um", "dm", "interface", "rpctype", "rt", "entryid")   # tracegroup.COLUMNS


def _interleave(rng, trace_of_row):
    """File order of rows whose per-trace order is already right: traces interleave, each trace keeps its row order."""
    u = rng.random(trace_of_row.shape[0])
    by_trace = np.lexsort((u, trace_of_row))                 # rows grouped by trace, u ascending inside a trace
    key = np.empty_like(u)
    key[np.argsort(trace_of_row, kind="stable")] = u[by_trace]
    return np.argsort(key, kind="stable")


def make_trace_table(seed=5, n_ms=24, n_traces=300):
    """Small processed span table covering what the trace grouping must get right (tests/golden/ref_preprocess.npz):
    interleaved traces with traceid gaps; one-row traces; the same rows in a different order (another runtime);
    one runtime under two entries whose lower entry's trace has the higher traceid and other timings (so the
    representative matters); negative rt; buckets on both sides of a 30000 boundary; the drop_wrong_edges anomalies of
    make_span_tables; an entry-id gap (entries 0, 1, 2, 4, 6).  -> dict(columns={TRACE_COLUMNS: int64 [R]},
    resource_index [(bucket, ms)] for every bucket and microservice, resource_values [len, 8] float64, n_ms)."""
    from .pertgraph import drop_wrong_edges, get_root_ms

    def root_kept(tab):              # misc.py:204 / :306 look the root up among the surviving rows (KeyError otherwise)
        root = get_root_ms(tab)
        keep = drop_wrong_edges(tab, root)
        return root in set(tab["um"][keep]) | set(tab["dm"][keep])

    rng = np.random.default_rng(seed)
    pats = make_span_tables(seed, 30, n_ms=n_ms, calls=(2, 12)) + make_span_tables(seed + 1, 3, n_ms=n_ms, calls=(1, 1))
    pats = [t for t in pats if root_kept(t)]
    rev = [{k: v[::-1].copy() for k, v in t.items()} for t in pats if len(t["um"]) > 2]
    pats.append(next(t for t in rev if root_kept(t)))            # same rows as a pattern, reversed: another runtime
    entries = np.array([0, 1, 2, 4, 6])
    pat_entry = entries[rng.integers(0, len(entries), len(pats))]
    shared = 5                                                   # pattern filed under entries 6 and 1 (see below)
    pat_entry[shared] = 6
    weights = 1.0 / np.arange(1, len(pats) + 1)
    weights[len(pats) - 4:] = 0.5                                # the one-row and reversed patterns occur too
    pick = rng.choice(len(pats), size=n_traces - 1, p=weights / weights.sum())
    tids = np.sort(rng.choice(3 * n_traces, size=n_traces, replace=False))      # gaps
    traces = []
    for i, p in enumerate(pick):
        traces.append((int(tids[i]), int(p), int(pat_entry[p])))
    traces.append((int(tids[-1]), shared, 1))   # highest traceid, lower entry: the representative of `shared`
    cols = {k: [] for k in TRACE_COLUMNS}
    for n, (tid, p, ent) in enumerate(traces):
        tab = pats[p]
        m = len(tab["um"])
        t0 = int(rng.integers(29990, 30010)) if n % 3 else int(rng.integers(0, 90000))   # around the 30000 boundary
        off = tab["timestamp"] - tab["timestamp"].min()
        root = int(np.argmax(np.abs(tab["rt"])))
        if n == len(traces) - 1:
            off = off[::-1].copy()                               # other timings for the late representative
            j = int(np.argmin(off))
            off[root], off[j] = off[j], off[root]                  # the root call still starts first
        rt = tab["rt"].copy()
        jit = rng.integers(-3, 4, m)
        jit[root] = 0
        rt = np.where(np.arange(m) == root, rt, rt + jit)
        cols["traceid"].append(np.full(m, tid))
        cols["timestamp"].append(t0 + off)
        cols["rpcid"].append(tab["rpcid"])
        cols["um"].append(tab["um"])
        cols["dm"].append(tab["dm"])
        cols["interface"].append(tab["interface"])
        cols["rpctype"].append(rng.integers(0, 6, m) if n % 2 else tab["rpctype"])
        cols["rt"].append(rt)
        cols["entryid"].append(np.full(m, ent))
    cols = {k: np.concatenate(v).astype(np.int64) for k, v in cols.items()}
    order = _interleave(rng, cols["traceid"])
    cols = {k: v[order] for k, v in cols.items()}
    buckets = np.unique(np.array([(cols["timestamp"][cols["traceid"] == t].min() // 30000) * 30000
                                  for t in np.unique(cols["traceid"])]))
    index = [(int(b), ms) for b in buckets for ms in range(n_ms)]
    values = rng.random((len(index), N_FEAT - 1))
    return {"columns": cols, "resource_index": index, "resource_values": values, "n_ms": n_ms}


def make_random_trace_table(seed, n_traces, rows=(20, 40), n_patterns=2000, n_entries=64, n_ms=4096, n_if=1024,
                            long_rows=0, n_long=0, span=300000):
    """Large processed span table for scale tests and timing, generated without a Python loop over traces.
    ``n_patterns`` call sequences (lengths uniform in ``rows``; ``n_long`` more of ``long_rows`` rows) are drawn with a
    Zipf-like law, so runtimes repeat heavily; a pattern belongs to one entry, a few to two.  Row 0 of every trace is its
    root call (smallest timestamp, largest |rt|), rpcids are unique inside a trace, traceids have gaps and the rows of
    all traces interleave.  -> dict of TRACE_COLUMNS, int64 [R]."""
    rng = np.random.default_rng(seed)
    lens = rng.integers(rows[0], rows[1] + 1, n_patterns)
    if n_long:
        lens = np.concatenate([lens, np.full(n_long, long_rows)])
    P = lens.shape[0]
    pptr = np.concatenate([[0], np.cumsum(lens)])
    um = rng.integers(0, n_ms, pptr[-1])
    dm = (um + rng.integers(1, n_ms, pptr[-1])) % n_ms           # no self loop: every representative keeps rows
    itf = rng.integers(0, n_if, pptr[-1])
    pat_entry = rng.integers(0, n_entries, P)
    w = 1.0 / np.arange(1, P + 1) ** 0.8
    pick = rng.choice(P, size=n_traces, p=w / w.sum())
    if n_long:
        pick[rng.choice(n_traces, n_long, replace=False)] = np.arange(n_patterns, P)
    ent = pat_entry[pick]
    other = rng.random(n_traces) < 0.02                           # a pattern met under a second entry
    ent[other] = (ent[other] + 1 + rng.integers(0, n_entries - 1, int(other.sum()))) % n_entries
    tids = np.sort(rng.choice(2 * n_traces + 7, size=n_traces, replace=False)) + 3
    tl = lens[pick]
    tr = np.repeat(np.arange(n_traces), tl)
    start = np.concatenate([[0], np.cumsum(tl)])[:-1]
    pos = np.arange(tr.shape[0]) - start[tr]
    src = pptr[pick][tr] + pos
    t0 = rng.integers(0, span, n_traces)[tr]
    first = pos == 0
    ts = t0 + np.where(first, 0, rng.integers(0, 9, tr.shape[0]))
    rt = np.where(first, 1000 + rng.integers(0, 500, tr.shape[0]),
                  rng.integers(-400, 400, tr.shape[0]))
    cols = {"traceid": tids[tr], "timestamp": ts, "rpcid": pos, "um": um[src], "dm": dm[src], "interface": itf[src],
            "rpctype": rng.integers(0, 8, tr.shape[0]), "rt": rt, "entryid": ent[tr]}
    order = _interleave(rng, tr)
    return {k: np.ascontiguousarray(v[order], dtype=np.int64) for k, v in cols.items()}


def make_raw_tables(seed=0, dotted_rpcid=False):
    """Deterministic raw CSV text of the Alibaba MSCallGraph / MSResource schema (the input of the reference's
    get_df(), preprocess.py:191-266) -> {"callgraph": {file name: text}, "resource": {file name: text}}.
    Call-graph files carry the leading unnamed index column; rows of a trace are interleaved with other traces.  Every
    trace's first timestamp is unique and the only timestamp ties are rows of one trace that differ in um (and, for
    the two-"(?)" case, in the sign of rt), so the reference's unstable sort cannot decide the result.  Covers:
      exact duplicate rows within one file and across files; negative rt; null string cells (um, interface, rpctype,
      and rpcid when ``dotted_rpcid``); a numeric rpcid column (some files written as "1.0", which pyarrow reads as
      floats) or dotted-string rpcids;
      entry detection: one candidate, several resolved by um == "(?)", several with zero or two "(?)", none;
      resource coverage exactly 0.6 (kept) and 4/7 (dropped); entries with 100 traces (dropped) and 101 (kept);
      resource microservices in no trace; resource groups of 1..5 rows, NaN usages, an all-NaN group and the Kahan
      group [1e16, 1, 1, -1e16] (mean 0.5), groups split across two files, rows with a null timestamp or msname."""
    rng = np.random.default_rng(seed)
    res_ms = [f"MS_{k:03d}" for k in range(24)]              # microservices with resource rows (and "USER")
    bare_ms = [f"NR_{k:02d}" for k in range(6)]               # microservices without
    types = ["rpc", "mc", "db", "mq"]
    traces = []                                               # (rows, kind); a row: dict of the call columns

    def rpcid(k):
        return f"0.1.{k}" if dotted_rpcid else str(k)

    def body(n, ms):
        """n child rows over microservices ``ms`` (all of them used), |rt| < 1000."""
        rows, prev = [], ms[0]
        for k in range(max(n, len(ms) - 1)):
            nxt = ms[(k + 1) % len(ms)]
            rows.append(dict(um=prev, dm=nxt, rpctype=types[rng.integers(len(types))],
                             interface=f"IF_{rng.integers(40):02d}", rpcid=rpcid(k + 1),
                             rt=int(rng.integers(1, 1000)) * (-1 if rng.random() < 0.3 else 1)))
            prev = nxt
        return rows

    def entry(um, dm, itf, rt):
        return dict(um=um, dm=dm, rpctype="http", interface=itf, rpcid=rpcid(0), rt=rt)

    def plain(dm, itf, um="USER", cover=None):
        rt = int(rng.integers(1000, 5000)) * (-1 if rng.random() < 0.2 else 1)
        ms = cover if cover is not None else [dm] + list(rng.choice(res_ms, size=int(rng.integers(2, 5)),
                                                                      replace=False))
        rows = [[entry(um, dm, itf, rt)]] + [[r] for r in body(int(rng.integers(2, 6)), ms)]
        if cover is None and rng.random() < 0.1:              # null string cells in a child row
            rows[-1][0][("um", "interface", "rpctype")[rng.integers(3)]] = None
        return rows

    for _ in range(95):
        traces.append(plain("MS_001", "IF_A"))
    for _ in range(6):                                        # two candidates, one of them "(?)": resolved
        t = plain("MS_001", "IF_A")
        t[0].append(dict(t[0][0], um="(?)"))
        traces.append(t)
    for _ in range(100):
        traces.append(plain("MS_002", "IF_B"))
    for _ in range(98):
        traces.append(plain("MS_003", "IF_C"))
    for k in range(3):                                        # coverage 3/5 = 0.6: kept
        traces.append(plain("MS_003", "IF_C", um="MS_004", cover=["MS_003", "MS_005", bare_ms[k], bare_ms[k + 1]]))
    for k in range(3):                                        # coverage 4/7: dropped
        traces.append(plain("MS_003", "IF_C", um="MS_004",
                            cover=["MS_003", "MS_005", "MS_006", bare_ms[k], bare_ms[k + 1], bare_ms[k + 2]]))
    for _ in range(3):                                        # two candidates, none "(?)": dropped
        t = plain("MS_007", "IF_D", um="MS_008")
        t[0].append(dict(t[0][0], um="MS_009"))
        traces.append(t)
    for _ in range(3):                                        # two "(?)" candidates (rt and -rt): dropped
        t = plain("MS_007", "IF_D", um="(?)")
        t[0].append(dict(t[0][0], um="(?)", rt=-t[0][0]["rt"]))
        traces.append(t)
    for _ in range(3):                                        # no http row at the first timestamp: dropped
        t = plain("MS_007", "IF_D")
        t[0][0]["rpctype"] = "rpc"
        traces.append(t)

    if dotted_rpcid:
        traces[0][-1][0]["rpcid"] = None                     # a null string rpcid (a child row)
    # interleave: every group of rows (tie partners share one group) gets a unique timestamp, in trace order
    order = rng.permutation(len(traces))
    events = []
    for rank, ti in enumerate(order):
        t0 = rank * 40.0
        for j in range(len(traces[ti])):
            events.append((t0 + j * rng.uniform(5, 60) if j else t0, ti, j))
    events.sort()
    base = 1_700_000_000_000 + seed * 10_000_000
    out_rows = []
    for k, (_, ti, j) in enumerate(events):
        for r in traces[ti][j]:
            out_rows.append(dict(r, traceid=f"tr{ti:04d}x{seed}", timestamp=base + 7 * k))
    # duplicates: within the same file and across files
    files = [[], [], []]
    for r in out_rows:
        files[int(rng.integers(3))].append(r)
    for _ in range(12):
        f = int(rng.integers(3))
        src = files[f][int(rng.integers(len(files[f])))]
        files[f].insert(int(rng.integers(len(files[f]) + 1)), dict(src))
    for _ in range(12):
        f, g = (int(v) for v in rng.choice(3, size=2, replace=False))
        files[g].insert(int(rng.integers(len(files[g]) + 1)), dict(files[f][int(rng.integers(len(files[f])))]))

    def cell(v):
        return "" if v is None else str(v)

    def rpc_cell(v, float_file):
        if v is None:
            return ""
        return f"{v}.0" if float_file and not dotted_rpcid else v

    callgraph = {}
    for f, rows in enumerate(files):
        lines = [",traceid,timestamp,rpcid,um,rpctype,dm,interface,rt"]
        for i, r in enumerate(rows):
            lines.append(",".join([str(1000 * f + i), r["traceid"], str(r["timestamp"]), rpc_cell(r["rpcid"], f == 2),
                                   cell(r["um"]), cell(r["rpctype"]), r["dm"], cell(r["interface"]), str(r["rt"])]))
        callgraph[f"MSCallGraph_{f}.csv"] = "\n".join(lines) + "\n"

    # resources: groups per (timestamp, msname) of 1..5 instance rows, split over two files
    extra = [f"MS_R{k}" for k in range(3)]                    # resourced, in no trace
    res_files = [[], []]
    b0 = base // 30000 * 30000                                # the traces' buckets are b0 and b0 + 30000
    ts_list = [b0 - 30000, b0, b0 + 30000]
    for ts in ts_list:
        for m in res_ms + extra + ["USER"]:
            n = int(rng.integers(1, 6))
            for i in range(n):
                cpu = None if rng.random() < 0.1 else float(rng.random())
                mem = None if rng.random() < 0.1 else float(rng.random() * 2)
                res_files[int(rng.integers(2))].append((ts, m, f"{m}_i{i}", cpu, mem))
    t3 = b0 + 60000
    res_files[0] += [(t3, "MS_000", "k0", 1e16, 0.25), (t3, "MS_000", "k1", 1.0, 0.5), (t3, "MS_000", "k2", 1.0, None),
                     (t3, "MS_000", "k3", -1e16, 0.125), (t3, "MS_001", "n0", None, None),
                     (t3, "MS_001", "n1", None, None), (None, "MS_002", "z0", 0.5, 0.5), (t3, None, "z1", 0.5, 0.5)]
    resource = {}
    for f, rows in enumerate(res_files):
        lines = ["timestamp,msname,msinstanceid,nodeid,instance_cpu_usage,instance_memory_usage"]
        for ts, m, inst, cpu, mem in rows:
            lines.append(",".join([cell(ts), cell(m), inst, f"node{len(lines) % 7}",
                                   "" if cpu is None else repr(cpu), "" if mem is None else repr(mem)]))
        resource[f"MSResource_{f}.csv"] = "\n".join(lines) + "\n"
    return {"callgraph": callgraph, "resource": resource}


def make_random_raw_tables(seed, n_traces, rows=(4, 56), n_entries=64, n_ms=3000, n_if=512, dup=0.05):
    """Large dictionary-encoded raw tables (rawtable.RawTables) for scale tests: heavy timestamp ties across traces
    (timestamps drawn from a narrow range), ``dup`` of the rows repeated exactly, entry rows with "(?)" tie partners,
    traces without an entry, partial resource coverage and resource groups of 1..8 rows with NaN usages."""
    from .rawtable import RawTables

    rng = np.random.default_rng(seed)
    lens = rng.integers(rows[0], rows[1] + 1, size=n_traces)
    R = int(lens.sum())
    tr = np.repeat(np.arange(n_traces), lens)
    first = np.concatenate([[0], np.cumsum(lens)[:-1]])
    is_first = np.zeros(R, bool)
    is_first[first] = True
    ent = rng.integers(n_entries, size=n_traces)
    start = rng.integers(0, n_traces * 4, size=n_traces)
    ts = start[tr] + rng.integers(0, 200, size=R) * (~is_first)
    rt = rng.integers(-900, 900, size=R)
    rt[first] = rng.integers(1000, 3000, size=n_traces) * np.where(rng.random(n_traces) < 0.2, -1, 1)
    ms_names = sorted({f"m{k:05d}" for k in range(n_ms - 1)} | {"(?)"})
    q = ms_names.index("(?)")
    um = rng.integers(n_ms, size=R)
    dm = rng.integers(n_ms, size=R)
    dm[first] = (ent * 7) % n_ms
    um[first] = np.where(rng.random(n_traces) < 0.5, q, um[first])
    itf = rng.integers(n_if, size=R)
    itf[first] = ent % n_if
    rty = rng.integers(1, 4, size=R)                          # 0 = "http"
    rty[first] = np.where(rng.random(n_traces) < 0.95, 0, 1)
    rpc = rng.integers(0, 64, size=R)
    cols = dict(traceid=tr, timestamp=ts, rpcid=rpc, um=um, rpctype=rty, dm=dm, interface=itf, rt=rt)
    # "(?)" tie partners of some entry rows, and exact duplicates
    tie = first[rng.random(n_traces) < 0.2]
    dup_rows = rng.integers(R, size=int(dup * R))
    extra = np.concatenate([tie, dup_rows])
    for k, v in cols.items():
        add = v[extra].copy()
        if k == "um":
            add[:len(tie)] = np.where(add[:len(tie)] == q, 0, q)
        cols[k] = np.concatenate([v, add])
    perm = rng.permutation(len(cols["traceid"]))
    cols = {k: v[perm] for k, v in cols.items()}
    # resources: about 80 % of the microservices, 1..8 rows per (timestamp, ms) group
    have = np.flatnonzero(rng.random(n_ms) < 0.8)
    n_ts = 4
    gm = np.repeat(have, n_ts)
    gt = np.tile(np.arange(n_ts) * 30000, len(have))
    cnt = rng.integers(1, 9, size=len(gm))
    r_ms, r_ts = np.repeat(gm, cnt), np.repeat(gt, cnt)
    K = len(r_ms)
    cpu, mem = rng.random(K), rng.random(K) * 1e3
    cpu[rng.random(K) < 0.05] = np.nan
    mem[rng.random(K) < 0.05] = np.nan
    rp = rng.permutation(K)
    resources = dict(timestamp=r_ts[rp], msname=r_ms[rp], instance_cpu_usage=cpu[rp], instance_memory_usage=mem[rp])
    dicts = dict(traceid=[f"t{k}" for k in range(n_traces)], interface=[f"i{k}" for k in range(n_if)],
                 rpcid=list(range(64)), rpctype=["http", "rpc", "mc", "db"], ms=ms_names)
    return RawTables(cols, resources, dicts)
