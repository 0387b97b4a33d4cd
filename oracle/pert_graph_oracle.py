"""CPU oracle for PERT-graph construction (SURVEY.md section 8f row N2).  TEST INFRASTRUCTURE ONLY: nothing under
pert_gnn_kdd23_b200/ imports this file.

Restates, in plain Python loops (small cases only):
  get_root_ms        <- misc.py:138-142  (GraphConstruct.get_root_spanID)
  drop_wrong_edges   <- misc.py:87-105
  span_graph         <- misc.py:190-219 (get_span_edge_index)
  pert_graph         <- misc.py:221-319 (get_pert_edge_index: stage chains, call / return edges in time order)
                        + :113-136,159-175 (min DFS depth -> the long-cast node_depth tensor)
  canonical_form     -- relabelling-invariant description of a PERT graph, used to compare with the reference's own
                        outputs: its node numbering follows pandas value_counts() / Python set iteration order,
                        which no specification fixes; stage nodes of one microservice are always consecutive.
Parity pinned: tests/golden/ref_pert.npz holds what the reference's GraphConstruct itself returned on
synthetic.make_span_tables(11) (oracle/gen_golden_pert.py runs it); tests/test_pert_graph.py checks this file against
it row by row (cleaning, root) and graph by graph (canonical form)."""
import numpy as np

from .index_oracle import dfs_min_depth, node_depth_tensor


def get_root_ms(t):
    """misc.py:138-142: `um` of the first row whose |rt| is the trace's maximum AND whose timestamp is its minimum."""
    a = np.abs(t["rt"])
    hit = np.nonzero((a == a.max()) & (t["timestamp"] == t["timestamp"].min()))[0]
    if hit.size == 0:
        raise IndexError("no root row")          # the reference: .iloc[0] on an empty frame
    return int(t["um"][hit[0]])


def drop_wrong_edges(t, root):
    """misc.py:87-105 -> indices of the rows that survive, in table order."""
    keep = [i for i in range(len(t["um"])) if t["um"][i] != t["dm"][i]]                     # :89 self loops
    seen, k2 = set(), []
    for i in keep:                                                                          # :92 rpcid, keep first
        if int(t["rpcid"][i]) not in seen:
            seen.add(int(t["rpcid"][i]))
            k2.append(i)
    k3 = [i for i in k2 if t["dm"][i] != root]                                              # :95 calls into the root
    last = {}
    for i in k3:                                                                            # :97 (um, dm), keep last
        last[(int(t["um"][i]), int(t["dm"][i]))] = i
    k4 = [i for i in k3 if last[(int(t["um"][i]), int(t["dm"][i]))] == i]
    seen, k5 = set(), []
    for i in k4:                                                                            # :100-103 unordered pair
        key = frozenset((int(t["um"][i]), int(t["dm"][i])))
        if key not in seen:
            seen.add(key)
            k5.append(i)
    return np.array(k5, dtype=np.int64)


def pert_graph(um, dm, interface, rpctype, t_start, t_end, root):
    """misc.py:221-319 with the canonical node numbering of csrc/pertgraph.cu:
    callers by (calls descending, id ascending), then leaves by id ascending.
    -> ms_id [n] i64, edge_index [2,4r] i64, edge_attr [4r,4] i64, node_depth [n,1] i64, root_nid."""
    r = len(um)
    calls = {}
    for u in um:
        calls[int(u)] = calls.get(int(u), 0) + 1
    callers = sorted(calls, key=lambda m: (-calls[m], m))
    leaves = sorted(set(int(d) for d in dm) - set(calls))
    stages, ms_id, edges, attrs = {}, [], [], []
    n = 0
    for m in callers:                                                   # :238-250
        k = 2 * calls[m] + 1
        stages[m] = list(range(n, n + k))
        for a, b in zip(stages[m], stages[m][1:]):
            edges.append([a, b])
            attrs.append([0, 0, 1, 1])
        ms_id += [m] * k
        n += k
    for m in leaves:                                                    # :251-257
        stages[m] = [n]
        ms_id.append(m)
        n += 1
    for m in sorted(calls):                                             # :271 groupby("um"): ascending keys
        ev = []
        for i in range(r):                                              # :278-289 rows of the group in table order
            if int(um[i]) != m:
                continue
            ev.append((int(t_start[i]), "start", int(dm[i]), int(interface[i]), int(rpctype[i])))
            ev.append((int(t_end[i]), "end", int(dm[i]), 0, 0))
        for i, (_t, mode, d, itf, rpc) in enumerate(sorted(ev, key=lambda e: e[0])):   # :290-302 (stable sort)
            if mode == "start":
                edges.append([stages[m][i], stages[d][0]])
                attrs.append([itf, rpc, 1, 0])
            else:
                edges.append([stages[d][-1], stages[m][i + 1]])
                attrs.append([itf, rpc, 0, 0])
    ei = np.array(edges, dtype=np.int64).reshape(-1, 2).T.copy()
    ea = np.array(attrs, dtype=np.int64).reshape(-1, 4)
    root_nid = stages[int(root)][0]                                     # :308
    depth = node_depth_tensor(dfs_min_depth(ei, n, root_nid))           # :159-175 + long cast :368
    return np.array(ms_id, dtype=np.int64), ei, ea, depth, root_nid


def span_graph(um, dm, interface, rpctype, root):
    """misc.py:190-219 get_span_edge_index (+ depth :113-175): torch.unique(sorted=True, return_inverse=True) over the
    [2, r] um/dm matrix.  -> ms_id [n], edge_index [2,r], edge_attr [r,2], node_depth [n,1], root_nid.  Fully
    specified by the reference, so this is compared bit for bit."""
    both = np.stack([np.asarray(um, dtype=np.int64), np.asarray(dm, dtype=np.int64)])
    ms_id, inv = np.unique(both.reshape(-1), return_inverse=True)
    ei = inv.reshape(2, -1).astype(np.int64)
    root_nid = int(np.searchsorted(ms_id, root))
    assert ms_id[root_nid] == root
    ea = np.stack([np.asarray(interface, dtype=np.int64), np.asarray(rpctype, dtype=np.int64)], axis=1)
    depth = node_depth_tensor(dfs_min_depth(ei, len(ms_id), root_nid))
    return ms_id.astype(np.int64), ei, ea, depth, root_nid


def canonical_form(ms_id, edge_index, edge_attr, node_depth):
    """-> (sorted node tuples (ms, stage, depth), sorted edge tuples (ms_s, stage_s, ms_d, stage_d, attr...)).
    `stage` = position of the node inside its microservice's consecutive block."""
    ms_id = np.asarray(ms_id).reshape(-1)
    stage = np.zeros(len(ms_id), dtype=np.int64)
    for i in range(1, len(ms_id)):
        stage[i] = stage[i - 1] + 1 if ms_id[i] == ms_id[i - 1] else 0
    # a microservice owns exactly one block
    starts = ms_id[stage == 0]
    assert len(np.unique(starts)) == len(starts), "microservice split over several blocks"
    nd = np.asarray(node_depth).reshape(-1)
    nodes = sorted((int(ms_id[i]), int(stage[i]), int(nd[i])) for i in range(len(ms_id)))
    ei, ea = np.asarray(edge_index), np.asarray(edge_attr)
    edges = sorted((int(ms_id[s]), int(stage[s]), int(ms_id[d]), int(stage[d])) + tuple(int(v) for v in ea[e])
                   for e, (s, d) in enumerate(ei.T))
    return nodes, edges
