"""Fused TransformerConv kernels against a float64 reference on graphs built to reach every branch of the staged-tile
kernels (csrc/tconv_tile.cu) and of the per-row gather kernels (csrc/tconv.cu): in- and out-hubs that overflow the
staged edge capacity, isolated nodes and edgeless batches, duplicate edges and self loops, sharp logits, graphs larger
than a tile, a batch whose N % B == 0 size hint is wrong, whole-graph tiles that overflow their edge capacity, PERT-like
attributes (interface 0 on 3 of 4 edges), interface ids >= 2^22, and step-engine batches whose tiles cut graphs.

The reference (ref_tconv) is checked against the oracle conv once; the graph builders assert the structure they exist
for against a restatement of the tile geometry, so a case that stops reaching its branch fails instead of passing
vacuously.  The reference, the builders and the bar-sensitivity checks run on the CPU; the kernel comparisons are
marked gpu."""
import math
from dataclasses import dataclass, field

import numpy as np
import pytest
import torch

from oracle.model_oracle import OracleTransformerConv, scatter, segment_softmax
from tests.helpers import RTOL, assert_close, assert_grads_close

gpu = pytest.mark.gpu

TILE_WIDTHS = (32, 64, 128)                      # staged-tile kernels (tconv_tile.cu)
ALL_WIDTHS = (4, 8, 16, 32, 64, 96, 128, 192, 256)
NODE_BAR = 1e-5          # out, alpha, dq, dk, dv: element-wise with an RMS floor (tests/helpers.py:elem_err)
SHARP_BAR = 1e-4         # the same at logits of +-100: fp32 rounding of a logit moves exp() by |logit| * 6e-8
HUB_BAR = 4e-5           # the same for the hub graphs: the hub's dq / dk is one fp32 sum over 2,400 edges (measured
                         # up to 1.7e-5 on an H100, per-row and staged kernels alike)
TABLE_BAR = 1e-4         # dt_if, dt_rpc: float atomics over thousands of mixed-sign terms
BIG_ID = 1 << 22         # the staged kernels pack interface id | rpc id << 22 (tconv_tile.cu:PACK_ID)


# ---------------------------------------------------------------------------------------------------------- reference
def ref_tconv(q, k, v, s, src, dst, if_id, rpc_id, t_if, t_rpc):
    """TransformerConv message passing in the precision of its inputs: e_t = t_if[a] + t_rpc[b],
    alpha = softmax_dst(<q_i, k_j + e_t> / sqrt(H)), out_i = sum alpha_t (v_j + e_t) + s_i.  -> (out, alpha [E])."""
    N, H = q.shape
    kj, vj = k.index_select(0, src), v.index_select(0, src)
    if t_if is not None:
        e = t_if.index_select(0, if_id) + t_rpc.index_select(0, rpc_id)
        kj, vj = kj + e, vj + e
    logit = (q.index_select(0, dst) * kj).sum(-1) / math.sqrt(H)
    alpha = segment_softmax(logit, dst, N)
    out = scatter(alpha.view(-1, 1) * vj, dst, N, "sum")
    return (out + s if s is not None else out), alpha


# ---------------------------------------------------------------------------------------------------------- geometry
def tile_geom(H, n_rpc, N, E, B):
    """csrc/tconv_tile.cu:tile_geom restated -> (T nodes per tile, ecap staged edges per tile, two CTAs per SM)."""
    budget2, budget1 = 115712.0 - 160, 231424.0 - 160
    deg = E / N if N > 0 else 1.0
    per_node = 4.0 * (2.0 * H + 1.0 + 0.5 + 4.0 * deg)
    fixed = 64.0 + 4.0 * n_rpc * H + 4.0 * 4.0 * 12.0

    def fit(b):
        return int((b - fixed) / per_node)

    T = fit(budget2)
    avg = N / B if B > 0 else 0.0
    uniform = B > 0 and N % B == 0
    two = T >= 64 and (avg == 0.0 or (avg <= T if uniform else avg <= 0.6 * T))
    if not two:
        T = fit(budget1)
    if uniform and avg <= T:
        T = T // (N // B) * (N // B)
    T = max(1, min(T, N, 65535))
    ecap = (int(deg * T + 0.999) + 8 + 3) // 4 * 4
    return T, ecap, two


def tile_fits(H, n_rpc, deg):
    """Node capacity of a two-CTA tile and of a whole-SM tile at average degree `deg`."""
    per_node = 4.0 * (2.0 * H + 1.0 + 0.5 + 4.0 * deg)
    fixed = 64.0 + 4.0 * n_rpc * H + 4.0 * 4.0 * 12.0
    return int((115712.0 - 160 - fixed) / per_node), int((231424.0 - 160 - fixed) / per_node)


def fixed_tiles(g, H, n_rpc, hint):
    """The fixed T-node tiles ops.tconv runs with: list of (first node, end node, edges of the tile's targets)."""
    T, ecap, _ = tile_geom(H, n_rpc, g.N, g.E, g.B if hint else 0)
    indeg = np.bincount(g.dst, minlength=g.N)
    return [(n0, min(n0 + T, g.N), int(indeg[n0:n0 + T].sum())) for n0 in range(0, g.N, T)], T, ecap


# ---------------------------------------------------------------------------------------------------------- builders
@dataclass
class Graph:
    sizes: list                      # nodes per graph, graph-major node numbering
    src: np.ndarray
    dst: np.ndarray
    if_id: np.ndarray                # interface id per edge (COO order)
    rpc_u: np.ndarray                # uniform [0,1) per edge: rpc id = floor(rpc_u * n_rpc) spreads over all types
    n_if: int = 64
    logit_scale: float = 1.0         # scale of q, k and the tables (sharp logits)
    notes: dict = field(default_factory=dict)

    @property
    def N(self):
        return int(sum(self.sizes))

    @property
    def E(self):
        return int(self.src.size)

    @property
    def B(self):
        return len(self.sizes)

    def rpc_id(self, n_rpc):
        return np.minimum((self.rpc_u * n_rpc).astype(np.int64), n_rpc - 1)


def _random_edges(rng, sizes, deg, edge_counts=None):
    src, dst, off = [], [], 0
    for gi, n in enumerate(sizes):
        m = int(round(deg * n)) if edge_counts is None else int(edge_counts[gi])
        if n > 0 and m > 0:
            src.append(off + rng.integers(0, n, m))
            dst.append(off + rng.integers(0, n, m))
        off += n
    cat = lambda xs: np.concatenate(xs).astype(np.int64) if xs else np.zeros(0, np.int64)
    return cat(src), cat(dst)


def _finish(rng, sizes, src, dst, n_if=64, **kw):
    order = rng.permutation(src.size)                      # COO order unrelated to the CSR order
    src, dst = src[order], dst[order]
    return Graph(sizes, src, dst, rng.integers(0, n_if, src.size).astype(np.int64), rng.random(src.size), n_if=n_if,
                 **kw)


def build_in_hub(seed=1):
    rng = np.random.default_rng(seed)
    sizes = [150] * 40
    src, dst = _random_edges(rng, sizes, 3.0)
    hub = 3 * 150 + 17                                     # node 17 of graph 3
    hs = 3 * 150 + rng.integers(0, 150, 2400)
    return _finish(rng, sizes, np.concatenate([src, hs]), np.concatenate([dst, np.full(2400, hub)]),
                   notes={"hub": hub})


def build_out_hub(seed=2):
    rng = np.random.default_rng(seed)
    sizes = [150] * 40
    src, dst = _random_edges(rng, sizes, 3.0)
    hub = 7 * 150 + 3
    hd = 7 * 150 + rng.integers(0, 150, 2400)
    return _finish(rng, sizes, np.concatenate([src, np.full(2400, hub)]), np.concatenate([dst, hd]),
                   notes={"hub": hub})


def build_isolated(seed=3):
    """A third of the nodes receive nothing (out = skip), another third send nothing."""
    rng = np.random.default_rng(seed)
    sizes = [120] * 30
    src, dst, off = [], [], 0
    for n in sizes:
        role = rng.integers(0, 3, n)                       # 0: no in-edges, 1: no out-edges, 2: both
        may_recv = off + np.flatnonzero(role != 0)
        may_send = off + np.flatnonzero(role != 1)
        m = 3 * n
        src.append(rng.choice(may_send, m))
        dst.append(rng.choice(may_recv, m))
        off += n
    return _finish(rng, sizes, np.concatenate(src), np.concatenate(dst))


def build_empty(seed=4):
    """No edges at all: every output row is its skip row, every gradient but the skip's is zero."""
    rng = np.random.default_rng(seed)
    return _finish(rng, [100] * 20, np.zeros(0, np.int64), np.zeros(0, np.int64))


def build_duplicates(seed=5):
    """Every edge repeated 1-4 times with the same attributes (identical logits tie), plus self loops."""
    rng = np.random.default_rng(seed)
    sizes = [100] * 40
    src, dst = _random_edges(rng, sizes, 1.5)
    n = src.size
    ifs, rpu = rng.integers(0, 64, n), rng.random(n)
    rep = rng.integers(1, 5, n)
    src, dst, ifs, rpu = (np.repeat(a, rep) for a in (src, dst, ifs, rpu))
    loops = rng.choice(sum(sizes), 1500, replace=False)
    src, dst = np.concatenate([src, loops]), np.concatenate([dst, loops])
    ifs, rpu = np.concatenate([ifs, rng.integers(0, 64, 1500)]), np.concatenate([rpu, rng.random(1500)])
    order = rng.permutation(src.size)
    return Graph(sizes, src[order], dst[order], ifs[order].astype(np.int64), rpu[order])


def build_sharp(seed=6):
    """q, k and the tables scaled by 4: logits of +-100, beyond fp32 exp's range without the max shift."""
    rng = np.random.default_rng(seed)
    sizes = [150] * 40
    src, dst = _random_edges(rng, sizes, 3.0)
    return _finish(rng, sizes, src, dst, logit_scale=4.0)


def build_big_graph(seed=7):
    """Ordinary graphs around one larger than a two-CTA tile and one larger than a whole-SM tile (at every tile width)."""
    rng = np.random.default_rng(seed)
    sizes = [100] * 12 + [1500] + [100] * 12 + [4000] + [100] * 6
    src, dst = _random_edges(rng, sizes, 3.0)
    return _finish(rng, sizes, src, dst)


def build_lying_hint(seed=8):
    """N % B == 0 but graphs of 150 and 250 nodes alternate in pairs: the fixed tiles (T a multiple of N / B) cut graphs."""
    rng = np.random.default_rng(seed)
    sizes = [150, 150, 250, 250] * 6
    src, dst = _random_edges(rng, sizes, 3.0)
    return _finish(rng, sizes, src, dst)


def build_dense(seed=9):
    """Equal node counts (whole-graph fixed tiles) but every 8th graph has 5x the edges: its tile overflows ecap."""
    rng = np.random.default_rng(seed)
    sizes = [150] * 40
    counts = [150 * 3 * (5 if g % 8 == 3 else 1) for g in range(40)]
    src, dst = _random_edges(rng, sizes, 3.0, counts)
    return _finish(rng, sizes, src, dst)


def build_pert_like(seed=10):
    """PERT graphs' attributes: interface 0 on 3 of 4 edges (chain and return edges), the rest spread over 1024 ids."""
    rng = np.random.default_rng(seed)
    sizes = [150] * 40
    src, dst = _random_edges(rng, sizes, 3.0)
    g = _finish(rng, sizes, src, dst, n_if=1024)
    g.if_id = np.where(rng.random(g.E) < 0.75, 0, g.if_id)
    return g


BUILDERS = {"in_hub": build_in_hub, "out_hub": build_out_hub, "isolated": build_isolated, "empty": build_empty,
            "duplicates": build_duplicates, "sharp": build_sharp, "big_graph": build_big_graph,
            "lying_hint": build_lying_hint, "dense": build_dense, "pert_like": build_pert_like}
_CACHE = {}


def graph(name):
    if name not in _CACHE:
        _CACHE[name] = BUILDERS[name]()
    return _CACHE[name]


# ---------------------------------------------------------------------------------------------------------- CPU tests
def test_reference_matches_oracle_conv():
    """ref_tconv with tables = the two halves of lin_edge applied to the embeddings == OracleTransformerConv, forward
    and every gradient (fp64)."""
    g = build_in_hub()
    N, H = g.N, 16
    torch.manual_seed(0)
    oc = OracleTransformerConv(H, H, edge_dim=2 * H).double()
    x = torch.randn(N, H, dtype=torch.float64)
    if_emb = torch.randn(g.n_if, H, dtype=torch.float64, requires_grad=True)
    rpc_emb = torch.randn(8, H, dtype=torch.float64, requires_grad=True)
    src, dst = torch.from_numpy(g.src), torch.from_numpy(g.dst)
    ia, ib = torch.from_numpy(g.if_id), torch.from_numpy(g.rpc_id(8))
    gout = torch.randn(N, H, dtype=torch.float64)
    ee = torch.cat([if_emb[ia], rpc_emb[ib]], dim=1)
    yo, alpha_o = oc(x, torch.stack([src, dst]), ee, return_alpha=True)
    yo.backward(gout)

    with torch.no_grad():
        We = oc.lin_edge.weight
        q, k, v, s = (lin(x) for lin in (oc.lin_query, oc.lin_key, oc.lin_value, oc.lin_skip))
        t_if, t_rpc = if_emb @ We[:, :H].t(), rpc_emb @ We[:, H:].t()
    leaves = [t.clone().requires_grad_() for t in (q, k, v, t_if, t_rpc)]
    out, alpha = ref_tconv(leaves[0], leaves[1], leaves[2], s, src, dst, ia, ib, leaves[3], leaves[4])
    out.backward(gout)
    dq, dk, dv, dt_if, dt_rpc = (t.grad for t in leaves)
    close = lambda a, b: torch.testing.assert_close(a, b, rtol=1e-10, atol=1e-10)
    close(out, yo)
    close(alpha, alpha_o)
    close(dq.t() @ x, oc.lin_query.weight.grad)
    close(dq.sum(0), oc.lin_query.bias.grad)
    close(dk.t() @ x, oc.lin_key.weight.grad)
    close(dv.t() @ x, oc.lin_value.weight.grad)
    close(dv.sum(0), oc.lin_value.bias.grad)
    close(dt_if @ We[:, :H], if_emb.grad)
    close(dt_rpc @ We[:, H:], rpc_emb.grad)
    close(torch.cat([dt_if.t() @ if_emb.detach(), dt_rpc.t() @ rpc_emb.detach()], dim=1), oc.lin_edge.weight.grad)


def test_builder_in_hub():
    g = build_in_hub()
    indeg = np.bincount(g.dst, minlength=g.N)
    assert indeg[g.notes["hub"]] >= 2000 and indeg.argmax() == g.notes["hub"]
    for H in TILE_WIDTHS:
        for n_rpc in (1, 8, 9):
            for hint in (True, False):
                _, T, ecap = fixed_tiles(g, H, n_rpc, hint)
                assert indeg[g.notes["hub"]] > ecap, (H, n_rpc, hint)     # more than the whole tile may stage


def test_builder_out_hub():
    g = build_out_hub()
    outdeg = np.bincount(g.src, minlength=g.N)
    assert outdeg[g.notes["hub"]] >= 2000
    for H in TILE_WIDTHS:
        for hint in (True, False):
            assert outdeg[g.notes["hub"]] > fixed_tiles(g, H, 8, hint)[2]


def test_builder_isolated_and_empty():
    g = build_isolated()
    indeg, outdeg = np.bincount(g.dst, minlength=g.N), np.bincount(g.src, minlength=g.N)
    assert (indeg == 0).sum() > g.N // 4 and (outdeg == 0).sum() > g.N // 4
    assert ((indeg > 0) & (outdeg > 0)).sum() > g.N // 4
    assert build_empty().E == 0 and build_empty().N > 0


def test_builder_duplicates():
    g = build_duplicates()
    pairs = g.src * g.N + g.dst
    _, counts = np.unique(pairs, return_counts=True)
    assert (counts >= 2).sum() > 1000 and (g.src == g.dst).sum() >= 1500
    # duplicates carry the same attributes, so their logits tie exactly
    key = np.stack([g.src, g.dst, g.if_id, g.rpc_id(8)], 1)
    assert np.unique(key, axis=0).shape[0] < g.E - 1000


def test_builder_sharp_logits():
    g = build_sharp()
    q, k, v, s, t_if, t_rpc, _ = make_inputs(g, 32, 8, with_tables=True, dtype=torch.float64)
    src, dst = torch.from_numpy(g.src), torch.from_numpy(g.dst)
    e = t_if[torch.from_numpy(g.if_id)] + t_rpc[torch.from_numpy(g.rpc_id(8))]
    logit = (q[dst] * (k[src] + e)).sum(-1) / math.sqrt(32)
    assert float(logit.abs().max()) > 88.8                 # fp32 exp overflows above 88.7
    _, alpha = ref_tconv(q, k, v, s, src, dst, torch.from_numpy(g.if_id), torch.from_numpy(g.rpc_id(8)), t_if, t_rpc)
    amax = scatter(alpha, dst, g.N, "max")
    indeg = np.bincount(g.dst, minlength=g.N)
    assert float((amax[torch.from_numpy(indeg >= 2)] > 0.99).double().mean()) > 0.5   # one edge takes the weight


def test_builder_big_graph():
    g = build_big_graph()
    big = sorted(g.sizes)[-2:]
    for H in TILE_WIDTHS:
        for n_rpc in (1, 8, 9):
            t2, t1 = tile_fits(H, n_rpc, g.E / g.N)
            assert big[0] > t2 and big[1] > t1, (H, n_rpc, t2, t1)
            for hint in (True, False):
                assert fixed_tiles(g, H, n_rpc, hint)[1] < big[1]


def _cut_graphs(sizes, T):
    starts = np.cumsum([0] + list(sizes))
    return sum(1 for a, b in zip(starts[:-1], starts[1:]) if a // T != (b - 1) // T)


def test_builder_lying_hint():
    g = build_lying_hint()
    assert g.N % g.B == 0 and len(set(g.sizes)) == 2
    for H in TILE_WIDTHS:
        for n_rpc in (1, 8, 9):
            T, _, _ = tile_geom(H, n_rpc, g.N, g.E, g.B)
            assert g.N // g.B <= T and T % (g.N // g.B) == 0      # the hint holds: fixed tiles of "whole graphs"
            assert _cut_graphs(g.sizes, T) > 0, (H, n_rpc, T)         # ... which cut real graphs


def test_builder_dense():
    g = build_dense()
    assert len(set(g.sizes)) == 1
    for H in TILE_WIDTHS:
        for n_rpc in (1, 8, 9):
            tiles, T, ecap = fixed_tiles(g, H, n_rpc, True)
            assert T % g.sizes[0] == 0 and _cut_graphs(g.sizes, T) == 0
            assert any(ne > ecap for _, _, ne in tiles), (H, n_rpc)


def test_builder_pert_like():
    g = build_pert_like()
    frac0 = float((g.if_id == 0).mean())
    assert 0.72 < frac0 < 0.78
    for n_rpc in (1, 8, 9, 40):
        assert np.unique(g.rpc_id(n_rpc)).size == n_rpc


def _ref_grads(g, H, n_rpc, with_tables, gout_seed=0, mutate=None):
    q, k, v, s, t_if, t_rpc, gout = make_inputs(g, H, n_rpc, with_tables, dtype=torch.float64)
    src, dst = torch.from_numpy(g.src), torch.from_numpy(g.dst)
    ia, ib = torch.from_numpy(g.if_id), torch.from_numpy(g.rpc_id(n_rpc))
    if mutate is not None:
        src, dst, ia, ib = mutate(src, dst, ia, ib)
    return _ref_run(q, k, v, s, t_if, t_rpc, src, dst, ia, ib, gout)


def test_bars_see_a_dropped_hub_edge():
    """The node bar fails when one of the hub's 2400 in-edges is missing."""
    g = build_in_hub()
    true = _ref_grads(g, 32, 8, True)
    e0 = int(np.flatnonzero(g.dst == g.notes["hub"])[0])
    keep = torch.ones(g.E, dtype=torch.bool)
    keep[e0] = False
    bad = _ref_grads(g, 32, 8, True, mutate=lambda s, d, a, b: (s[keep], d[keep], a[keep], b[keep]))
    for name in ("out", "dq"):
        with pytest.raises(AssertionError):
            assert_close(bad[name], true[name], rtol=NODE_BAR, what=name)


def test_bars_see_a_masked_interface_id():
    """The bars fail when interface ids are read as id & (2^22 - 1), the packing defect of the staged kernels."""
    g = large_id_graph()
    H = 8
    t_full = torch.randn(BIG_ID + 64, H, generator=torch.Generator().manual_seed(3))
    ia = torch.from_numpy(g.if_id)
    uniq, inv = torch.unique(torch.cat([ia, ia & (BIG_ID - 1)]), return_inverse=True)
    q, k, v, s, _, t_rpc, gout = make_inputs(g, H, 8, True, table_rows=1)
    src, dst, ib = torch.from_numpy(g.src), torch.from_numpy(g.dst), torch.from_numpy(g.rpc_id(8))
    true, bad = (_ref_run(q, k, v, s, t_full[uniq], t_rpc, src, dst, ids, ib, gout) for ids in (inv[:g.E], inv[g.E:]))
    for name in ("out", "alpha", "dq", "dk", "dt_rpc"):
        with pytest.raises(AssertionError):
            assert_close(bad[name], true[name], rtol=NODE_BAR if name != "dt_rpc" else TABLE_BAR, what=name)


# ---------------------------------------------------------------------------------------------------------- inputs
def make_inputs(g, H, n_rpc, with_tables, dtype=torch.float32, seed=0, table_rows=None):
    """Seeded q, k, v, skip, tables and upstream gradient (CPU, `dtype`); the interface table has `table_rows` rows
    (default g.n_if; callers with a 2^22-row table build it themselves)."""
    gen = torch.Generator().manual_seed(seed * 1000 + H)
    c = g.logit_scale
    q, k = (torch.randn(g.N, H, generator=gen) * c for _ in range(2))
    v, s, gout = (torch.randn(g.N, H, generator=gen) for _ in range(3))
    t_if = t_rpc = None
    if with_tables:
        t_rpc = torch.randn(n_rpc, H, generator=gen) * c
        t_if = torch.randn(g.n_if if table_rows is None else table_rows, H, generator=gen) * c
    cast = lambda t: None if t is None else t.to(dtype)
    return cast(q), cast(k), cast(v), cast(s), cast(t_if), cast(t_rpc), cast(gout)


def _ref_run(q, k, v, s, t_if, t_rpc, src, dst, ia, ib, gout):
    """float64 reference forward + backward -> dict of tensors (alpha in COO order)."""
    leaves = [t.detach().double().requires_grad_() if t is not None else None for t in (q, k, v, t_if, t_rpc)]
    out, alpha = ref_tconv(leaves[0], leaves[1], leaves[2], s.double(), src, dst, ia, ib, leaves[3], leaves[4])
    out.backward(gout.double())
    r = {"out": out.detach(), "alpha": alpha.detach()}
    for name, t in zip(("dq", "dk", "dv", "dt_if", "dt_rpc"), leaves):
        if t is not None:
            r[name] = t.grad if t.grad is not None else torch.zeros_like(t)
    return r


def large_id_graph(seed=11):
    """A small batch whose interface ids include 0, 2^22 - 1, 2^22 and 2^22 + 63 (rpc ids <= 6)."""
    rng = np.random.default_rng(seed)
    sizes = [100] * 12
    src, dst = _random_edges(rng, sizes, 3.0)
    pool = np.array([0, 1, 5, BIG_ID - 1, BIG_ID, BIG_ID + 1, BIG_ID + 5, BIG_ID + 63], dtype=np.int64)
    g = _finish(rng, sizes, src, dst, n_if=BIG_ID + 64)
    g.if_id = pool[rng.integers(0, pool.size, g.E)]
    g.rpc_u = rng.random(g.E) * 7.0 / 8.0                  # rpc ids 0..6 of n_rpc = 8
    return g


# ---------------------------------------------------------------------------------------------------------- GPU runs
def run_cuda(g, H, n_rpc, with_tables, hint=True, ld=None, t_if_dev=None):
    """One forward + backward through the C-ABI entries ops.tconv calls (pert_tconv_fwd / pert_tconv_bwd; fixed tiles).
    ld > H stores every node plane and gradient with that row stride, which the staged kernels decline: the per-row
    kernels then run at any width.  -> dict of CPU tensors, alpha in CSR order."""
    from pert_gnn_kdd23_b200 import _lib
    from pert_gnn_kdd23_b200.index import build_index

    call, ptr, st = _lib.call, _lib.ptr, _lib.stream()
    ld = H if ld is None else ld
    N, E = g.N, g.E
    dev = torch.device("cuda")
    q, k, v, s, t_if, t_rpc, gout = make_inputs(g, H, n_rpc, with_tables, table_rows=1 if t_if_dev is not None else None)
    if t_if_dev is not None:
        t_if = t_if_dev
    ei = torch.from_numpy(np.stack([g.src, g.dst])).to(dev)
    ea = torch.from_numpy(np.stack([g.if_id, g.rpc_id(n_rpc)], 1)).to(dev) if with_tables else None
    gi = build_index(ei, N, ea, g.n_if if with_tables else 0, n_rpc if with_tables else 0).check()

    def plane(*ts):                                         # [len(ts), N, ld] with the rows in the first H columns
        p = torch.zeros(len(ts), N, ld, device=dev)
        for i, t in enumerate(ts):
            p[i, :, :H] = t.to(dev)
        return p

    pl, gp = plane(q, k, v, s), plane(gout)[0]
    t_if = t_if.to(dev).contiguous() if with_tables else None
    t_rpc = t_rpc.to(dev).contiguous() if with_tables else None
    n = n_rpc if with_tables else 0
    B = g.B if hint else 0
    out = torch.full((N, ld), float("nan"), device=dev)
    alpha = torch.full((max(E, 1),), float("nan"), device=dev)
    csr_if = gi.csr_if if with_tables else None
    csr_rpc = gi.csr_rpc if with_tables else None
    call("pert_tconv_fwd", ptr(pl[0]), ptr(pl[1]), ptr(pl[2]), ptr(pl[3]), ld, ptr(gi.rowptr), ptr(gi.csr_src),
         ptr(csr_if), ptr(csr_rpc), ptr(t_if), ptr(t_rpc), ptr(out), ld, ptr(alpha), n, N, E, B, H, st)
    d = torch.full((3, N, ld), float("nan"), device=dev)
    dsp = torch.empty(max(E, 1), device=dev)
    rpc_ws = torch.empty(16 * N, device=dev) if with_tables else None
    dt_if = torch.zeros_like(t_if) if with_tables else None
    dt_rpc = torch.zeros_like(t_rpc) if with_tables else None
    call("pert_tconv_bwd", ptr(gp), ld, ptr(pl[0]), ptr(pl[1]), ptr(pl[2]), ld, ptr(gi.rowptr), ptr(gi.csr_src),
         ptr(csr_if), ptr(csr_rpc), ptr(gi.colptr), ptr(gi.csc_pos), ptr(gi.csc_dst), ptr(t_if), ptr(t_rpc),
         ptr(alpha), ptr(d[0]), ptr(d[1]), ptr(d[2]), ld, ptr(dsp), ptr(rpc_ws), ptr(dt_if), ptr(dt_rpc), n, N, E, B, H,
         st)
    torch.cuda.synchronize()
    r = {"out": out[:, :H].cpu(), "alpha": alpha[:E].cpu(), "dq": d[0, :, :H].cpu(), "dk": d[1, :, :H].cpu(),
         "dv": d[2, :, :H].cpu(), "perm": gi.perm.long().cpu()}
    if with_tables:
        r["dt_if"], r["dt_rpc"] = dt_if, dt_rpc.cpu()         # dt_if stays on the device (2^22-row tables)
    return r


def reference_for(g, H, n_rpc, with_tables):
    src, dst = torch.from_numpy(g.src), torch.from_numpy(g.dst)
    q, k, v, s, t_if, t_rpc, gout = make_inputs(g, H, n_rpc, with_tables)
    return _ref_run(q, k, v, s, t_if, t_rpc, src, dst, torch.from_numpy(g.if_id), torch.from_numpy(g.rpc_id(n_rpc)),
                    gout)


def compare(got, want, tag, node_bar=NODE_BAR):
    assert_close(got["out"], want["out"], rtol=node_bar, what=f"{tag} out")
    if got["alpha"].numel():
        assert_close(got["alpha"], want["alpha"][got["perm"]], rtol=node_bar, what=f"{tag} alpha")
    for name in ("dq", "dk", "dv"):
        assert_close(got[name], want[name], rtol=node_bar, what=f"{tag} {name}")
    for name in ("dt_if", "dt_rpc"):
        if name in want:
            assert_close(got[name].cpu(), want[name], rtol=TABLE_BAR, what=f"{tag} {name}")


def _case(name, H, n_rpc=8, with_tables=True, hint=True, ld=None):
    g = graph(name)
    bar = {"sharp": SHARP_BAR, "in_hub": HUB_BAR, "out_hub": HUB_BAR}.get(name, NODE_BAR)
    tag = f"{name} H={H} n_rpc={n_rpc} tables={with_tables} hint={hint} ld={ld or H}"
    compare(run_cuda(g, H, n_rpc, with_tables, hint, ld), reference_for(g, H, n_rpc, with_tables), tag, bar)


@gpu
@pytest.mark.parametrize("H", ALL_WIDTHS)
@pytest.mark.parametrize("name", list(BUILDERS))
def test_tconv_structure_every_width(name, H):
    _case(name, H)


# 16 KiB / (4 H) + 1 rpc types: the staged kernels decline the rpc table and the per-row kernels run
_BIG_RPC = {H: 16384 // (4 * H) + 1 for H in ALL_WIDTHS}


@gpu
@pytest.mark.parametrize("variant", ["no_tables", "rpc1", "rpc9", "rpc_big", "no_hint"])
@pytest.mark.parametrize("H", [32, 64, 128, 96])
@pytest.mark.parametrize("name", list(BUILDERS))
def test_tconv_structure_variants(name, H, variant):
    """n_rpc = 8 runs the rpc_ws fast path of the source pass, 9 its shared-memory atomics."""
    kw = {"no_tables": dict(with_tables=False), "rpc1": dict(n_rpc=1), "rpc9": dict(n_rpc=9),
          "rpc_big": dict(n_rpc=_BIG_RPC[H]), "no_hint": dict(hint=False)}[variant]
    _case(name, H, **kw)


@gpu
@pytest.mark.parametrize("H", TILE_WIDTHS)
@pytest.mark.parametrize("name", list(BUILDERS))
def test_tconv_structure_per_row_kernels_at_tile_widths(name, H):
    """Row stride H + 4: the staged kernels return PERT_ERR_UNSUPPORTED and the per-row kernels run at 32 / 64 / 128."""
    _case(name, H, ld=H + 4)


@gpu
@pytest.mark.parametrize("H", TILE_WIDTHS)
def test_tconv_interface_ids_beyond_22_bits(H):
    """Interface ids 2^22 - 1, 2^22, 2^22 + 63 in a table of 2^22 + 64 rows.  dt_if is compared on the referenced
    rows; every other row must stay exactly zero."""
    g = large_id_graph()
    n_rpc = 8
    gen = torch.Generator(device="cuda").manual_seed(H)
    t_if_dev = torch.randn(g.n_if, H, device="cuda", generator=gen)
    got = run_cuda(g, H, n_rpc, True, t_if_dev=t_if_dev)
    ia = torch.from_numpy(g.if_id)
    uniq, inv = torch.unique(ia, return_inverse=True)
    q, k, v, s, _, t_rpc, gout = make_inputs(g, H, n_rpc, True, table_rows=1)
    want = _ref_run(q, k, v, s, t_if_dev[uniq.cuda()].cpu(), t_rpc, torch.from_numpy(g.src), torch.from_numpy(g.dst),
                    inv, torch.from_numpy(g.rpc_id(n_rpc)), gout)
    dt_if = got.pop("dt_if")
    got["dt_if"] = dt_if[uniq.cuda()].cpu()
    compare(got, want, f"ids >= 2^22 H={H}")
    rest = torch.ones(g.n_if, dtype=torch.bool, device="cuda")
    rest[uniq.cuda()] = False
    assert int(torch.count_nonzero(dt_if[rest])) == 0
    del got, dt_if, t_if_dev
    torch.cuda.empty_cache()


@gpu
def test_dropin_forward_with_more_than_2_22_edges():
    """TransformerConv.forward(x, edge_index, edge_attr) uses each edge's row as its interface id: E = 2^22 + 2^14
    edges at H = 32 against the oracle conv in float64 on the device."""
    from pert_gnn_kdd23_b200.nn import TransformerConv

    H, Din, De, n, B = 32, 16, 8, 256, 256                  # 65,536 nodes, average in-degree 64
    N = B * n
    gen = torch.Generator(device="cuda").manual_seed(0)
    E = BIG_ID + (1 << 14)
    g_of = torch.randint(0, B, (E,), device="cuda", generator=gen)
    src = g_of * n + torch.randint(0, n, (E,), device="cuda", generator=gen)
    dst = g_of * n + torch.randint(0, n, (E,), device="cuda", generator=gen)
    ei = torch.stack([src, dst])
    torch.manual_seed(0)
    oc = OracleTransformerConv(Din, H, edge_dim=De).double().cuda()
    cc = TransformerConv(Din, H, edge_dim=De)
    cc.load_state_dict({k: v.float() for k, v in oc.state_dict().items()})
    cc = cc.cuda()
    x = torch.randn(N, Din, device="cuda", generator=gen)
    ea = torch.randn(E, De, device="cuda", generator=gen)
    gout = torch.randn(N, H, device="cuda", generator=gen)
    xc = x.clone().requires_grad_()
    yc = cc(xc, ei, ea)
    yc.backward(gout)
    xo = x.double().requires_grad_()
    yo = oc(xo, ei, ea.double())
    yo.backward(gout.double())
    # the node and edge linears run on the 3xTF32 tensor cores here: the model bar, as test_tconv_generic_edge_features
    assert_close(yc, yo, rtol=RTOL, what="drop-in out")
    assert_close(xc.grad, xo.grad, rtol=RTOL, what="drop-in dx")
    assert_grads_close(cc.named_parameters(), oc.named_parameters(), RTOL)


# ---------------------------------------------------------------------------------------------------------- engine
def _data(rng, n, m, L=6, extra=None, if_zero_frac=0.0):
    from pert_gnn_kdd23_b200.synthetic import make_graph

    d = make_graph(rng, n, m, L)
    if extra is not None:                                  # (src, dst) local ids of added edges
        s, t = extra
        ea = np.stack([rng.integers(0, 1024, s.size), rng.integers(0, 8, s.size)], 1)
        d.edge_index = torch.cat([d.edge_index, torch.from_numpy(np.stack([s, t]).astype(np.int64))], 1)
        d.edge_attr = torch.cat([d.edge_attr, torch.from_numpy(ea.astype(np.int64))], 0)
    if if_zero_frac:
        zero = torch.from_numpy(rng.random(d.edge_attr.size(0)) < if_zero_frac)
        d.edge_attr[zero, 0] = 0
    return d


def _hub_batch(cfg, seed):
    """Jittered graph sizes with an in-hub (2000 in-edges) in one graph and an out-hub in another."""
    from pert_gnn_kdd23_b200.data import Batch
    from pert_gnn_kdd23_b200.synthetic import CONFIGS

    rng = np.random.default_rng(seed)
    base = CONFIGS[cfg]["nodes"] or 150
    sizes = [max(2, int(base * (0.8 + 0.4 * rng.random()))) for _ in range(24)]
    if sum(sizes) % len(sizes) == 0:
        sizes[0] += 1
    dl = []
    for gi, n in enumerate(sizes):
        extra = None
        if gi == 2:
            extra = (rng.integers(0, n, 2000), np.full(2000, n // 2))
        elif gi == 5:
            extra = (np.full(2000, n // 3), rng.integers(0, n, 2000))
        dl.append(_data(rng, n, 3 * n, extra=extra))
    return Batch.from_data_list(dl)


def _assert_cut_tiles(b, H):
    N, E, B = b.x.size(0), b.edge_index.size(1), b.num_graphs
    T, _, _ = tile_geom(H, 8, N, E, B)
    assert not (N % B == 0 and N // B <= T), "batch would run whole-graph fixed tiles, not tiles that cut graphs"


@gpu
@pytest.mark.parametrize("cfg", [1, 2, 3])
def test_engine_hubs_on_cut_tiles(cfg):
    from pert_gnn_kdd23_b200.synthetic import CONFIGS
    from tests.test_gpu_fullsize import _full_parity

    b = _hub_batch(cfg, 100 + cfg)
    _assert_cut_tiles(b, CONFIGS[cfg]["hidden"])
    _full_parity(cfg, None, f"cfg{cfg} hubs", batch=b)


@gpu
def test_engine_lying_hint_cfg2():
    from pert_gnn_kdd23_b200.data import Batch
    from tests.test_gpu_fullsize import _full_parity

    rng = np.random.default_rng(21)
    sizes = [150, 150, 250, 250] * 6
    b = Batch.from_data_list([_data(rng, n, 3 * n) for n in sizes])
    N, E, B = b.x.size(0), b.edge_index.size(1), b.num_graphs
    T, _, _ = tile_geom(64, 8, N, E, B)
    assert N % B == 0 and N // B <= T and _cut_graphs(sizes, T) > 0
    _full_parity(2, None, "cfg2 lying hint", batch=b)


@gpu
def test_engine_mixed_sizes_cfg3():
    """1-node edgeless graphs, 2-node graphs, ordinary graphs and one larger than a whole-SM tile (cut into pieces)."""
    from pert_gnn_kdd23_b200.data import Batch
    from tests.test_gpu_fullsize import _full_parity

    rng = np.random.default_rng(22)
    sizes = [1, 2, 100, 1, 120, 2, 90, 700, 1, 110, 2, 100, 1]
    b = Batch.from_data_list([_data(rng, n, 3 * n if n > 2 else n - 1) for n in sizes])
    N, E = b.x.size(0), b.edge_index.size(1)
    assert 700 > tile_fits(128, 8, E / N)[1]
    _assert_cut_tiles(b, 128)
    _full_parity(3, None, "cfg3 mixed sizes", batch=b)


@gpu
def test_engine_pert_like_attributes_cfg2():
    from pert_gnn_kdd23_b200.data import Batch
    from tests.test_gpu_fullsize import _full_parity

    rng = np.random.default_rng(23)
    b = Batch.from_data_list([_data(rng, 200, 600, L=8, if_zero_frac=0.75) for _ in range(32)])
    assert 0.7 < float((b.edge_attr[:, 0] == 0).double().mean()) < 0.8
    _full_parity(2, None, "cfg2 PERT-like attributes", batch=b)


@gpu
def test_engine_single_node_graphs():
    from pert_gnn_kdd23_b200.data import Batch
    from tests.test_gpu_fullsize import _full_parity

    rng = np.random.default_rng(24)
    b = Batch.from_data_list([_data(rng, 1, 0, L=1) for _ in range(32)])
    assert b.edge_index.size(1) == 0
    _full_parity(2, None, "cfg2 single-node graphs", batch=b)
