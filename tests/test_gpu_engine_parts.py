"""-m gpu tests of the step engine's own kernels (csrc/engine.cu) against fp64 on their own inputs
(tests/engine_parts_ref.py): the fused global head at every kernel and padded width, from one graph to 131,075, with
uniform, hot and last-row entry ids and three kinds of d_global; the edge-table GEMMs on both sides of the split-K
switch and across the grouped-launch boundaries; the parameter pack and the gradient unpack bit for bit.

The batches are built as tensors: single-node, edgeless graphs for the head, and 4-node trees whose edges cover every
interface row (plus a hot row 0) for the tables.  The engine's intermediates come from pert_model_workspace_offset.
The largest error of each quantity as a fraction of its bar is printed at the end of the module (pytest -s)."""
import ctypes
import math

import pytest
import torch

from tests import engine_parts_ref as R

pytestmark = pytest.mark.gpu

KERNEL_WIDTHS = (4, 8, 16, 32, 64, 96, 128, 192, 256)
PADDED_WIDTHS = (5, 48, 100, 200)
CAT_ROWS = 6
N_ENTRY = 37
PERT_ERR_RANGE = -3
WORST = {}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if WORST:
        print("\nlargest error as a fraction of its bar:")
        for k in sorted(WORST):
            print(f"  {k:28s} {WORST[k]:.3g}")


def _check(what, got, ref, bar, tag):
    w = R.worst(got, ref, bar)
    WORST[what] = max(WORST.get(what, 0.0), w)
    assert w <= 1.0, f"{tag} {what}: {w:.3g} of its bar"


def _model(H, L=2, F=4, n_if=8, n_rpc=4, seed=0):
    from pert_gnn_kdd23_b200.model import SAGEDeterministic

    torch.manual_seed(seed)
    m = SAGEDeterministic(F, [CAT_ROWS], N_ENTRY - 1, n_if - 1, n_rpc - 1, H, L, 0.0).cuda()
    return m, m.engine()


class _Batch:
    """Device tensors of one batch and its graph index."""

    def __init__(self, model, n_nodes, batch, entry_id, src=None, dst=None, if_id=None, rpc_id=None, seed=0):
        from pert_gnn_kdd23_b200.index import build_index

        g = torch.Generator().manual_seed(seed)
        N, B = n_nodes, entry_id.numel()
        self.N, self.B = N, B
        self.x = torch.randn(N, model.in_channels, generator=g).cuda()
        self.cat_X = torch.randint(0, CAT_ROWS, (N, 1), generator=g).cuda()
        self.entry_id = entry_id.cuda()
        self.batch = batch.cuda()
        self.pnn = torch.bincount(batch, minlength=B).float()[batch].cuda()
        self.probs = torch.ones(N).cuda()
        if src is None:
            ei, ea = torch.empty(2, 0, dtype=torch.int64), torch.empty(0, 2, dtype=torch.int64)
        else:
            ei, ea = torch.stack([src, dst]), torch.stack([if_id, rpc_id], 1)
        self.E = ei.size(1)
        self.index = build_index(ei.cuda(), N, ea.cuda(), model.interface_embeds.num_embeddings,
                                 model.rpctype_embeds.num_embeddings).check()
        self.index.num_graphs = B

    def forward(self, eng, training):
        with torch.no_grad():
            g, _ = eng.forward(self.x, self.cat_X, self.entry_id, self.probs, self.pnn, self.batch, self.index,
                               training)
        return g.reshape(-1)

    def backward(self, eng, dg, grads):
        with torch.no_grad():
            eng.backward(dg.cuda(), None, grads=grads)
        torch.cuda.synchronize()


def _edgeless(model, ids, seed=0):
    B = ids.numel()
    return _Batch(model, B, torch.arange(B), ids, seed=seed)


def _trees(model, n_if, n_rpc, min_graphs=8, seed=0):
    """4-node trees (node j's parent drawn from the nodes before it) with at least 2 max(n_if, n_rpc) edges; the
    interface ids cover every row once and put the rest of the edges on row 0, the rpc ids cover every row."""
    g = torch.Generator().manual_seed(seed)
    G = max(min_graphs, math.ceil(2 * max(n_if, n_rpc) / 3))
    base = torch.arange(G).repeat_interleave(3) * 4
    j = torch.tensor([1, 2, 3]).repeat(G)
    par = (torch.rand(3 * G, generator=g) * j).long()
    src, dst = base + par, base + j
    E = src.numel()
    if_id = torch.cat([torch.arange(n_if), torch.zeros(E - n_if, dtype=torch.int64)])[torch.randperm(E, generator=g)]
    rpc_id = torch.cat([torch.arange(n_rpc), torch.randint(0, n_rpc, (E - n_rpc,), generator=g)])
    rpc_id = rpc_id[torch.randperm(E, generator=g)]
    ids = torch.randint(0, N_ENTRY, (G,), generator=g)
    return _Batch(model, 4 * G, torch.arange(G).repeat_interleave(4), ids, src, dst, if_id, rpc_id, seed=seed)


def _ws(eng, b, which, layer, shape):
    off = eng.lib.pert_model_workspace_offset(ctypes.byref(eng.desc), b.N, b.E, b.B, which, layer)
    assert off >= 0, (which, layer, off)
    n = math.prod(shape)
    return eng.ws[off:off + n].view(shape).cpu()


def _flat_mat(flat, off, rows, cols):
    return flat[off:off + rows * cols].view(rows, cols)


# ------------------------------------------------------------------------------------------------------ head
def _entry_ids(mode, B, g):
    if mode == "uniform":
        return torch.randint(0, N_ENTRY, (B,), generator=g)
    return torch.full((B,), 3 if mode == "hot" else N_ENTRY - 1, dtype=torch.int64)


def _d_global(mode, B, g):
    if mode == "gauss":
        return torch.randn(B, generator=g)
    if mode == "zero_sum":        # the gradient of a fitted median: +-tau / B, summing to 0 exactly
        d = torch.full((B,), 0.3 / B)
        d[1::2] = -d[1::2]
        if B % 2:
            d[-1] = 0.0
        return d
    d = torch.randn(B, generator=g)
    d[torch.randperm(B, generator=g)[:B // 2]] = 0.0
    return d


def _head_fwd_check(eng, b, g_pred, flat, tag):
    d, H, Hp, B = eng.desc, eng.desc.H, eng.Hp, b.B
    W1, b1, W2, b2, ent = R.head_params(d, Hp, flat)
    z = _ws(eng, b, 2, 0, (B, 2 * Hp))
    h1 = _ws(eng, b, 1, 0, (B, Hp))
    ids = b.entry_id.cpu()
    assert torch.equal(z[:, Hp:], ent[ids]), f"{tag}: the entry half of z is not entry_embeds[entry_id]"
    assert int((z[:, H:Hp] != 0).sum()) == 0
    pre, pre_bar, pred, pred_bar = R.head_fwd_ref(z, W1, b1, W2, b2, h1)
    _check("head h1", h1, torch.relu(pre), pre_bar, tag)
    _check("head global_pred", g_pred.cpu(), pred, pred_bar, tag)
    return z, h1


def _head_case(model, eng, B, ent_mode, dg_mode, seed):
    d, H, Hp = eng.desc, eng.desc.H, eng.Hp
    tag = f"H={H} B={B} {ent_mode}/{dg_mode}"
    g = torch.Generator().manual_seed(seed)
    ids = _entry_ids(ent_mode, B, g)
    b = _edgeless(model, ids, seed)
    flat = eng.fp.flat.detach().cpu()
    model.train()
    gp = b.forward(eng, True)
    torch.cuda.synchronize()
    z, h1 = _head_fwd_check(eng, b, gp, flat, tag)
    dg = _d_global(dg_mode, B, g)
    grads = torch.zeros_like(eng.fp.flat)
    b.backward(eng, dg, grads)
    gc = grads.cpu()
    W1, _, W2, _, _ = R.head_params(d, Hp, flat)
    ref = R.head_bwd_ref(dg, z, h1, W1, W2, ids, d.n_entry)
    _check("head dpool", _ws(eng, b, 3, 0, (B, Hp)), *ref["dpool"], tag)
    got = {"entry": _flat_mat(gc, d.off_entry, d.n_entry, H), "W1": _flat_mat(gc, d.off_g1_w, H, 2 * H),
           "b1": gc[d.off_g1_b:d.off_g1_b + H], "W2": gc[d.off_g2_w:d.off_g2_w + H], "b2": gc[d.off_g2_b:d.off_g2_b + 1]}
    cut = {"entry": lambda t: t[:, :H], "W1": lambda t: torch.cat([t[:H, :H], t[:H, Hp:Hp + H]], 1),
           "b1": lambda t: t[:H], "W2": lambda t: t[:H], "b2": lambda t: t}
    for k, v in got.items():
        rv, bar = ref[k]
        _check(f"head d{k}", v, cut[k](rv), cut[k](bar), tag)
    # eval: BatchNorm on the running statistics, the same head kernel
    model.eval()
    gp = b.forward(eng, False)
    torch.cuda.synchronize()
    _head_fwd_check(eng, b, gp, flat, tag + " eval")


COMBOS = (("uniform", "gauss"), ("hot", "zero_sum"), ("last", "half_zero"))


@pytest.mark.parametrize("B", [1, 7, 8, 9, 4097])
@pytest.mark.parametrize("H", KERNEL_WIDTHS + PADDED_WIDTHS)
def test_head(H, B):
    model, eng = _model(H)
    for i, (em, dm) in enumerate(COMBOS):
        _head_case(model, eng, B, em, dm, seed=100 * B + i)


@pytest.mark.parametrize("H", [64, 256])
def test_head_large_batch(H):
    """131,075 graphs: 16,385 CTAs add into every head weight gradient, and a hot entry row takes one atomic each."""
    model, eng = _model(H)
    for i, (em, dm) in enumerate(COMBOS[:2]):
        _head_case(model, eng, 131075, em, dm, seed=i)


def test_head_entry_id_out_of_range():
    """An entry id >= n_entry raises PERT_ERR_RANGE in the status word; the head reads and writes row 0 in its place,
    and nothing lands outside the entry table (the id points into a guard region behind the gradient buffer)."""
    model, eng = _model(16)
    d, H, Hp = eng.desc, eng.desc.H, eng.Hp
    n = eng.fp.flat.numel()
    bad = N_ENTRY + (n - d.off_entry - N_ENTRY * H) // H + 2    # its row starts behind the flat buffer
    ids = torch.arange(1, 9)
    ids[3] = bad
    b = _edgeless(model, ids)
    model.train()
    b.index.status.zero_()
    gp = b.forward(eng, True)
    torch.cuda.synchronize()
    assert int(b.index.status.item()) == PERT_ERR_RANGE
    flat = eng.fp.flat.detach().cpu()
    safe = ids.clone()
    safe[3] = 0
    W1, b1, W2, b2, ent = R.head_params(d, Hp, flat)
    z = _ws(eng, b, 2, 0, (8, 2 * Hp))
    h1 = _ws(eng, b, 1, 0, (8, Hp))
    assert torch.equal(z[:, Hp:], ent[safe])
    guard = torch.zeros(n + 64 * H, device="cuda")
    grads = guard[:n]
    dg = torch.randn(8)
    b.backward(eng, dg, grads)
    assert int((guard[n:] != 0).sum()) == 0, "the backward wrote behind the gradient buffer"
    ref = R.head_bwd_ref(dg, z, h1, W1, W2, safe, d.n_entry)
    gc = grads.cpu()
    _check("head dentry", _flat_mat(gc, d.off_entry, d.n_entry, H), ref["entry"][0][:, :H], ref["entry"][1][:, :H],
           "out-of-range id")


# ------------------------------------------------------------------------------------------------------ edge tables
N_CONVS = (2, 3, 4, 6, 7, 8)
SMALL_IF = (1, 2, 511, 512, 513)
TABLE_CASES = ([(H, N_CONVS[i % 6], SMALL_IF[i % 5], (1, 8, 64)[i % 3]) for i, H in enumerate(KERNEL_WIDTHS)] +
               [(32, L, 513, 8) for L in N_CONVS] +
               [(5, 3, 512, 8), (100, 4, 511, 64), (200, 2, 2, 1)] +
               [(16, 3, 4099, 64), (64, 7, 4099, 1), (16, 2, 100003, 8), (64, 3, 100003, 8)])


@pytest.mark.parametrize("H,L,n_if,n_rpc", TABLE_CASES)
def test_edge_tables(H, L, n_if, n_rpc):
    model, eng = _model(H, L, n_if=n_if, n_rpc=n_rpc)
    d, Hp = eng.desc, eng.Hp
    tag = f"H={H} L={L} n_if={n_if} n_rpc={n_rpc}"
    b = _trees(model, n_if, n_rpc)
    flat = eng.fp.flat.detach().cpu()
    model.train()
    b.forward(eng, True)
    grads = torch.zeros_like(eng.fp.flat)
    b.backward(eng, torch.randn(b.B, generator=torch.Generator().manual_seed(1)), grads)
    gc = grads.cpu()
    dts = {"if": [], "rpc": []}
    Ws = {"if": [], "rpc": []}
    for l in range(L):
        if_p, rpc_p, weA, weB = R.edge_params(d, Hp, flat, l)
        _check("t_if", _ws(eng, b, 4, l, (n_if, Hp)), *R.table_fwd_ref(if_p, weA), tag)
        _check("t_rpc", _ws(eng, b, 5, l, (n_rpc, Hp)), *R.table_fwd_ref(rpc_p, weB), tag)
        dt_if, dt_rpc = _ws(eng, b, 6, l, (n_if, Hp)), _ws(eng, b, 7, l, (n_rpc, Hp))
        assert int(dt_if.abs().sum(1).gt(0).sum()) > 0, f"{tag}: no interface row of conv {l} has a gradient"
        dweA, dweB = _ws(eng, b, 10, l, (Hp, Hp)), _ws(eng, b, 11, l, (Hp, Hp))
        _check(f"dWeA (split-K {R.split_k(n_if)})", dweA, *R.table_wgrad_ref(dt_if, if_p, R.split_k(n_if)), tag)
        _check("dWeB", dweB, *R.table_wgrad_ref(dt_rpc, rpc_p, 1), tag)
        # lin_edge.weight.grad: the two halves unpacked into the zero gradient buffer, bit for bit
        want = torch.cat([dweA[:d.H, :d.H], dweB[:d.H, :d.H]], 1)
        assert torch.equal(_flat_mat(gc, d.off_we[l], d.H, 2 * d.H), want), f"{tag}: lin_edge.weight.grad of conv {l}"
        dts["if"].append(dt_if)
        dts["rpc"].append(dt_rpc)
        Ws["if"].append(weA)
        Ws["rpc"].append(weB)
    for key, off, n in (("if", d.off_if, n_if), ("rpc", d.off_rpc, n_rpc)):
        ref, bar = R.table_dgrad_ref(dts[key], Ws[key])
        _check(f"d {key}_emb", _flat_mat(gc, off, n, d.H), ref[:, :d.H], bar[:, :d.H], tag)


# ------------------------------------------------------------------------------------------------------ pack / unpack
def _F_of(Hp, pad):
    """in_channels with (pad) or without conv-0 pad columns: k0 = F + Hp rounded up to 8."""
    F = (-Hp) % 8 or 8
    return F + 1 if pad else F


PACK_CASES = ([(H, (2, 5, 6, 8)[i % 4], pad) for i, H in enumerate(KERNEL_WIDTHS + PADDED_WIDTHS)
               for pad in (False, True)] + [(64, L, pad) for L in (2, 5, 6, 8) for pad in (False, True)])


@pytest.mark.parametrize("H,L,pad", PACK_CASES)
def test_pack_and_unpack(H, L, pad):
    from pert_gnn_kdd23_b200 import _lib

    Hp = _lib.lib().pert_model_width(H)
    F = _F_of(Hp, pad)
    model, eng = _model(H, L, F=F)
    d = eng.desc
    assert (d.k0 > F + Hp) == pad
    tag = f"H={H} L={L} F={F}"
    b = _trees(model, d.n_if, d.n_rpc)
    flat = eng.fp.flat.detach().cpu()
    model.train()
    n_packed = eng.lib.pert_model_packed_bytes(ctypes.byref(d)) // 4
    for G0 in (None, torch.randn(eng.fp.flat.numel(), generator=torch.Generator().manual_seed(H))):
        b.forward(eng, True)
        torch.cuda.synchronize()
        assert torch.equal(eng.ws[:n_packed].cpu(), R.packed_restatement(d, Hp, L, flat)), f"{tag}: packed region"
        grads = torch.zeros_like(eng.fp.flat) if G0 is None else G0.cuda()
        b.backward(eng, torch.randn(b.B, generator=torch.Generator().manual_seed(2)), grads)
        gc = grads.cpu()
        for l in range(L):
            K = d.k0 if l == 0 else Hp
            packed = R.conv_unpack(d, Hp, l, _ws(eng, b, 8, l, (4 * Hp, K)), _ws(eng, b, 9, l, (4 * Hp,)),
                                   _ws(eng, b, 10, l, (Hp, Hp)), _ws(eng, b, 11, l, (Hp, Hp)))
            got = R.conv_param_views(d, l, gc)
            base = R.conv_param_views(d, l, G0) if G0 is not None else None
            for k, v in packed.items():
                want = v if base is None else base[k] + v          # float32 addition, as k_unpack's +=
                assert torch.equal(got[k], want), f"{tag} conv {l} {k} ({'G0 +' if base is not None else 'zero +'})"
