"""CPU tests of tests/engine_parts_ref.py and of the engine's new workspace offsets: the offsets against a restatement of
engine.cu carve(); every fp64 reference against autograd of the oracle's head and lin_edge; every bar against a float32
restatement of its kernel's summation order under several random atomic orders; and every bar against the defects it
exists to catch."""
import ctypes
import math

import numpy as np
import pytest
import torch

from oracle.model_oracle import OracleSAGEDeterministic
from pert_gnn_kdd23_b200 import _lib
from tests import engine_parts_ref as R

F, CAT_ROWS, N_ENTRY, N_IF, N_RPC = 9, (16, 5), 11, 40, 3
KERNEL_WIDTHS = (4, 8, 16, 32, 64, 96, 128, 192, 256)


def _model(H, L=2, n_if=N_IF, n_rpc=N_RPC, seed=0):
    """-> (CPU SAGEDeterministic, its engine, fp64 oracle with the same parameters)."""
    from pert_gnn_kdd23_b200.model import SAGEDeterministic

    torch.manual_seed(seed)
    args = (F, list(CAT_ROWS), N_ENTRY - 1, n_if - 1, n_rpc - 1, H, L, 0.0)
    m = SAGEDeterministic(*args)
    with torch.no_grad():
        for p in m.parameters():
            p.normal_()
    o = OracleSAGEDeterministic(*args).double()
    o.load_state_dict({k: v.double() for k, v in m.state_dict().items()})
    return m, m.engine(), o


# ------------------------------------------------------------------------------------------------------ offsets
def _carve(d, Hp, N, E, B):
    """engine.cu carve() restated: {(which, layer): offset in floats} of the tensors pert_model_workspace_offset
    exposes."""
    lib = _lib.lib()
    H, L = d.H, d.n_convs
    off = 0

    def take(n):
        nonlocal off
        o = off
        off += R.al64(n)
        return o

    def take_tensors():
        for i in range(d.n_cat):
            take(d.cat_rows[i] * Hp)
        for n in (d.n_entry, d.n_if, d.n_rpc):
            take(n * Hp)
        for _ in range(2 * (L - 1) + 1):
            take(Hp)
        take(2 * Hp * Hp)
        take(Hp)
        take(Hp)

    K = [d.k0 if l == 0 else Hp for l in range(L)]
    got = {}
    for l in range(L):
        for n in (4 * Hp * K[l], 4 * Hp, 4 * Hp * K[l]) + (Hp * Hp,) * 4:
            take(n)
    if Hp != H:
        take_tensors()
    for l in range(L):
        for which, n in ((8, 4 * Hp * K[l]), (9, 4 * Hp), (10, Hp * Hp), (11, Hp * Hp), (6, d.n_if * Hp),
                         (7, d.n_rpc * Hp)):
            got[which, l] = take(n)
    for _ in range(L - 1):
        take(4 * Hp)                      # bn_dsums: 2Hp doubles
    if Hp != H:
        take_tensors()
    for l in range(L):
        got[4, l] = take(d.n_if * Hp)
        got[5, l] = take(d.n_rpc * Hp)
        if l == 0:
            take(N * K[0])
        take(4 * N * Hp)
        take(N * Hp)
        if l + 1 < L:
            got[0, l + 1] = take(N * Hp)
        take(E)
        take(2 * Hp)
    take(lib.pert_bn_workspace_bytes(N, Hp) // 4 + 16)
    take(B * Hp)                          # pool
    got[2, 0] = take(2 * B * Hp)
    got[1, 0] = take(B * Hp)
    take(4 * N * Hp)                      # dplanes
    take(N * max(d.k0, Hp))               # dx
    take(E)                               # dsp
    take(N * 16)                          # rpc_ws (PERT_TCONV_RPC_WS_FLOATS)
    take(2 * Hp)                          # sums
    got[3, 0] = take(B * Hp)
    return got


@pytest.mark.parametrize("H", [8, 48, 128, 200])
@pytest.mark.parametrize("L", [2, 3])
def test_workspace_offsets(H, L):
    """Codes 2..11 land where carve() puts their tensors, at kernel and padded widths; codes 0 and 1 are unchanged; a
    layer outside [0, n_convs) and an unknown code are refused."""
    from pert_gnn_kdd23_b200.model import SAGEDeterministic

    lib = _lib.lib()
    eng = SAGEDeterministic(F, list(CAT_ROWS), N_ENTRY - 1, N_IF - 1, N_RPC - 1, H, L, 0.0).engine()
    d = eng.desc
    for N, E, B in ((0, 0, 0), (100, 300, 4), (5000, 20000, 64)):
        want = _carve(d, eng.Hp, N, E, B)
        for (which, layer), off in want.items():
            assert lib.pert_model_workspace_offset(ctypes.byref(d), N, E, B, which, layer) == off, (which, layer)
        for which in range(4, 12):
            for layer in (-1, L):
                assert lib.pert_model_workspace_offset(ctypes.byref(d), N, E, B, which, layer) == -1, (which, layer)
        assert lib.pert_model_workspace_offset(ctypes.byref(d), N, E, B, 12, 0) == -1
        assert lib.pert_model_workspace_offset(ctypes.byref(d), N, E, B, 0, 0) == -1
        assert lib.pert_model_workspace_offset(ctypes.byref(d), N, E, B, 3, 0) + B * eng.Hp <= \
            lib.pert_model_workspace_bytes(ctypes.byref(d), N, E, B) // 4


# ------------------------------------------------------------------------------------------------------ pack layout
@pytest.mark.parametrize("H", [5, 8, 100, 128])
@pytest.mark.parametrize("L", [2, 3])
def test_pack_restatement(H, L):
    """The restated packed region has pert_model_packed_bytes / 4 floats; conv_unpack inverts conv_pack; the pad mask
    marks exactly the slots no parameter reaches."""
    m, eng, _ = _model(H, L)
    d, Hp, flat = eng.desc, eng.Hp, eng.fp.flat.detach()
    packed = R.packed_restatement(d, Hp, L, flat)
    assert packed.numel() == eng.lib.pert_model_packed_bytes(ctypes.byref(d)) // 4
    pad = R.packed_pad_mask(d, Hp, L, flat.numel())
    assert int((packed[pad] != 0).sum()) == 0
    assert int((~pad).sum()) == int((packed != 0).sum())       # every parameter was drawn nonzero
    for l in range(L):
        w4, b4, weA, weB = R.conv_pack(d, Hp, l, flat)
        back = R.conv_unpack(d, Hp, l, w4, b4, weA, weB)
        views = R.conv_param_views(d, l, flat)
        for k, v in views.items():
            assert torch.equal(back[k], v), (l, k)
            assert torch.equal(v, dict(m.convs[l].named_parameters())[k].detach()), (l, k)
    G0 = np.random.default_rng(1).standard_normal(64).astype(np.float32)
    pk = np.random.default_rng(2).standard_normal(64).astype(np.float32)
    assert np.array_equal(R.unpack_f32(G0, pk), G0 + pk)
    assert not np.array_equal(R.unpack_f32(G0, pk, defect="overwrite"), G0 + pk)


# ------------------------------------------------------------------------------------------------------ references
def _head_inputs(eng, B, seed=0):
    d, Hp = eng.desc, eng.Hp
    g = torch.Generator().manual_seed(seed)
    W1, b1, W2, b2, ent = R.head_params(d, Hp, eng.fp.flat.detach())
    ids = torch.randint(0, d.n_entry, (B,), generator=g)
    pool = torch.zeros(B, Hp)
    pool[:, :d.H] = torch.randn(B, d.H, generator=g)
    z = torch.cat([pool, ent[ids]], 1)
    dg = torch.randn(B, generator=g)
    return z, W1, b1, W2, b2, ids, dg


@pytest.mark.parametrize("H", [5, 16])
def test_head_refs_match_oracle_autograd(H):
    _, eng, o = _model(H)
    Hp, B = eng.Hp, 13
    z, W1, b1, W2, b2, ids, dg = _head_inputs(eng, B)
    pool = z[:, :H].double().requires_grad_()
    zo = torch.cat([pool, o.entry_embeds(ids)], 1)
    pre_o = o.global_linear1(zo)
    h1_o = torch.relu(pre_o)
    g_o = o.global_linear2(h1_o).reshape(-1)
    (g_o * dg.double()).sum().backward()
    h1 = R._pad(h1_o.detach(), (B, Hp))
    pre, _, pred, _ = R.head_fwd_ref(z, W1, b1, W2, b2, h1)
    torch.testing.assert_close(pre[:, :H], pre_o.detach(), rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(pred, g_o.detach(), rtol=1e-12, atol=1e-12)
    r = R.head_bwd_ref(dg, z, h1, W1, W2, ids, N_ENTRY)
    want = {"dpool": pool.grad, "entry": o.entry_embeds.weight.grad, "W1": o.global_linear1.weight.grad,
            "b1": o.global_linear1.bias.grad, "W2": o.global_linear2.weight.grad.reshape(-1),
            "b2": o.global_linear2.bias.grad}
    got = {k: v[0] for k, v in r.items()}
    got["dpool"], got["entry"] = got["dpool"][:, :H], got["entry"][:, :H]
    got["W1"] = torch.cat([got["W1"][:H, :H], got["W1"][:H, Hp:Hp + H]], 1)
    got["b1"], got["W2"] = got["b1"][:H], got["W2"][:H]
    for k in want:
        torch.testing.assert_close(got[k], want[k], rtol=1e-12, atol=1e-12, msg=k)


@pytest.mark.parametrize("H", [5, 16])
def test_table_refs_match_oracle_autograd(H):
    L = 3
    _, eng, o = _model(H, L)
    d, Hp, flat = eng.desc, eng.Hp, eng.fp.flat.detach()
    g = torch.Generator().manual_seed(3)
    E = 57
    ea = torch.stack([torch.randint(0, N_IF, (E,), generator=g), torch.randint(0, N_RPC, (E,), generator=g)], 1)
    emb = torch.cat([o.interface_embeds(ea[:, 0]), o.rpctype_embeds(ea[:, 1])], 1)
    des = [torch.randn(E, H, generator=g).double() for _ in range(L)]
    loss = 0
    for l in range(L):
        e = o.convs[l].lin_edge(emb)
        if_p, rpc_p, weA, weB = R.edge_params(d, Hp, flat, l)
        t_if, _ = R.table_fwd_ref(if_p, weA)
        t_rpc, _ = R.table_fwd_ref(rpc_p, weB)
        torch.testing.assert_close((t_if[ea[:, 0]] + t_rpc[ea[:, 1]])[:, :H], e.detach(), rtol=1e-12, atol=1e-12)
        loss = loss + (e * des[l]).sum()
    loss.backward()
    dts_if, dts_rpc, wa, wb = [], [], [], []
    for l in range(L):
        if_p, rpc_p, weA, weB = R.edge_params(d, Hp, flat, l)
        dt_if = torch.zeros(N_IF, Hp, dtype=torch.float64).index_add_(0, ea[:, 0], R._pad(des[l], (E, Hp)))
        dt_rpc = torch.zeros(N_RPC, Hp, dtype=torch.float64).index_add_(0, ea[:, 1], R._pad(des[l], (E, Hp)))
        dA, _ = R.table_wgrad_ref(dt_if, if_p, R.split_k(N_IF))
        dB, _ = R.table_wgrad_ref(dt_rpc, rpc_p, 1)
        torch.testing.assert_close(torch.cat([dA[:H, :H], dB[:H, :H]], 1), o.convs[l].lin_edge.weight.grad,
                                   rtol=1e-12, atol=1e-12)
        dts_if.append(dt_if)
        dts_rpc.append(dt_rpc)
        wa.append(weA)
        wb.append(weB)
    torch.testing.assert_close(R.table_dgrad_ref(dts_if, wa)[0][:, :H], o.interface_embeds.weight.grad,
                               rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(R.table_dgrad_ref(dts_rpc, wb)[0][:, :H], o.rpctype_embeds.weight.grad,
                               rtol=1e-12, atol=1e-12)


# ------------------------------------------------------------------------------------------------------ bars
def _head_fwd_worst(eng, B, defect=None, seed=0):
    z, W1, b1, W2, b2, ids, dg = _head_inputs(eng, B, seed)
    W1k = W1
    if defect == "entry_at_H":
        W1k = R.pad_w1(torch.cat([W1[:eng.desc.H, :eng.desc.H], W1[:eng.desc.H, eng.Hp:eng.Hp + eng.desc.H]], 1),
                       eng.Hp, entry_col=eng.desc.H)
    h1, pred = R.head_fwd_f32(z, W1k, b1, W2, b2, defect=defect if defect == "slice" else None)
    h1 = torch.from_numpy(h1)
    pre, pre_bar, pr, pr_bar = R.head_fwd_ref(z, W1, b1, W2, b2, h1)
    return max(R.worst(h1, torch.relu(pre), pre_bar), R.worst(pred, pr, pr_bar))


def _head_bwd_worst(eng, B, rng, defect=None, seed=0):
    z, W1, b1, W2, b2, ids, dg = _head_inputs(eng, B, seed)
    ids[: B // 2] = 0                                  # a hot row
    z[: B // 2, eng.Hp:] = R.head_params(eng.desc, eng.Hp, eng.fp.flat.detach())[4][0]
    h1, _ = R.head_fwd_f32(z, W1, b1, W2, b2)
    got = R.head_bwd_f32(dg, z, h1, W1, W2, ids, eng.desc.n_entry, rng=rng, defect=defect)
    ref = R.head_bwd_ref(dg, z, torch.from_numpy(h1), W1, W2, ids, eng.desc.n_entry)
    return max(R.worst(got[k], *ref[k]) for k in ref)


def _table_worst(eng, l, n_rows, rng, defect=None):
    d, Hp, flat = eng.desc, eng.Hp, eng.fp.flat.detach()
    if_p, _, weA, weB = R.edge_params(d, Hp, flat, l)
    g = torch.Generator().manual_seed(l)
    dT = R._pad(torch.randn(n_rows, d.H, generator=g), (n_rows, Hp))
    emb = R._pad(torch.randn(n_rows, d.H, generator=g), (n_rows, Hp))
    ks = R.split_k(n_rows)
    gemm = lambda A, Bt, k=1: torch.from_numpy(R.small_gemm_f32(A, Bt, k, rng, defect))
    w = [R.worst(gemm(if_p, weB if defect == "swap" else weA), *R.table_fwd_ref(if_p, weA)),
         R.worst(gemm(dT.T, emb.T, ks), *R.table_wgrad_ref(dT, emb, ks))]
    # d emb over the layers: one small GEMM per layer, the layers added atomically in a random order
    Ws = [R.edge_params(d, Hp, flat, k)[2] for k in range(eng.n_convs)]
    dTs = [dT * (k + 1) for k in range(eng.n_convs)]
    parts = [R.small_gemm_f32(t, W.T, 1, rng, defect) for t, W in zip(dTs, Ws)]
    w.append(R.worst(R._atomic_sum(parts, rng), *R.table_dgrad_ref(dTs, Ws)))
    return max(w)


@pytest.mark.parametrize("H", [4, 5, 16, 100, 192, 200, 256])
def test_head_fwd_bars_pass_f32_restatement(H):
    _, eng, _ = _model(H)
    assert _head_fwd_worst(eng, 11) <= 1.0


@pytest.mark.parametrize("H", [4, 5, 8, 16])
@pytest.mark.parametrize("B", [1, 7, 9, 17])
def test_head_bwd_bars_pass_f32_restatement(H, B):
    _, eng, _ = _model(H)
    for seed in range(3):
        assert _head_bwd_worst(eng, B, np.random.default_rng(seed), seed=seed) <= 1.0


@pytest.mark.parametrize("H,n_rows", [(4, 1), (5, 2), (16, 511), (8, 513), (32, 600)])
def test_table_bars_pass_f32_restatement(H, n_rows):
    _, eng, _ = _model(H, 3)
    for seed in range(3):
        assert _table_worst(eng, 1, n_rows, np.random.default_rng(seed)) <= 1.0


@pytest.mark.parametrize("defect,H,how", [
    ("entry_at_H", 5, "head_fwd"), ("entry_at_H", 100, "head_fwd"),
    ("slice", 192, "head_fwd"), ("slice", 256, "head_fwd"),
    ("drop_tail", 8, "head_bwd"), ("no_mask", 8, "head_bwd"), ("no_mask", 5, "head_bwd"),
    ("split_floor", 8, "table"), ("swap", 16, "table"),
    ("tf32", 4, "table"), ("tf32", 16, "table"), ("tf32", 64, "table"), ("tf32", 256, "table"),
])
def test_bars_reject_defects(defect, H, how):
    _, eng, _ = _model(H, 3)
    if how == "head_fwd":
        w = _head_fwd_worst(eng, 11, defect)
    elif how == "head_bwd":
        w = _head_bwd_worst(eng, 9, np.random.default_rng(0), defect)
    else:
        w = _table_worst(eng, 1, 513 if defect == "split_floor" else 24, np.random.default_rng(0), defect)
    assert w > 1.0, f"{defect} at H={H} stays within its bar ({w:.3g})"
