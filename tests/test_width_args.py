"""CPU tests of the padded hidden width (include/pertgnn.h, pert_model_width): the width rule, the workspace of a padded
model (the Hp-wide one plus the zero-padded copies of the other tensors), the descriptor checks, the unchanged
attention-kernel widths and the launch counts of the engine at the widths that run unpadded."""
import ctypes

import pytest

from pert_gnn_kdd23_b200 import _lib

KERNEL_WIDTHS = (4, 8, 16, 32, 64, 96, 128, 192, 256)
F, L, CAT_ROWS, N_ENTRY, N_IF, N_RPC = 9, 3, (16, 5), 8, 40, 3


def width_rule(H):
    return min((w for w in KERNEL_WIDTHS if w >= H), default=-2) if H >= 1 else -2


def _desc(H, k0_width=None):
    from pert_gnn_kdd23_b200._lib import PertModelDesc

    d = PertModelDesc()
    d.F, d.H, d.n_convs, d.n_cat = F, H, L, len(CAT_ROWS)
    for i, r in enumerate(CAT_ROWS):
        d.cat_rows[i] = r
    d.n_entry, d.n_if, d.n_rpc = N_ENTRY, N_IF, N_RPC
    d.k0 = (F + (k0_width or width_rule(H)) + 7) // 8 * 8
    d.bn_eps, d.bn_momentum = 1e-5, 0.1
    return d


def _al64(n):
    return (max(n, 1) + 63) // 64 * 64


def _padded_copies_floats(Hp):
    """Floats of one set of zero-padded copies: embeddings, BatchNorm gamma / beta, local_linear, global_linear1/2."""
    rows = list(CAT_ROWS) + [N_ENTRY, N_IF, N_RPC]
    return (sum(_al64(r * Hp) for r in rows) + 2 * (L - 1) * _al64(Hp) + _al64(Hp) + _al64(2 * Hp * Hp) +
            2 * _al64(Hp))


def test_model_width_rule():
    lib = _lib.lib()
    for H in range(0, 301):
        assert lib.pert_model_width(H) == width_rule(H), H
    assert lib.pert_model_width(-5) == -2


def test_tconv_supported_width_unchanged():
    lib = _lib.lib()
    for H in range(0, 301):
        assert lib.pert_tconv_supported_width(H) == int(H in KERNEL_WIDTHS), H


@pytest.mark.parametrize("H", [1, 3, 10, 48, 50, 80, 100, 129, 200, 255])
def test_workspace_of_padded_width(H):
    lib = _lib.lib()
    Hp = width_rule(H)
    assert Hp != H
    d, dp = _desc(H), _desc(Hp)
    extra = 4 * _padded_copies_floats(Hp)
    for N, E, B in ((0, 0, 0), (100, 300, 4), (5000, 20000, 64)):
        got = lib.pert_model_workspace_bytes(ctypes.byref(d), N, E, B)
        assert got == lib.pert_model_workspace_bytes(ctypes.byref(dp), N, E, B) + 2 * extra, (N, E, B)
        # saved activations are laid out at Hp, behind the parameter copies
        for which, layer in ((0, 1), (0, L - 1), (1, 0)):
            off = lib.pert_model_workspace_offset(ctypes.byref(d), N, E, B, which, layer)
            offp = lib.pert_model_workspace_offset(ctypes.byref(dp), N, E, B, which, layer)
            assert off == offp + 2 * extra // 4
    assert lib.pert_model_packed_bytes(ctypes.byref(d)) == lib.pert_model_packed_bytes(ctypes.byref(dp)) + extra


@pytest.mark.parametrize("H", KERNEL_WIDTHS)
def test_workspace_of_kernel_width_has_no_copies(H):
    """At Hp = H nothing is added: the packed region is the conv packs alone."""
    lib = _lib.lib()
    d = _desc(H)
    packs = 0
    for l in range(L):
        K = d.k0 if l == 0 else H
        packs += 2 * _al64(4 * H * K) + _al64(4 * H) + 4 * _al64(H * H)    # W4, W4^T, b4, lin_edge halves
    assert lib.pert_model_packed_bytes(ctypes.byref(d)) == 4 * packs


def test_descriptor_checks():
    lib = _lib.lib()
    ws = lambda d: lib.pert_model_workspace_bytes(ctypes.byref(d), 10, 10, 1)
    assert ws(_desc(48)) > 0 and ws(_desc(256)) > 0 and ws(_desc(1)) > 0
    assert ws(_desc(48, k0_width=48)) == -1          # conv 0's input must hold the Hp-wide embedding block
    assert ws(_desc(257, k0_width=257)) == -1        # above 256: refused, as before
    assert ws(_desc(0, k0_width=4)) == -1


@pytest.mark.parametrize("H", KERNEL_WIDTHS + (10, 48, 200))
@pytest.mark.parametrize("layers", [2, 3, 8])
def test_launch_counts(H, layers):
    """launches_forward / _backward: exactly the formula of the unpadded engine at its widths; one pack launch more in
    each direction at a padded width."""
    from pert_gnn_kdd23_b200.model import SAGEDeterministic

    m = SAGEDeterministic(F, list(CAT_ROWS), N_ENTRY - 1, N_IF - 1, N_RPC - 1, H, layers, 0.0)
    eng = m.engine()
    Hp = width_rule(H)
    assert eng.Hp == Hp and eng.desc.H == H and eng.desc.k0 == (F + Hp + 7) // 8 * 8
    assert tuple(eng.bn_running.shape) == (layers - 1, 2, Hp)
    assert tuple(m.bns[0].running_mean.shape) == (H,)
    lib = eng.lib
    N = 5000
    eng._saved = (None,) * 8 + (N, 0, 0, 0.0)

    n, count = 0, 0                                      # pack launches of the unpadded engine
    for l in range(layers):
        count += 24 if l == 0 else 16
        if count + 24 > 96 or l == layers - 1:
            n, count = n + 1, 0
    pack = n + int(Hp != H)
    applies = 0 if lib.pert_bn_linear_fwd_planes_supported(N, Hp, Hp) else layers - 1
    fwd = pack + (layers + 5) // 6 + len(CAT_ROWS) + 1 + 2 * layers + applies + 1 + 1
    linear = sum(1 if lib.pert_linear_bwd_planes_supported(N, Hp, eng.desc.k0 if l == 0 else Hp, Hp) else 2
                 for l in range(layers))
    bwd = 1 + 1 + 2 * layers + linear + 2 * (layers - 1) + len(CAT_ROWS) + (layers + 2) // 3 + pack
    assert eng.launches_forward() == fwd
    assert eng.launches_backward() == bwd


def test_tconv_c_entries_reject_bad_logical_width():
    """pert_tconv_fwd_c / _bwd_c: 1 <= C <= H, else PERT_ERR_BADARG before any CUDA call (host pointers, never read)."""
    lib = _lib.lib()
    buf = ctypes.create_string_buffer(64)
    p = ctypes.addressof(buf) + (-ctypes.addressof(buf)) % 16
    for C in (0, -1, 65):
        assert lib.pert_tconv_fwd_c(p, p, p, None, 64, p, None, None, None, None, None, p, 64, None, 0, 1, 0, 0, 64, C,
                                    None) == -1, C
        assert lib.pert_tconv_bwd_c(p, 64, p, p, p, 64, p, None, None, None, p, None, None, None, None, None, p, p, p,
                                    64, None, None, None, None, 0, 1, 0, 0, 64, C, None) == -1, C
