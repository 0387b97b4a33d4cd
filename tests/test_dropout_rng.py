"""CPU tests of the engine's dropout: the Philox4x32-10 restatement against the Random123 known-answer vectors, the
statistics and exact thresholds of the mask contract, the C-ABI argument checks, and the masked oracle forward."""
import ctypes
import math

import numpy as np
import pytest
import torch

from tests.dropout_ref import dropout_mask, oracle_forward, philox4x32_10, scale_of, threshold

N_BIG, H_BIG = 51200, 64     # cfg2's node count and width


@pytest.mark.parametrize("ctr, key, want", [
    ((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
     (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
])
def test_philox_known_answers(ctr, key, want):
    got = tuple(int(w) for w in philox4x32_10(ctr, key))
    assert got == want, [hex(w) for w in got]


@pytest.mark.parametrize("p", [0.1, 0.5, 0.9])
def test_kept_fraction(p):
    keep = dropout_mask(0x1234_5678_9abc_def0, 3, 1, N_BIG, H_BIG, p)
    n = keep.size
    sigma = math.sqrt(p * (1 - p) / n)
    assert abs(keep.mean() - (1 - p)) <= 6 * sigma, (keep.mean(), 1 - p, sigma)


def test_masks_differ_across_layer_step_seed():
    p, n = 0.5, N_BIG * H_BIG
    sigma = math.sqrt(0.25 / n)
    base = dropout_mask(7, 5, 0, N_BIG, H_BIG, p)
    for seed, step, layer in ((7, 5, 1), (7, 6, 0), (8, 5, 0), (7 + 2 ** 32, 5, 0), (7, 5 + 2 ** 32, 0)):
        other = dropout_mask(seed, step, layer, N_BIG, H_BIG, p)
        agree = float((base == other).mean())
        assert abs(agree - 0.5) <= 6 * sigma, (seed, step, layer, agree)


def test_threshold_and_scale_exact():
    assert threshold(0.0) == 0
    assert threshold(1.0) == 2 ** 32
    assert threshold(2.0 ** -32) == 1
    assert threshold(0.5) == 2 ** 31
    assert scale_of(1.0) == 0.0 and scale_of(0.0) == 1.0 and scale_of(0.5) == 2.0
    assert dropout_mask(1, 0, 0, 8, 8, 0.0).all()
    assert not dropout_mask(1, 0, 0, 8, 8, 1.0).any()


def test_mask_layout():
    """Column col + j of row r takes word j of the float4 group r*(H/4) + col/4."""
    N, H, seed, step, layer = 3, 8, 99, 4, 2
    m = dropout_mask(seed, step, layer, N, H, 0.5)
    for r in range(N):
        for c4 in range(H // 4):
            w = philox4x32_10((r * (H // 4) + c4, layer, step, 0), (seed, 0))
            for j in range(4):
                assert m[r, 4 * c4 + j] == (int(w[j]) >= 2 ** 31)


def _desc(H=64):
    from pert_gnn_kdd23_b200.engine import PertModelDesc

    d = PertModelDesc()
    d.F, d.H, d.n_convs, d.n_cat = 9, H, 3, 1
    d.cat_rows[0] = 16
    d.n_entry, d.n_if, d.n_rpc = 8, 8, 8
    d.k0 = (9 + H + 7) // 8 * 8
    d.bn_eps, d.bn_momentum = 1e-5, 0.1
    return d


def test_abi_dropout_argument_checks():
    """The dropout arguments are rejected with PERT_ERR_BADARG before any CUDA call (null device pointers)."""
    from pert_gnn_kdd23_b200 import _lib

    L = _lib.lib()
    assert L.pert_version() == 2005
    d = _desc()
    state = (ctypes.c_longlong * 2)(1, 0)          # host memory: never read, the calls are rejected first

    def fwd(p, st, N=100, training=1):
        return L.pert_model_forward(ctypes.byref(d), *([None] * 9), N, 0, 1, *([None] * 5), 0, training, p, st,
                                    None, None, None, None, None, None)

    def bwd(p, training=1):
        return L.pert_model_backward(ctypes.byref(d), *([None] * 7), 100, 0, 1, *([None] * 8), 0, training, p,
                                     None, None, None, None)

    for p in (float("nan"), -0.1, 1.5, float("inf")):
        assert fwd(p, state) == -1, p
        assert fwd(p, state, training=0) == -1, p
        assert bwd(p) == -1, p
    assert fwd(0.5, None) == -1                      # training with p > 0 needs the {seed, step} state
    assert fwd(0.5, state, N=(1 << 32) // 16) == -1  # N*H/4 = 2^32 groups overflow the counter word


def test_oracle_masks_equal_torch_dropout():
    """oracle_forward with the masks torch's F.dropout drew reproduces the oracle's own F.dropout forward.  The masks
    are recovered as F.dropout(ones) != 0 under the same seed (torch's mask does not depend on the input values)."""
    from oracle.model_oracle import OracleSAGEDeterministic
    from pert_gnn_kdd23_b200.synthetic import model_args
    from tests.helpers import forward_args, make_batch

    torch.manual_seed(0)
    oracle = OracleSAGEDeterministic(*model_args(2)).train()
    oracle.dropout = 0.3
    a = forward_args(make_batch(2, 4))
    N, H = a[0].size(0), oracle.bns[0].num_features
    n_bn = len(oracle.bns)
    state = {k: v.clone() for k, v in oracle.state_dict().items()}
    torch.manual_seed(11)
    g_ref, l_ref = oracle(*a)
    oracle.load_state_dict(state)                    # undo the running-statistics update of that forward
    torch.manual_seed(11)
    masks = {f"bn{i}": torch.nn.functional.dropout(torch.ones(N, H), p=0.3, training=True) != 0 for i in range(n_bn)}
    assert 0.6 < float(masks["bn0"].float().mean()) < 0.8
    g, l = oracle_forward(oracle, *a, dropout_masks=masks)
    torch.testing.assert_close(g, g_ref, rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(l, l_ref, rtol=1e-5, atol=1e-6)
    # p = 1: everything after the first BatchNorm sees zeros, like F.dropout(p=1)
    oracle.dropout = 1.0
    g1, l1 = oracle_forward(oracle, *a, dropout_masks={k: torch.ones_like(v) for k, v in masks.items()})
    torch.manual_seed(0)
    g1_ref, l1_ref = oracle_forward(oracle, *a)
    torch.testing.assert_close(g1, g1_ref)
    torch.testing.assert_close(l1, l1_ref)
    # eval mode: masks are ignored
    oracle.eval()
    torch.testing.assert_close(oracle_forward(oracle, *a, dropout_masks=masks)[0], oracle(*a)[0])
