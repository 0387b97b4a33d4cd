"""CPU tests of the multi-quantile global head: the refusals of every _q entry point (made with NULL device pointers,
so a call that got past its checks would fault -- none may), the workspace of a head with n_out outputs, the
constructor's level checks, the state_dict of a quantile model, how steps and metrics resolve ``tau``, the ctypes
signatures, and the float32 restatements of tests/quantile_ref.py against their fp64 references and bars."""
import ctypes
import math

import numpy as np
import pytest
import torch

from pert_gnn_kdd23_b200 import _lib
from tests import quantile_ref as Q

BADARG = -1
F, L, CAT_ROWS, N_ENTRY, N_IF, N_RPC = 9, 3, (16, 5), 8, 40, 3


def _desc(H):
    d = _lib.PertModelDesc()
    d.F, d.H, d.n_convs, d.n_cat = F, H, L, len(CAT_ROWS)
    for i, r in enumerate(CAT_ROWS):
        d.cat_rows[i] = r
    d.n_entry, d.n_if, d.n_rpc = N_ENTRY, N_IF, N_RPC
    Hp = _lib.lib().pert_model_width(H)
    d.k0 = (F + Hp + 7) // 8 * 8
    d.bn_eps, d.bn_momentum = 1e-5, 0.1
    return d


def _al64(n):
    return (max(n, 1) + 63) // 64 * 64


def _levels(*t):
    return (ctypes.c_float * max(len(t), 1))(*t)


# ------------------------------------------------------------------------------------------------------ C-ABI
def test_max_quantiles_matches_header():
    from pert_gnn_kdd23_b200 import model

    assert _lib.MAX_QUANTILES == model.MAX_QUANTILES == 8


@pytest.mark.parametrize("H", [16, 64, 5, 100])
def test_workspace_q_sizes(H):
    """n_out = 1 is the plain layout; above it the workspace grows only where the padded copy of global_linear2 and its
    gradient hold n_out rows (Hp > H), and the offsets behind them shift by as much."""
    lib = _lib.lib()
    d = _desc(H)
    Hp = lib.pert_model_width(H)
    N, E, B = 1000, 3000, 64
    base = lib.pert_model_workspace_bytes(ctypes.byref(d), N, E, B)
    packed = lib.pert_model_packed_bytes(ctypes.byref(d))
    assert base > 0 and packed > 0
    assert lib.pert_model_workspace_bytes_q(ctypes.byref(d), 1, N, E, B) == base
    assert lib.pert_model_packed_bytes_q(ctypes.byref(d), 1) == packed
    for which in range(0, 12):
        for layer in (0, 1, 2):
            assert lib.pert_model_workspace_offset_q(ctypes.byref(d), 1, N, E, B, which, layer) == \
                lib.pert_model_workspace_offset(ctypes.byref(d), N, E, B, which, layer)
    for T in range(2, 9):
        grow = 4 * (_al64(T * Hp) - _al64(Hp)) if Hp != H else 0
        assert lib.pert_model_workspace_bytes_q(ctypes.byref(d), T, N, E, B) == base + 2 * grow
        assert lib.pert_model_packed_bytes_q(ctypes.byref(d), T) == packed + grow
        h1 = lib.pert_model_workspace_offset_q(ctypes.byref(d), T, N, E, B, 1, 0)
        assert h1 == lib.pert_model_workspace_offset(ctypes.byref(d), N, E, B, 1, 0) + 2 * grow // 4


def test_model_q_refusals():
    """n_out outside 1..8 and what the plain forms refuse, before any CUDA call (NULL device pointers throughout)."""
    lib = _lib.lib()
    d = _desc(16)
    fwd_args = lambda: [None] * 9 + [10, 20, 2] + [None] * 5 + [1 << 30, 1, 0.0] + [None] * 8
    bwd_args = lambda: [None] * 7 + [10, 20, 2] + [None] * 7 + [None, 1 << 30, 1, 0.0] + [None] * 5
    for T in (0, -1, 9, 100):
        assert lib.pert_model_workspace_bytes_q(ctypes.byref(d), T, 10, 20, 2) == BADARG
        assert lib.pert_model_packed_bytes_q(ctypes.byref(d), T) == BADARG
        assert lib.pert_model_workspace_offset_q(ctypes.byref(d), T, 10, 20, 2, 1, 0) == BADARG
        assert lib.pert_model_forward_q(ctypes.byref(d), T, *fwd_args()) == BADARG
        assert lib.pert_model_backward_q(ctypes.byref(d), T, *bwd_args()) == BADARG
    for T in (1, 4, 8):
        assert lib.pert_model_workspace_bytes_q(None, T, 10, 20, 2) == BADARG
        assert lib.pert_model_workspace_bytes_q(ctypes.byref(d), T, -1, 20, 2) == BADARG
        assert lib.pert_model_workspace_offset_q(ctypes.byref(d), T, 10, 20, 2, 12, 0) == BADARG
        # valid n_out, NULL params / workspace: refused as the plain forms refuse them
        assert lib.pert_model_forward_q(ctypes.byref(d), T, *fwd_args()) == BADARG
        assert lib.pert_model_backward_q(ctypes.byref(d), T, *bwd_args()) == BADARG
        a = fwd_args()
        a[19] = float("nan")                                       # dropout NaN
        assert lib.pert_model_forward_q(ctypes.byref(d), T, *a) == BADARG
    bad = _desc(16)
    bad.n_convs = 1
    assert lib.pert_model_workspace_bytes_q(ctypes.byref(bad), 2, 10, 20, 2) == BADARG
    assert lib.pert_model_forward_q(ctypes.byref(bad), 2, *fwd_args()) == BADARG


BAD_LEVELS = [(), (0.5, 0.5), (0.9, 0.5), (-0.1, 0.5), (0.5, 1.5), (float("nan"),), (0.1, float("nan")),
              (0.5, float("inf"))]


def test_loss_and_metrics_q_refusals():
    lib = _lib.lib()
    good = _levels(0.5, 0.9)
    acc = 1     # never dereferenced: every call below is refused before any launch
    for T in (0, -3, 9):
        assert lib.pert_pinball_loss_q(1, 1, _levels(*[0.1 * i for i in range(9)]), T, 4, 1.0, None, None, None,
                                       None) == BADARG
        assert lib.pert_eval_metrics_q(1, 1, _levels(*[0.1 * i for i in range(9)]), T, 4, acc, None, None) == BADARG
    for lv in BAD_LEVELS:
        T = len(lv)
        assert lib.pert_pinball_loss_q(1, 1, _levels(*lv), T, 4, 1.0, None, None, None, None) == BADARG, lv
        assert lib.pert_eval_metrics_q(1, 1, _levels(*lv), T, 4, acc, None, None) == BADARG, lv
    assert lib.pert_pinball_loss_q(1, 1, None, 2, 4, 1.0, None, None, None, None) == BADARG
    assert lib.pert_eval_metrics_q(1, 1, None, 2, 4, acc, None, None) == BADARG
    for T, lv in ((1, _levels(0.5)), (2, good)):
        # what the plain forms refuse
        assert lib.pert_pinball_loss_q(None, 1, lv, T, 4, 1.0, None, None, None, None) == BADARG
        assert lib.pert_pinball_loss_q(1, None, lv, T, 4, 1.0, None, None, None, None) == BADARG
        assert lib.pert_pinball_loss_q(1, 1, lv, T, 0, 1.0, None, None, None, None) == BADARG
        assert lib.pert_pinball_loss_q(1, 1, lv, T, 2 ** 31, 1.0, None, None, None, None) == BADARG
        assert lib.pert_eval_metrics_q(None, 1, lv, T, 4, acc, None, None) == BADARG
        assert lib.pert_eval_metrics_q(1, None, lv, T, 4, acc, None, None) == BADARG
        assert lib.pert_eval_metrics_q(1, 1, lv, T, 4, None, None, None) == BADARG
        assert lib.pert_eval_metrics_q(1, 1, lv, T, -1, acc, None, None) == BADARG
        assert lib.pert_eval_metrics_q(1, 1, lv, T, 2 ** 31, acc, None, None) == BADARG
        assert lib.pert_eval_metrics_q(1, 1, lv, T, 0, acc, None, None) == 0     # B = 0: nothing to add, no launch
    # the levels 0 and 1 themselves are quantiles
    assert lib.pert_eval_metrics_q(1, 1, _levels(0.0, 1.0), 2, 0, acc, None, None) == 0


def test_signatures_bound():
    lib = _lib.lib()
    sig = _lib.SIGNATURES
    I, P, LL, F_ = ctypes.c_int, ctypes.c_void_p, ctypes.c_longlong, ctypes.c_float
    assert sig["pert_model_forward_q"][1] == [P, I] + sig["pert_model_forward_live"][1][1:]
    assert sig["pert_model_backward_q"][1] == [P, I] + sig["pert_model_backward_live"][1][1:]
    assert sig["pert_model_workspace_bytes_q"] == (LL, [P, I, LL, LL, LL])
    assert sig["pert_model_packed_bytes_q"] == (LL, [P, I])
    assert sig["pert_model_workspace_offset_q"] == (LL, [P, I, LL, LL, LL, I, I])
    assert sig["pert_pinball_loss_q"] == (I, [P, P, P, I, LL, F_, P, P, P, P])
    assert sig["pert_eval_metrics_q"] == (I, [P, P, P, I, LL, P, P, P])
    for name in sig:
        if name.endswith("_q"):
            fn = getattr(lib, name)
            assert fn.argtypes == sig[name][1] and fn.restype == sig[name][0]


# ------------------------------------------------------------------------------------------------------ model
def _model(**kw):
    from pert_gnn_kdd23_b200.model import SAGEDeterministic

    torch.manual_seed(0)
    return SAGEDeterministic(F, list(CAT_ROWS), N_ENTRY - 1, N_IF - 1, N_RPC - 1, 16, 3, 0.1, **kw)


@pytest.mark.parametrize("bad", [(), [0.5] * 9, (0.5, 0.5), (0.9, 0.1), (-0.01,), (1.01,), (float("nan"),),
                                 0.5, "0.5", (0.1, None)])
def test_constructor_refuses_bad_levels(bad):
    with pytest.raises((ValueError, TypeError)):
        _model(quantiles=bad)


def test_constructor_levels_and_state_dict():
    plain = _model()
    assert plain.quantiles is None
    q = _model(quantiles=[0.5, 0.9, np.float32(0.95), 0.99])
    assert q.quantiles == (0.5, 0.9, float(np.float32(0.95)), 0.99)
    assert all(type(t) is float for t in q.quantiles)
    assert list(q.state_dict()) == list(plain.state_dict())
    sd, sp = q.state_dict(), plain.state_dict()
    for k in sd:
        if k.startswith("global_linear2."):
            continue
        assert sd[k].shape == sp[k].shape, k
    H = plain.hidden_channels
    assert sd["global_linear2.weight"].shape == (4, H) and sd["global_linear2.bias"].shape == (4,)
    assert sp["global_linear2.weight"].shape == (1, H) and sp["global_linear2.bias"].shape == (1,)
    one = _model(quantiles=(0.5,))
    assert one.quantiles == (0.5,)
    # one level: the reference's parameters, drawn in the same order from the same seed
    for (k, a), (_, b) in zip(one.state_dict().items(), plain.state_dict().items()):
        assert torch.equal(a, b), k
    edges = _model(quantiles=(0.0, 1.0))
    assert edges.quantiles == (0.0, 1.0)
    assert len(_model(quantiles=[i / 10 for i in range(1, 9)]).quantiles) == 8


def test_tau_resolution():
    from pert_gnn_kdd23_b200.train import EvalMetrics, resolve_tau

    plain, q = _model(), _model(quantiles=(0.5, 0.9, 0.95, 0.99))
    assert resolve_tau(plain) == (0.5,)
    assert resolve_tau(plain, None) == (0.5,)
    assert resolve_tau(plain, 0.95) == (0.95,)
    assert resolve_tau(plain, [0.3]) == (0.3,)
    with pytest.raises(ValueError):
        resolve_tau(plain, (0.5, 0.9))
    assert resolve_tau(q) == (0.5, 0.9, 0.95, 0.99)
    assert resolve_tau(q, [0.5, 0.9, 0.95, 0.99]) == q.quantiles
    for bad in (0.5, (0.5, 0.9), (0.5, 0.9, 0.95, 0.98), (0.99, 0.95, 0.9, 0.5)):
        with pytest.raises(ValueError):
            resolve_tau(q, bad)
    one = _model(quantiles=(0.9,))
    assert resolve_tau(one) == (0.9,) and resolve_tau(one, 0.9) == (0.9,)
    with pytest.raises(ValueError):
        resolve_tau(one, 0.5)
    # EvalMetrics holds the levels; its accumulators are 4T + 1 doubles (CPU tensors suffice to check the layout)
    m = EvalMetrics("cpu")
    assert m.levels == (0.5,) and m.tau == 0.5 and m.acc.numel() == 5
    m = EvalMetrics("cpu", 0.95)
    assert m.levels == (0.95,) and m.tau == 0.95
    m = EvalMetrics("cpu", q.quantiles)
    assert m.levels == q.quantiles and m.acc.numel() == 17
    m.acc.copy_(torch.arange(17, dtype=torch.float64))
    m.count = 2
    assert m.result() == ((0.0, 2.0, 4.0, 6.0), (0.5, 2.5, 4.5, 6.5), (1.0, 3.0, 5.0, 7.0))
    assert m.coverage() == (1.5, 3.5, 5.5, 7.5)
    assert m.crossing() == 8.0


def test_steps_refuse_mismatched_tau_before_any_launch():
    """The steps resolve tau before they touch the model or the device (the model here lives on the CPU)."""
    from pert_gnn_kdd23_b200 import train

    q = _model(quantiles=(0.5, 0.9))
    for call in (lambda: train.train_step(q, None, None, 0.5),
                 lambda: train.fused_train_step(q, None, None, (0.1, 0.9)),
                 lambda: train.GraphedTrainStep(q, None, 0.9),
                 lambda: train.BucketedTrainStep(q, None, (0.5,)),
                 lambda: train.eval_step(q, None, 0.5),
                 lambda: train.evaluate(q, [], "cpu", 0.5),
                 lambda: train.evaluate_bucketed(q, [], "cpu", 0.5)):
        with pytest.raises(ValueError):
            call()
    assert train.GraphedTrainStep(q, None).tau == (0.5, 0.9)
    assert train.BucketedTrainStep(_model(), None).tau == (0.5,)


def test_torch_quantile_loss_levels():
    from pert_gnn_kdd23_b200.train import torch_quantile_loss

    y = torch.tensor([3.0, 5.0, 8.0])
    p1 = torch.tensor([4.0, 5.0, 6.0])
    assert torch.equal(torch_quantile_loss(y, p1), torch_quantile_loss(y, p1, 0.5))
    taus = (0.1, 0.5, 0.9)
    pT = torch.tensor([[4.0, 2.0, 9.0], [5.0, 5.0, 5.0], [6.0, 8.5, 7.0]])
    got = float(torch_quantile_loss(y, pT, taus))
    ref = np.mean([max(t * (yb - p), (t - 1) * (yb - p)) for yb, row in zip(y.tolist(), pT.tolist())
                   for t, p in zip(taus, row)])
    assert abs(got - ref) <= 1e-6 * abs(ref)
    # one level as a sequence is the scalar loss on the single column
    assert torch.allclose(torch_quantile_loss(y, p1[:, None], (0.3,)), torch_quantile_loss(y, p1, 0.3))


# ------------------------------------------------------------------------------------------------------ restatements
@pytest.mark.parametrize("Hp,T", [(16, 1), (48, 3), (100, 4), (256, 8)])
def test_head_fwd_restatement_within_bar_and_defects_outside(Hp, T):
    rng = np.random.default_rng(Hp * 10 + T)
    B = 64
    h1 = np.maximum(rng.standard_normal((B, Hp)), 0).astype(np.float32)
    W2 = rng.standard_normal((T, Hp)).astype(np.float32)
    b2 = rng.standard_normal(T).astype(np.float32)
    ref, bar = Q.head_fwd_ref_q(torch.from_numpy(h1), torch.from_numpy(W2), torch.from_numpy(b2))
    from tests.engine_parts_ref import worst

    assert worst(Q.head_fwd_f32(h1, W2, b2), ref, bar) <= 1
    if T > 1:
        for defect in ("row0", "bias0", "stride1"):
            assert worst(Q.head_fwd_f32(h1, W2, b2, defect), ref, bar) > 1, defect


def test_head_bwd_reference_reduces_to_one_output():
    """At T = 1 the T-level reference is the one-output reference of tests/engine_parts_ref.py, bars included up to the
    dh rounding (1 there, T = 1 here)."""
    from tests.engine_parts_ref import head_bwd_ref

    rng = np.random.default_rng(3)
    B, Hp, n_entry = 37, 48, 9
    dg = torch.from_numpy(rng.standard_normal(B).astype(np.float32))
    z = torch.from_numpy(rng.standard_normal((B, 2 * Hp)).astype(np.float32))
    h1 = torch.from_numpy(np.maximum(rng.standard_normal((B, Hp)), 0).astype(np.float32))
    W1 = torch.from_numpy(rng.standard_normal((Hp, 2 * Hp)).astype(np.float32))
    W2 = torch.from_numpy(rng.standard_normal(Hp).astype(np.float32))
    ids = torch.from_numpy(rng.integers(0, n_entry, B))
    one = head_bwd_ref(dg, z, h1, W1, W2, ids, n_entry)
    q = Q.head_bwd_ref_q(dg[:, None], z, h1, W1, W2[None, :], ids, n_entry)
    for k in one:
        r1, b1 = one[k]
        rq, bq = q[k]
        assert torch.allclose(rq.reshape(r1.shape), r1, rtol=1e-12, atol=1e-12), k
        assert torch.allclose(bq.reshape(b1.shape), b1, rtol=1e-9, atol=0), k


@pytest.mark.parametrize("B,T", [(1, 2), (257, 3), (1000, 4), (5000, 8)])
def test_pinball_restatement_within_bar_and_defects_outside(B, T):
    y, yhat = Q.quantile_data(B, T, seed=B + T)
    taus = [0.0, 0.5, 0.9, 0.95, 0.99, 0.995, 0.999, 1.0][:T] if T < 8 else [0.0, 0.1, 0.5, 0.9, 0.95, 0.99, 0.999, 1.0]
    taus = sorted(set(taus))
    yhat = yhat[:, :len(taus)]
    T = len(taus)
    for live in (None, max(1, B // 2)):
        ref = Q.pinball_q_ref(y, yhat, taus, 0.125, live)
        n = (B if live is None else live) * T
        rl, rd = Q.pinball_q_worst(*Q.pinball_q_f32(y, yhat, taus, 0.125, live), *ref, n)
        assert rl <= 1 and rd <= 1, (rl, rd)
        for defect in ("per_graph", "level0"):
            rl, rd = Q.pinball_q_worst(*Q.pinball_q_f32(y, yhat, taus, 0.125, live, defect), *ref, n)
            assert max(rl, rd) > 1, defect


def test_metrics_reference_counts():
    y = np.array([10, 20, 30, 40], np.int64)
    yhat = np.array([[9, 10, 11], [20, 25, 19], [31, 31, 31], [50, 45, 60]], np.float32)
    out = Q.metrics_q_ref(y, yhat, (0.1, 0.5, 0.9))
    assert out.shape == (13,)
    assert list(out[3::4][:3]) == [3.0, 4.0, 3.0]          # y <= yhat per level (ties count)
    assert out[12] == 2.0                                  # rows 1 and 3 cross
    assert out[0] == 1 + 0 + 1 + 10 and math.isclose(out[1], 0.1 + 0 + 1 / 30 + 10 / 40, rel_tol=1e-6)
    assert Q.metrics_q_ref(y, yhat[:, :1], (0.5,))[4] == 0.0
