"""CPU tests of the fp64 references and bars of tests/loss_adam_ref.py: the pinball reference agrees with autograd of
the reference loss, the float32 restatement of each kernel passes its bar, and each bar rejects the restatement carrying
a defect the GPU tests are meant to catch."""
import math

import numpy as np
import pytest
import torch

from oracle.model_oracle import torch_quantile_loss
from tests.loss_adam_ref import (U, adam_f32, adam_grad, adam_hyper, adam_state, adam_worst, f32, loss_data,
                                 metrics_bar, metrics_f64_terms, metrics_ref, metrics_terms, pinball_f32,
                                 pinball_ref, pinball_worst)


@pytest.mark.parametrize("tau", [0.0, 0.05, 0.5, 0.95, 1.0])
@pytest.mark.parametrize("B", [1, 7, 300])
def test_pinball_ref_matches_autograd(B, tau):
    y, yhat = loss_data(B, seed=B)
    yt = torch.tensor(y.astype(np.float32).astype(np.float64))
    yh = torch.tensor(yhat.astype(np.float64), requires_grad=True)
    loss = torch_quantile_loss(yt, yh, f32(tau))
    loss.backward()
    ref_loss, ref_d = pinball_ref(y, yhat, tau)
    assert abs(float(loss) - ref_loss) <= 1e-14 * abs(ref_loss)
    np.testing.assert_allclose(ref_d, yh.grad.numpy(), rtol=1e-15, atol=0)
    if B >= 3:   # loss_data makes the first two graphs ties
        assert ref_d[0] == 0.5 * (1 - 2 * f32(tau)) / B


def test_pinball_ref_live_and_ghosts():
    y, yhat = loss_data(64, seed=1)
    yhat[40:] = np.nan
    loss, d = pinball_ref(y, yhat, 0.95, grad_scale=0.125, live=40)
    full, dfull = pinball_ref(y[:40], yhat[:40], 0.95, grad_scale=0.125)
    assert loss == full and np.array_equal(d[:40], dfull) and not d[40:].any()
    assert np.isnan(pinball_ref(y, yhat, 0.95, live=1000)[0])   # live above B is clamped to B: the NaNs are in


@pytest.mark.parametrize("B", [1, 255, 257, 4096, 65537])
@pytest.mark.parametrize("tau", [0.0, 0.05, 0.95, 1.0])
def test_pinball_bars_pass_f32_restatement(B, tau):
    y, yhat = loss_data(B, seed=B + 7)
    for gs in (1.0, 0.125):
        for live in (None, max(1, B // 2)):
            rl, rd = pinball_worst(*pinball_f32(y, yhat, tau, gs, live), *pinball_ref(y, yhat, tau, gs, live),
                                   B if live is None else live)
            assert rl <= 1 and rd <= 1, (gs, live, rl, rd)


@pytest.mark.parametrize("defect", ["capacity", "tie0", "tie_neg_tau"])
def test_pinball_bars_reject_defects(defect):
    B, live, tau = 4096, 3000, 0.95
    y, yhat = loss_data(B, seed=3)
    rl, rd = pinball_worst(*pinball_f32(y, yhat, tau, 0.125, live, defect), *pinball_ref(y, yhat, tau, 0.125, live),
                           live)
    assert max(rl, rd) > 1e3, (defect, rl, rd)


def test_metrics_terms_are_float32_and_bar():
    B = 20000
    y, yhat = loss_data(B, seed=5)
    assert (y > 2 ** 24).any() and (y.astype(np.float32).astype(np.int64) != y).any()
    terms = metrics_terms(y, yhat, 0.95)
    assert all(t.dtype == np.float32 for t in terms)
    ref = metrics_ref(y, yhat, 0.95)
    # the correct terms summed in another order (numpy's pairwise double sum) pass the bar
    for t, r in zip(terms, ref):
        assert abs(float(np.sum(t.astype(np.float64))) - r) <= metrics_bar(B) * r
    # terms built in double on the exact int64 y (no float32 promotion) fail it: y > 2^24 is not a float32
    for t, r in zip(metrics_f64_terms(y, yhat, 0.95), ref):
        assert abs(math.fsum(t.tolist()) - r) > 10 * metrics_bar(B) * r


BETAS = [(0.9, 0.999), (0.5, 0.9)]


def _adam_run(n, hp, steps, seed):
    """(state before the last step, its step count) after running the float32 restatement through ``steps``."""
    rng = np.random.default_rng(seed)
    p, g = adam_state(n, seed)
    m = np.zeros(n, np.float32)
    v = np.zeros(n, np.float32)
    for t in steps[:-1]:
        p, m, v = adam_f32(p, g, m, v, t, hp)
        g = adam_grad(n, rng)
    return p, g, m, v, steps[-1]


@pytest.mark.parametrize("betas", BETAS)
@pytest.mark.parametrize("wd,gs", [(0.0, 1.0), (1e-2, 0.125)])
def test_adam_bars_pass_f32_restatement(betas, wd, gs):
    hp = adam_hyper(lr=1e-3, betas=betas, weight_decay=wd, grad_scale=gs)
    seq = [1, 2, 3, 10, 100, 10 ** 4, 2 ** 24 + 1]
    for k in range(1, len(seq) + 1):
        p, g, m, v, t = _adam_run(4096, hp, seq[:k], seed=k)
        w = adam_worst(p, g, m, v, t, hp, adam_f32(p, g, m, v, t, hp))
        assert max(w) <= 1, (t, w)


@pytest.mark.parametrize("defect,t", [("bc_off_by_one", 2), ("bc_off_by_one", 10), ("adamw", 3),
                                      ("eps_in_sqrt", 2), ("fp32_bc", 2)])
def test_adam_bars_reject_defects(defect, t):
    hp = adam_hyper(lr=1e-3, betas=(0.9, 0.999), weight_decay=1e-2 if defect == "adamw" else 0.0, grad_scale=0.125)
    p, g, m, v, t = _adam_run(1 << 16, hp, list(range(1, t + 1)), seed=11)
    w = adam_worst(p, g, m, v, t, hp, adam_f32(p, g, m, v, t, hp, defect))
    assert w[2] > 1, (defect, t, w)
    assert max(adam_worst(p, g, m, v, t, hp, adam_f32(p, g, m, v, t, hp))) <= 1


def test_fp32_bias_correction_error_at_small_steps():
    """What the float32 corrections cost: 1 - 0.999f^t formed in float32 is off by a few 1e-6 relative at t = 2 and 5,
    about 50 u, while the correction from double rounds once (u)."""
    b2 = np.float32(0.999)
    for t in (2, 5):
        exact = 1.0 - float(b2) ** t
        bc32 = float(np.float32(1) - b2 ** np.float32(t))
        assert abs(bc32 - exact) / exact > 20 * U
        assert abs(float(np.float32(exact)) - exact) / exact <= U


@pytest.mark.parametrize("B", [2 ** 31, 2 ** 32 + 5])
def test_loss_and_metrics_reject_batches_above_int_max(B):
    """The kernels index graphs with 32-bit counts; a larger B is refused before any launch (dummy non-NULL pointers,
    never read)."""
    from pert_gnn_kdd23_b200 import _lib

    L = _lib.lib()
    assert L.pert_pinball_loss(1, 1, 0.5, B, 1.0, 1, 1, None) == -1
    assert L.pert_pinball_loss_live(1, 1, 0.5, B, 1.0, 1, 1, 1, None) == -1
    assert L.pert_eval_metrics(1, 1, 0.5, B, 1, None) == -1
    assert L.pert_eval_metrics_live(1, 1, 0.5, B, 1, 1, None) == -1
