"""The pinball loss (``pert_pinball_loss`` / ``_live``), the eval metrics (``pert_eval_metrics`` / ``_live``), the Adam
step (``pert_adam_step``) and both forms of the fused data-parallel Adam (``pert_allreduce_adam`` at world = 1) against
the fp64 references of tests/loss_adam_ref.py, whose docstrings derive every bar.

Covered edges: the pinball kernel's single 256-thread block and its strided loop (B up to 10^6), tau at 0 and 1, exact
ties, grad_scale != 1, NULL outputs, padded batches with NaN / inf in the ghost slots and live counts below and above
the capacity; the metric kernel's 64-block cap (B > 16384) and accumulation across calls; Adam's scalar sizes, block
edges and a 3M-float buffer, weight decay, grad_scale, two beta pairs, gradients from 1e-12 to 1e3 and step counts up to
2^24 + 1.  The module prints the largest error of each quantity as a fraction of its bar."""
import math
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from pert_gnn_kdd23_b200 import _lib
from tests.loss_adam_ref import (adam_f32, adam_grad, adam_hyper, adam_state, adam_worst, f32, loss_data,
                                 metrics_bar, metrics_terms, pinball_ref, pinball_worst)

pytestmark = pytest.mark.gpu

WORST = {}


def _note(name, r):
    WORST[name] = max(WORST.get(name, 0.0), float(r))


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nworst error / bar: " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(WORST.items())))


def _L():
    return _lib.lib()


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _pinball(y, yhat, tau, gs, *, loss=True, dyhat=True, live=None, plain=False):
    """One call on device copies; outputs pre-filled with NaN so that every unwritten slot shows."""
    B = y.numel()
    lo = torch.full((1,), float("nan"), device="cuda") if loss else None
    d = torch.full((B,), float("nan"), device="cuda") if dyhat else None
    p = _lib.ptr
    if plain:
        rc = _L().pert_pinball_loss(p(y), p(yhat), f32(tau), B, f32(gs), p(lo), p(d), _lib.stream())
    else:
        rc = _L().pert_pinball_loss_live(p(y), p(yhat), f32(tau), B, f32(gs), p(lo), p(d), p(live), _lib.stream())
    assert rc == 0
    torch.cuda.synchronize()
    return (float(lo.item()) if loss else None), (d.cpu().numpy() if dyhat else None)


TAUS = [0.0, 0.05, 0.5, 0.95, 1.0]


@pytest.mark.parametrize("B", [1, 31, 32, 33, 255, 256, 257, 4096, 65537, 10 ** 6])
def test_pinball_matches_fp64(B):
    y, yhat = loss_data(B, seed=B)
    yd, yhd = _dev(y), _dev(yhat)
    for tau in TAUS:
        for gs in (1.0, 0.125):
            loss, d = _pinball(yd, yhd, tau, gs, plain=True)
            rl, rd = pinball_worst(loss, d, *pinball_ref(y, yhat, tau, gs), B)
            _note("pinball_loss", rl)
            _note("pinball_dyhat", rd)
            assert rl <= 1 and rd <= 1, (tau, gs, loss, rl, rd)


def test_pinball_null_outputs_and_null_live():
    B = 4097
    y, yhat = loss_data(B, seed=9)
    yd, yhd = _dev(y), _dev(yhat)
    for tau in (0.05, 0.95):
        loss, d = _pinball(yd, yhd, tau, 0.125, plain=True)
        assert np.float32(_pinball(yd, yhd, tau, 0.125, dyhat=False, plain=True)[0]).tobytes() == \
            np.float32(loss).tobytes()
        assert np.array_equal(_pinball(yd, yhd, tau, 0.125, loss=False, plain=True)[1].view(np.int32),
                              d.view(np.int32))
        l2, d2 = _pinball(yd, yhd, tau, 0.125, live=None)          # _live with live = NULL is the plain call
        assert np.float32(l2).tobytes() == np.float32(loss).tobytes()
        assert np.array_equal(d2.view(np.int32), d.view(np.int32))


@pytest.mark.parametrize("live", [1, 255, 3000, 4095, 5000])
def test_pinball_live_ghosts(live):
    """A padded batch: ghost slots (y = 1, yhat = NaN / +inf / -inf) must not reach the loss and get dyhat = 0; a live
    count above the capacity is clamped to it."""
    B = 4096
    y, yhat = loss_data(B, seed=live)
    bl = min(B, live)
    y[bl:] = 1
    yhat[bl:] = np.resize(np.array([np.nan, np.inf, -np.inf], np.float32), B - bl)
    yd, yhd = _dev(y), _dev(yhat)
    word = torch.tensor([12345, live], dtype=torch.int64, device="cuda")
    for tau in (0.0, 0.5, 0.95, 1.0):
        for gs in (1.0, 0.125):
            loss, d = _pinball(yd, yhd, tau, gs, live=word)
            assert math.isfinite(loss) and not d[bl:].any() and np.isfinite(d).all()
            rl, rd = pinball_worst(loss, d, *pinball_ref(y, yhat, tau, gs, live=live), bl)
            _note("pinball_loss", rl)
            _note("pinball_dyhat", rd)
            assert rl <= 1 and rd <= 1, (tau, gs, rl, rd)
            if live >= B:
                lp, dp = _pinball(yd, yhd, tau, gs, plain=True)
                assert np.float32(lp).tobytes() == np.float32(loss).tobytes() and np.array_equal(dp, d)


def _ratio(got, ref, rel_bar):
    """|got - ref| as a fraction of rel_bar * ref; a zero reference must come out exactly 0."""
    if ref == 0:
        return 0.0 if got == 0 else math.inf
    return abs(got - ref) / (rel_bar * ref)


def _metrics(y, yhat, tau, acc, live=None):
    rc = _L().pert_eval_metrics_live(_lib.ptr(y), _lib.ptr(yhat), f32(tau), y.numel(), _lib.ptr(acc), _lib.ptr(live),
                                     _lib.stream())
    assert rc == 0


@pytest.mark.parametrize("B", [1, 255, 256, 257, 16383, 16384, 16385, 10 ** 6])
def test_eval_metrics_accumulate_matches_fp64(B):
    """Three calls accumulate into one acc (the last through the plain entry); each sum against the exactly rounded sum
    of every float32 term so far."""
    acc = torch.zeros(3, dtype=torch.float64, device="cuda")
    terms = [[], [], []]
    for k in range(3):
        y, yhat = loss_data(B, seed=100 * B + k)
        if k < 2:
            _metrics(_dev(y), _dev(yhat), 0.95, acc)
        else:
            assert _L().pert_eval_metrics(_lib.ptr(_dev(y)), _lib.ptr(_dev(yhat)), f32(0.95), B, _lib.ptr(acc),
                                          _lib.stream()) == 0
        for lst, t in zip(terms, metrics_terms(y, yhat, 0.95)):
            lst.append(t.astype(np.float64))
        got = acc.cpu().tolist()
        for name, g, lst in zip(("mae", "mape", "qloss"), got, terms):
            ref = math.fsum(np.concatenate(lst).tolist())
            r = _ratio(g, ref, metrics_bar((k + 1) * B))
            _note("metrics_" + name, r)
            assert r <= 1, (name, k, g, ref, r)


def test_eval_metrics_empty_and_live_ghosts():
    acc = torch.tensor([1.5, -2.25, 3.0], dtype=torch.float64, device="cuda")
    # B = 0 returns before any launch, so dummy y / yhat / live pointers are never read
    assert _L().pert_eval_metrics(1, 1, f32(0.5), 0, _lib.ptr(acc), _lib.stream()) == 0
    assert _L().pert_eval_metrics_live(1, 1, f32(0.5), 0, _lib.ptr(acc), 1, _lib.stream()) == 0
    assert acc.cpu().tolist() == [1.5, -2.25, 3.0]
    B = 20000
    for live in (12345, 16385, 30000):
        y, yhat = loss_data(B, seed=live)
        bl = min(B, live)
        y[bl:] = 1
        yhat[bl:] = np.nan
        acc.zero_()
        _metrics(_dev(y), _dev(yhat), 0.05, acc, torch.tensor([7, live], dtype=torch.int64, device="cuda"))
        got = acc.cpu().tolist()
        for name, g, t in zip(("mae", "mape", "qloss"), got, metrics_terms(y[:bl], yhat[:bl], 0.05)):
            ref = math.fsum(t.astype(np.float64).tolist())
            r = _ratio(g, ref, metrics_bar(bl))
            _note("metrics_" + name, r)
            assert r <= 1, (live, name, g, ref)


STEPS = [1, 2, 3, 10, 100, 10 ** 4, 2 ** 24 + 1]
CONFIGS = [(wd, gs, betas) for wd in (0.0, 1e-2) for gs in (1.0, 0.125) for betas in ((0.9, 0.999), (0.5, 0.9))]


def _adam_step(p, g, m, v, t, hp):
    rc = _L().pert_adam_step(_lib.ptr(p), _lib.ptr(g), _lib.ptr(m), _lib.ptr(v), p.numel(), hp["lr"], hp["b1"],
                             hp["b2"], hp["eps"], hp["wd"], t, hp["gs"], _lib.stream())
    assert rc == 0


@pytest.mark.parametrize("n", [1, 3, 4, 255, 256, 257, 3_000_001])
def test_adam_step_matches_fp64(n):
    """Each step is checked from the kernel's own float32 state before it, at step counts 1, 2, 3, 10, 100, 10^4 and
    2^24 + 1 (which float32 cannot represent)."""
    configs = CONFIGS if n < 10 ** 6 else [CONFIGS[0], CONFIGS[-1]]
    for c, (wd, gs, betas) in enumerate(configs):
        hp = adam_hyper(lr=1e-3, betas=betas, weight_decay=wd, grad_scale=gs)
        rng = np.random.default_rng(1000 * n + c)
        p, g = adam_state(n, seed=n + c)
        pd, md, vd = _dev(p), torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
        for t in STEPS:
            before = [x.cpu().numpy() for x in (pd, md, vd)]
            _adam_step(pd, _dev(g), md, vd, t, hp)
            out = [x.cpu().numpy() for x in (pd, md, vd)]
            wm, wv, wdl = adam_worst(before[0], g, before[1], before[2], t, hp, out)
            _note("adam_m", wm)
            _note("adam_v", wv)
            _note("adam_delta", wdl)
            if t == 2:
                _note("adam_delta_t2", wdl)
            assert max(wm, wv, wdl) <= 1, (wd, gs, betas, t, wm, wv, wdl)
            g = adam_grad(n, rng)


def test_adam_bias_correction_is_double():
    """At t = 2 the kernel's update sits within the fp64 bar, which the float32 corrections (1 - powf(beta, t)) miss:
    the same state run through the float32 restatement with either correction brackets the kernel."""
    n = 1 << 18
    hp = adam_hyper(lr=1e-3, betas=(0.9, 0.999), grad_scale=0.125)
    p, g = adam_state(n, seed=2)
    pd, md, vd = _dev(p), torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
    _adam_step(pd, _dev(g), md, vd, 1, hp)
    g2 = adam_grad(n, np.random.default_rng(3))
    before = [x.cpu().numpy() for x in (pd, md, vd)]
    _adam_step(pd, _dev(g2), md, vd, 2, hp)
    out = [x.cpu().numpy() for x in (pd, md, vd)]
    ref_p = before[0].astype(np.float64)
    from tests.loss_adam_ref import adam_ref

    delta_ref = adam_ref(before[0], g2, before[1], before[2], 2, hp)[0] - ref_p
    nz = np.abs(delta_ref) > 1e-6
    rel = np.abs((out[0].astype(np.float64) - ref_p) - delta_ref)[nz] / np.abs(delta_ref[nz])
    _note("adam_t2_update_rel_err", rel.max())     # a relative error, not a fraction of a bar
    assert adam_worst(before[0], g2, before[1], before[2], 2, hp, out)[2] <= 1
    assert adam_worst(before[0], g2, before[1], before[2], 2, hp,
                      adam_f32(before[0], g2, before[1], before[2], 2, hp, "fp32_bc"))[2] > 1


def test_fused_adam_trajectory_matches_torch_adam_fp64():
    """30 FusedAdam steps with weight decay and grad_scale on a small model's FlatParams against torch.optim.Adam on
    float64 copies fed the same float32 gradients: checks the argument order and the step counter.  Bar: each step adds
    at most an ulp of p (2u |p|) and the per-step state drift grows by at most 16u of that step's update, so after T
    steps T (2u |p| + 16u sum_t |delta_t|)."""
    from pert_gnn_kdd23_b200.train import FlatParams, FusedAdam
    from tests.loss_adam_ref import U

    torch.manual_seed(0)
    lin_c = torch.nn.Sequential(torch.nn.Linear(37, 19), torch.nn.Linear(19, 3)).cuda()
    lin_o = torch.nn.Sequential(torch.nn.Linear(37, 19), torch.nn.Linear(19, 3)).double()
    lin_o.load_state_dict({k: v.double().cpu() for k, v in lin_c.state_dict().items()})
    fp = FlatParams(lin_c)
    opt_c = FusedAdam(fp, lr=1e-3, weight_decay=1e-2)
    opt_o = torch.optim.Adam(lin_o.parameters(), lr=f32(1e-3), betas=(f32(0.9), f32(0.999)), eps=f32(1e-8),
                             weight_decay=f32(1e-2))
    T = 30
    sum_delta = [torch.zeros_like(q) for q in lin_o.parameters()]
    for _ in range(T):
        before = [q.detach().clone() for q in lin_o.parameters()]
        for pc, po in zip(lin_c.parameters(), lin_o.parameters()):
            g = 0.01 * torch.randn(po.shape)
            pc.grad.copy_(g.cuda())
            po.grad = g.double() * 0.125
        opt_o.step()
        opt_c.step(grad_scale=0.125)
        for s, q, b in zip(sum_delta, lin_o.parameters(), before):
            s += (q.detach() - b).abs()
    assert opt_c.t == T
    for pc, po, s in zip(lin_c.parameters(), lin_o.parameters(), sum_delta):
        err = (pc.detach().double().cpu() - po.detach()).abs()
        bar = T * (2 * U * po.detach().abs() + 16 * U * s)
        r = float((err / bar).max())
        _note("fused_adam_trajectory", r)
        assert r <= 1, r


@pytest.mark.parametrize("mode", ["ag", "rs"])
def test_allreduce_adam_world1(mode):
    """Both forms of pert_allreduce_adam at world = 1 (the form is read from PERT_PEER_MODE once per process, so each
    runs in its own process: tests/peer_adam_world1.py): bit-identical to pert_adam_step and within the fp64 bar."""
    here = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, PERT_PEER_MODE=mode)
    r = subprocess.run([sys.executable, os.path.join(here, "peer_adam_world1.py")], capture_output=True, text=True,
                       timeout=600, env=env)
    assert "PEER_WORLD1_OK" in r.stdout, (mode, r.stdout[-3000:], r.stderr[-3000:])
    for k, v in re.findall(r"(\w+)=([0-9.e+-]+)", r.stdout.split("PEER_WORLD1_OK", 1)[1]):
        if k.startswith("worst_"):
            _note(f"peer_{mode}_{k[6:]}", float(v))
