"""CPU tests of the conformal calibration's refusals: every PERT_ERR_BADARG case of pert_calib_offsets /
pert_calib_apply (made with NULL or dummy device pointers, so a call that got past its checks would fault -- none may),
the workspace size, and the host errors of Calibration, Calibration.fit, calibrate and predict(calibration=...)."""
import ctypes

import pytest
import torch

from pert_gnn_kdd23_b200 import _lib

BADARG = -1
DUMMY = 1                                     # a non-NULL pointer that is never dereferenced


def _taus(*t):
    return (ctypes.c_double * max(len(t), 1))(*t)


def _fit(**kw):
    a = dict(y=DUMMY, yhat=DUMMY, group=DUMMY, n=1000, T=2, taus=_taus(0.5, 0.9), n_groups=8, min_count=1, off=DUMMY,
             count=DUMMY, own=DUMMY, ws=DUMMY, ws_bytes=1 << 40, status=DUMMY, stream=None)
    a.update(kw)
    return _lib.lib().pert_calib_offsets(a["y"], a["yhat"], a["group"], a["n"], a["T"], a["taus"], a["n_groups"],
                                         a["min_count"], a["off"], a["count"], a["own"], a["ws"], a["ws_bytes"],
                                         a["status"], a["stream"])


def test_workspace_bytes():
    lib = _lib.lib()
    a = lib.pert_calib_workspace_bytes(1000, 2, 8)
    assert a > 4 * 1000 * 2
    assert lib.pert_calib_workspace_bytes(10 ** 6, 4, 8) > lib.pert_calib_workspace_bytes(10 ** 6, 2, 8)
    assert lib.pert_calib_workspace_bytes(1000, 2, 10 ** 4) > a
    assert lib.pert_calib_workspace_bytes(1000, 2, 0) > 0
    for n, T, G in ((0, 2, 8), (-1, 2, 8), (1000, 0, 8), (1000, 9, 8), (1000, 2, -1), (1 << 28, 8, 8),
                    (1000, 2, 1 << 31)):
        assert lib.pert_calib_workspace_bytes(n, T, G) == BADARG, (n, T, G)


@pytest.mark.parametrize("field", ["y", "yhat", "off", "count", "own", "ws", "status", "taus"])
def test_offsets_refuse_null_pointers(field):
    assert _fit(**{field: None}) == BADARG


def test_offsets_refuse_bad_sizes():
    assert _fit(n=0) == BADARG and _fit(n=-5) == BADARG
    assert _fit(n=1 << 30, T=2) == BADARG                       # n T = 2^31
    for T in (0, -1, 9):
        assert _fit(T=T, taus=_taus(*[0.1 * i for i in range(9)])) == BADARG
    assert _fit(n_groups=-1) == BADARG
    assert _fit(n_groups=1 << 31) == BADARG
    assert _fit(min_count=0) == BADARG and _fit(min_count=-3) == BADARG
    need = _lib.lib().pert_calib_workspace_bytes(1000, 2, 8)
    assert _fit(ws_bytes=need - 1) == BADARG


@pytest.mark.parametrize("levels", [(0.5, 0.5), (0.9, 0.5), (-0.1, 0.5), (0.5, 1.5), (float("nan"), 0.5),
                                    (0.1, float("nan")), (0.5, float("inf"))])
def test_offsets_refuse_bad_levels(levels):
    assert _fit(taus=_taus(*levels)) == BADARG


def test_offsets_refuse_a_global_row_that_cannot_be_formed():
    assert _fit(T=1, taus=_taus(1.0)) == BADARG                 # no finite set reaches tau = 1
    assert _fit(n=98, T=1, taus=_taus(0.99)) == BADARG          # 0.99 needs 99 graphs
    assert _fit(n=18, T=2, taus=_taus(0.5, 0.95)) == BADARG


def test_apply_refusals():
    lib = _lib.lib()
    ap = lambda yhat, Q, T, off, rows: lib.pert_calib_apply(yhat, None, Q, T, off, rows, 1, None, None)  # noqa: E731
    assert ap(DUMMY, -1, 2, DUMMY, 3) == BADARG
    assert ap(None, 5, 2, DUMMY, 3) == BADARG
    for T in (0, 9, -2):
        assert ap(DUMMY, 5, T, DUMMY, 3) == BADARG
    assert ap(DUMMY, 1 << 30, 2, DUMMY, 3) == BADARG
    assert ap(DUMMY, 5, 2, DUMMY, 0) == BADARG
    assert ap(DUMMY, 5, 2, DUMMY, 1 << 31) == BADARG
    # nothing to do: no launch, no CUDA call
    assert ap(None, 0, 2, None, 0) == 0
    assert lib.pert_calib_apply(DUMMY, None, 5, 2, None, 0, 0, None, None) == 0


# ------------------------------------------------------------------------------------------------------ host side
def test_min_calibration_size():
    from pert_gnn_kdd23_b200.train import min_calibration_size

    assert min_calibration_size(0.99) == 99 and min_calibration_size(0.95) == 19
    assert min_calibration_size(0.5) == 1 and min_calibration_size(0.0) == 1
    assert min_calibration_size(1.0) is None
    for tau in (0.3, 0.9, 0.95, 0.99, 0.999):
        n = min_calibration_size(tau)
        k = lambda m: max(1, -(-(m + 1) * tau // 1))                      # noqa: E731
        assert k(n) <= n and k(n - 1) > n - 1


def _cpu_set(n=200, T=2):
    return torch.zeros(n, dtype=torch.int64), torch.zeros(n, T), torch.zeros(n, dtype=torch.int64)


def test_fit_host_errors():
    from pert_gnn_kdd23_b200.train import Calibration

    y, yhat, e = _cpu_set()
    with pytest.raises(ValueError, match="strictly increasing"):
        Calibration.fit(y, yhat, e, (0.9, 0.5), 4)
    with pytest.raises(ValueError, match="strictly increasing"):
        Calibration.fit(y, yhat, e, (0.5, 1.5), 4)
    with pytest.raises(ValueError, match="levels"):
        Calibration.fit(y, torch.zeros(200, 9), e, tuple(0.1 * i for i in range(9)), 4)
    with pytest.raises(ValueError, match="by must be"):
        Calibration.fit(y, yhat, e, (0.5, 0.9), 4, by="trace")
    with pytest.raises(ValueError, match="min_count"):
        Calibration.fit(y, yhat, e, (0.5, 0.9), 4, min_count=0)
    with pytest.raises(ValueError, match="n_groups"):
        Calibration.fit(y, yhat, e, (0.5, 0.9), -1)
    with pytest.raises(ValueError, match="predictions"):
        Calibration.fit(y, torch.zeros(200, 3), e, (0.5, 0.9), 4)
    with pytest.raises(ValueError, match="no calibration graphs"):
        Calibration.fit(y[:0], yhat[:0], e[:0], (0.5, 0.9), 4)
    with pytest.raises(ValueError, match="at least n = 99"):
        Calibration.fit(y[:50], yhat[:50], e[:50], (0.5, 0.99), 4)
    with pytest.raises(ValueError, match="level 1.0"):
        Calibration.fit(y, yhat, e, (0.5, 1.0), 4)
    with pytest.raises(ValueError, match="one entry id per graph"):
        Calibration.fit(y, yhat, e[:10], (0.5, 0.9), 4)
    with pytest.raises(_lib.PertGnnError, match="CUDA device"):
        Calibration.fit(y, yhat, e, (0.5, 0.9), 4)                  # host tensors: no CPU fallback


def test_calibration_constructor_checks():
    from pert_gnn_kdd23_b200.train import Calibration

    off, cnt, own = torch.zeros(5, 2), torch.zeros(5, dtype=torch.int32), torch.zeros(5, 2, dtype=torch.int8)
    c = Calibration((0.5, 0.9), off, cnt, own)
    assert c.levels == (0.5, 0.9) and c.n_groups == 4 and c.by == "entry" and c.min_count == 1
    with pytest.raises(ValueError):
        Calibration((0.5,), off, cnt, own)
    with pytest.raises(ValueError):
        Calibration((0.5, 0.9), off.double(), cnt, own)
    with pytest.raises(ValueError):
        Calibration((0.5, 0.9), off, cnt[:4], own)
    with pytest.raises(ValueError):
        Calibration((0.5, 0.9), off, cnt, own[:, :1])
    with pytest.raises(ValueError):
        Calibration((0.5, 0.9), off, cnt, own, by="trace")


def _model(quantiles=None):
    from pert_gnn_kdd23_b200.model import SAGEDeterministic
    from pert_gnn_kdd23_b200.synthetic import model_args

    torch.manual_seed(0)
    return SAGEDeterministic(*model_args(1), quantiles=quantiles)


def test_levels_of_a_calibration_must_match_the_model():
    """predict / eval_step / evaluate_bucketed refuse a calibration of other levels before any device work."""
    from pert_gnn_kdd23_b200.train import Calibration, _calibrated_levels, eval_step, evaluate_bucketed, predict

    T4 = (0.5, 0.9, 0.95, 0.99)
    c2 = Calibration((0.5, 0.9), torch.zeros(3, 2), torch.zeros(3, dtype=torch.int32),
                     torch.zeros(3, 2, dtype=torch.int8))
    c1 = Calibration((0.95,), torch.zeros(3, 1), torch.zeros(3, dtype=torch.int32),
                     torch.zeros(3, 1, dtype=torch.int8))
    mq, m1 = _model(T4), _model()
    with pytest.raises(ValueError):
        predict(mq, None, [0], [0], calibration=c2)
    with pytest.raises(ValueError):
        eval_step(mq, None, calibration=c2)
    with pytest.raises(ValueError):
        evaluate_bucketed(mq, [], "cpu", calibration=c2)
    with pytest.raises(ValueError):
        predict(m1, None, [0], [0], calibration=c2)                 # one output, two levels
    with pytest.raises(ValueError):
        eval_step(m1, None, tau=0.5, calibration=c1)                # evaluated at 0.5, calibrated at 0.95
    with pytest.raises(TypeError):
        predict(mq, None, [0], [0], calibration=object())
    assert _calibrated_levels(mq, None, None) == T4


def test_host_calibration_is_refused_before_any_launch():
    """A calibration whose tensors are on the host (e.g. reloaded with map_location="cpu") with the right levels is
    refused by predict, eval_step and evaluate_bucketed before any work, and the apply refuses host tensors itself."""
    from pert_gnn_kdd23_b200.train import Calibration, _calib_apply, _calibrated_levels, eval_step, evaluate_bucketed
    from pert_gnn_kdd23_b200.train import predict

    T4 = (0.5, 0.9, 0.95, 0.99)
    host = Calibration(T4, torch.zeros(3, 4), torch.zeros(3, dtype=torch.int32), torch.zeros(3, 4, dtype=torch.int8))
    one = Calibration((0.95,), torch.zeros(3, 1), torch.zeros(3, dtype=torch.int32),
                      torch.zeros(3, 1, dtype=torch.int8))
    mq, m1 = _model(T4), _model()
    was = mq.training
    for call in (lambda: predict(mq, None, [0], [0], calibration=host),
                 lambda: eval_step(mq, None, calibration=host),
                 lambda: evaluate_bucketed(mq, [], "cpu", calibration=host),
                 lambda: predict(m1, None, [0], [0], calibration=one),
                 lambda: _calibrated_levels(m1, 0.95, one)):
        with pytest.raises(_lib.PertGnnError, match="host"):
            call()
    assert mq.training == was
    with pytest.raises(_lib.PertGnnError, match="one CUDA device"):
        _calib_apply(torch.zeros(5, 4), torch.zeros(5, dtype=torch.int64), host.offsets, False)
    moved = host.to("cpu")
    assert moved.levels == T4 and moved.by == host.by and torch.equal(moved.offsets, host.offsets)
    with pytest.raises(ValueError, match="one device"):
        Calibration(T4, torch.zeros(3, 4), torch.zeros(3, dtype=torch.int32, device="meta"),
                    torch.zeros(3, 4, dtype=torch.int8))


def test_calibrate_host_errors():
    from pert_gnn_kdd23_b200.train import calibrate

    with pytest.raises(ValueError):
        calibrate(_model((0.5, 0.9)), [], "cpu", tau=0.5)           # tau differs from the model's levels
