"""CPU tests of the conformal predictive distribution's refusals: every PERT_ERR_BADARG case of pert_cpd_fit /
pert_cpd_tail / pert_cpd_quantile (made with NULL or dummy device pointers, so a call that got past its checks would
fault -- none may), the workspace size, and the host errors of ScoreDistribution, its fit and queries,
fit_distribution and score_traces, host tensors included."""
import ctypes

import pytest
import torch

from pert_gnn_kdd23_b200 import _lib

BADARG = -1
DUMMY = 1                                     # a non-NULL pointer that is never dereferenced


def _taus(*t):
    return (ctypes.c_double * max(len(t), 1))(*t)


def _fit(**kw):
    a = dict(y=DUMMY, yhat=DUMMY, ld=2, col=1, group=DUMMY, n=1000, G=8, scores=DUMMY, ptr=DUMMY, ws=DUMMY,
             ws_bytes=1 << 40, status=DUMMY, stream=None)
    a.update(kw)
    return _lib.lib().pert_cpd_fit(a["y"], a["yhat"], a["ld"], a["col"], a["group"], a["n"], a["G"], a["scores"],
                                   a["ptr"], a["ws"], a["ws_bytes"], a["status"], a["stream"])


def _tail(**kw):
    a = dict(scores=DUMMY, ptr=DUMMY, G=8, min_count=1, yhat=DUMMY, ld=1, col=0, group=DUMMY, Q=100, x=DUMMY, S=2,
             y=None, ge=DUMMY, gt=DUMMY, row=DUMMY, status=DUMMY, stream=None)
    a.update(kw)
    return _lib.lib().pert_cpd_tail(a["scores"], a["ptr"], a["G"], a["min_count"], a["yhat"], a["ld"], a["col"],
                                    a["group"], a["Q"], a["x"], a["S"], a["y"], a["ge"], a["gt"], a["row"],
                                    a["status"], a["stream"])


def _quantile(**kw):
    a = dict(scores=DUMMY, ptr=DUMMY, G=8, min_count=1, yhat=DUMMY, ld=1, col=0, group=DUMMY, Q=100,
             taus=_taus(0.5, 0.99), L=2, out=DUMMY, status=DUMMY, stream=None)
    a.update(kw)
    return _lib.lib().pert_cpd_quantile(a["scores"], a["ptr"], a["G"], a["min_count"], a["yhat"], a["ld"], a["col"],
                                        a["group"], a["Q"], a["taus"], a["L"], a["out"], a["status"], a["stream"])


def test_workspace_bytes():
    lib = _lib.lib()
    a = lib.pert_cpd_workspace_bytes(1000, 8)
    assert a > 2 * 4 * 2 * 1000                                     # two ping-pong buffers of 2n keys
    assert lib.pert_cpd_workspace_bytes(10 ** 6, 8) > a
    assert lib.pert_cpd_workspace_bytes(1000, 10 ** 4) > a
    assert lib.pert_cpd_workspace_bytes(1, 0) > 0
    for n, G in ((0, 8), (-1, 8), (1 << 30, 8), (1000, -1), (1000, 2 ** 31 - 2)):
        assert lib.pert_cpd_workspace_bytes(n, G) == BADARG, (n, G)
    assert lib.pert_cpd_workspace_bytes((1 << 30) - 1, 0) > 0


@pytest.mark.parametrize("field", ["y", "yhat", "scores", "ptr", "ws", "status"])
def test_fit_refuses_null_pointers(field):
    assert _fit(**{field: None}) == BADARG


def test_fit_refuses_bad_sizes():
    assert _fit(n=0) == BADARG and _fit(n=-5) == BADARG
    assert _fit(n=1 << 30) == BADARG                                # n >= 2^31 / 2
    assert _fit(G=-1) == BADARG and _fit(G=2 ** 31 - 2) == BADARG
    assert _fit(ld=0) == BADARG and _fit(col=-1) == BADARG and _fit(col=2) == BADARG
    need = _lib.lib().pert_cpd_workspace_bytes(1000, 8)
    assert _fit(ws_bytes=need - 1) == BADARG


def test_tail_refusals():
    for field in ("scores", "ptr", "yhat", "status", "ge", "gt", "row"):
        assert _tail(**{field: None}) == BADARG, field
    assert _tail(Q=-1) == BADARG
    assert _tail(S=0) == BADARG
    assert _tail(Q=1 << 30, S=2) == BADARG                          # Q S = 2^31
    assert _tail(G=-1) == BADARG and _tail(G=2 ** 31 - 2) == BADARG
    assert _tail(min_count=0) == BADARG
    assert _tail(ld=0) == BADARG and _tail(col=1) == BADARG and _tail(col=-1) == BADARG
    assert _tail(x=None, y=None) == BADARG                          # neither thresholds nor labels
    assert _tail(x=DUMMY, y=DUMMY, S=1) == BADARG                   # both
    assert _tail(x=None, y=DUMMY, S=2) == BADARG                    # labels are one per request
    assert _tail(Q=0, scores=None, ptr=None, yhat=None, ge=None, gt=None, row=None, status=None) == 0  # nothing to do


def test_quantile_refusals():
    for field in ("scores", "ptr", "yhat", "status", "out", "taus"):
        assert _quantile(**{field: None}) == BADARG, field
    for L in (0, 9, -1):
        assert _quantile(L=L, taus=_taus(*[0.1 * i for i in range(9)])) == BADARG
    for lv in ((0.5, 0.5), (0.9, 0.5), (-0.1, 0.5), (0.5, 1.5), (float("nan"), 0.5), (0.5, float("inf"))):
        assert _quantile(taus=_taus(*lv)) == BADARG, lv
    assert _quantile(Q=-1) == BADARG and _quantile(Q=1 << 30) == BADARG
    assert _quantile(min_count=0) == BADARG and _quantile(G=-1) == BADARG
    assert _quantile(ld=3, col=3) == BADARG
    assert _quantile(Q=0, out=None) == 0


# ------------------------------------------------------------------------------------------------------ host side
def _dist(device="cpu"):
    from pert_gnn_kdd23_b200.train import ScoreDistribution

    return ScoreDistribution(0.5, torch.zeros(20, device=device), torch.tensor([0, 5, 10, 10, 20], device=device))


def test_constructor_checks():
    from pert_gnn_kdd23_b200.train import ScoreDistribution

    d = _dist()
    assert d.n_groups == 3 and d.level == 0.5 and d.by == "entry" and d.min_count == 1 and d.column == 0
    assert d.counts.tolist() == [5, 5, 0, 10] and d.device == torch.device("cpu")
    s, p = torch.zeros(20), torch.tensor([0, 5, 10, 10, 20])
    for kw in (dict(level=1.5), dict(by="trace"), dict(min_count=0), dict(column=-1)):
        a = dict(level=0.5, by="entry", min_count=1, column=0)
        a.update(kw)
        with pytest.raises(ValueError):
            ScoreDistribution(a["level"], s, p, a["by"], a["min_count"], a["column"])
    with pytest.raises(ValueError):
        ScoreDistribution(0.5, s.double(), p)
    with pytest.raises(ValueError):
        ScoreDistribution(0.5, s, p.int())
    with pytest.raises(ValueError):
        ScoreDistribution(0.5, s, p[:1])
    with pytest.raises(ValueError, match="one device"):
        ScoreDistribution(0.5, s, p.to("meta"))
    moved = d.to("cpu")
    assert torch.equal(moved.scores, d.scores) and torch.equal(moved.ptr, d.ptr) and moved.level == d.level


def test_fit_host_errors():
    from pert_gnn_kdd23_b200.train import ScoreDistribution

    y, yhat, e = torch.zeros(200, dtype=torch.int64), torch.zeros(200, 3), torch.zeros(200, dtype=torch.int64)
    fit = ScoreDistribution.fit
    with pytest.raises(ValueError, match="level"):
        fit(y, yhat, e, 4, 1.5, column=0)
    with pytest.raises(ValueError, match="by must be"):
        fit(y, yhat, e, 4, 0.5, by="trace", column=0)
    with pytest.raises(ValueError, match="min_count"):
        fit(y, yhat, e, 4, 0.5, min_count=0, column=0)
    with pytest.raises(ValueError, match="n_groups"):
        fit(y, yhat, e, -1, 0.5, column=0)
    with pytest.raises(ValueError, match="no held-out graphs"):
        fit(y[:0], yhat[:0], e[:0], 4, 0.5, column=0)
    with pytest.raises(ValueError, match="predictions"):
        fit(y, yhat[:10], e, 4, 0.5, column=0)
    with pytest.raises(ValueError, match="column="):
        fit(y, yhat, e, 4, 0.5)                                     # three columns, none named
    with pytest.raises(ValueError, match="column 3"):
        fit(y, yhat, e, 4, 0.5, column=3)
    with pytest.raises(ValueError, match="one entry id per graph"):
        fit(y, yhat, e[:10], 4, 0.5, column=0)
    with pytest.raises(_lib.PertGnnError, match="CUDA device"):
        fit(y, yhat, e, 4, 0.5, column=1)                           # host tensors: no CPU fallback
    with pytest.raises(_lib.PertGnnError, match="CUDA device"):
        fit(y, yhat[:, 0], None, 0, 0.5, by="global")


def test_queries_refuse_host_tensors_before_any_launch():
    d = _dist()
    yh, ent = torch.zeros(7), torch.zeros(7, dtype=torch.int64)
    for call in (lambda: d.tail(yh, ent, 100.0), lambda: d.pvalues(yh, ent, ent),
                 lambda: d.quantile(yh, ent, (0.5, 0.9))):
        with pytest.raises(_lib.PertGnnError, match="host"):
            call()
    with pytest.raises(ValueError, match="strictly increasing"):
        d.quantile(yh, ent, (0.9, 0.5))
    with pytest.raises(ValueError, match="levels"):
        d.quantile(yh, ent, tuple(0.1 * i for i in range(9)))


def _model(quantiles=None):
    from pert_gnn_kdd23_b200.model import SAGEDeterministic
    from pert_gnn_kdd23_b200.synthetic import model_args

    torch.manual_seed(0)
    return SAGEDeterministic(*model_args(1), quantiles=quantiles)


def test_fit_distribution_levels():
    from pert_gnn_kdd23_b200.train import _base_level, fit_distribution

    T4 = (0.5, 0.9, 0.95, 0.99)
    mq, m1 = _model(T4), _model()
    with pytest.raises(ValueError, match="level="):
        fit_distribution(mq, [], "cpu")                             # four levels, none named
    with pytest.raises(ValueError, match="level="):
        fit_distribution(mq, [], "cpu", level=0.8)
    assert _base_level(mq, 0.95) == (0.95, 2) and _base_level(mq, 0.5) == (0.5, 0)
    assert _base_level(m1, None) == (0.5, 0) and _base_level(m1, 0.95) == (0.95, 0)
    with pytest.raises(ValueError, match="differs"):
        _base_level(_model((0.9,)), 0.5)
    assert _base_level(_model((0.9,)), None) == (0.9, 0)


def test_score_traces_refusals():
    from pert_gnn_kdd23_b200.train import score_traces

    with pytest.raises(TypeError):
        score_traces(_model(), [], "cpu", object())
    with pytest.raises(_lib.PertGnnError, match="move it"):
        score_traces(_model(), [], "cpu", _dist())                  # a distribution on the host
