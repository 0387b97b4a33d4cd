"""CPU tests of the score window's refusals: every PERT_ERR_BADARG case of pert_cpd_merge (NULL or dummy device
pointers, so a call that got past its checks would fault -- none may), its workspace size, and the host errors of
ScoreDistribution's log, insert, evict and add_traces.  After each refused update the distribution is unchanged."""
import pytest
import torch

from pert_gnn_kdd23_b200 import _lib

BADARG = -1
DUMMY = 1                                     # a non-NULL pointer that is never dereferenced


def _merge(**kw):
    a = dict(scores=DUMMY, ptr=DUMMY, G_old=8, n_old=2000, d_scores=DUMMY, d_ptr=DUMMY, G_new=8, n_delta=200, sign=1,
             out=DUMMY, out_ptr=DUMMY, ws=DUMMY, ws_bytes=1 << 40, status=DUMMY, stream=None)
    a.update(kw)
    return _lib.lib().pert_cpd_merge(a["scores"], a["ptr"], a["G_old"], a["n_old"], a["d_scores"], a["d_ptr"],
                                     a["G_new"], a["n_delta"], a["sign"], a["out"], a["out_ptr"], a["ws"],
                                     a["ws_bytes"], a["status"], a["stream"])


def test_workspace_bytes():
    lib = _lib.lib()
    a = lib.pert_cpd_merge_workspace_bytes(8, 8, 2000, 200)
    assert a > 0
    assert lib.pert_cpd_merge_workspace_bytes(8, 10 ** 5, 2000, 200) > a          # grows with the rows
    assert lib.pert_cpd_merge_workspace_bytes(0, 0, 1, 1) > 0
    assert lib.pert_cpd_merge_workspace_bytes(8, 8, 2 ** 31 - 2, 1) > 0            # a removal may start at the bound
    for args in ((-1, 8, 2000, 200), (8, 7, 2000, 200), (8, 2 ** 31 - 2, 2000, 200), (8, 8, 0, 200),
                 (8, 8, 2000, 0), (8, 8, 2000, -1), (8, 8, 2 ** 31, 1), (8, 8, 2 ** 30, 2 ** 30 + 5)):
        assert lib.pert_cpd_merge_workspace_bytes(*args) == BADARG, args


@pytest.mark.parametrize("field", ["scores", "ptr", "d_scores", "d_ptr", "out", "out_ptr", "ws", "status"])
def test_merge_refuses_null_pointers(field):
    assert _merge(**{field: None}) == BADARG


def test_merge_refuses_bad_sizes():
    assert _merge(G_new=7) == BADARG                                  # G shrinks
    assert _merge(G_old=-1) == BADARG and _merge(G_new=2 ** 31 - 2, G_old=8) == BADARG
    for sign in (0, 2, -2):
        assert _merge(sign=sign) == BADARG, sign
    assert _merge(n_old=0) == BADARG and _merge(n_delta=0) == BADARG and _merge(n_delta=-3) == BADARG
    assert _merge(n_old=2 ** 30, n_delta=2 ** 30) == BADARG           # the result reaches 2^31 scores (n = 2^30)
    assert _merge(sign=-1, n_delta=2000) == BADARG                    # a removal that leaves nothing
    assert _merge(sign=-1, n_delta=2001) == BADARG
    need = _lib.lib().pert_cpd_merge_workspace_bytes(8, 8, 2000, 200)
    assert _merge(ws_bytes=need - 1) == BADARG


# ------------------------------------------------------------------------------------------------------ host side
def _logged(device="cpu", n=10, G=3):
    from pert_gnn_kdd23_b200.train import ScoreDistribution

    log = (torch.arange(n, dtype=torch.int64), torch.zeros(n), torch.arange(n, dtype=torch.int64) % G,
           torch.arange(n, dtype=torch.int64))
    return ScoreDistribution(0.5, torch.zeros(2 * n, device=device), torch.zeros(G + 2, dtype=torch.int64),
                             log=tuple(t.to(device) for t in log))


def _state(d):
    return (d.scores, d.ptr, d.log, d.n_groups)


def _unchanged(d, s):
    a = _state(d)
    assert a[0] is s[0] and a[1] is s[1] and a[3] == s[3]
    assert (a[2] is None) == (s[2] is None) and (a[2] is None or all(x is y for x, y in zip(a[2], s[2])))


def test_constructor_log_checks():
    from pert_gnn_kdd23_b200.train import ScoreDistribution

    d = _logged()
    assert d.log_y.tolist() == list(range(10)) and d.log_ts.dtype == torch.int64 and d.log_yhat.dtype == torch.float32
    assert _logged().to("cpu").log_entry.tolist() == d.log_entry.tolist()
    s, p = torch.zeros(20), torch.zeros(5, dtype=torch.int64)
    y, yh, e, t = d.log
    for bad in ((y, yh, e), (y.int(), yh, e, t), (y, yh.double(), e, t), (y, yh, e, t[:9]), (y, yh, e, t.float()),
                (y[:5], yh[:5], e[:5], t[:5]), [y, yh, e, None]):
        with pytest.raises(ValueError):
            ScoreDistribution(0.5, s, p, log=bad)
    with pytest.raises(ValueError, match="device"):
        ScoreDistribution(0.5, s, p, log=(y, yh, e, t.to("meta")))
    with pytest.raises(TypeError):
        ScoreDistribution(0.5, s, p, "entry", 1, 0, (y, yh, e, t))    # keyword only
    g = ScoreDistribution(0.5, torch.zeros(10), torch.tensor([0, 10]), by="global", log=d.log)
    assert g.log_y.numel() == 10                                      # by="global": n scores for n graphs
    assert ScoreDistribution(0.5, s, p).log is None and ScoreDistribution(0.5, s, p).log_ts is None


def test_evict_refusals_leave_it_unchanged():
    from pert_gnn_kdd23_b200.train import ScoreDistribution

    plain = ScoreDistribution(0.5, torch.zeros(20), torch.tensor([0, 5, 10, 10, 20]))
    with pytest.raises(ValueError, match="needs a log"):
        plain.evict(5)
    d = _logged()
    s = _state(d)
    with pytest.raises(ValueError, match="without a score"):
        d.evict(10)                                                   # every ts is < 10
    _unchanged(d, s)
    assert d.evict(0) == 0                                            # nothing older: nothing to do
    _unchanged(d, s)
    with pytest.raises(_lib.PertGnnError, match="host"):
        d.evict(5)                                                    # a table on the host: no CPU fallback
    _unchanged(d, s)


def test_insert_refusals_leave_it_unchanged():
    from pert_gnn_kdd23_b200.train import ScoreDistribution

    k = 4
    y, yh, e, t = torch.zeros(k, dtype=torch.int64), torch.zeros(k), torch.zeros(k, dtype=torch.int64), \
        torch.zeros(k, dtype=torch.int64)
    plain = ScoreDistribution(0.5, torch.zeros(20), torch.tensor([0, 5, 10, 10, 20]))
    with pytest.raises(ValueError, match="needs a log"):
        plain.insert(y, yh, e, t)
    d = _logged()
    s = _state(d)
    cases = [
        (ValueError, "shrink", lambda: d.insert(y, yh, e, t, n_groups=2)),
        (ValueError, "ts must be", lambda: d.insert(y, yh, e, t[:3])),
        (ValueError, "ts must be", lambda: d.insert(y, yh, e, t.int())),
        (ValueError, "ts must be", lambda: d.insert(y, yh, e, None)),
        (ValueError, "no graphs", lambda: d.insert(y[:0], yh[:0], e[:0], t[:0])),
        (ValueError, "predictions", lambda: d.insert(y, yh[:3], e, t)),
        (ValueError, "entry id", lambda: d.insert(y, yh, e[:3], t)),
        (ValueError, "base column", lambda: ScoreDistribution(0.5, d.scores, d.ptr, column=2, log=d.log).insert(
            y, torch.zeros(k, 2), e, t)),
        (_lib.PertGnnError, "host", lambda: d.insert(y, yh, e, t)),
        (_lib.PertGnnError, "host", lambda: d.insert(y, yh, e, t, n_groups=9)),
    ]
    for exc, match, call in cases:
        with pytest.raises(exc, match=match):
            call()
        _unchanged(d, s)


def test_fit_ts_checks():
    from pert_gnn_kdd23_b200.train import ScoreDistribution

    y, yhat, e = torch.zeros(200, dtype=torch.int64), torch.zeros(200), torch.zeros(200, dtype=torch.int64)
    for ts in (torch.zeros(199, dtype=torch.int64), torch.zeros(200, dtype=torch.int32), [0] * 200):
        with pytest.raises(ValueError, match="ts must be"):
            ScoreDistribution.fit(y, yhat, e, 4, 0.5, ts=ts)
    with pytest.raises(_lib.PertGnnError, match="CUDA device"):
        ScoreDistribution.fit(y, yhat, e, 4, 0.5, ts=torch.zeros(200, dtype=torch.int64))


def test_add_traces_refusals():
    from pert_gnn_kdd23_b200.train import ScoreDistribution

    plain = ScoreDistribution(0.5, torch.zeros(20), torch.tensor([0, 5, 10, 10, 20]))
    with pytest.raises(ValueError, match="needs a log"):
        plain.add_traces(None, None, [0, 1])
    d = _logged()
    s = _state(d)
    with pytest.raises(_lib.PertGnnError, match="host"):
        d.add_traces(None, None, [0, 1])                              # refused before any forward
    _unchanged(d, s)
