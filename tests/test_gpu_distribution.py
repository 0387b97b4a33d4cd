"""GPU tests of the conformal predictive distribution (csrc/cpd.cu, train.ScoreDistribution, fit_distribution and
score_traces).

- The fitted table is bit-equal to np.sort per row (tests/cpd_ref.py), and two fits are bit-identical, from one graph
  to 10^7, on one group, 64 uniform entries, 10^4 sparse entries and a Zipf set where one entry holds 90 %, around the
  one-CTA tier bound (4096) and the tile size (8192), with keys sharing their top byte, 10^6 equal scores, ties, +-0,
  subnormals and +-1e30, and by="global".
- Tail counts and rows are bit-equal to the restatement, at thresholds equal to stored scores, +-0 and +-inf, and
  with entries on both sides of min_count; the probabilities and p-values follow from them.
- The quantile is bit-equal to Calibration.fit + pert_calib_apply at the levels both answer, and +inf exactly where
  the restatement has no bound.
- Validity on fresh exchangeable graphs: p-values and tail brackets within 4 binomial sigma.
- NaN predictions, NaN thresholds, out-of-range ids and host tensors raise.
- End to end on a pattern store: fit_distribution, predict (plain and what-if), tail, quantile and score_traces
  against their restatements; predict, calibrate and evaluate_bucketed unchanged by the new calls.
"""
import math

import numpy as np
import pytest
import torch

from pert_gnn_kdd23_b200 import _lib, ops
from tests import cpd_ref as R
from tests.test_gpu_calibration import _trained, store4096  # noqa: F401 -- the module's store fixture

pytestmark = pytest.mark.gpu

# (n, grouping, n_groups, score kind, columns of the prediction tensor)
CASES = [
    (1, "one", 1, "ties", 1),
    (2, "one", 1, "extreme", 1),
    (99, "uniform", 64, "ties", 1),
    (4095, "one", 1, "normal", 1),
    (4096, "one", 1, "extreme", 1),
    (4097, "one", 1, "ties", 3),
    (8191, "uniform", 2, "normal", 1),
    (8192, "one", 1, "normal", 1),
    (8193, "zipf", 64, "ties", 1),
    (12289, "global", 0, "extreme", 1),
    (10 ** 5, "sparse", 10 ** 4, "extreme", 1),
    (10 ** 5, "uniform", 64, "top_byte", 4),
    (10 ** 6, "zipf", 10 ** 4, "normal", 1),
    (10 ** 6, "one", 1, "equal", 1),
    (10 ** 6, "uniform", 64, "top_byte", 1),
    (10 ** 6, "global", 0, "normal", 1),
    (10 ** 7, "zipf", 10 ** 4, "ties", 1),
    (10 ** 7, "uniform", 64, "normal", 2),
    (10 ** 7, "sparse", 10 ** 4, "normal", 1),
]


def _make(n, grouping, G, score_kind, seed):
    rng = np.random.default_rng(seed)
    kind = "uniform" if grouping in ("one", "global") else grouping
    y, yhat, g = R.make_set(rng, n, max(G, 1), kind, score_kind)
    return y, yhat, (None if grouping == "global" else g)


def _fit(y, yhat, g, G, min_count=1, T=1, column=0):
    """ScoreDistribution.fit of yhat placed at column ``column`` of a [n, T] prediction tensor."""
    from pert_gnn_kdd23_b200.train import ScoreDistribution

    yh = torch.from_numpy(yhat).cuda()
    if T > 1:
        full = torch.randn(yh.numel(), T, device="cuda")
        full[:, column] = yh
        yh = full
    yd = torch.from_numpy(y).cuda()
    if g is None:
        return ScoreDistribution.fit(yd, yh, None, 0, 0.5, by="global", column=column if T > 1 else None)
    return ScoreDistribution.fit(yd, yh, torch.from_numpy(g).cuda(), G, 0.5, min_count=min_count,
                                 column=column if T > 1 else None)


def _bits(t):
    return t.detach().cpu().numpy().view(np.int32)


@pytest.mark.parametrize("n,grouping,G,score_kind,T", CASES)
def test_table_bit_equal_to_np_sort(n, grouping, G, score_kind, T):
    y, yhat, g = _make(n, grouping, G, score_kind, seed=n + T)
    d = _fit(y, yhat, g, G, T=T, column=T - 1)
    tab, ptr = R.table(y, yhat, g, 0 if g is None else G)
    assert np.array_equal(d.ptr.cpu().numpy(), ptr)
    got = _bits(d.scores)
    bad = np.flatnonzero(got != tab.view(np.int32))
    assert bad.size == 0, (bad[:5], d.scores.cpu().numpy()[bad[:5]], tab[bad[:5]])
    assert d.column == (T - 1) and d.n_groups == (0 if g is None else G)
    again = _fit(y, yhat, g, G, T=T, column=T - 1)
    assert np.array_equal(_bits(again.scores), got) and torch.equal(again.ptr, d.ptr)


def _query_set(tab, ptr, G, Q, rng):
    """Predictions, ids on both sides of [0, G), thresholds: stored scores + yhat (c equal to a stored score), +-0 +
    yhat, +-inf and random values."""
    yhat = rng.normal(1000, 200, Q).astype(np.float32)
    ids = rng.integers(-3, G + 4, Q)
    x = (rng.normal(1000, 300, (Q, 4))).astype(np.float32)
    pick = tab[rng.integers(0, tab.size, Q)]
    x[:, 0] = (yhat + pick).astype(np.float32)
    back = (x[:, 0] - yhat).astype(np.float32)
    x[back != pick, 0] = yhat[back != pick]                       # keep c exact: else c = 0 (+-0 below)
    x[:, 1] = np.where(rng.random(Q) < 0.5, yhat, -0.0)
    x[: Q // 8, 2] = np.inf
    x[Q // 8: Q // 4, 2] = -np.inf
    return yhat, ids, x.astype(np.float32)


@pytest.mark.parametrize("kind,min_count", [("uniform", 1), ("zipf", 80), ("sparse", 6250)])
def test_tail_counts_bit_equal(kind, min_count):
    rng = np.random.default_rng(7)
    G, n, Q = 256, 2 * 10 ** 5, 3 * 10 ** 5
    y, yh_fit, g = R.make_set(rng, n, G, kind, "ties" if kind == "uniform" else "normal")
    y = (y + 1000).astype(np.int64)
    d = _fit(y, yh_fit, g, G, min_count=min_count)
    tab, ptr = R.table(y, yh_fit, g, G)
    cnt = np.diff(ptr)[:G]
    if min_count > 1:                                              # entries on both sides of min_count
        assert ((cnt > 0) & (cnt < min_count)).any() and (cnt >= min_count).any()
    yhat, ids, x = _query_set(tab, ptr, G, Q, rng)
    yd, idd, xd = (torch.from_numpy(a).cuda() for a in (yhat, ids, x))
    ge, gt, row, _ = d._tail_counts(yd, idd, x=xd)
    w_ge, w_gt, w_row = R.tail(tab, ptr, min_count, yhat, ids, x=x)
    assert np.array_equal(row.cpu().numpy(), w_row)
    assert np.array_equal(ge.cpu().numpy(), w_ge) and np.array_equal(gt.cpu().numpy(), w_gt)
    lo, hi = d.tail(yd, idd, xd)
    w_lo, w_hi = R.probabilities(w_ge, w_gt, w_row, ptr)
    assert lo.dtype == torch.float64 and lo.shape == (Q, 4)
    assert np.array_equal(lo.cpu().numpy(), w_lo) and np.array_equal(hi.cpu().numpy(), w_hi)
    lo1, hi1 = d.tail(yd, idd, xd[:, 0].contiguous())                # [Q] thresholds -> [Q]
    assert lo1.shape == (Q,) and np.array_equal(hi1.cpu().numpy(), w_hi[:, 0])
    lo_s, _ = d.tail(yd, idd, 1000.0)                               # one SLO for every request
    assert np.array_equal(lo_s.cpu().numpy(), R.probabilities(*R.tail(tab, ptr, min_count, yhat, ids,
                                                                        x=np.full(Q, 1000.0)), ptr)[0][:, 0])
    labels = rng.integers(0, 3000, Q)
    p = d.pvalues(yd, idd, torch.from_numpy(labels).cuda())
    assert np.array_equal(p.cpu().numpy(), R.pvalues(tab, ptr, min_count, yhat, ids, labels))
    # predictions as a [Q, T] column: the same counts with no copy of the column
    full = torch.randn(Q, 3, device="cuda")
    full[:, 2] = yd
    d2 = type(d)(d.level, d.scores, d.ptr, d.by, min_count, column=2)
    assert torch.equal(d2._tail_counts(full, idd, x=xd)[0], ge)


LEVELS = (0.0, 0.1, 0.5, 0.9, 0.95, 0.99, 0.999)


@pytest.mark.parametrize("kind,min_count", [("zipf", 1), ("uniform", 1562), ("sparse", 12500)])
def test_quantile_equals_calibration(kind, min_count):
    from pert_gnn_kdd23_b200.train import Calibration, _calib_apply

    rng = np.random.default_rng(3)
    G, n, Q = 64, 10 ** 5, 2 * 10 ** 5
    y, yh_fit, g = R.make_set(rng, n, G, kind, "normal")
    d = _fit(y, yh_fit, g, G, min_count=min_count)
    L = len(LEVELS)
    cal = Calibration.fit(torch.from_numpy(y).cuda(), torch.from_numpy(np.repeat(yh_fit[:, None], L, 1)).cuda(),
                          torch.from_numpy(g).cuda(), LEVELS, G, min_count=min_count)
    yhat = rng.normal(1000, 200, Q).astype(np.float32)
    ids = rng.integers(-2, G + 3, Q)
    yd, idd = torch.from_numpy(yhat).cuda(), torch.from_numpy(ids).cuda()
    got = d.quantile(yd, idd, LEVELS)
    want = yd[:, None].repeat(1, L).contiguous()
    _calib_apply(want, idd, cal.offsets, False)
    assert np.array_equal(_bits(got), _bits(want))
    tab, ptr = R.table(y, yh_fit, g, G)
    assert np.array_equal(_bits(got), R.quantile(tab, ptr, min_count, yhat, ids, LEVELS).view(np.int32))
    assert np.isfinite(got.cpu().numpy()).all()


def test_quantile_is_inf_exactly_where_no_bound_exists():
    rng = np.random.default_rng(4)
    G, n = 8, 500                                                  # 0.999 needs 999 graphs; 0.99 only the global row
    y, yh_fit, g = R.make_set(rng, n, G, "uniform", "normal")
    d = _fit(y, yh_fit, g, G)
    yhat = rng.normal(1000, 200, 1000).astype(np.float32)
    ids = rng.integers(-1, G + 1, 1000)
    lv = (0.5, 0.99, 0.999)                                        # k = 251, 496, 501 on the global row of 500
    got = d.quantile(torch.from_numpy(yhat).cuda(), torch.from_numpy(ids).cuda(), lv).cpu().numpy()
    tab, ptr = R.table(y, yh_fit, g, G)
    want = R.quantile(tab, ptr, 1, yhat, ids, lv)
    assert np.array_equal(got.view(np.int32), want.view(np.int32))
    assert np.isinf(got[:, 2]).all() and np.isfinite(got[:, :2]).all()


def _exchangeable(seed, n, G):
    """Latencies with an entry-dependent scale around a biased, noisy prediction; fit and test from the same law."""
    rng = np.random.default_rng(seed)
    w = 1.0 / np.arange(1, G + 1)
    e = rng.choice(G, size=n, p=w / w.sum())
    scale = 5.0 + 3.0 * e
    y = np.round(200 + scale * rng.lognormal(0.0, 0.6, n)).astype(np.int64)
    yhat = (200 + 1.2 * scale + rng.normal(0, 0.3, n) * scale).astype(np.float32)
    return y, yhat, e


def test_validity_on_exchangeable_graphs():
    """For one fitted table the share of test graphs with p <= alpha centres on the table's conditional level, which
    itself varies with the held-out draw by a binomial sigma over its m graphs: sigma is that of the difference of the
    two independent sets, sqrt(a (1 - a) (1 / n_test + 1 / m))."""
    G, n = 40, 2 * 10 ** 5
    yf, hf, ef = _exchangeable(1, n, G)
    yt, ht, et = _exchangeable(2, n, G)
    d = _fit(yf, hf, ef, G)
    yd, ed = torch.from_numpy(ht).cuda(), torch.from_numpy(et).cuda()
    p = d.pvalues(yd, ed, torch.from_numpy(yt).cuda()).cpu().numpy()
    for a in (0.01, 0.05, 0.1):
        sig = math.sqrt(a * (1 - a) * 2 / n)
        assert (p <= a).mean() <= a + 4 * sig, a
        cnt = d.counts.cpu().numpy()
        for grp in np.flatnonzero(np.bincount(et, minlength=G) >= 5000):
            sel = et == grp
            sg = math.sqrt(a * (1 - a) * (1 / sel.sum() + 1 / cnt[grp]))
            assert (p[sel] <= a).mean() <= a + 4 * sg, (a, grp)
    rng = np.random.default_rng(9)
    x = (ht + rng.normal(1.0, 1.0, n) * (5.0 + 3.0 * et)).astype(np.float32)
    lo, hi = d.tail(yd, ed, torch.from_numpy(x).cuda())
    exceed = (yt.astype(np.float32) > x).mean()
    lo_m, hi_m = float(lo.mean()), float(hi.mean())
    sig = math.sqrt(max(exceed * (1 - exceed), 1e-4) / n)
    assert lo_m - 4 * sig <= exceed <= hi_m + 4 * sig, (lo_m, exceed, hi_m)


def test_errors_raise():
    rng = np.random.default_rng(3)
    y, yhat, g = R.make_set(rng, 5000, 16, "uniform")
    yhat[1234] = np.nan
    with pytest.raises(_lib.PertGnnError, match="NaN"):
        _fit(y, yhat, g, 16)
    yhat[1234] = 0.0
    for bad in (16, -1):
        g[77] = bad
        with pytest.raises(_lib.PertGnnError, match="entry id"):
            _fit(y, yhat, g, 16)
    g[77] = 3
    d = _fit(y, yhat, g, 16)                                      # the same set, repaired, fits
    q = torch.zeros(10, device="cuda")
    ids = torch.zeros(10, dtype=torch.int64, device="cuda")
    x = torch.full((10,), 100.0, device="cuda")
    x[3] = float("nan")
    with pytest.raises(_lib.PertGnnError, match="NaN"):
        d.tail(q, ids, x)
    qn = q.clone()
    qn[5] = float("nan")
    with pytest.raises(_lib.PertGnnError, match="NaN"):
        d.quantile(qn, ids, 0.5)
    with pytest.raises(_lib.PertGnnError, match="NaN"):
        d.pvalues(qn, ids, ids)
    d.tail(q, ids, 100.0)                                         # clean operands pass
    # host or other-device operands are refused before any launch
    l0 = ops.LAUNCHES["n"]
    for call in (lambda: d.tail(q.cpu(), ids, 100.0), lambda: d.tail(q, ids.cpu(), 100.0),
                 lambda: d.tail(q, ids, x.cpu()), lambda: d.pvalues(q, ids, ids.cpu()),
                 lambda: d.quantile(q.cpu(), ids, 0.5), lambda: d.to("cpu").quantile(q, ids, 0.5)):
        with pytest.raises(_lib.PertGnnError):
            call()
    assert ops.LAUNCHES["n"] == l0


# ------------------------------------------------------------------------------------------------------ end to end
def test_end_to_end_on_a_pattern_store(store4096, monkeypatch):  # noqa: F811
    from pert_gnn_kdd23_b200 import train
    from pert_gnn_kdd23_b200.store import StoreLoader
    from pert_gnn_kdd23_b200.train import (ScoreDistribution, calibrate, eval_step, evaluate_bucketed,
                                           fit_distribution, predict, score_traces)
    from tests.helpers import assert_close

    art, store = store4096
    taus = (0.5, 0.9, 0.95, 0.99)
    m = _trained(store, taus)
    ids = np.arange(len(store))
    cal_ids, test_ids = ids[0::2], ids[1::2]
    ent = store._h_trace_entry.astype(np.int64)
    ts = np.array([int(art["tr2data"][k]["timestamp"]) for k in store.trace_keys], dtype=np.int64)
    G = m.entry_embeds.num_embeddings

    # the calls the distribution must leave as they were
    predict(m, store, ent[test_ids], ts[test_ids], batch_size=512, asof=True)
    l0 = ops.LAUNCHES["n"]
    plain = predict(m, store, ent[test_ids], ts[test_ids], batch_size=512, asof=True)
    plain_launches = ops.LAUNCHES["n"] - l0
    loader = StoreLoader(store, test_ids, 300)
    for _ in range(2):
        evaluate_bucketed(m, loader, "cuda")
    l0 = ops.LAUNCHES["n"]
    plain_e = evaluate_bucketed(m, loader, "cuda")
    plain_e_launches = ops.LAUNCHES["n"] - l0
    cal_loader = StoreLoader(store, cal_ids, 300)
    calibrate(m, cal_loader, "cuda")
    l0 = ops.LAUNCHES["n"]
    cal0 = calibrate(m, cal_loader, "cuda")
    cal_launches = ops.LAUNCHES["n"] - l0

    # fit: the table is the restatement's on the predictions the fit received
    seen, real = [], train._replayed_predictions

    def spy(*a, **k):
        out = real(*a, **k)
        seen.append(tuple(t.clone() for t in out))
        return out

    monkeypatch.setattr(train, "_replayed_predictions", spy)
    d = fit_distribution(m, cal_loader, "cuda", level=0.9)
    assert d.level == 0.9 and d.column == 1 and d.n_groups == G
    y_c, yh_c, e_c = (t.cpu().numpy() for t in seen[0])
    tab, ptr = R.table(y_c, yh_c[:, 1], e_c, G)
    assert np.array_equal(_bits(d.scores), tab.view(np.int32)) and np.array_equal(d.ptr.cpu().numpy(), ptr)
    assert int(d.counts[-1]) == len(cal_ids)
    with pytest.raises(ValueError):
        fit_distribution(m, cal_loader, "cuda")                    # four levels: name one

    # predict + tail / quantile, plain and what-if, against the restatement on the same predictions
    slo = np.stack([np.full(len(test_ids), 300.0), np.full(len(test_ids), 600.0)], 1).astype(np.float32)
    ent_d = torch.from_numpy(ent[test_ids]).cuda()
    res_ms = np.unique([mm for _, mm in art["resource_index"]])
    rng = np.random.default_rng(5)
    o_ms = rng.choice(res_ms, max(1, res_ms.size // 10), replace=False)
    ov = (np.zeros(o_ms.size, dtype=np.int64), o_ms, np.full((o_ms.size, 8), 1.2))
    whatif = predict(m, store, ent[test_ids], ts[test_ids], batch_size=512, asof=True, overrides=ov,
                     scenario_ids=np.zeros(len(test_ids), dtype=np.int64))
    for pred in (plain, whatif):
        assert pred.shape == (len(test_ids), 4)
        ph = pred.cpu().numpy()[:, 1]
        lo, hi = d.tail(pred, ent_d, torch.from_numpy(slo).cuda())
        w = R.tail(tab, ptr, 1, ph, ent[test_ids], x=slo)
        w_lo, w_hi = R.probabilities(*w, ptr)
        assert np.array_equal(lo.cpu().numpy(), w_lo) and np.array_equal(hi.cpu().numpy(), w_hi)
        q = d.quantile(pred, ent_d, (0.5, 0.99, 0.999))
        assert np.array_equal(_bits(q), R.quantile(tab, ptr, 1, ph, ent[test_ids], (0.5, 0.99, 0.999)).view(np.int32))

    # score_traces: the p-values of the replayed forward, against those of eager eval_step predictions
    p = score_traces(m, loader, "cuda", d)
    y_t, yh_t, e_t = (t.cpu().numpy() for t in seen[-1])
    assert np.array_equal(p.cpu().numpy(), R.pvalues(tab, ptr, 1, yh_t[:, 1], e_t, y_t))
    eager, ys, es = [], [], []
    m.eval()
    with torch.no_grad():
        for b in loader:
            g_, _ = m(*train.model_inputs(b))
            eager.append(g_[:, 1].clone())
            ys.append(b.y.reshape(-1))
            es.append(b.entry_id.reshape(-1))
    m.train()
    eager = torch.cat(eager)
    assert_close(torch.from_numpy(yh_t[:, 1]).cuda(), eager, what="score_traces predictions vs eager eval")
    p_eager = d.pvalues(eager, torch.cat(es), torch.cat(ys)).cpu().numpy()
    step = 1.0 / (np.diff(ptr)[R.rows_of(ptr, 1, e_t, e_t.size)] + 1)
    diff = np.abs(p.cpu().numpy() - p_eager)
    assert (diff <= 2 * step + 1e-12).all() and (diff > 0).mean() <= 0.01
    monkeypatch.undo()

    # saved as plain tensors, reloaded on the host: refused until moved back
    import io

    buf = io.BytesIO()
    torch.save({"level": d.level, "scores": d.scores, "ptr": d.ptr, "by": d.by, "min_count": d.min_count,
                "column": d.column}, buf)
    buf.seek(0)
    s = torch.load(buf, map_location="cpu")
    host = ScoreDistribution(s["level"], s["scores"], s["ptr"], s["by"], s["min_count"], s["column"])
    with pytest.raises(_lib.PertGnnError, match="host"):
        host.tail(plain, ent_d, 300.0)
    back = host.to("cuda")
    assert torch.equal(back.tail(plain, ent_d, 300.0)[1], d.tail(plain, ent_d, 300.0)[1])

    # a one-level distribution of the same model's median, and the global grouping
    dg = fit_distribution(m, cal_loader, "cuda", level=0.5, by="global")
    assert dg.n_groups == 0 and int(dg.counts[-1]) == len(cal_ids)

    # the calls without the distribution: same launches and results as before it
    l0 = ops.LAUNCHES["n"]
    again = predict(m, store, ent[test_ids], ts[test_ids], batch_size=512, asof=True)
    assert ops.LAUNCHES["n"] - l0 == plain_launches
    assert_close(again, plain, what="predict() before and after the distribution calls")
    l0 = ops.LAUNCHES["n"]
    again_e = evaluate_bucketed(m, loader, "cuda")
    assert ops.LAUNCHES["n"] - l0 == plain_e_launches
    for gv, wv in zip(again_e, plain_e):
        for a, b in zip(gv, wv):
            assert abs(a - b) <= 1e-5 * abs(b), (gv, wv)
    l0 = ops.LAUNCHES["n"]
    cal1 = calibrate(m, cal_loader, "cuda")
    assert ops.LAUNCHES["n"] - l0 == cal_launches
    assert_close(cal1.offsets, cal0.offsets, what="calibrate() before and after the distribution calls")
    assert torch.equal(cal1.counts, cal0.counts)
