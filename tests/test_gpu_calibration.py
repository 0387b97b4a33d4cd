"""GPU tests of the conformal calibration (csrc/calib.cu, train.Calibration / calibrate, and the calibration= paths of
predict, eval_step and evaluate_bucketed).

- The fit's offsets, counts and own flags are bit-equal to tests/calib_ref.py, and two runs are bit-identical, from
  one graph to 10^7, at T in {1, 2, 3, 4, 8}, around the one-CTA tier bound (4096 graphs) and the tile size (8192), on
  one group, 64 uniform entries, 10^4 entries with many empty ones and a Zipf set where one entry holds 90 %, with
  tied scores, +-0, subnormals and +-1e30.
- A NaN prediction and an out-of-range entry id raise through the status word.
- The apply is bit-equal to the fp32 restatement, with and without the running max; ghost rows stay; unseen ids
  read the global row.
- In-sample and out-of-sample coverage meet the conformal bounds.
- End to end on a pattern store: predict and evaluate_bucketed with a calibration against their restatements.
"""
import math

import numpy as np
import pytest
import torch

from pert_gnn_kdd23_b200 import _lib, ops
from tests import calib_ref as R

pytestmark = pytest.mark.gpu

LEVELS = {1: (0.95,), 2: (0.0, 0.5), 3: (0.1, 0.5, 0.9), 4: (0.5, 0.9, 0.95, 0.99),
          8: (0.0, 0.1, 0.25, 0.5, 0.75, 0.9, 0.95, 0.999)}

# (n, T, grouping, n_groups, score kind, min_count); levels: LEVELS[T] except where n is too small for them
CASES = [
    (1, 1, "one", 1, "ties", 1),
    (2, 2, "one", 1, "extreme", 1),
    (99, 4, "uniform", 64, "ties", 1),
    (100, 4, "uniform", 64, "normal", 1),
    (4095, 3, "one", 1, "normal", 1),
    (4096, 3, "one", 1, "extreme", 1),
    (4097, 3, "one", 1, "ties", 1),
    (8191, 2, "uniform", 2, "normal", 1),
    (8192, 8, "one", 1, "normal", 1),
    (8193, 8, "zipf", 64, "ties", 1),
    (12289, 4, "global", 0, "extreme", 1),
    (10 ** 5, 8, "sparse", 10 ** 4, "extreme", 1),
    (10 ** 5, 4, "uniform", 16, "normal", 6250),          # min_count inside the sizes of large-tier entries
    (10 ** 5, 4, "zipf", 64, "ties", 156),                 # ... and of the small-tier entries beside a hot one
    (10 ** 6, 4, "zipf", 10 ** 4, "normal", 1),
    (10 ** 6, 2, "uniform", 64, "ties", 1),
    (10 ** 6, 1, "sparse", 10 ** 4, "normal", 800),        # ... and of small-tier entries
    (10 ** 7, 2, "zipf", 10 ** 4, "ties", 1),
    (10 ** 7, 1, "uniform", 64, "normal", 1),
]


def _levels(n, T):
    if n == 1:
        return (0.5,)
    if n == 2:
        return (0.0, 0.5)
    return LEVELS[T]                  # n = 99 and 100 at T = 4 keep 0.99: there the global row's k is n


def _make(n, T, grouping, G, score_kind, seed):
    rng = np.random.default_rng(seed)
    kind = "uniform" if grouping in ("one", "global") else grouping
    y, yhat, g = R.make_set(rng, n, T, max(G, 1), kind, score_kind)
    return y, yhat, (None if grouping == "global" else g)


def _bits(t):
    return t.detach().cpu().numpy().view(np.int32)


def _fit(y, yhat, g, taus, G, min_count=1):
    from pert_gnn_kdd23_b200.train import Calibration

    dev = "cuda"
    yd, yh = torch.from_numpy(y).to(dev), torch.from_numpy(yhat).to(dev)
    if g is None:
        return Calibration.fit(yd, yh, None, taus, 0, by="global")
    return Calibration.fit(yd, yh, torch.from_numpy(g).to(dev), taus, G, min_count=min_count)


@pytest.mark.parametrize("n,T,grouping,G,score_kind,min_count", CASES)
def test_offsets_bit_equal_to_reference(n, T, grouping, G, score_kind, min_count):
    taus = _levels(n, T)
    y, yhat, g = _make(n, len(taus), grouping, G, score_kind, seed=n + 7 * T)
    cal = _fit(y, yhat, g, taus, G, min_count)
    off, cnt, own = R.offsets(y, yhat, g, 0 if g is None else G, taus, min_count)
    assert cal.offsets.shape == off.shape and cal.levels == taus
    got = cal.offsets.cpu().numpy()
    bad = np.flatnonzero(got.view(np.int32) != off.view(np.int32))
    assert bad.size == 0, (bad[:5], got.reshape(-1)[bad[:5]], off.reshape(-1)[bad[:5]])
    assert np.array_equal(cal.counts.cpu().numpy(), cnt)
    assert np.array_equal(cal.own.cpu().numpy(), own)
    if min_count > 1:                 # the rule decides: some entries fall back only because of min_count
        assert (R.offsets(y, yhat, g, G, taus, 1)[2][:G] > own[:G]).any() and own[:G].any()
    again = _fit(y, yhat, g, taus, G, min_count)
    assert np.array_equal(_bits(again.offsets), _bits(cal.offsets))
    assert torch.equal(again.own, cal.own) and torch.equal(again.counts, cal.counts)


def test_errors_raise_through_status():
    rng = np.random.default_rng(3)
    y, yhat, g = R.make_set(rng, 5000, 2, 16, "uniform")
    yhat[1234, 1] = np.nan
    with pytest.raises(_lib.PertGnnError, match="NaN"):
        _fit(y, yhat, g, (0.5, 0.9), 16)
    yhat[1234, 1] = 0.0
    g[77] = 16
    with pytest.raises(_lib.PertGnnError, match="entry id"):
        _fit(y, yhat, g, (0.5, 0.9), 16)
    g[77] = -1
    with pytest.raises(_lib.PertGnnError, match="entry id"):
        _fit(y, yhat, g, (0.5, 0.9), 16)
    g[77] = 3
    _fit(y, yhat, g, (0.5, 0.9), 16)                      # the same set, repaired, fits


@pytest.mark.parametrize("T", [1, 2, 3, 4, 8])
def test_apply_bit_equal(T):
    from pert_gnn_kdd23_b200.train import _calib_apply

    rng = np.random.default_rng(T)
    G, Q = 50, 300001
    off = rng.normal(0, 30, (G + 1, T)).astype(np.float32)
    q = rng.normal(0, 100, (Q, T)).astype(np.float32)
    grp = rng.integers(-3, G + 5, Q)                      # unseen ids on both sides read the global row
    offd, gd = torch.from_numpy(off).cuda(), torch.from_numpy(grp).cuda()
    shape = (Q, T) if T > 1 else (Q,)
    for monotone in (False, True):
        x = torch.from_numpy(q).cuda().reshape(shape).contiguous()
        _calib_apply(x, gd, offd, monotone)
        want = R.apply(q.reshape(shape), grp, off, monotone=monotone)
        assert np.array_equal(x.cpu().numpy().view(np.int32), want.view(np.int32)), monotone
    x = torch.from_numpy(q).cuda().reshape(shape).contiguous()
    _calib_apply(x, gd, None, True)                       # no table: only the running max
    assert np.array_equal(x.cpu().numpy().view(np.int32), R.apply(q.reshape(shape), grp, None, True).view(np.int32))
    live = torch.tensor([0, 123457], dtype=torch.int64, device="cuda")
    x = torch.from_numpy(q).cuda().reshape(shape).contiguous()
    _calib_apply(x, gd, offd, True, live=live)
    want = R.apply(q.reshape(shape), grp, off, monotone=True, live=123457)
    assert np.array_equal(x.cpu().numpy().view(np.int32), want.view(np.int32))
    assert np.array_equal(x.cpu().numpy()[123457:].view(np.int32), q.reshape(shape)[123457:].view(np.int32))


def test_in_sample_coverage():
    rng = np.random.default_rng(11)
    G, taus = 10 ** 4, LEVELS[4]
    y, yhat, g = R.make_set(rng, 10 ** 6, 4, G, "zipf")
    yhat = (np.round(yhat * 16) / 16).astype(np.float32)  # on a 1/16 grid: y - yhat and yhat + c are exact, r = 0
    cal = _fit(y, yhat, g, taus, G)
    off, cnt, own = (t.cpu().numpy() for t in (cal.offsets, cal.counts, cal.own))
    r = R.roundtrip_slack(y, yhat)
    assert (r == 0).all(), r
    c = (yhat + off[g]).astype(np.float32)
    ok = y.astype(np.float32)[:, None] <= c
    for t, tau in enumerate(taus):
        cov = np.bincount(g, weights=ok[:, t], minlength=G)
        k = np.array([R.k_of(int(m), tau) for m in cnt[:G]])
        mine = own[:G, t] == 1
        assert (cov[mine] >= k[mine] - r[t]).all()
        # the global row on its own, over every graph
        assert (y.astype(np.float32) <= (yhat[:, t] + off[G, t]).astype(np.float32)).sum() >= R.k_of(len(y), tau)


def _exchangeable(seed, n, G):
    """Latencies with an entry-dependent scale and a predictor that is biased low and noisy per level (so its raw
    levels cross); fit and test sets drawn from the same law."""
    rng = np.random.default_rng(seed)
    w = 1.0 / np.arange(1, G + 1)
    e = rng.choice(G, size=n, p=w / w.sum())
    scale = 5.0 + 3.0 * e
    y = np.round(200 + scale * rng.lognormal(0.0, 0.6, n)).astype(np.int64)
    base = 200 + scale[:, None] * np.array([0.8, 1.2, 1.5, 1.9])[None, :]
    yhat = (base + rng.normal(0, 0.3, (n, 4)) * scale[:, None]).astype(np.float32)
    return y, yhat, e


def test_out_of_sample_coverage():
    from pert_gnn_kdd23_b200.train import EvalMetrics, _calib_apply

    G, n, taus = 40, 2 * 10 ** 5, LEVELS[4]
    yf, hf, ef = _exchangeable(1, n, G)
    yt, ht, et = _exchangeable(2, n, G)
    cal = _fit(yf, hf, ef, taus, G)
    cnt = cal.counts.cpu().numpy()
    for monotone in (False, True):
        x = torch.from_numpy(ht).cuda()
        _calib_apply(x, torch.from_numpy(et).cuda(), cal.offsets, monotone)
        m = EvalMetrics("cuda", taus)
        m.update(torch.from_numpy(yt).cuda(), x)
        cov = m.coverage()
        for t, tau in enumerate(taus):
            sig = math.sqrt(tau * (1 - tau) / n)
            assert cov[t] >= tau - 4 * sig, (monotone, t, cov)
            if not monotone:
                assert cov[t] <= tau + 1 / (n + 1) + 4 * sig, (t, cov)
        if monotone:
            assert m.crossing() == 0.0
        else:
            assert m.crossing() > 0.0                     # the raw levels do cross: the running max has work to do
        if monotone:
            continue
        xc = x.cpu().numpy()
        for grp in np.flatnonzero(np.bincount(et, minlength=G) >= 5000):
            sel = et == grp
            nt = int(sel.sum())
            for t, tau in enumerate(taus):
                if not cal.own[grp, t]:
                    continue
                c = float((yt[sel].astype(np.float32) <= xc[sel, t]).mean())
                sig = math.sqrt(tau * (1 - tau) / nt)
                assert tau - 4 * sig <= c <= tau + 1 / (int(cnt[grp]) + 1) + 4 * sig, (grp, t, c)


# ------------------------------------------------------------------------------------------------------ end to end
@pytest.fixture(scope="module")
def store4096():
    from pert_gnn_kdd23_b200.store import PatternStore
    from pert_gnn_kdd23_b200.synthetic import make_pert_artifacts

    art, _ = make_pert_artifacts(seed=3, n_entries=64, n_traces=4096, device="cuda")
    return art, PatternStore.from_artifacts(art, "cuda")


def _trained(store, quantiles, steps=6):
    from pert_gnn_kdd23_b200.model import SAGEDeterministic
    from pert_gnn_kdd23_b200.store import StoreLoader
    from pert_gnn_kdd23_b200.synthetic import model_args
    from pert_gnn_kdd23_b200.train import FlatParams, FusedAdam, fused_train_step

    torch.manual_seed(0)
    args = list(model_args(2))
    args[2] = max(args[2], int(store.id_bounds()["entry"]) - 1)
    m = SAGEDeterministic(*args, quantiles=quantiles).cuda()
    opt = FusedAdam(FlatParams(m), lr=3e-3)
    loader = StoreLoader(store, list(range(len(store))), 256, shuffle=True, generator=torch.Generator().manual_seed(1))
    for i, d in enumerate(loader):
        if i >= steps:
            break
        fused_train_step(m, opt, d, tau=quantiles or 0.95)
    return m


def _capture_apply_input(monkeypatch):
    """Records a copy of the predictions every pert_calib_apply of train.py receives.  The engine's forward adds some
    float sums with atomics, so two predict calls agree to rounding, not bit for bit; the apply is compared bit for bit
    against the numpy restatement on the predictions it was given."""
    from pert_gnn_kdd23_b200 import train

    seen, real = [], train._calib_apply

    def spy(yhat, group, off, monotone, live=None):
        seen.append(yhat.clone())
        return real(yhat, group, off, monotone, live)

    monkeypatch.setattr(train, "_calib_apply", spy)
    return seen


def test_end_to_end_on_a_pattern_store(store4096, monkeypatch):
    from pert_gnn_kdd23_b200.store import StoreLoader
    from pert_gnn_kdd23_b200.train import EvalMetrics, calibrate, eval_step, evaluate_bucketed, predict
    from tests.helpers import assert_close

    art, store = store4096
    taus = LEVELS[4]
    m = _trained(store, taus)
    ids = np.arange(len(store))
    cal_ids, test_ids = ids[0::2], ids[1::2]
    ent = store._h_trace_entry.astype(np.int64)
    ts = np.array([int(art["tr2data"][k]["timestamp"]) for k in store.trace_keys], dtype=np.int64)

    plain0 = predict(m, store, ent[test_ids], ts[test_ids], batch_size=512, asof=True)
    l0 = ops.LAUNCHES["n"]
    plain1 = predict(m, store, ent[test_ids], ts[test_ids], batch_size=512, asof=True)
    plain_launches = ops.LAUNCHES["n"] - l0
    loader = StoreLoader(store, test_ids, 300)
    for _ in range(2):                                     # eager, then captured: the next call replays
        evaluate_bucketed(m, loader, "cuda")
    l0 = ops.LAUNCHES["n"]
    plain_e = evaluate_bucketed(m, loader, "cuda")
    plain_e_launches = ops.LAUNCHES["n"] - l0

    cal = calibrate(m, StoreLoader(store, cal_ids, 300), "cuda", max_graphs=32)
    assert cal.levels == taus and cal.n_groups == m.entry_embeds.num_embeddings
    own = cal.own.cpu().numpy()
    assert own[:, 3].sum() < own[:, 0].sum()               # ~32 graphs per entry: the 0.99 level falls back
    assert int(cal.counts[-1]) == len(cal_ids)

    seen = _capture_apply_input(monkeypatch)
    l0 = ops.LAUNCHES["n"]
    got = predict(m, store, ent[test_ids], ts[test_ids], batch_size=512, asof=True, calibration=cal)
    assert ops.LAUNCHES["n"] - l0 == plain_launches + 1 and len(seen) == 1
    assert_close(seen[0], plain1, what="the predictions the apply received vs predict()")
    want = R.apply(seen[0].cpu().numpy(), ent[test_ids], cal.offsets.cpu().numpy())
    assert np.array_equal(got.cpu().numpy().view(np.int32), want.view(np.int32))
    mono = predict(m, store, ent[test_ids], ts[test_ids], batch_size=512, asof=True, calibration=cal, monotone=True)
    want = R.apply(seen[1].cpu().numpy(), ent[test_ids], cal.offsets.cpu().numpy(), monotone=True)
    assert np.array_equal(mono.cpu().numpy().view(np.int32), want.view(np.int32))
    monkeypatch.undo()

    # a calibration saved as plain tensors and reloaded on the host is refused until it is moved to the device
    import io

    from pert_gnn_kdd23_b200.train import Calibration

    buf = io.BytesIO()
    torch.save({"levels": cal.levels, "offsets": cal.offsets, "counts": cal.counts, "own": cal.own, "by": cal.by,
                "min_count": cal.min_count}, buf)
    buf.seek(0)
    d = torch.load(buf, map_location="cpu")
    host = Calibration(d["levels"], d["offsets"], d["counts"], d["own"], d["by"], d["min_count"])
    with pytest.raises(_lib.PertGnnError, match="host"):
        predict(m, store, ent[test_ids], ts[test_ids], batch_size=512, asof=True, calibration=host)
    back = host.to("cuda")
    assert torch.equal(back.offsets, cal.offsets) and torch.equal(back.own, cal.own) and back.by == cal.by
    assert predict(m, store, ent[:8], ts[:8], asof=True, calibration=back).shape == (8, 4)

    # evaluation: graph-replayed with the calibration against the eager eval_step
    cal2 = calibrate(m, StoreLoader(store, cal_ids, 300), "cuda", min_count=40)
    assert cal2.offsets.shape == cal.offsets.shape and not torch.equal(cal2.offsets, cal.offsets)
    for c in (cal, cal2, cal):
        want_m = EvalMetrics("cuda", taus)
        m.eval()
        for d in loader:
            eval_step(m, d, None, want_m, calibration=c)
        m.train()
        for rep in range(3):
            got_e = evaluate_bucketed(m, loader, "cuda", calibration=c)
            for gv, wv in zip(got_e, want_m.result()):
                for a, b in zip(gv, wv):
                    assert abs(a - b) <= 1e-5 * abs(b), (rep, gv, wv)
    st = m.__dict__["_bucketed_eval_calibrated"]
    assert st.replays > 0 and st.capture_error is None
    evaluate_bucketed(m, loader, "cuda", calibration=cal)
    cov = st.metrics.coverage()
    evaluate_bucketed(m, loader, "cuda", calibration=cal, monotone=True)
    assert st.metrics.crossing() == 0.0
    evaluate_bucketed(m, loader, "cuda")
    raw = m.__dict__["_bucketed_eval"].metrics.coverage()
    n_test = len(test_ids)
    print(f"\ncalibration end to end: {n_test} held-out traces, levels {taus}: coverage raw "
          f"{tuple(round(c, 4) for c in raw)}, calibrated {tuple(round(c, 4) for c in cov)}")
    for t, tau in enumerate(taus):
        assert cov[t] >= tau - 4 * math.sqrt(tau * (1 - tau) / n_test), (t, cov)

    # the calls without the new arguments: the same results and launches as before any calibrated call
    l0 = ops.LAUNCHES["n"]
    plain2 = predict(m, store, ent[test_ids], ts[test_ids], batch_size=512, asof=True)
    assert ops.LAUNCHES["n"] - l0 == plain_launches
    assert_close(plain2, plain1, what="predict() before and after the calibrated calls")
    l0 = ops.LAUNCHES["n"]
    again = evaluate_bucketed(m, loader, "cuda")
    assert ops.LAUNCHES["n"] - l0 == plain_e_launches
    for gv, wv in zip(again, plain_e):                     # the forward adds some float sums with atomics
        for a, b in zip(gv, wv):
            assert abs(a - b) <= 1e-5 * abs(b), (gv, wv)


def test_one_level_model(store4096, monkeypatch):
    from pert_gnn_kdd23_b200.store import StoreLoader
    from pert_gnn_kdd23_b200.train import calibrate, predict
    from tests.helpers import assert_close

    art, store = store4096
    m = _trained(store, None, steps=3)
    ids = np.arange(len(store))
    cal = calibrate(m, StoreLoader(store, ids[0::2], 300), "cuda", tau=0.95)
    assert cal.levels == (0.95,) and cal.offsets.shape == (m.entry_embeds.num_embeddings + 1, 1)
    ent = store._h_trace_entry.astype(np.int64)[ids[1::2]]
    ts = np.array([int(art["tr2data"][k]["timestamp"]) for k in store.trace_keys], dtype=np.int64)[ids[1::2]]
    plain = predict(m, store, ent, ts, asof=True)
    seen = _capture_apply_input(monkeypatch)
    got = predict(m, store, ent, ts, asof=True, calibration=cal)
    assert got.shape == (len(ent),) and plain.shape == got.shape
    assert_close(seen[0], plain, what="the predictions the apply received vs predict()")
    want = R.apply(seen[0].cpu().numpy(), ent, cal.offsets.cpu().numpy())
    assert np.array_equal(got.cpu().numpy().view(np.int32), want.view(np.int32))
