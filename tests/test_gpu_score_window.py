"""GPU tests of the score window (csrc/cpd.cu pert_cpd_merge, ScoreDistribution.insert / evict / add_traces).

- Seeded random sequences of inserts and evicts over windows of 1 to 10^7 graphs, with deltas of 1, 4095/4096/4097,
  8191/8192/8193 and 10^5 graphs, on 64 uniform entries, 10^4 sparse entries and a Zipf mix where one entry holds 90 %,
  with ties, +-0, subnormals, +-1e30 and 10^6 equal scores, G growth mid-sequence, by="global" and a base column of
  [n, T] predictions.  After every step the table is bit-equal to ScoreDistribution.fit over the surviving log and to
  the numpy restatement (tests/cpd_window_ref.py), the log equals the restatement's, and a second run of the same
  sequence is bit-identical.
- A removal the table does not hold raises through the status word and leaves the old tensors in place; so do a NaN
  prediction and an out-of-range entry id on insert.
- End to end on a store built with from_trace_groups: fit with ts, then append_traces -> grow_embeddings ->
  add_traces(evict_before=cut) -> evict_traces(cut); the p-values, the table, the log against a fresh forward, and
  the existing calls' launches and results unchanged.
"""
import numpy as np
import pytest
import torch

from pert_gnn_kdd23_b200 import _lib, ops
from tests import cpd_ref as R
from tests import cpd_window_ref as W

pytestmark = pytest.mark.gpu


def _bits(t):
    return t.detach().cpu().numpy().view(np.int32)


def _batch(rng, k, G, mix, score_kind, t, spread=1):
    kind = "uniform" if mix in ("one", "global") else mix
    y, yhat, g = R.make_set(rng, k, max(G, 1), kind, score_kind)
    return y, yhat, g, t + rng.integers(0, spread, k).astype(np.int64)


def _dev(batch, T=1, column=0, seed=0):
    """The batch on the device, the prediction at column ``column`` of a [k, T] tensor."""
    y, yhat, g, ts = batch
    yh = torch.from_numpy(yhat).cuda()
    if T > 1:
        full = torch.randn(yh.numel(), T, device="cuda", generator=torch.Generator("cuda").manual_seed(seed))
        full[:, column] = yh
        yh = full
    return (torch.from_numpy(y).cuda(), yh, torch.from_numpy(g).cuda(), torch.from_numpy(ts).cuda())


def _assert_contract(d, w, check_restated_merge):
    """The table is the fit over the surviving log and the restatement's; the log is the restatement's."""
    from pert_gnn_kdd23_b200.train import ScoreDistribution

    for got, want in zip(d.log, w.log):
        got = got.cpu().numpy()
        assert got.dtype == want.dtype and np.array_equal(got.view(np.int32) if got.dtype == np.float32 else got,
                                                          want.view(np.int32) if want.dtype == np.float32 else want)
    ref = ScoreDistribution.fit(d.log_y, d.log_yhat, d.log_entry if d.by == "entry" else None, d.n_groups, d.level,
                                by=d.by)
    assert torch.equal(d.ptr, ref.ptr) and np.array_equal(_bits(d.scores), _bits(ref.scores))
    tab, ptr = w.table()
    assert np.array_equal(d.ptr.cpu().numpy(), ptr) and np.array_equal(_bits(d.scores), tab.view(np.int32))
    if check_restated_merge:
        assert np.array_equal(w.ptr, ptr) and np.array_equal(w.tab.view(np.int32), tab.view(np.int32))


# (window, deltas cycled through the inserts, mix, G, score kind, columns of the predictions)
SEQS = [
    (1, (1, 4095, 4096, 4097), "uniform", 64, "ties", 1),
    (10 ** 4, (8191, 8192, 8193, 1), "zipf", 64, "extreme", 1),
    (10 ** 5, (10 ** 5, 4096, 1), "sparse", 10 ** 4, "extreme", 1),
    (10 ** 5, (8192, 4097), "global", 0, "ties", 1),
    (10 ** 5, (4095, 10 ** 5), "uniform", 64, "normal", 3),
    (10 ** 6, (10 ** 5, 1, 8193), "zipf", 10 ** 4, "normal", 1),
    (10 ** 6, (10 ** 5, 4096), "one", 1, "equal", 1),
    (10 ** 7, (10 ** 5, 1), "zipf", 10 ** 4, "ties", 1),
    (10 ** 7, (10 ** 5,), "uniform", 64, "normal", 2),
    (10 ** 7, (8192,), "sparse", 10 ** 4, "normal", 1),
]


@pytest.mark.parametrize("n,deltas,mix,G,score_kind,T", SEQS)
def test_random_update_sequences(n, deltas, mix, G, score_kind, T):
    from pert_gnn_kdd23_b200.train import ScoreDistribution

    rng = np.random.default_rng(n + len(deltas) + G)
    by = "global" if mix == "global" else "entry"
    col = T - 1
    first = _batch(rng, n, G, mix, score_kind, 0, spread=4)
    w = W.Window(*first, G, group=by == "entry")
    y, yh, e, ts = _dev(first, T, col)
    kw = dict(by=by, column=col if T > 1 else None, ts=ts)
    runs = [ScoreDistribution.fit(y, yh, e if by == "entry" else None, G, 0.5, **kw) for _ in range(2)]
    small = n <= 10 ** 6
    _assert_contract(runs[0], w, small)
    t, grown = 4, False
    steps = 7 if n <= 10 ** 6 else 4
    for step in range(steps):
        if step % 3 == 2:                                        # evict the oldest bucket (or two)
            cut = int(w.log[3].min()) + 1 + int(rng.integers(0, 2))
            if (w.log[3] < cut).all():
                cut = int(w.log[3].min()) + 1
            if (w.log[3] < cut).all():
                continue
            k = w.evict(cut)
            assert [d.evict(cut) for d in runs] == [k, k]
        else:
            G_new = w.G
            if step == 3 and by == "entry" and not grown:        # ids of new entries arrive mid-sequence
                G_new, grown = w.G + 5, True
            k = deltas[(step // 3 * 2 + step % 3) % len(deltas)]
            b = _batch(rng, k, G_new, mix, score_kind, t)
            if G_new > w.G:
                b[2][: max(1, k // 2)] = rng.integers(w.G, G_new, max(1, k // 2))
            w.insert(*b, n_groups=G_new)
            yb, yhb, eb, tb = _dev(b, T, col, seed=step)
            for d in runs:
                d.insert(yb, yhb, eb if by == "entry" else None, tb, n_groups=G_new)
            t += 1
        _assert_contract(runs[0], w, small)
        assert runs[0].n_groups == (w.G if by == "entry" else 0)
        assert torch.equal(runs[0].ptr, runs[1].ptr) and torch.equal(runs[0].scores.view(torch.int32),
                                                                     runs[1].scores.view(torch.int32))
        for a, b in zip(runs[0].log, runs[1].log):
            assert torch.equal(a, b)


def test_queries_read_the_updated_table():
    """tail, pvalues and quantile of an updated window equal those of a distribution fitted on its log."""
    from pert_gnn_kdd23_b200.train import ScoreDistribution

    rng = np.random.default_rng(2)
    d = ScoreDistribution.fit(*_dev(_batch(rng, 5000, 16, "zipf", "ties", 0, 3))[:3], 16, 0.9,
                              ts=_dev(_batch(rng, 5000, 16, "zipf", "ties", 0, 3))[3])
    d.insert(*_dev(_batch(rng, 3000, 20, "uniform", "ties", 3)), n_groups=20)
    d.evict(2)
    ref = ScoreDistribution.fit(d.log_y, d.log_yhat, d.log_entry, d.n_groups, 0.9)
    q = torch.from_numpy(rng.normal(1000, 200, 4000).astype(np.float32)).cuda()
    ids = torch.from_numpy(rng.integers(-1, 22, 4000)).cuda()
    lab = torch.from_numpy(rng.integers(0, 3000, 4000)).cuda()
    for a, b in zip(d.tail(q, ids, 1100.0), ref.tail(q, ids, 1100.0)):
        assert torch.equal(a, b)
    assert torch.equal(d.pvalues(q, ids, lab), ref.pvalues(q, ids, lab))
    assert torch.equal(d.quantile(q, ids, (0.5, 0.99)), ref.quantile(q, ids, (0.5, 0.99)))


def test_failed_updates_leave_the_old_tensors():
    from pert_gnn_kdd23_b200.train import ScoreDistribution

    rng = np.random.default_rng(4)
    y, yh, e, ts = _dev(_batch(rng, 20000, 32, "uniform", "normal", 0, 4))        # (almost) distinct scores
    d = ScoreDistribution.fit(y, yh, e, 32, 0.5, ts=ts)
    # a log whose evicted scores the table does not hold: the merge's status word refuses it
    bad_yh = d.log_yhat.clone()
    old = d.log_ts < 1
    bad_yh[old] = bad_yh[old] + 0.25                              # scores no graph of the table has
    bad = ScoreDistribution(d.level, d.scores, d.ptr, log=(d.log_y, bad_yh, d.log_entry, d.log_ts))
    state = (bad.scores, bad.ptr, bad.log)
    with pytest.raises(_lib.PertGnnError, match="not all in the table"):
        bad.evict(1)
    assert bad.scores is state[0] and bad.ptr is state[1] and all(a is b for a, b in zip(bad.log, state[2]))
    # one copy too many of a value the table holds
    dup = (d.log_y.clone(), d.log_yhat.clone(), d.log_entry.clone(), d.log_ts.clone())
    i = int(torch.nonzero(old)[0])
    j = int(torch.nonzero(~old)[0])
    for t in dup[:3]:
        t[j] = t[i]                                               # row j restates row i
    dup[3][j] = 0
    s_i = d.log_y[i].float() - d.log_yhat[i]
    assert int(((d.log_y.float() - d.log_yhat) == s_i).sum()) == 1    # whose score the table holds once
    bad2 = ScoreDistribution(d.level, d.scores, d.ptr, log=dup)
    with pytest.raises(_lib.PertGnnError, match="not all in the table"):
        bad2.evict(1)
    # insert: a NaN prediction or an entry id past n_groups
    state = (d.scores, d.ptr, d.log)
    yb, yhb, eb, tb = _dev(_batch(rng, 100, 32, "uniform", "ties", 5))
    yhb[7] = float("nan")
    with pytest.raises(_lib.PertGnnError, match="NaN"):
        d.insert(yb, yhb, eb, tb)
    yhb[7] = 0.0
    eb[3] = 40
    with pytest.raises(_lib.PertGnnError, match="entry id"):
        d.insert(yb, yhb, eb, tb, n_groups=40)
    assert d.scores is state[0] and d.ptr is state[1] and all(a is b for a, b in zip(d.log, state[2]))
    d.insert(yb, yhb, eb, tb, n_groups=41)                        # the same batch with room for id 40 goes in
    assert d.n_groups == 41 and d.log_y.numel() == 20100
    # refused before any launch: operands on another device than the table
    l0 = ops.LAUNCHES["n"]
    for call in (lambda: d.insert(yb.cpu(), yhb, eb, tb), lambda: d.insert(yb, yhb, eb, tb.cpu()),
                 lambda: d.to("cpu").evict(3)):
        with pytest.raises(_lib.PertGnnError):
            call()
    assert ops.LAUNCHES["n"] == l0


# ------------------------------------------------------------------------------------------------------ end to end
def _time_chunks(cols, n_chunks):
    """The trace table cut into chunks of whole traces by their first timestamp."""
    tid = cols["traceid"]
    u, inv = np.unique(tid, return_inverse=True)
    first = np.full(u.size, np.iinfo(np.int64).max)
    np.minimum.at(first, inv, cols["timestamp"])
    edges = np.quantile(first, np.linspace(0, 1, n_chunks + 1)[1:-1])
    c = np.searchsorted(edges, first, side="right")[inv]
    return [{k: v[c == j].copy() for k, v in cols.items()} for j in range(n_chunks)]


def test_end_to_end_serving_loop(monkeypatch):
    from pert_gnn_kdd23_b200 import train
    from pert_gnn_kdd23_b200.model import SAGEDeterministic
    from pert_gnn_kdd23_b200.store import StoreLoader
    from pert_gnn_kdd23_b200.synthetic import make_random_trace_table
    from pert_gnn_kdd23_b200.train import (ScoreDistribution, calibrate, fit_distribution, grow_embeddings, predict,
                                           score_traces)
    from tests.helpers import assert_close
    from tests.test_gpu_trace_evict import _store

    cols = make_random_trace_table(23, 6000, rows=(1, 8), n_patterns=220, n_entries=10, n_ms=64, n_if=16,
                                   span=300000)
    chunks = _time_chunks(cols, 4)
    chunks[3]["entryid"][chunks[3]["entryid"] == 3] = 10                    # entry 10 is new to the store
    s = _store(chunks[0], "span", ([(0, 3)], np.ones((1, 8))), 64)
    torch.manual_seed(0)
    m = SAGEDeterministic(9, [64], 7, 32, 6, 32, 2, 0.0).cuda()
    grow_embeddings(m, store=s, seed=1)
    ids = np.arange(len(s))
    ts = s.t["trace_ts"][torch.from_numpy(ids).cuda()]
    d = fit_distribution(m, StoreLoader(s, ids, 64), "cuda", ts=ts)
    assert d.log_y.numel() == len(s) and torch.equal(d.log_ts, ts)
    sid = ids.copy()                                                         # the store index of every log row

    seen, real = [], train._replayed_predictions

    def spy(*a, **k):
        out = real(*a, **k)
        seen.append(tuple(t.clone() for t in out))
        return out

    monkeypatch.setattr(train, "_replayed_predictions", spy)
    for j in (1, 2, 3):
        new = s.append_traces(chunks[j])
        grow_embeddings(m, store=s, seed=j)
        new_ids = np.arange(new.start, new.stop)
        bts = s.t["trace_ts"].cpu().numpy()
        cut = int(np.quantile(bts, 0.3)) + 1
        before = ScoreDistribution(d.level, d.scores, d.ptr, d.by, d.min_count, d.column)
        log_ts = d.log_ts.cpu().numpy()
        p = d.add_traces(m, s, new_ids, evict_before=cut, batch_size=64)
        y_n, yh_n, e_n = seen[-1]
        assert torch.equal(p, before.pvalues(yh_n, e_n, y_n))            # test, then insert
        assert p.dtype == torch.float64 and p.numel() == new_ids.size
        # the logged ŷ of the chunk against a fresh forward on the same store state (a trace's inputs follow its
        # entry's live pattern mix, which the next append or evict re-weights)
        kept_new = torch.from_numpy(bts[new_ids] >= cut).cuda()
        _, yh_fresh, _ = real(m, StoreLoader(s, new_ids, 64), "cuda", 32, "check")
        assert_close(d.log_yhat[d.log_yhat.numel() - int(kept_new.sum()):], yh_fresh[kept_new, 0],
                     what="logged predictions vs a fresh forward")
        remap = s.evict_traces(cut)
        kept = np.concatenate([log_ts, bts[new_ids]]) >= cut
        sid = remap[np.concatenate([sid, new_ids])]
        assert np.array_equal(sid >= 0, kept)
        sid = sid[kept]
        assert d.n_groups == m.entry_embeds.num_embeddings
        assert d.log_y.numel() == len(s) == sid.size
        # the table is the fit of its log; the log's labels, entries and buckets are the store's survivors'
        ref = ScoreDistribution.fit(d.log_y, d.log_yhat, d.log_entry, d.n_groups, d.level)
        assert torch.equal(d.ptr, ref.ptr) and np.array_equal(_bits(d.scores), _bits(ref.scores))
        y_f, _, e_f = real(m, StoreLoader(s, sid, 64), "cuda", 32, "check")
        assert torch.equal(d.log_y, y_f) and torch.equal(d.log_entry, e_f)
        assert torch.equal(d.log_ts, s.t["trace_ts"][torch.from_numpy(sid).cuda()])
    assert 10 < m.entry_embeds.num_embeddings
    monkeypatch.undo()

    # the calls without the new arguments: same launches and results before and after another update
    ids = np.arange(len(s))
    ent = s._h_trace_entry.astype(np.int64)
    q_ts = s.t["trace_ts"].cpu().numpy()
    loader = StoreLoader(s, ids, 64)

    def calls():
        out, n = [], []
        for f in (lambda: predict(m, s, ent, q_ts, batch_size=256, asof=True),
                  lambda: calibrate(m, loader, "cuda").offsets,
                  lambda: fit_distribution(m, loader, "cuda").scores,
                  lambda: score_traces(m, loader, "cuda", d0)):
            l0 = ops.LAUNCHES["n"]
            out.append(f())
            n.append(ops.LAUNCHES["n"] - l0)
        return out, n

    d0 = ScoreDistribution(d.level, d.scores, d.ptr, d.by, d.min_count, d.column)
    calls()                                                                   # warm the graph cache
    out0, n0 = calls()
    d.add_traces(m, s, ids[-50:])
    out1, n1 = calls()
    assert n0 == n1
    assert_close(out1[0], out0[0], what="predict before and after add_traces")
    assert_close(out1[1], out0[1], what="calibrate before and after add_traces")
    assert out1[2].numel() == out0[2].numel()
    step = 1.0 / (d0.counts[-1].item() + 1)
    assert (out1[3] - out0[3]).abs().max().item() <= 2 * step + 1e-12
