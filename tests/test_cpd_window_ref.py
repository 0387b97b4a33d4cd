"""CPU tests of the score-window restatement (tests/cpd_window_ref.py): the merged table equals the fit over the log
after every insert and evict, and the brute form, on ties, +-0, subnormals, +-1e30, empty rows, single-score rows, G
growth and the global grouping; each defect switch changes a result the GPU tests compare bit for bit."""
import numpy as np
import pytest

from tests import cpd_ref as R
from tests import cpd_window_ref as W


def _bits(a):
    return np.asarray(a, dtype=np.float32).view(np.int32)


def _same(a, b):
    return a[1].size == b[1].size and np.array_equal(a[1], b[1]) and np.array_equal(_bits(a[0]), _bits(b[0]))


def _batch(rng, k, G, score_kind, kind="uniform", t=0):
    y, yhat, g = R.make_set(rng, k, max(G, 1), kind, score_kind)
    return y, yhat, g % max(G, 1), np.full(k, t, np.int64) + rng.integers(0, 3, k)


def _run(seed, G, score_kind, group=True, grow=0, defect=None, steps=8, k=60, kind="uniform"):
    """A seeded sequence of inserts and evicts on a vectorised window, a brute one and (with ``defect``) a broken
    one; -> the list of (table, log) after every step of each."""
    rng = np.random.default_rng(seed)
    first = _batch(rng, k, G, score_kind, kind)
    wins = [W.Window(*first, G, group=group, defect=d, brute=b)
            for d, b in ((None, False), (None, True), (defect, False))]
    out = [[] for _ in wins]
    t = 3
    for step in range(steps):
        if step % 3 == 2:
            cut = t - 4
            for w in wins:
                try:
                    w.evict(cut)
                except ValueError:
                    pass
        else:
            G_new = wins[0].G + (grow if step == 3 else 0)
            batch = _batch(rng, int(rng.integers(1, 2 * k)), G_new, score_kind, kind, t)
            for w in wins:
                w.insert(*batch, n_groups=G_new)
            t += 2
        for w, o in zip(wins, out):
            o.append(((w.tab.copy(), w.ptr.copy()), [a.copy() for a in w.log]))
    return out


@pytest.mark.parametrize("score_kind", ["normal", "ties", "extreme", "equal"])
@pytest.mark.parametrize("G,group,grow", [(8, True, 0), (5, True, 3), (0, False, 0), (1, True, 0), (40, True, 2)])
def test_merge_equals_fit_on_the_log_and_the_brute_form(score_kind, G, group, grow):
    if not group:
        G = 0
    fast, brute, _ = _run(11 + G, G, score_kind, group, grow)
    rng_w = W.Window(*_batch(np.random.default_rng(0), 5, max(G, 1), score_kind), G, group=group)
    assert rng_w.table()[1].size == (G if group else 0) + 2
    for (tf, lf), (tb, lb) in zip(fast, brute):
        assert _same(tf, tb)
        for a, b in zip(lf, lb):
            assert np.array_equal(a.view(np.int64) if a.dtype == np.int64 else _bits(a),
                                  b.view(np.int64) if b.dtype == np.int64 else _bits(b))


def test_every_step_equals_the_fit_of_its_log():
    rng = np.random.default_rng(5)
    w = W.Window(*_batch(rng, 200, 16, "extreme", "sparse"), 16)
    for step in range(20):
        if step % 4 == 3:
            w.evict(int(np.median(w.log[3])))
        else:
            w.insert(*_batch(rng, int(rng.integers(1, 50)), 16 + step, "extreme", "zipf", step), n_groups=16 + step)
        tab, ptr = w.table()
        assert np.array_equal(ptr, w.ptr) and np.array_equal(_bits(tab), _bits(w.tab)), step


def test_edge_rows_and_values():
    """Empty rows, single-score rows, +-0 (one key), subnormals and +-1e30 in insert and remove."""
    y = np.array([0, 0, 1, 2, 0, 0], np.int64)
    yh = np.array([0.0, -0.0, 1e-40, -1e30, 1e30, 0.0], np.float32)
    g = np.array([0, 0, 2, 2, 3, 0], np.int64)
    ts = np.array([0, 1, 2, 3, 4, 5], np.int64)
    w = W.Window(y, yh, g, ts, 5)
    assert np.diff(w.ptr)[[1, 4]].tolist() == [0, 0]                 # empty rows
    w.insert(np.array([5], np.int64), np.array([5.0], np.float32), np.array([4], np.int64), np.array([6]))
    assert np.diff(w.ptr)[4] == 1                                   # a single-score row
    for cut in (1, 3, 5, 6):
        w.evict(cut)
        tab, ptr = w.table()
        assert np.array_equal(ptr, w.ptr) and np.array_equal(_bits(tab), _bits(w.tab)), cut
    with pytest.raises(ValueError, match="empty"):
        w.evict(100)
    with pytest.raises(ValueError, match="shrinks"):
        w.insert(y, yh, g, ts, n_groups=2)


def test_a_removal_the_table_lacks_is_refused():
    tab, ptr = R.table(np.array([1, 2], np.int64), np.zeros(2, np.float32), np.array([0, 0]), 1)
    dtab, dptr = R.table(np.array([3], np.int64), np.zeros(1, np.float32), np.array([0]), 1)
    with pytest.raises(ValueError):
        W.merge(tab, ptr, dtab, dptr, -1)
    with pytest.raises(ValueError):
        W.merge_brute(tab, ptr, dtab, dptr, -1)
    two, tptr = R.table(np.array([1, 1], np.int64), np.zeros(2, np.float32), np.array([0, 0]), 1)
    with pytest.raises(ValueError):                                 # one copy in the table, two in the delta
        W.merge(tab, ptr, two, tptr, -1)


@pytest.mark.parametrize("defect", ["skip_global", "old_g_at_gold", "remove_all", "unstable"])
def test_each_defect_changes_a_compared_result(defect):
    fast, _, broken = _run(3, 6, "ties", grow=2 if defect == "old_g_at_gold" else 0, defect=defect, steps=9, k=80)
    differs = False
    for (tf, lf), (tb, lb) in zip(fast, broken):
        differs |= not _same(tf, tb) or any(not np.array_equal(a, b) for a, b in zip(lf, lb))
    assert differs, defect
