"""CPU tests of the conformal-calibration restatement (tests/calib_ref.py): the vectorised form agrees with a brute-force
sort of every group on sets with ties, +-0, subnormals, empty groups and groups of one graph; the k rule and the
fallback behave as the contract says; and every defect switch changes the result on a set the GPU tests use, so
their bit-equality would catch the defect."""
import numpy as np
import pytest

from tests import calib_ref as R

TAUS = [(0.5,), (0.0, 0.9), (0.1, 0.5, 0.9), (0.5, 0.9, 0.95, 0.99), (0.0, 0.1, 0.25, 0.5, 0.75, 0.9, 0.95, 0.999)]


def _same(a, b):
    return np.array_equal(np.asarray(a).view(np.int32) if np.asarray(a).dtype == np.float32 else a,
                          np.asarray(b).view(np.int32) if np.asarray(b).dtype == np.float32 else b)


@pytest.mark.parametrize("kind", ["uniform", "sparse", "zipf"])
@pytest.mark.parametrize("score_kind", ["normal", "ties", "extreme"])
@pytest.mark.parametrize("taus", TAUS)
def test_vectorised_equals_brute_force(kind, score_kind, taus):
    rng = np.random.default_rng(hash((kind, score_kind, len(taus))) % 2 ** 32)
    n, G = 3000, 300
    y, yhat, g = R.make_set(rng, n, len(taus), G, kind, score_kind)
    g[:5] = np.arange(5) + G - 5          # a few groups of one graph at the end of the id range
    for min_count in (1, 3, 40):
        got = R.offsets(y, yhat, g, G, taus, min_count)
        want = R.offsets_brute(y, yhat, g, G, taus, min_count)
        for a, b in zip(got, want):
            assert _same(a, b)
    assert (got[1][:G] == 0).any() or kind == "uniform"     # empty groups present


def test_global_only_and_small_sets():
    rng = np.random.default_rng(1)
    for n in (1, 2, 5, 19, 99, 100):
        y, yhat, _ = R.make_set(rng, n, 2, 1, "uniform", "ties")
        taus = (0.0, 0.5)
        got = R.offsets(y, yhat, None, 0, taus)
        want = R.offsets_brute(y, yhat, None, 0, taus)
        for a, b in zip(got, want):
            assert _same(a, b)
        assert got[1].tolist() == [n] and got[2].tolist() == [[1, 1]]


def test_k_rule_and_fallback():
    assert [R.k_of(m, 0.99) for m in (98, 99, 100)] == [99, 99, 100]
    assert not R.own_of(98, 0.99, 1, False) and R.own_of(99, 0.99, 1, False)
    assert R.k_of(5, 0.0) == 1 and R.own_of(1, 0.0, 1, False)
    assert not R.own_of(10, 0.5, 11, False) and R.own_of(10, 0.5, 11, True)
    # a group of 3 at 0.9: k = 4 > 3 -> the global offset; at 0.5: k = 2, its second smallest score
    y = np.array([10, 20, 30, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0], dtype=np.int64)
    yhat = np.zeros((20, 2), dtype=np.float32)
    g = np.array([0, 0, 0] + [1] * 17, dtype=np.int64)
    off, cnt, own = R.offsets(y, yhat, g, 2, (0.5, 0.9))
    assert cnt.tolist() == [3, 17, 20]
    assert off[0, 0] == 20 and own[0, 0] == 1
    assert own[0, 1] == 0 and off[0, 1] == off[2, 1]
    # -0 and +0 are one value: the score of y = 0, yhat = 0 is +0
    s = R.scores(np.array([0]), np.array([[0.0]], dtype=np.float32))
    assert np.signbit(s).sum() == 0


def test_apply_restatement():
    off = np.array([[1.0, -5.0], [2.0, 3.0], [0.5, 0.25]], dtype=np.float32)     # two entries and the global row
    yhat = np.array([[1, 2], [1, 2], [1, 2], [1, 2]], dtype=np.float32)
    g = np.array([0, 1, 7, -1])
    got = R.apply(yhat, g, off)
    assert got.tolist() == [[2, -3], [3, 5], [1.5, 2.25], [1.5, 2.25]]
    assert R.apply(yhat, g, off, monotone=True).tolist() == [[2, 2], [3, 5], [1.5, 2.25], [1.5, 2.25]]
    assert R.apply(yhat, g, off, live=2).tolist() == [[2, -3], [3, 5], [1, 2], [1, 2]]
    assert R.apply(yhat, g, None, monotone=True).tolist() == yhat.tolist()
    assert R.apply(np.array([1, 2], np.float32), np.array([0, 1]), off[:, :1]).tolist() == [2, 4]


def _defect_set():
    rng = np.random.default_rng(7)
    n, G = 20000, 256                     # ~78 graphs per entry: the 0.99 level falls back to the global row
    y, yhat, g = R.make_set(rng, n, 4, G, "uniform")
    return y, yhat, g, G, (0.5, 0.9, 0.95, 0.99)


@pytest.mark.parametrize("defect", ["k_n", "no_fallback"])
def test_fit_defects_change_the_offsets(defect):
    y, yhat, g, G, taus = _defect_set()
    good = R.offsets(y, yhat, g, G, taus)
    bad = R.offsets(y, yhat, g, G, taus, defect=defect)
    assert not _same(good[0], bad[0])


@pytest.mark.parametrize("defect", ["running_min", "row_shift"])
def test_apply_defects_change_the_result(defect):
    y, yhat, g, G, taus = _defect_set()
    off, _, _ = R.offsets(y, yhat, g, G, taus)
    rng = np.random.default_rng(8)
    q = rng.normal(0, 100, (5000, 4)).astype(np.float32)
    qg = rng.integers(0, G, 5000)
    assert not _same(R.apply(q, qg, off, monotone=True), R.apply(q, qg, off, monotone=True, defect=defect))


def test_in_sample_coverage_bound_of_the_restatement():
    y, yhat, g, G, taus = _defect_set()
    off, cnt, own = R.offsets(y, yhat, g, G, taus)
    cal = R.apply(yhat, g, off)
    r = R.roundtrip_slack(y, yhat)
    for grp in range(G):
        m = g == grp
        for t, tau in enumerate(taus):
            if own[grp, t]:
                covered = int((y[m].astype(np.float32) <= cal[m, t]).sum())
                assert covered >= R.k_of(int(cnt[grp]), tau) - int(r[t])
