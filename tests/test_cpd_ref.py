"""CPU tests of the numpy restatement of the conformal predictive distribution (tests/cpd_ref.py): the vectorised
table, tail counts and quantiles agree with the brute-force forms on ties, +-0, subnormals, +-1e30, empty groups and
groups of one; the quantile equals the calibration's restatement where both answer; each defect switch changes a
result the GPU tests compare bit for bit."""
import numpy as np
import pytest

from tests import calib_ref
from tests import cpd_ref as R


def _edge_set():
    """Ties, +-0, subnormals, +-1e30; group 0 empty, group 1 of one graph, group 4 out of every query's min_count."""
    y = np.array([0, 0, 1, 2, 2, 0, 1, 0, 0, 2, 1, 1, 0], dtype=np.int64)
    yhat = np.array([0.0, -0.0, 1e-40, -1e-40, 1e30, -1e30, 1.0, 2.5, 0.0, 2.0, 0.5, -1.0, 1e-40], dtype=np.float32)
    g = np.array([1, 2, 2, 2, 3, 3, 3, 3, 2, 3, 4, 4, 2], dtype=np.int64)
    return y, yhat, g, 6


def _queries(tab, G):
    """Predictions, ids on both sides of [0, G) and thresholds equal to stored scores, +-0, +-inf and between."""
    rng = np.random.default_rng(0)
    stored = np.unique(tab)
    Q = 40
    yhat = rng.choice(np.array([0.0, -0.0, 1.0, 1e-40, -2.5], np.float32), Q)
    ids = rng.integers(-2, G + 3, Q)
    pool = np.concatenate([stored, [0.0, -0.0, np.inf, -np.inf, 0.25, 1e-41]]).astype(np.float32)
    x = (rng.choice(pool, (Q, 3)) + yhat[:, None]).astype(np.float32)
    x[:, 0] = rng.choice(pool, Q)
    return yhat, ids, x


@pytest.mark.parametrize("grouped", [True, False])
def test_table_matches_brute(grouped):
    y, yhat, g, G = _edge_set()
    gg = g if grouped else None
    a, pa = R.table(y, yhat, gg, G)
    b, pb = R.table_brute(y, yhat, gg, G)
    assert np.array_equal(pa, pb) and np.array_equal(a.view(np.int32), b.view(np.int32))
    assert not np.signbit(a[a == 0]).any()                           # -0 canonicalised
    assert pa[-1] == (2 * y.size if grouped else y.size)
    if grouped:
        assert pa[1] - pa[0] == 0 and pa[2] - pa[1] == 1             # an empty group and a group of one


@pytest.mark.parametrize("min_count", [1, 2, 5])
def test_tail_matches_brute(min_count):
    y, yhat, g, G = _edge_set()
    tab, ptr = R.table(y, yhat, g, G)
    qh, ids, x = _queries(tab, G)
    for kw in (dict(x=x), dict(x=x[:, :1]), dict(y=np.abs(ids) % 3)):
        got = R.tail(tab, ptr, min_count, qh, ids, **kw)
        want = R.tail_brute(tab, ptr, min_count, qh, ids, **kw)
        for a, b in zip(got, want):
            assert np.array_equal(a, b), kw
    ge, gt, row = R.tail(tab, ptr, min_count, qh, ids, x=x)
    assert (ge >= gt).all()
    lo, hi = R.probabilities(ge, gt, row, ptr)
    assert ((0 <= lo) & (lo < hi) & (hi <= 1)).all()
    assert (row[(ids < 0) | (ids >= G)] == G).all()
    assert (row[ids == 0] == G).all()                               # the empty group falls back


def test_quantile_matches_brute_and_the_calibration():
    y, yhat, g, G = _edge_set()
    tab, ptr = R.table(y, yhat, g, G)
    qh, ids, _ = _queries(tab, G)
    levels = (0.0, 0.1, 0.5, 0.9, 0.95)
    for min_count in (1, 3):
        got = R.quantile(tab, ptr, min_count, qh, ids, levels)
        assert np.array_equal(got.view(np.int32), R.quantile_brute(tab, ptr, min_count, qh, ids, levels).view(np.int32))
    # where the calibration can fit (0.9 needs 9 graphs: n = 13), the quantile is its offset added as the apply adds it
    lv = (0.0, 0.5, 0.9)
    off, _, _ = calib_ref.offsets(y, np.repeat(yhat[:, None], len(lv), 1), g, G, lv, min_count=2)
    want = calib_ref.apply(np.repeat(qh[:, None], len(lv), 1), ids, off)
    assert np.array_equal(R.quantile(tab, ptr, 2, qh, ids, lv).view(np.int32), want.view(np.int32))
    # 0.95 needs 19 graphs: no finite bound anywhere, +inf exactly
    assert np.isinf(R.quantile(tab, ptr, 1, qh, ids, (0.95,))).all()


def test_pvalue_definition():
    y, yhat, g, G = _edge_set()
    tab, ptr = R.table(y, yhat, g, G)
    # every held-out graph scored against its own row: p = (1 + #{s_i >= s}) / (m + 1) > 0 and <= 1
    p = R.pvalues(tab, ptr, 1, yhat, g, y)
    assert ((p > 0) & (p <= 1)).all()
    ge, gt, row = R.tail_brute(tab, ptr, 1, yhat, g, y=y)
    m = ptr[row + 1] - ptr[row]
    assert np.array_equal(p, (ge[:, 0] + 1) / (m + 1))


@pytest.mark.parametrize("defect", ["swap_ge_gt", "no_plus1", "k_n", "no_fallback", "row_shift"])
def test_defects_are_caught(defect):
    """Each defect changes a result the GPU tests compare bit for bit against the restatement."""
    rng = np.random.default_rng(5)
    y, yhat, g = R.make_set(rng, 3000, 16, "zipf", "normal")
    g[g == 3] = 4                                                   # group 3 empty
    tab, ptr = R.table(y, yhat, g, 16)
    qh = yhat[:500]
    ids = np.concatenate([g[:495], [3, 3, -1, 16, 99]])
    x = np.stack([y[:500].astype(np.float32), qh + 1.0], 1)
    mc = 150
    if defect in ("swap_ge_gt", "no_fallback", "row_shift"):
        assert any(not np.array_equal(a, b) for a, b in zip(R.tail(tab, ptr, mc, qh, ids, x=x),
                                                            R.tail(tab, ptr, mc, qh, ids, x=x, defect=defect)))
    if defect in ("no_plus1", "swap_ge_gt"):
        assert not np.array_equal(R.pvalues(tab, ptr, mc, qh, ids, y[:500]),
                                  R.pvalues(tab, ptr, mc, qh, ids, y[:500], defect=defect))
    if defect in ("k_n", "no_fallback", "row_shift"):
        levels = (0.1, 0.5, 0.9, 0.99)
        assert not np.array_equal(R.quantile(tab, ptr, mc, qh, ids, levels).view(np.int32),
                                  R.quantile(tab, ptr, mc, qh, ids, levels, defect=defect).view(np.int32))


def test_make_set_kinds():
    rng = np.random.default_rng(1)
    y, yhat, _ = R.make_set(rng, 10000, 4, "uniform", "top_byte")
    keys = R.scores(y, yhat).view(np.uint32) ^ np.uint32(0x80000000)
    assert np.unique(keys >> 24).size == 1 and np.unique((keys >> 16) & 255).size > 64
    y, yhat, _ = R.make_set(rng, 1000, 4, "uniform", "equal")
    assert np.unique(R.scores(y, yhat)).size == 1
