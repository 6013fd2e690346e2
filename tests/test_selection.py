"""Feature selection on the CPU: the numpy restatement (tests/selection_oracle.py) pinned to the PySpark doctest, scipy and
scikit-learn; b200flow.selection's incomplete gamma and beta pinned to scipy; the selection rules; and the host half of
b200flow/selection.py against the restatement bit for bit."""
import math

import numpy as np
import pytest
from scipy import special, stats

import selection_oracle as so
from b200flow import selection as bs


def _classes(n, D, k, seed, shift=0.3):
    rng = np.random.default_rng(seed)
    y = rng.integers(0, k, n).astype(np.float64)
    x = rng.normal(size=(n, D)) + shift * y[:, None] * rng.normal(size=D)
    return x, y


def _categorical(n, D, k, seed):
    rng = np.random.default_rng(seed)
    y = rng.integers(0, k, n).astype(np.float64)
    x = rng.integers(0, 4, (n, D)).astype(np.float64)
    x[:, ::3] = np.minimum(x[:, ::3] + (y[:, None] > 0), 4)          # every third feature depends on the label
    return x, y


def test_pyspark_doctest_known_answer():
    x = np.array([[0, 0, 1], [1, 0, 1], [2, 1, 1], [3, 1, 1]], np.float64)
    y = np.array([0, 0, 1, 1], np.float64)
    p, dof, st = so.chi_square(x, y)
    assert list(dof) == [3, 1, 0]
    assert st[0] == 4.0 and st[2] == 0.0 and p[2] == 1.0
    assert abs(p[0] - 0.2614641299491107) < 1e-15


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_chi_square_equals_scipy(seed):
    x, y = _categorical(3000, 7, 3 + seed, seed)
    p, dof, st = so.chi_square(x, y)
    for j in range(x.shape[1]):
        _, t = so.contingency(x[:, j:j + 1], y)
        s, pv, df, _ = stats.chi2_contingency(t[0], correction=False)
        assert dof[j] == df
        assert abs(st[j] - s) <= 1e-10 * s
        assert abs(p[j] - pv) <= 1e-12


def test_anova_and_f_value_equal_scipy_and_sklearn():
    fs = pytest.importorskip("sklearn.feature_selection")
    x, y = _classes(5000, 9, 5, 4, shift=0.02)
    p, dof, f = so.anova(x, y)
    fk, pk = fs.f_classif(x, y)
    for j in range(x.shape[1]):
        fo, po = stats.f_oneway(*[x[y == c, j] for c in range(5)])
        assert abs(f[j] - fo) <= 1e-10 * fo and abs(f[j] - fk[j]) <= 1e-10 * fk[j]
        assert abs(p[j] - po) <= 1e-12 and abs(p[j] - pk[j]) <= 1e-12
    assert list(dof) == [4999] * 9
    rng = np.random.default_rng(5)
    yc = x[:, 0] * 0.01 + x[:, 3] * 0.03 + rng.normal(size=5000)
    p, dof, f = so.f_value(x, yc)
    fr, pr = fs.f_regression(x, yc)
    assert np.all(np.abs(f - fr) <= 1e-10 * fr) and np.all(np.abs(p - pr) <= 1e-12)
    assert list(dof) == [4998] * 9


def test_selection_rules_equal_sklearn_without_ties():
    fs = pytest.importorskip("sklearn.feature_selection")
    x, y = _classes(400, 30, 3, 6, shift=0.15)
    p, _, _ = so.anova(x, y)
    assert len(set(p)) == len(p)
    for mode, t, sk in (("fpr", 0.05, fs.SelectFpr(fs.f_classif, alpha=0.05)),
                        ("fdr", 0.2, fs.SelectFdr(fs.f_classif, alpha=0.2)),
                        ("fwe", 0.5, fs.SelectFwe(fs.f_classif, alpha=0.5)),
                        ("numTopFeatures", 7, fs.SelectKBest(fs.f_classif, k=7))):
        want = list(np.flatnonzero(sk.fit(x, y).get_support()))
        assert bs.select(p, mode, t) == want == so.select(p, mode, t), mode
        assert want, mode


def test_selection_rules_with_ties_nan_and_empty_results():
    p = np.array([0.5, np.nan, 0.01, 0.5, 0.01, 0.2, np.nan])
    assert bs.select(p, "numTopFeatures", 3) == [2, 4, 5]
    assert bs.select(p, "numTopFeatures", 4) == [0, 2, 4, 5]        # ties by index
    assert bs.select(p, "numTopFeatures", 6) == [0, 1, 2, 3, 4, 5]  # NaN last, the lower index first
    assert bs.select(p, "numTopFeatures", 50) == list(range(7))
    assert bs.select(p, "percentile", 0.3) == [2, 4]                # (7 * 0.3).toInt = 2
    assert bs.select(p, "percentile", 0.99) == [0, 1, 2, 3, 4, 5]   # (7 * 0.99).toInt = 6
    assert bs.select(p, "fpr", 0.01) == [] and bs.select(p, "fpr", 0.0100001) == [2, 4]
    assert bs.select(p, "fwe", 0.05) == [] and bs.select(p, "fwe", 0.08) == [2, 4]
    assert bs.select(p, "fdr", 0.001) == []
    assert bs.select(p, "fdr", 0.04) == [2, 4]                      # 0.01 <= 0.04 * 2 / 7, 0.2 > 0.04 * 3 / 7
    assert bs.select(p, "fdr", 1.0) == [0, 2, 3, 4, 5]              # NaN never passes
    for mode, t in (("numTopFeatures", 3), ("numTopFeatures", 4), ("numTopFeatures", 6), ("percentile", 0.3), ("fpr", 0.3),
                    ("fwe", 0.5), ("fdr", 0.5), ("fdr", 1.0)):
        assert bs.select(p, mode, t) == so.select(p, mode, t), mode


def test_special_functions_equal_scipy():
    for dof in (1, 2, 3, 7, 22, 118, 1000, 25000, 1e6, 4.9e6, 5e6):
        a = dof / 2.0
        for x in (1e-300, 1e-8, 0.1, 0.5 * a, a - 3 * math.sqrt(a), a - 1, a, a + 1, a + 1.5, a + math.sqrt(a),
                  a + 5 * math.sqrt(a), a + 12 * math.sqrt(a), 2 * a + 50, 1e3 * a + 1e3):
            if x >= 0.0:
                assert abs((1.0 - bs.gamma_p(a, x)) - (1.0 - special.gammainc(a, x))) <= 1e-12, (dof, x)
    for d1, d2 in ((1, 1), (1, 2), (2, 10), (22, 100), (255, 3), (4, 1e4)):
        for f in (1e-9, 0.01, 0.5, 0.9, 1.0, 1.3, 2.0, 5.0, 30.0, 1e3, 1e8):
            want = special.betainc(d1 / 2.0, d2 / 2.0, d1 * f / (d1 * f + d2))
            assert abs((1.0 - bs.f_cdf(f, d1, d2)) - (1.0 - want)) <= 1e-12, (d1, d2, f)


D2_LARGE = (1e5, 5e5, 9e5, 4.9e6, 5e6)       # up to n for KDD-full, where scipy's betainc is no reference at 1e-12


def _f_tail_even(f, d1, d2):
    """1 - cdf of F(d1, d2) at f for even d1, in 60-digit decimal arithmetic from the closed form
    (1 - x)^b sum over j < a of (b)_j x^j / j!, a = d1 / 2, b = d2 / 2, x = d1 f / (d1 f + d2)."""
    from decimal import Decimal, localcontext
    with localcontext() as ctx:
        ctx.prec = 60
        F, D1, D2 = Decimal(f), Decimal(d1), Decimal(d2)
        x, y, b = D1 * F / (D1 * F + D2), D2 / (D1 * F + D2), D2 / 2
        term = s = Decimal(1)
        for j in range(1, d1 // 2):
            term = term * (b + j - 1) * x / j
            s += term
        return float((b * y.ln()).exp() * s)


@pytest.mark.parametrize("d2", (1.0, 2.0, 10.0, 1e4) + D2_LARGE)
def test_f_tail_equals_the_exact_closed_form_for_even_d1(d2):
    for d1 in (2, 4, 22, 118, 254):
        for f in (1e-9, 0.01, 0.5, 0.9, 1.0, 1.1, 1.3, 2.0, 5.0, 30.0, 1e3, 1e8):
            assert abs((1.0 - bs.f_cdf(f, float(d1), d2)) - _f_tail_even(f, d1, d2)) <= 1e-12, (d1, d2, f)


@pytest.mark.parametrize("d2", D2_LARGE)
def test_f_tail_equals_a_40_digit_evaluation_for_odd_d1(d2):
    """odd d1 (d1 = 1 is every F-value test) has no finite closed form: the reference is the positive hypergeometric form
    I_x(a, b) = x^a y^b / (a B(a, b)) 2F1(a + b, 1; a + 1; x) at 40 digits, itself checked against the closed form."""
    mp = pytest.importorskip("mpmath")

    def cdf(f, d1):
        with mp.workdps(40):
            F = mp.mpf(f)
            x, y, a, b = d1 * F / (d1 * F + d2), mp.mpf(d2) / (d1 * F + d2), mp.mpf(d1) / 2, mp.mpf(d2) / 2
            return float(1 - x ** a * y ** b / (a * mp.beta(a, b)) * mp.hyp2f1(a + b, 1, a + 1, x))

    assert abs(cdf(1.3, 22) - _f_tail_even(1.3, 22, d2)) <= 1e-15
    for d1 in (1, 3, 21):
        for f in (1e-9, 0.01, 0.5, 1.0, 1.3, 2.0, 5.0, 30.0):
            assert abs((1.0 - bs.f_cdf(f, float(d1), d2)) - cdf(f, d1)) <= 1e-12, (d1, d2, f)


def test_dictionaries_merge_at_the_distinct_value_limit():
    """10,000 distinct values across two ranks are accepted, 10,001 are refused on every rank, and so is a column one rank
    alone flagged as overflowing."""
    def export(keys, overflow=0.0):
        row = np.full(bs.MAX_CATEGORIES + 2, np.inf)
        k = np.sort(np.asarray(keys, np.float64))[:bs.MAX_CATEGORIES + 1]
        row[:len(k)] = k
        row[-1] = overflow
        return row[None, :]

    a, b = export(np.arange(0.0, 6000.0)), export(np.arange(4000.0, 10000.0))
    d = bs.merge_dictionaries([a, b], "test")
    assert len(d) == 1 and np.array_equal(d[0], np.arange(10000.0))
    with pytest.raises(bs.TooManyValuesError, match="more than 10000 distinct values in column 0"):
        bs.merge_dictionaries([a, export(np.arange(4000.0, 10001.0))], "test")
    with pytest.raises(bs.TooManyValuesError, match="column 1"):
        bs.merge_dictionaries([np.concatenate([a, a]), np.concatenate([b, export([1.0], overflow=1.0)])], "test")
    assert len(so.dictionary(np.arange(10001.0) % 10000)) == 10000 and len(so.dictionary(np.arange(10001.0))) == 10001


def test_p_is_exactly_zero_where_one_minus_cdf_rounds_to_zero():
    assert 1.0 - bs.chi2_cdf(1e4, 3.0) == 0.0 and 1.0 - bs.chi2_cdf(800.0, 1.0) == 0.0
    assert 1.0 - bs.f_cdf(1e6, 3.0, 1e6) == 0.0 and 1.0 - bs.f_cdf(math.inf, 3.0, 10.0) == 0.0
    assert bs.chi2_cdf(0.0, 4.0) == 0.0 and bs.f_cdf(0.0, 2.0, 5.0) == 0.0
    assert math.isnan(bs.chi2_cdf(math.nan, 2.0)) and math.isnan(bs.f_cdf(math.nan, 2.0, 5.0))


def test_degenerate_statistics():
    x = np.array([[1.0, 5.0, 2.0], [1.0, 5.0, 3.0], [2.0, 5.0, 2.5], [2.0, 5.0, 4.0]])
    y = np.array([0.0, 0.0, 1.0, 1.0])
    p, _, f = so.anova(x, y)
    assert f[0] == math.inf and p[0] == 0.0                         # constant within each class, different between
    assert math.isnan(f[1]) and math.isnan(p[1])                    # constant: 0 / 0
    res = bs.anova_from_totals(*_anova_totals(x, y))
    assert res.p_values[0] == 0.0 and math.isnan(res.p_values[1])


def test_minus_zero_and_plus_zero_are_one_category():
    x = np.array([[0.0], [-0.0], [1.0], [-0.0]])
    y = np.array([0.0, 1.0, 0.0, 1.0])
    d = so.dictionary(x[:, 0])
    assert len(d) == 2 and str(d[0]) == "0.0"
    _, t = so.contingency(x, y)
    assert t[0].tolist() == [[1, 2], [1, 0]]


def test_large_mean_needs_two_passes():
    rng = np.random.default_rng(4)
    n = 20000
    y = rng.integers(0, 3, n).astype(np.float64)
    x = (1e9 + rng.normal(size=n) + 0.05 * y).reshape(-1, 1)
    _, _, f = so.anova(x, y)
    fo, _ = stats.f_oneway(*[x[y == c, 0] - 1e9 for c in range(3)])
    assert abs(f[0] - float(fo)) <= 1e-3 * float(fo)                # the class means' rounding at 1e9 bounds SSB
    # the one-pass form (raw sums of squares) loses the within-class spread at this mean
    ss = float((x[:, 0] * x[:, 0]).sum()) - float(x[:, 0].sum()) ** 2 / n
    ssb = sum(float(x[y == c, 0].sum()) ** 2 / (y == c).sum() for c in range(3)) - float(x[:, 0].sum()) ** 2 / n
    one_pass = (ssb / 2) / ((ss - ssb) / (n - 3))
    assert not abs(one_pass - float(fo)) <= 1e-2 * float(fo)


def _anova_totals(x, y):
    labels = so.dictionary(y)
    ids = np.searchsorted(labels, y)
    k = len(labels)
    sums = so.chain(so.group_sum_partials(x, ids, k, 0))
    cnt = np.bincount(ids, minlength=k)
    return sums, cnt, so.chain(so.centered_partials(x, ids, k, sums / cnt.astype(float)[:, None], None, 0.0, 0))


def test_host_half_equals_the_restatement_bit_for_bit():
    x, y = _categorical(6000, 6, 4, 9)
    res = bs.chi_square_from_counts(so.contingency(x, y)[1])
    for a, b in zip((res.p_values, res.dof, res.statistics), so.chi_square(x, y)):
        assert a.tobytes() == np.asarray(b).astype(a.dtype).tobytes()
    x, y = _classes(6000, 5, 4, 10, shift=0.05)
    res = bs.anova_from_totals(*_anova_totals(x, y))
    for a, b in zip((res.p_values, res.dof, res.statistics), so.anova(x, y)):
        assert a.tobytes() == np.asarray(b).astype(a.dtype).tobytes()
    yc = x[:, 1] * 0.02 + np.random.default_rng(1).normal(size=6000)
    n, D = x.shape
    mx = so.chain(so.group_sum_partials(x, None, 1, 0))[0] * (1.0 / n)
    my = so.chain(so.group_sum_partials(yc.reshape(-1, 1), None, 1, 0))[0, 0] * (1.0 / n)
    t = so.chain(so.centered_partials(x, None, 1, mx[None, :], yc, my, 0))[0]
    res = bs.f_value_from_totals(t[:D], t[D:2 * D], float(t[2 * D]), n)
    for a, b in zip((res.p_values, res.dof, res.statistics), so.f_value(x, yc)):
        assert a.tobytes() == np.asarray(b).astype(a.dtype).tobytes()
    assert np.allclose(so.variances(x), x.var(0, ddof=1), rtol=1e-12)


def test_shim_parameters_are_validated():
    from pyspark.ml.feature import (ChiSqSelector, IllegalArgumentException, UnivariateFeatureSelector,
                                    VarianceThresholdSelector, _check_selection)
    s = UnivariateFeatureSelector(featuresCol="f", outputCol="o", labelCol="l")
    assert s.getSelectionMode() == "numTopFeatures" and s.getSelectionThreshold() is None
    assert s.setFeatureType("categorical") is s and s.getFeatureType() == "categorical"
    with pytest.raises(IllegalArgumentException, match="Unsupported combination"):
        s.setLabelType("continuous")._fit(None)
    with pytest.raises(IllegalArgumentException, match="featureType"):
        UnivariateFeatureSelector()._fit(None)
    with pytest.raises(IllegalArgumentException, match="selectionMode"):
        UnivariateFeatureSelector(selectionMode="kbest").setFeatureType("continuous").setLabelType("continuous")._fit(None)
    for mode, t in (("numTopFeatures", 0), ("percentile", 1.5), ("fpr", -0.1), ("fdr", 2.0), ("fwe", math.nan)):
        with pytest.raises(IllegalArgumentException):
            _check_selection(mode, t)
    assert _check_selection("percentile", 0.0) == 0.0
    c = ChiSqSelector(numTopFeatures=5)
    assert (c.getNumTopFeatures(), c.getSelectorType(), c.getPercentile(), c.getFpr(), c.getFdr(), c.getFwe()) == \
        (5, "numTopFeatures", 0.1, 0.05, 0.05, 0.05)
    with pytest.raises(IllegalArgumentException):
        ChiSqSelector(selectorType="fpr", fpr=3.0)._fit(None)
    with pytest.raises(IllegalArgumentException, match="varianceThreshold"):
        VarianceThresholdSelector(varianceThreshold=-1.0)._fit(None)
    assert VarianceThresholdSelector().getVarianceThreshold() == 0.0
