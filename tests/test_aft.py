"""AFTSurvivalRegression on the CPU: the numpy restatement (tests/aft_oracle.py) against scipy's Weibull fit and
censored log-likelihood, central differences of its gradient, the quantile formula, and the shim's params, validators
and refusals."""
import math

import numpy as np
import pytest
import torch

import aft_oracle as ao


def test_uncensored_intercept_only_fit_equals_scipy_weibull():
    stats = pytest.importorskip("scipy.stats")
    rng = np.random.default_rng(1)
    t = stats.weibull_min.rvs(1.7, scale=3.0, size=4000, random_state=rng)
    x = np.ones((4000, 1))                                    # a constant feature: inv = 0, the intercept-only model
    coef, b, sigma, _ = ao.fit(x, t, np.ones(4000), max_iter=500, tol=1e-12)
    shape, _, scale = stats.weibull_min.fit(t, floc=0)
    assert coef[0] == 0.0
    assert abs(1.0 / sigma - shape) <= 1e-4 * shape and abs(math.exp(b) - scale) <= 1e-4 * scale


def test_censored_fit_minimises_the_weibull_likelihood():
    stats = pytest.importorskip("scipy.stats")
    optimize = pytest.importorskip("scipy.optimize")
    x, t, c, _, _ = ao.weibull_data(20000, 3, 2, censor_rate=0.35)
    assert 0.15 < 1.0 - c.mean() < 0.45
    coef, b, sigma, _ = ao.fit(x, t, c, max_iter=500, tol=1e-14)

    def nll(p):
        lam = np.exp(x @ p[:3] + p[3])
        k = 1.0 / math.exp(p[4])
        return -np.sum(c * stats.weibull_min.logpdf(t, k, scale=lam) + (1 - c) * stats.weibull_min.logsf(t, k, scale=lam))

    start = np.concatenate([coef, [b, math.log(sigma)]])
    res = optimize.minimize(nll, start + 0.05, method="BFGS", options={"gtol": 1e-8})
    assert np.max(np.abs(res.x - start)) <= 1e-5, (res.x, start)
    assert nll(start) <= res.fun + 1e-6 * abs(res.fun)


@pytest.mark.parametrize("fi", [True, False])
def test_gradient_equals_central_differences(fi):
    x, t, c, _, _ = ao.weibull_data(300, 4, 3)
    rng = np.random.default_rng(4)
    v = np.concatenate([rng.normal(0, 0.3, 4), [0.8, -0.2]])
    _, g = ao.objective(v, x, t, c, fi)
    h = 1e-6
    for j in range(v.shape[0]):
        if j == 4 and not fi:
            assert g[j] == 0.0
            continue
        e = np.zeros_like(v)
        e[j] = h
        fd = (ao.objective(v + e, x, t, c, fi)[0] - ao.objective(v - e, x, t, c, fi)[0]) / (2 * h)
        assert abs(fd - g[j]) <= 1e-7 * max(1.0, abs(g[j])), j


def test_an_overflowing_point_is_rejected():
    x, t, c, _, _ = ao.weibull_data(200, 2, 5)
    f, g = ao.objective(np.array([0.0, 0.0, 0.0, -8.0]), x, t, c, True)     # sigma = e^-8: e^z overflows
    assert f == math.inf and not g.any()


def test_quantile_formula_is_the_weibull_ppf():
    stats = pytest.importorskip("scipy.stats")
    x = np.random.default_rng(6).normal(0, 1, (5, 3))
    coef, b, sigma = np.array([0.3, -0.2, 0.1]), 1.1, 0.6
    probs = [0.01, 0.3, 0.5, 0.99]
    q = ao.quantiles(x, coef, b, sigma, probs)
    lam = np.exp(x @ coef + b)
    want = np.stack([stats.weibull_min.ppf(p, 1.0 / sigma, scale=lam) for p in probs], 1)
    assert np.allclose(q, want, rtol=1e-12)
    from b200flow.aft import quantile_factors
    assert np.allclose(quantile_factors(probs, sigma), (-np.log1p(-np.array(probs))) ** sigma, rtol=1e-14)


class _Frame:
    """the columns AFTSurvivalRegression._fit reads, on the host"""

    def __init__(self, x, t, c):
        from pyspark.sql import ColumnData
        self._cols = {"features": ColumnData("vector", torch.as_tensor(x), "f64"),
                      "label": ColumnData("numeric", torch.as_tensor(t, dtype=torch.float64), "f64"),
                      "censor": ColumnData("numeric", torch.as_tensor(c, dtype=torch.float64), "f64")}

    def _column_tensor(self, name):
        return self._cols[name].data


def test_defaults_and_param_validation():
    from pyspark.ml.feature import IllegalArgumentException
    from pyspark.ml.regression import AFTSurvivalRegression, AFTSurvivalRegressionModel
    s = AFTSurvivalRegression()
    want = {"featuresCol": "features", "labelCol": "label", "predictionCol": "prediction", "censorCol": "censor",
            "quantileProbabilities": [0.01, 0.05, 0.1, 0.25, 0.5, 0.75, 0.9, 0.95, 0.99], "quantilesCol": None,
            "fitIntercept": True, "maxIter": 100, "tol": 1e-6, "aggregationDepth": 2, "maxBlockSizeInMB": 0.0}
    assert {k: s.getOrDefault(k) for k in want} == want
    p = AFTSurvivalRegression(maxIter=0, tol=0.0, fitIntercept=False, quantileProbabilities=[0.5])._check()
    assert (p.max_iter, p.tol, p.fit_intercept, p.quantile_probabilities) == (0, 0.0, False, [0.5])
    for bad in ({"maxIter": -1}, {"maxIter": 1.5}, {"tol": -1e-9}, {"aggregationDepth": 1}, {"maxBlockSizeInMB": -1.0},
                {"quantileProbabilities": []}, {"quantileProbabilities": [0.0, 0.5]},
                {"quantileProbabilities": [0.5, 1.0]}, {"quantileProbabilities": [float("nan")]}):
        with pytest.raises(IllegalArgumentException):
            AFTSurvivalRegression(**bad)._check()
    with pytest.raises(TypeError):
        AFTSurvivalRegression(weightCol="w")
    assert AFTSurvivalRegressionModel._all_defaults()["censorCol"] == "censor"


def test_refusals_before_any_device_work():
    """bad params and missing columns raise before the features reach the device"""
    from pyspark.ml.feature import IllegalArgumentException
    from pyspark.ml.regression import AFTSurvivalRegression
    df = _Frame(np.ones((4, 2)), [1.0, 2.0, 3.0, 4.0], [1.0, 0.0, 1.0, 1.0])
    with pytest.raises(IllegalArgumentException, match="quantileProbabilities"):
        AFTSurvivalRegression(quantileProbabilities=[0.0]).fit(df)
    with pytest.raises(IllegalArgumentException, match="does not exist"):
        AFTSurvivalRegression(censorCol="nope").fit(df)
    with pytest.raises(IllegalArgumentException, match="does not exist"):
        AFTSurvivalRegression(labelCol="nope").fit(df)
