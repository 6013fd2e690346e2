"""FMRegressor on the CPU: the numpy restatement (tests/fm_regression_oracle.py) against the PySpark doctest's known
answer, central differences of the squared loss, and the shim's params and refusals."""
import numpy as np
import pytest
import torch

import fm_oracle as fo
import fm_regression_oracle as fro


def test_the_restatement_reproduces_the_pyspark_doctest():
    X, y = fro.doctest_data()
    w, hist, it = fro.fit(X, y, k=2, seed=16)
    V, lin, b = fo.split(w, 1, 2, True, True)
    d = fro.DOCTEST
    pred = fo.raw(w, np.array(d["x"])[:, None], 1, 2)
    assert np.max(np.abs(pred - np.array(d["prediction"]))) <= 1e-14 * 4
    assert abs(b - d["intercept"]) <= 1e-14
    r = fo.JavaRandom(16)
    # D = 1: the factor gradient is 0 up to the rounding of its two sums, which adamW's epsilon turns into steps of 1e-10
    assert np.max(np.abs(V.reshape(-1) - [r.next_gaussian() * 0.01, r.next_gaussian() * 0.01])) <= 1e-8
    assert it == len(hist) and hist[0] == np.mean(y * y)


def test_the_factor_two_matters():
    """with g = r - y the same loop misses the doctest's printed predictions"""
    X, y = fro.doctest_data()
    orig = fro.sums
    try:
        def half(*a, **kw):
            loss, g = orig(*a, **kw)
            return loss, g / 2
        fro.sums = half
        w, _, _ = fro.fit(X, y, k=2, seed=16)
    finally:
        fro.sums = orig
    assert np.max(np.abs(fo.raw(w, np.array(fro.DOCTEST["x"])[:, None], 1, 2) - fro.DOCTEST["prediction"])) > 1e-12


@pytest.mark.parametrize("fl,fi", [(True, True), (False, True), (True, False), (False, False)])
def test_gradient_equals_central_differences(fl, fi):
    rng = np.random.default_rng(3)
    D, k = 5, 3
    X = rng.normal(0.0, 1.0, (60, D)) * (rng.random((60, D)) < 0.6)
    y = rng.normal(0.0, 2.0, 60)
    w = rng.normal(0.0, 0.4, D * k + D * fl + fi)
    _, g = fro.sums(w, X, y, D, k, fl, fi)
    h = 1e-6
    for j in range(w.shape[0]):
        e = np.zeros_like(w)
        e[j] = h
        fd = (fro.sums(w + e, X, y, D, k, fl, fi)[0] - fro.sums(w - e, X, y, D, k, fl, fi)[0]) / (2 * h)
        assert abs(fd - g[j]) <= 1e-6 * max(1.0, abs(g[j])), j


def test_defaults_and_param_validation():
    from pyspark.ml.feature import IllegalArgumentException
    from pyspark.ml.regression import FMRegressionModel, FMRegressor
    s = FMRegressor()
    want = {"factorSize": 8, "fitIntercept": True, "fitLinear": True, "regParam": 0.0, "miniBatchFraction": 1.0,
            "initStd": 0.01, "maxIter": 100, "stepSize": 1.0, "tol": 1e-6, "solver": "adamW", "seed": None,
            "weightCol": None, "featuresCol": "features", "labelCol": "label", "predictionCol": "prediction"}
    assert {k: s.getOrDefault(k) for k in want} == want
    p = FMRegressor(factorSize=2, fitIntercept=False, fitLinear=False, regParam=0.5, miniBatchFraction=0.25, initStd=0.0,
                    maxIter=0, stepSize=0.1, tol=0.0, solver="gd", seed=16)._check()
    assert (p.factor_size, p.fit_intercept, p.fit_linear, p.reg_param, p.mini_batch_fraction, p.init_std, p.max_iter,
            p.step_size, p.tol, p.solver, p.seed) == (2, False, False, 0.5, 0.25, 0.0, 0, 0.1, 0.0, "gd", 16)
    assert FMRegressor()._check().seed == FMRegressor()._check().seed
    for bad in ({"factorSize": 0}, {"factorSize": 2.5}, {"regParam": -0.1}, {"initStd": -1.0}, {"miniBatchFraction": 0.0},
                {"miniBatchFraction": 1.5}, {"maxIter": -1}, {"maxIter": 1.5}, {"stepSize": 0.0}, {"tol": -1e-9},
                {"solver": "lbfgs"}, {"weightCol": "w"}):
        with pytest.raises(IllegalArgumentException):
            FMRegressor(**bad)._check()
    for foreign in ({"thresholds": [0.5, 0.5]}, {"probabilityCol": "p"}):
        with pytest.raises(TypeError):
            FMRegressor(**foreign)
    assert FMRegressionModel._all_defaults()["factorSize"] == 8


def test_weight_col_is_refused_at_fit():
    from pyspark.ml.feature import IllegalArgumentException
    from pyspark.ml.regression import FMRegressor
    from pyspark.sql import ColumnData

    class _Frame:
        _cols = {"features": ColumnData("vector", torch.zeros((4, 2), dtype=torch.float64), "f64"),
                 "label": ColumnData("numeric", torch.zeros(4, dtype=torch.float64), "f64")}

    with pytest.raises(IllegalArgumentException, match="weightCol"):
        FMRegressor(weightCol="w").fit(_Frame())
