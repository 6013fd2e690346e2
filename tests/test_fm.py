"""FMClassifier on the CPU: the numpy restatement (tests/fm_oracle.py) against the PySpark doctest's known answer,
java.util.Random, central differences, the pairwise identity, hand-computed gd and adamW steps, the mini-batch draw and
the shim's params and refusals."""
import math

import numpy as np
import pytest
import torch

import fm_oracle as fo


def test_java_random_gives_the_doctest_draws():
    from b200flow.fm import JavaRandom, init_factors
    r = fo.JavaRandom(11)
    assert [r.next_gaussian() * 0.01, r.next_gaussian() * 0.01] == [0.016270071762169862, -0.0051318174074211735]
    for seed in (0, 11, -5, 2 ** 40 + 3, 1841230984):
        a, b = fo.JavaRandom(seed), JavaRandom(seed)
        assert [a.next_gaussian() for _ in range(9)] == [b.next_gaussian() for _ in range(9)]
        assert np.array_equal(init_factors(3, 5, 0.01, seed).reshape(-1), fo.init_coefficients(3, 5, False, False, 0.01, seed))
    r = fo.JavaRandom(42)                                 # java.util.Random(42).nextInt() is -1170105035
    assert r.next(32) == -1170105035


def test_the_restatement_reproduces_the_pyspark_doctest():
    X, y = fo.doctest_data()
    w, hist, it = fo.fit(X, y, k=2, seed=11)
    V, lin, b = fo.split(w, 1, 2, True, True)
    d = fo.DOCTEST
    assert abs(b - d["intercept"]) <= 1e-12 * abs(d["intercept"])
    assert round(float(lin[0]), 4) == d["linear"][0]
    r = fo.JavaRandom(11)
    assert V.reshape(-1).tolist() == [r.next_gaussian() * 0.01, r.next_gaussian() * 0.01]     # D = 1: no factor gradient
    assert np.round(V.reshape(-1), 4).tolist() == d["factors"]
    raw = fo.raw(w, np.array(d["x"])[:, None], 1, 2)
    p = 1.0 / (1.0 + np.exp(-raw))
    assert np.max(np.abs(np.c_[1.0 - p, p] - np.array(d["probability"]))) <= 1e-12
    assert it == len(hist) == 100 and hist[0] == math.log(2.0)


def _problem(n, D, seed):
    rng = np.random.default_rng(seed)
    X = rng.normal(0.0, 1.0, (n, D)) * (rng.random((n, D)) < 0.6)
    y = (rng.random(n) < 0.4).astype(np.float64)
    return X, y


@pytest.mark.parametrize("fl,fi", [(True, True), (False, True), (True, False), (False, False)])
def test_gradient_equals_central_differences(fl, fi):
    X, y = _problem(60, 5, 3)
    D, k = 5, 3
    rng = np.random.default_rng(4)
    w = rng.normal(0.0, 0.4, D * k + D * fl + fi)
    _, g = fo.sums(w, X, y, D, k, fl, fi)
    h = 1e-6
    for j in range(w.shape[0]):
        e = np.zeros_like(w)
        e[j] = h
        fd = (fo.sums(w + e, X, y, D, k, fl, fi)[0] - fo.sums(w - e, X, y, D, k, fl, fi)[0]) / (2 * h)
        assert abs(fd - g[j]) <= 1e-6 * max(1.0, abs(g[j])), j


def test_pairwise_term_is_the_quadratic_form():
    X, _ = _problem(40, 6, 5)
    rng = np.random.default_rng(6)
    D, k = 6, 4
    V = rng.normal(0.0, 1.0, (D, k))
    w = np.concatenate([V.reshape(-1), np.zeros(D), [0.0]])
    want = 0.5 * (np.einsum("ni,ij,nj->n", X, V @ V.T, X) - (X * X) @ (V * V).sum(1))
    assert np.max(np.abs(fo.raw(w, X, D, k) - want)) <= 1e-12 * max(1.0, np.max(np.abs(want)))


def test_gd_and_adamw_steps_match_hand_computation():
    w = np.array([0.5, -1.0, 2.0])
    g = np.array([0.1, 0.2, -0.3])
    for reg in (0.0, 0.3):
        w1, rv = fo.GD(3)(w, g, 2.0, 4, reg)
        eta = 2.0 / 2.0
        assert np.array_equal(w1, w * (1 - eta * reg) - eta * g)
        n1 = np.sqrt(np.sum(w1 * w1))
        assert rv == 0.5 * reg * n1 * n1
        a = fo.AdamW(3)
        w1, _ = a(w, g, 0.5, 1, reg)
        # first step: m_hat = g, v_hat = g^2, so the step is 0.5 g / (|g| + eps), plus the decay reg w
        assert np.allclose(w1, w - (0.5 * g / (np.abs(g) + 1e-8) + reg * w), rtol=1e-15, atol=1e-15)
        w2, _ = a(w1, -g, 0.5, 2, reg)
        m = 0.9 * (0.1 * g) + 0.1 * (-g)
        v = 0.999 * (0.001 * g * g) + 0.001 * g * g
        mh, vh = m / (1 - 0.81), v / (1 - 0.999 ** 2)
        assert np.allclose(w2, w1 - (0.5 * mh / (np.sqrt(vh) + 1e-8) + reg * w1), rtol=1e-14, atol=1e-15)
        if reg > 0:                                       # the decay reaches every coefficient, the intercept included
            assert not np.allclose(w2, fo.AdamW(3)(fo.AdamW(3)(w, g, 0.5, 1, 0.0)[0], -g, 0.5, 2, 0.0)[0])


def test_the_batch_draw_keeps_the_fraction_and_an_empty_batch_skips_the_update():
    from b200flow.kmeans import philox
    keep = fo.batch_mask(20000, 0.3, 5)
    assert abs(keep.mean() - 0.3) < 0.015
    assert not np.array_equal(keep, fo.batch_mask(20000, 0.3, 6))
    assert fo.batch_mask(50, 1.0, 1).all()
    thr = math.floor(0.3 * 2 ** 32)
    assert keep[12345] == (philox(47, fo.PURPOSE_FMMB, 12345, 0)[0] < thr)
    # two rows at fraction 0.2: some iterations draw no row; they add no history entry and make no update
    X, y = fo.doctest_data()
    empty = [it for it in range(1, 21) if not fo.batch_mask(2, 0.2, it).any()]
    assert empty
    w, hist, n_up = fo.fit(X, y, k=2, seed=11, fraction=0.2, max_iter=20, tol=0.0, solver="gd")
    assert len(hist) == n_up == 20 - len(empty)


def test_fit_stops_on_the_relative_step():
    X, y = _problem(80, 4, 7)
    w, hist, it = fo.fit(X, y, k=2, solver="gd", step=0.5, tol=1e-3, max_iter=500)
    assert 2 <= it < 500 and len(hist) == it


class _Frame:
    """the two columns FMClassifier._fit reads, on the host"""

    def __init__(self, x, y, meta=None):
        from pyspark.sql import ColumnData
        self._cols = {"features": ColumnData("vector", torch.as_tensor(x), "f64"),
                      "label": ColumnData("numeric", torch.as_tensor(y, dtype=torch.float64), "f64", meta)}

    def _column_tensor(self, name):
        return self._cols[name].data


def test_defaults_and_param_validation():
    from pyspark.ml.classification import FMClassifier, FMClassificationModel
    from pyspark.ml.feature import IllegalArgumentException
    s = FMClassifier()
    want = {"factorSize": 8, "fitIntercept": True, "fitLinear": True, "regParam": 0.0, "miniBatchFraction": 1.0,
            "initStd": 0.01, "maxIter": 100, "stepSize": 1.0, "tol": 1e-6, "solver": "adamW", "thresholds": None,
            "seed": None, "weightCol": None, "featuresCol": "features", "labelCol": "label", "predictionCol": "prediction",
            "probabilityCol": "probability", "rawPredictionCol": "rawPrediction"}
    assert {k: s.getOrDefault(k) for k in want} == want
    p = FMClassifier(factorSize=2, fitIntercept=False, fitLinear=False, regParam=0.5, miniBatchFraction=0.25, initStd=0.0,
                     maxIter=0, stepSize=0.1, tol=0.0, solver="gd", seed=11)._check()
    assert (p.factor_size, p.fit_intercept, p.fit_linear, p.reg_param, p.mini_batch_fraction, p.init_std, p.max_iter,
            p.step_size, p.tol, p.solver, p.seed) == (2, False, False, 0.5, 0.25, 0.0, 0, 0.1, 0.0, "gd", 11)
    assert FMClassifier()._check().seed == FMClassifier()._check().seed
    for bad in ({"factorSize": 0}, {"factorSize": 2.5}, {"regParam": -0.1}, {"initStd": -1.0}, {"miniBatchFraction": 0.0},
                {"miniBatchFraction": 1.5}, {"maxIter": -1}, {"maxIter": 1.5}, {"stepSize": 0.0}, {"tol": -1e-9},
                {"solver": "lbfgs"}, {"weightCol": "w"}, {"thresholds": [0.4, 0.6]}):
        with pytest.raises(IllegalArgumentException):
            FMClassifier(**bad)._check()
    with pytest.raises(TypeError):
        FMClassifier(elasticNetParam=0.1)
    assert FMClassificationModel._all_defaults()["factorSize"] == 8


def test_two_classes_are_required_and_labels_must_be_valid():
    from pyspark.ml.classification import FMClassifier
    from pyspark.ml.feature import IllegalArgumentException
    x = np.zeros((4, 2))
    with pytest.raises(IllegalArgumentException, match="FMClassifier only supports binary classification. 3 classes "
                                                       "detected in label"):
        FMClassifier().fit(_Frame(x, [0, 1, 2, 1]))
    with pytest.raises(IllegalArgumentException, match="1 classes detected"):
        FMClassifier().fit(_Frame(x, [0, 0, 0, 0]))
    meta = {"ml_attr": {"type": "nominal", "vals": ["a", "b", "c"]}}
    with pytest.raises(IllegalArgumentException, match="3 classes detected"):
        FMClassifier().fit(_Frame(x, [0, 1, 1, 0], meta))
    for y in ([0, 1, -1, 1], [0, 1, 0.5, 1]):
        with pytest.raises(IllegalArgumentException, match="invalid label"):
            FMClassifier().fit(_Frame(x, y))
    with pytest.raises(IllegalArgumentException, match="weightCol"):
        FMClassifier(weightCol="w").fit(_Frame(x, [0, 1, 0, 1]))
