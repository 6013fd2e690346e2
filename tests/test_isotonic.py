"""IsotonicRegression on the CPU: the chunked restatement of the device's PAV against Spark's sequential one and against
scipy, Spark's doctest, hand-worked cases, java.util.Arrays.binarySearch at its edges, and the shim's params and
refusals (DESIGN.md §5p)."""
import math

import numpy as np
import pytest
import torch

import isotonic_oracle as io


def _data(kind, n, seed):
    rng = np.random.default_rng(seed)
    x = rng.uniform(0.0, 10.0, n)
    if kind == "ties":
        x = np.round(x, 1)
    y = {"increasing": x + rng.normal(0, 0.5, n), "decreasing": -x + rng.normal(0, 0.5, n),
         "noisy": rng.normal(0, 1.0, n), "ties": np.sin(x) + rng.normal(0, 0.3, n)}[kind]
    return y, x, rng.uniform(0.1, 3.0, n)


@pytest.mark.parametrize("C", [2, 3, 32, 1024])
@pytest.mark.parametrize("kind", ["increasing", "decreasing", "noisy", "ties"])
def test_chunked_equals_sequential(kind, C):
    y, x, w = _data(kind, 3000, C)
    for iso in (True, False):
        b0, p0 = io.fit(y, x, w, isotonic=iso)
        b1, p1 = io.fit(y, x, w, isotonic=iso, chunk=C)
        assert np.array_equal(b0, b1)
        assert np.allclose(p1, p0, rtol=1e-12, atol=0)


@pytest.mark.parametrize("kind", ["increasing", "noisy", "ties"])
def test_fit_agrees_with_scipy_on_the_unique_points(kind):
    from scipy.optimize import isotonic_regression
    y, x, w = _data(kind, 2000, 5)
    o = io._order(x)
    uy, ux, uw = io.make_unique(y[o].tolist(), x[o].tolist(), w[o].tolist())
    want = isotonic_regression(uy, weights=uw, increasing=True).x
    for chunk in (None, 3):
        b, p = io.fit(y, x, w, chunk=chunk)
        got = np.array([io.predict(v, b, p) for v in ux])
        assert np.allclose(got, want, rtol=1e-12, atol=1e-12)


def test_spark_doctest():
    b, p = io.fit([1.0, 0.0], [1.0, 0.0])
    assert b.tolist() == [0.0, 1.0] and p.tolist() == [0.0, 1.0]
    assert io.predict(-1.0, b, p) == 0.0


def test_hand_cases():
    # equal adjacent means pool (>=): one block, two output points
    b, p = io.fit([1.0, 1.0, 1.0], [0.0, 1.0, 2.0])
    assert b.tolist() == [0.0, 2.0] and p.tolist() == [1.0, 1.0]
    # antitonic keeps a decreasing series; isotonic pools it
    b, p = io.fit([3.0, 2.0, 1.0], [0.0, 1.0, 2.0], isotonic=False)
    assert b.tolist() == [0.0, 1.0, 2.0] and p.tolist() == [3.0, 2.0, 1.0]
    b, p = io.fit([3.0, 2.0, 1.0], [0.0, 1.0, 2.0])
    assert b.tolist() == [0.0, 2.0] and p.tolist() == [2.0, 2.0]
    # weights; a zero-weight row is dropped
    b, p = io.fit([2.0, 0.0, 1e9], [0.0, 1.0, 0.5], [3.0, 1.0, 0.0])
    assert b.tolist() == [0.0, 1.0] and p.tolist() == [1.5, 1.5]
    # -0.0 sorts first and == 0.0 pools the two: one point at -0.0
    b, p = io.fit([1.0, 3.0, 5.0], [0.0, -0.0, 1.0])
    assert b.tolist() == [0.0, 1.0] and math.copysign(1.0, b[0]) == -1.0 and p.tolist() == [2.0, 5.0]
    # one point is kept as it is by makeUnique; PAV's weights give (w y) / w
    b, p = io.fit([3.0], [2.0], [0.7])
    assert b.tolist() == [2.0] and p.tolist() == [(0.7 * 3.0) / 0.7]
    # two rows of one feature pool through makeUnique first
    b, p = io.fit([3.0, 1.0], [2.0, 2.0], [0.7, 0.3])
    s = (3.0 * 0.7 + 1.0 * 0.3) / (0.7 + 0.3)
    assert b.tolist() == [2.0] and p.tolist() == [(1.0 * s) / 1.0]
    # every weight 0: an empty model
    b, p = io.fit([1.0, 2.0], [0.0, 1.0], [0.0, 0.0])
    assert b.size == 0 and p.size == 0
    with pytest.raises(ValueError):
        io.fit([1.0], [0.0], [-1.0])


def test_binary_search_edges_and_host_predict():
    from b200flow import isotonic as biso
    b = np.array([-1.0, 0.0, 2.0, 5.0])
    p = np.array([0.5, 1.0, 3.0, 4.0])
    fit = biso.IsotonicFit(b, p)
    cases = {float("nan"): 4.0, float("inf"): 4.0, -float("inf"): 0.5, -3.0: 0.5, 9.0: 4.0, 2.0: 3.0, 5.0: 4.0,
             -1.0: 0.5, 1.0: 1.0 + (3.0 - 1.0) * (1.0 - 0.0) / (2.0 - 0.0)}
    for x, want in cases.items():
        assert io.predict(x, b, p) == want, x
        assert biso.predict_value(x, fit) == want, x
    # -0.0 orders before the boundary 0.0: not a hit, the interpolation from -1.0 gives the same value here
    assert io.binary_search(b, -0.0) == -2 and io.binary_search(b, 0.0) == 1
    assert biso.java_binary_search(b, -0.0) == -2 and biso.java_binary_search(b, float("nan")) == -5
    assert io.predict(-0.0, b, p) == 0.5 + (1.0 - 0.5) * (-0.0 - -1.0) / (0.0 - -1.0)
    rng = np.random.default_rng(1)
    for x in rng.uniform(-2, 6, 200):
        assert biso.predict_value(x, fit) == io.predict(x, b, p)
    with pytest.raises(ValueError, match="empty"):
        biso.predict_value(0.0, biso.IsotonicFit(np.zeros(0), np.zeros(0)))


def _frame(cols):
    from pyspark.sql import ColumnData, DataFrame
    n = next(iter(cols.values())).shape[0]
    return DataFrame(n, None, None, {}, {k: ColumnData("vector" if v.dim() == 2 else "numeric", v, "f64")
                                         for k, v in cols.items()})


def test_shim_params_and_refusals():
    from pyspark.ml.feature import IllegalArgumentException
    from pyspark.ml.regression import IsotonicRegression, IsotonicRegressionModel, _isotonic_feature
    from b200flow import isotonic as biso
    est = IsotonicRegression()
    assert est.getOrDefault("isotonic") is True and est.getOrDefault("featureIndex") == 0
    assert est.getOrDefault("featuresCol") == "features" and est.getOrDefault("weightCol") is None
    df = _frame({"features": torch.arange(12, dtype=torch.float64).reshape(4, 3), "s": torch.zeros(4, dtype=torch.float32),
                 "label": torch.zeros(4, dtype=torch.float64)})
    assert torch.equal(_isotonic_feature(IsotonicRegression(featureIndex=2), df), torch.tensor([2.0, 5.0, 8.0, 11.0],
                                                                                                 dtype=torch.float64))
    assert _isotonic_feature(IsotonicRegression(featuresCol="s"), df).dtype == torch.float32
    with pytest.raises(IllegalArgumentException, match="parameter featureIndex given invalid value -1"):
        IsotonicRegression(featureIndex=-1).fit(df)
    with pytest.raises(IllegalArgumentException, match="out of range"):
        IsotonicRegression(featureIndex=3).fit(df)
    with pytest.raises(IllegalArgumentException, match="does not exist"):
        IsotonicRegression(featuresCol="nope").fit(df)
    with pytest.raises(IllegalArgumentException, match="does not exist"):
        IsotonicRegression(weightCol="nope").fit(df)
    m = IsotonicRegressionModel(biso.IsotonicFit(np.array([0.0, 1.0]), np.array([0.0, 1.0])))
    assert m.numFeatures == 1 and m.boundaries.toArray().tolist() == [0.0, 1.0] and m.predict(-1.0) == 0.0
    assert m.predict(0.25) == 0.25
    with pytest.raises(IllegalArgumentException, match="empty"):
        IsotonicRegressionModel(biso.IsotonicFit(np.zeros(0), np.zeros(0))).predict(1.0)
    with pytest.raises(_lib_error()):
        biso.isotonic_fit(torch.zeros(3), torch.zeros(3, dtype=torch.float64))      # no CPU fallback


def _lib_error():
    from b200flow._lib import B200FlowError
    return B200FlowError


def test_scratch_query_is_host_only():
    from b200flow import _lib
    assert _lib.isotonic_scratch(0) > 0 and _lib.isotonic_scratch(1 << 20) > 100 * (1 << 20)
    with pytest.raises(_lib.B200FlowError):
        _lib.isotonic_scratch(1 << 32)
