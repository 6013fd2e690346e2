"""IsotonicRegression on the device (DESIGN.md §5p): the fit equals the chunked restatement bit for bit for forced and
default chunk sizes on increasing, decreasing, noisy, heavy-tie and adversarial-junction data up to millions of rows, and
Spark's sequential PAV to 1e-12; f32 features give the f64 model; the predict kernel equals the host predict bit for bit;
the shim with numeric and vector features, a forest's probability calibrated through featureIndex=1, and CrossValidator
over isotonic."""
import numpy as np
import pytest
import torch

import isotonic_oracle as io

pytestmark = pytest.mark.gpu

DEFAULT_CHUNK = 64          # kIsoChunk of csrc/isotonic.cu


def _data(kind, n, seed):
    rng = np.random.default_rng(seed)
    x = rng.uniform(0.0, 100.0, n)
    w = rng.uniform(0.1, 3.0, n)
    if kind == "increasing":
        y = x + rng.normal(0, 2.0, n)
    elif kind == "decreasing":
        y = -x + rng.normal(0, 2.0, n)
    elif kind == "noisy":
        y = rng.normal(0, 1.0, n)
    elif kind == "ties":
        x = np.floor(rng.exponential(3.0, n))                  # few distinct values, long runs
        y = np.tanh(x / 5) + rng.normal(0, 0.5, n)
        w[rng.random(n) < 0.05] = 0.0                          # zero weights are dropped
    else:                                                      # a heavy, very low point just right of the middle
        x = np.arange(n, dtype=np.float64)
        y = x.copy()
        w = np.ones(n)
        y[n // 2 + 1], w[n // 2 + 1] = -1e3 * n, 1e3
    return y, x, w


def _device_fit(y, x, w, iso=True, chunk=0, dtype=torch.float64):
    from b200flow import isotonic as biso
    t = lambda a, dt=torch.float64: torch.from_numpy(np.ascontiguousarray(a)).to("cuda", dt)      # noqa: E731
    return biso.isotonic_fit(t(x, dtype), t(y), None if w is None else t(w), isotonic=iso, chunk=chunk)


def _same(fit, b, p):
    assert fit.boundaries.view(np.int64).tolist() == b.view(np.int64).tolist()
    assert fit.predictions.view(np.int64).tolist() == p.view(np.int64).tolist()


@pytest.mark.parametrize("chunk", [2, 3, 32, 0])
@pytest.mark.parametrize("kind", ["increasing", "decreasing", "noisy", "ties", "junction"])
def test_fit_equals_chunked_restatement(kind, chunk):
    y, x, w = _data(kind, 20000, 3)
    C = chunk or DEFAULT_CHUNK
    for iso in (True, False):
        _same(_device_fit(y, x, w, iso, chunk), *io.fit(y, x, w, isotonic=iso, chunk=C))
    b0, p0 = io.fit(y, x, w)
    fit = _device_fit(y, x, w, True, chunk)
    assert np.array_equal(fit.boundaries, b0) and np.allclose(fit.predictions, p0, rtol=1e-12, atol=1e-300)


@pytest.mark.parametrize("kind,n", [("noisy", 1_000_000), ("ties", 3_000_000), ("junction", 1_000_000)])
def test_fit_at_scale(kind, n):
    y, x, w = _data(kind, n, 11)
    fit = _device_fit(y, x, w)
    _same(fit, *io.fit(y, x, w, chunk=DEFAULT_CHUNK))
    b0, p0 = io.fit(y, x, w)
    assert np.array_equal(fit.boundaries, b0) and np.allclose(fit.predictions, p0, rtol=1e-12, atol=1e-300)


def test_edges_f32_and_refusals():
    from b200flow import isotonic as biso
    y, x, w = _data("noisy", 5000, 4)
    x32 = x.astype(np.float32)
    a, b = _device_fit(y, x32, w, dtype=torch.float32), _device_fit(y, x32.astype(np.float64), w)
    _same(a, b.boundaries, b.predictions)
    _same(_device_fit([1.0, 0.0], [1.0, 0.0], None), np.array([0.0, 1.0]), np.array([0.0, 1.0]))
    _same(_device_fit([1.0, 3.0, 5.0], [0.0, -0.0, 1.0], None), *io.fit([1.0, 3.0, 5.0], [0.0, -0.0, 1.0]))
    _same(_device_fit([3.0], [2.0], [0.7]), *io.fit([3.0], [2.0], [0.7]))
    e = _device_fit([1.0, 2.0], [0.0, 1.0], [0.0, 0.0])
    assert e.boundaries.size == 0 and e.predictions.size == 0
    e = biso.isotonic_fit(torch.zeros(0, device="cuda"), torch.zeros(0, dtype=torch.float64, device="cuda"))
    assert e.boundaries.size == 0
    for bad in ((float("nan"), 0.0, 1.0), (0.0, float("inf"), 1.0), (0.0, 0.0, float("nan"))):
        with pytest.raises(ValueError, match="finite"):
            _device_fit([1.0, bad[0]], [0.0, bad[1]], [1.0, bad[2]])
    with pytest.raises(ValueError, match="Negative weight at point"):
        _device_fit([1.0, 2.0], [0.0, 1.0], [1.0, -0.5])
    with pytest.raises(ValueError, match="empty"):
        biso.isotonic_predict(torch.zeros(3, device="cuda"), e)


def test_predict_kernel_equals_host_predict():
    from b200flow import isotonic as biso
    y, x, w = _data("ties", 50000, 6)
    fit = _device_fit(y, x, w)
    b = fit.boundaries
    rng = np.random.default_rng(2)
    q = np.concatenate([rng.uniform(b[0] - 3, b[-1] + 3, 20000), b, (b[:-1] + b[1:]) / 2,
                        [np.nan, np.inf, -np.inf, -0.0, 0.0, 1e300, -1e300]])
    for dt in (torch.float64, torch.float32):
        qt = torch.from_numpy(q).to("cuda", dt)
        got = biso.isotonic_predict(qt, fit).cpu().numpy()
        want = np.array([biso.predict_value(v, fit) for v in qt.double().cpu().numpy()])
        assert got.view(np.int64).tolist() == want.view(np.int64).tolist()
        assert np.array_equal(want, [io.predict(v, fit.boundaries, fit.predictions) for v in qt.double().cpu().numpy()])
    strided = torch.from_numpy(np.stack([q, -q], 1)).cuda()[:, 1]
    assert torch.equal(biso.isotonic_predict(strided, fit), biso.isotonic_predict((-torch.from_numpy(q)).cuda(), fit))


def _frame(cols):
    from pyspark.sql import ColumnData, DataFrame
    from b200flow import synth
    n = next(iter(cols.values())).shape[0]
    rec, dicts = synth.make_kdd(n, 2, seed=1, device="cuda:0")
    df = DataFrame.fromRecords(rec, synth.kdd_schema(), dicts).select("duration")
    return df._with(cols={k: ColumnData("vector" if v.dim() == 2 else "numeric", v.cuda(), "f64") for k, v in cols.items()})


def test_shim_numeric_and_vector_features():
    from pyspark.ml.feature import IllegalArgumentException
    from pyspark.ml.regression import IsotonicRegression
    y, x, w = _data("increasing", 8000, 9)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a))     # noqa: E731
    vec = np.stack([np.sin(x), x, np.cos(x)], 1)
    df = _frame({"f": t(x), "features": t(vec), "label": t(y), "w": t(w)})
    b, p = io.fit(y, x, w, chunk=DEFAULT_CHUNK)
    for est in (IsotonicRegression(featuresCol="f", weightCol="w"), IsotonicRegression(featureIndex=1, weightCol="w")):
        m = est.fit(df)
        _same(m._fit_result, b, p)
        assert m.numFeatures == 1 and np.array_equal(m.boundaries.toArray(), b)
        assert np.array_equal(m.predictions.toArray(), p)
        pred = m.transform(df)._column_tensor("prediction").cpu().numpy()
        assert pred.view(np.int64).tolist() == [np.float64(m.predict(v)).view(np.int64) for v in x]
    m = IsotonicRegression(featureIndex=1, isotonic=False).fit(df)
    assert np.all(np.diff(m.predictions.toArray()) <= 0)
    m.setFeatureIndex(0)
    out = m.transform(df)._column_tensor("prediction").cpu().numpy()
    assert out.tolist() == [m.predict(v) for v in vec[:, 0]]
    with pytest.raises(IllegalArgumentException, match="already exists"):
        m.transform(m.transform(df))
    with pytest.raises(IllegalArgumentException, match="finite"):
        IsotonicRegression(featuresCol="f").fit(_frame({"f": t(np.array([0.0, np.nan])), "label": t(np.zeros(2))}))
    with pytest.raises(IllegalArgumentException, match="empty"):
        IsotonicRegression(featuresCol="f", weightCol="w").fit(
            _frame({"f": t(np.zeros(2)), "label": t(np.zeros(2)), "w": t(np.zeros(2))})).transform(df)


def test_calibrating_forest_probabilities():
    from pyspark.ml import Pipeline
    from pyspark.ml.classification import RandomForestClassifier
    from pyspark.ml.feature import VectorAssembler
    from pyspark.ml.regression import IsotonicRegression
    from test_tuning_gpu import _frame as kdd_frame
    df, feats = kdd_frame(30000, 2, seed=31)
    pipe = Pipeline(stages=[VectorAssembler(inputCols=feats, outputCol="features"),
                            RandomForestClassifier(labelCol="label_num", maxBins=70, numTrees=8, maxDepth=4, seed=5),
                            IsotonicRegression(featuresCol="probability", labelCol="label_num", featureIndex=1,
                                               predictionCol="calibrated")])
    pm = pipe.fit(df)
    out = pm.transform(df)
    cal = pm.stages[-1]
    score = out._column_tensor("probability")[:, 1].cpu().numpy()
    lab = out._column_tensor("label_num").cpu().numpy()
    _same(cal._fit_result, *io.fit(lab, score, chunk=DEFAULT_CHUNK))
    got = out._column_tensor("calibrated").cpu().numpy()
    assert got.min() >= 0.0 and got.max() <= 1.0
    order = np.argsort(score, kind="stable")
    assert np.all(np.diff(got[order]) >= 0)


def test_cross_validator_picks_isotonic_on_increasing_data():
    from pyspark.ml.evaluation import RegressionEvaluator
    from pyspark.ml.regression import IsotonicRegression
    from pyspark.ml.tuning import CrossValidator, ParamGridBuilder, TrainValidationSplit
    y, x, _ = _data("increasing", 20000, 12)
    df = _frame({"x": torch.from_numpy(x), "label": torch.from_numpy(y)})
    est = IsotonicRegression(featuresCol="x")
    grid = ParamGridBuilder().addGrid(est.isotonic, [True, False]).build()
    ev = RegressionEvaluator(metricName="rmse")
    cvm = CrossValidator(estimator=est, estimatorParamMaps=grid, evaluator=ev, numFolds=3, seed=7).fit(df)
    assert cvm.avgMetrics[0] < cvm.avgMetrics[1]
    assert cvm.bestModel.getOrDefault("isotonic") is True
    tvs = TrainValidationSplit(estimator=est, estimatorParamMaps=grid, evaluator=ev, trainRatio=0.75, seed=7).fit(df)
    assert tvs.validationMetrics[0] < tvs.validationMetrics[1]
