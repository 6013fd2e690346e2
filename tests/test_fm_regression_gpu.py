"""FMRegressor on the device: the squared-error instantiation of the fused factorization-machine kernel against the numpy
restatement (tests/fm_regression_oracle.py), with and without the linear and intercept blocks and with a mini-batch;
f32 features against their f64 copy; fits against the restatement's with both solvers; the PySpark doctest through
createDataFrame; and the shim under Pipeline and CrossValidator over factorSize x regParam."""
import math

import numpy as np
import pytest
import torch

import fm_oracle as fo
import fm_regression_oracle as fro

pytestmark = pytest.mark.gpu


def _problem(n, D, kf, seed):
    rng = np.random.default_rng(seed)
    x = rng.normal(0.0, 1.0, (n, D)) * rng.uniform(0.3, 2.0, D) * (rng.random((n, D)) < 0.7)
    y = rng.normal(0.0, 3.0, n)
    w = rng.normal(0.0, 0.6 / np.sqrt(D), D * (kf + 1) + 1)
    w[-1] = 0.7
    return np.ascontiguousarray(x), y, w


def _launch_totals(x, y, w, kf, fraction=1.0, seed=43, row_offset=0):
    """one launch at a global row offset that need not start a chunk, its partials chained in chunk order"""
    from b200flow import fm as bfm
    from b200flow._lib import call, ptr
    n, D = x.shape
    W = D * (kf + 1) + D + 3
    nc = (row_offset + n - 1) // 4096 - row_offset // 4096 + 1
    parts = torch.zeros((nc, 1, W), dtype=torch.float64, device="cuda")
    bfm.regression_loss_grad(torch.as_tensor(x).cuda(), torch.as_tensor(y).cuda(), torch.as_tensor(w).reshape(1, -1).cuda(),
                             kf, fraction, seed, row_offset, parts)
    tot = torch.zeros((1, W), dtype=torch.float64, device="cuda")
    call("b200flow_group_sums_chain", ptr(parts), nc, 1, W, ptr(tot))
    return tot.cpu().numpy()[0]


def _totals(x, y, w, kf, fraction=1.0, seed=43):
    from b200flow import dist as bdist, fm as bfm
    xt = torch.as_tensor(x).cuda()
    sh = bdist.Shards(xt.shape[0], 0, None, xt.device)
    return bfm.fm_regression_loss_grad_totals(xt, torch.as_tensor(y).cuda(), torch.as_tensor(w).reshape(1, -1).cuda(), kf,
                                              fraction, seed, sh).cpu().numpy()[0]


def _check(got, x, y, w, D, kf, fl=True, fi=True, keep=None):
    keep = np.ones(x.shape[0], bool) if keep is None else keep
    nv = D * kf
    parts = [got[2:2 + nv] - w[:nv] * np.repeat(got[3 + nv + D:3 + nv + 2 * D], kf)]
    if fl:
        parts.append(got[2 + nv:2 + nv + D])
    if fi:
        parts.append(got[2 + nv + D:3 + nv + D])
    g = np.concatenate(parts)
    ow = np.concatenate([w[:nv]] + ([w[nv:nv + D]] if fl else []) + ([w[-1:]] if fi else []))
    want_loss, want_g = fro.sums(ow, x[keep], y[keep], D, kf, fl, fi)
    assert got[1] == keep.sum()
    assert abs(got[0] - want_loss) <= 1e-12 * abs(want_loss)
    assert np.max(np.abs(g - want_g)) <= 1e-10 * max(1.0, np.max(np.abs(want_g)))


@pytest.mark.parametrize("n,D,kf", [(5000, 5, 4), (9001, 119, 8), (4097, 41, 3), (3000, 255, 32), (777, 1, 2)])
def test_loss_grad_equals_the_restatement(n, D, kf):
    x, y, w = _problem(n, D, kf, 11)
    _check(_totals(x, y, w, kf), x, y, w, D, kf)
    _check(_launch_totals(x, y, w, kf, row_offset=1000), x, y, w, D, kf)


@pytest.mark.parametrize("fl,fi", [(False, True), (True, False), (False, False)])
def test_loss_grad_without_the_linear_or_intercept_block(fl, fi):
    D, kf = 30, 5
    x, y, w = _problem(5000, D, kf, 12)
    if not fl:
        w[D * kf:D * kf + D] = 0.0
    if not fi:
        w[-1] = 0.0
    _check(_totals(x, y, w, kf), x, y, w, D, kf, fl, fi)


def test_mini_batch_partials_equal_the_restatement():
    D, kf, off = 20, 4, 1000
    x, y, w = _problem(9000, D, kf, 13)
    for fraction, it in ((0.5, 1), (0.1, 7)):
        keep = fo.batch_mask(x.shape[0], fraction, it, off)
        assert 0 < keep.sum() < x.shape[0]
        _check(_launch_totals(x, y, w, kf, fraction, 42 + it, off), x, y, w, D, kf, keep=keep)


def test_f32_features_equal_their_f64_copy_and_batches_chain_to_the_same_totals():
    from b200flow import selection
    D, kf = 41, 6
    x, y, w = _problem(20000, D, kf, 15)
    x32 = x.astype(np.float32)
    a = _totals(x32, y, w, kf)
    assert np.array_equal(a, _totals(x32.astype(np.float64), y, w, kf))
    assert np.array_equal(_totals(x32, y, w, kf, 0.5), _totals(x32.astype(np.float64), y, w, kf, 0.5))
    old = selection.PARTIALS_BUDGET
    selection.PARTIALS_BUDGET = (D * (kf + 1) + D + 3) * 8 * 2
    try:
        assert np.array_equal(_totals(x32, y, w, kf), a)
    finally:
        selection.PARTIALS_BUDGET = old


def test_the_classifier_partials_are_unchanged_beside_the_regressor():
    """the two instantiations share the products: with y in {0, 1} the factor-product sums differ only through g"""
    from b200flow import fm as bfm
    D, kf = 12, 3
    x, _, w = _problem(3000, D, kf, 16)
    y01 = (np.random.default_rng(2).random(3000) < 0.5).astype(np.int32)
    from b200flow import dist as bdist
    xt = torch.as_tensor(x).cuda()
    sh = bdist.Shards(3000, 0, None, xt.device)
    cls = bfm.fm_loss_grad_totals(xt, torch.as_tensor(y01).cuda(), torch.ones(1, dtype=torch.int32, device="cuda"),
                                  torch.as_tensor(w).reshape(1, -1).cuda(), kf, 1.0, 43, sh).cpu().numpy()[0]
    loss, g = fo.sums(w, x, y01.astype(np.float64), D, kf)
    assert abs(cls[0] - loss) <= 1e-12 * loss
    reg = _totals(x, y01.astype(np.float64), w, kf)
    assert cls[1] == reg[1] == 3000 and not np.array_equal(cls, reg)


FIT_CASES = [("adamW", 0.0, 1.0, True, True), ("adamW", 0.05, 1.0, True, False), ("gd", 0.01, 1.0, True, True),
             ("gd", 0.0, 0.5, False, True), ("adamW", 0.0, 0.3, True, True)]


@pytest.mark.parametrize("solver,reg,fraction,fl,fi", FIT_CASES)
def test_fit_matches_the_restatement(solver, reg, fraction, fl, fi):
    from b200flow import fm as bfm
    rng = np.random.default_rng(5)
    D, kf = 6, 3
    x = rng.normal(0.0, 1.0, (600, D))
    y = x[:, 0] * x[:, 1] + 0.5 * x[:, 2] + rng.normal(0, 0.5, 600)
    step = 0.05 if solver == "adamW" else 0.05
    p = bfm.FMParams(factor_size=kf, fit_linear=fl, fit_intercept=fi, reg_param=reg, mini_batch_fraction=fraction,
                     init_std=0.1, max_iter=40, step_size=step, tol=1e-9, solver=solver, seed=3)
    for dtype in (torch.float64, torch.float32):
        xd = x if dtype == torch.float64 else x.astype(np.float32).astype(np.float64)
        fit = bfm.fm_regression_fit(torch.as_tensor(xd).cuda().to(dtype), torch.as_tensor(y).cuda(), p)
        w, hist, it = fro.fit(xd, y, k=kf, fit_linear=fl, fit_intercept=fi, reg=reg, fraction=fraction, init_std=0.1,
                              max_iter=40, step=step, tol=1e-9, solver=solver, seed=3)
        V, lin, b = fo.split(w, D, kf, fl, fi)
        assert fit.iterations == it and len(fit.objective_history) == len(hist)
        assert np.max(np.abs(np.array(fit.objective_history) - hist)) <= 1e-10 * max(hist)
        for got, want in ((fit.factors, V), (fit.linear, lin), (np.array([fit.intercept]), np.array([b]))):
            assert np.max(np.abs(got - want)) <= 1e-9 * max(1.0, np.max(np.abs(want)))
        assert fl or not fit.linear.any()
        assert fi or fit.intercept == 0.0


def _spark():
    from pyspark.sql import SparkSession
    return SparkSession.builder.getOrCreate()


def test_the_pyspark_doctest_through_create_data_frame():
    from pyspark.ml.linalg import Vectors
    from pyspark.ml.regression import FMRegressor
    spark = _spark()
    df = spark.createDataFrame([(2.0, Vectors.dense(2.0)), (1.0, Vectors.dense(1.0)), (0.0, Vectors.dense(0.0))],
                               ["label", "features"])
    fm = FMRegressor(factorSize=2)
    fm.setSeed(16)
    model = fm.fit(df)
    assert model.getFactorSize() == 2 and model.numFeatures == 1
    d = fro.DOCTEST
    test0 = spark.createDataFrame([(Vectors.dense(v),) for v in d["x"]], ["features"])
    pred = model.transform(test0)._column_tensor("prediction").cpu().numpy()
    assert np.max(np.abs(pred - np.array(d["prediction"]))) <= 1e-12
    assert abs(model.intercept - d["intercept"]) <= 1e-12
    r = fo.JavaRandom(16)
    assert np.max(np.abs(model.factors.toArray().reshape(-1) - [r.next_gaussian() * 0.01, r.next_gaussian() * 0.01])) <= 1e-8
    assert model.predict(Vectors.dense(0.5)) == pred[1]


def _frame(x, y):
    from pyspark.sql import ColumnData, DataFrame
    from b200flow import synth
    rec, dicts = synth.make_kdd(x.shape[0], 2, seed=1, device="cuda:0")
    df = DataFrame.fromRecords(rec, synth.kdd_schema(), dicts).select("duration")
    return df._with(cols={"features": ColumnData("vector", torch.as_tensor(x).cuda(), "f64"),
                          "label": ColumnData("numeric", torch.as_tensor(np.asarray(y, np.float64)).cuda(), "f64")})


def test_refusals():
    from b200flow import _lib, fm as bfm
    from pyspark.ml.feature import IllegalArgumentException
    from pyspark.ml.regression import FMRegressor
    with pytest.raises(_lib.UnsupportedParamError):
        bfm.fm_regression_fit(torch.zeros((10, 256), dtype=torch.float64, device="cuda"), torch.zeros(10, device="cuda"),
                              bfm.FMParams())
    x = torch.ones((10, 3), dtype=torch.float64, device="cuda")
    y = torch.arange(10, dtype=torch.float64, device="cuda")
    with pytest.raises(ValueError, match="at least one row"):
        bfm.fm_regression_fit(x[:0], y[:0], bfm.FMParams())
    yb = y.clone()
    yb[2] = math.inf
    with pytest.raises(ValueError, match="finite labels"):
        bfm.fm_regression_fit(x, yb, bfm.FMParams())
    xb = x.clone()
    xb[3, 1] = math.nan
    with pytest.raises(ValueError, match="finite features"):
        bfm.fm_regression_fit(xb, y, bfm.FMParams())
    with pytest.raises(IllegalArgumentException):
        FMRegressor(factorSize=64).fit(_frame(np.zeros((10, 255)), np.arange(10.0)))
    m = FMRegressor(maxIter=0, seed=2).fit(_frame(np.ones((10, 3)), np.arange(10.0)))
    assert m.intercept == 0.0 and not m.linear.toArray().any()


def test_shim_pipeline_and_cross_validation():
    from pyspark.ml import Pipeline
    from pyspark.ml.evaluation import RegressionEvaluator
    from pyspark.ml.feature import StandardScaler, VectorAssembler
    from pyspark.ml.regression import FMRegressor
    from pyspark.ml.tuning import CrossValidator, ParamGridBuilder, fold_frames
    from pyspark.sql import ColumnData, DataFrame
    from b200flow import synth
    rec, dicts = synth.make_kdd(20000, 5, seed=7, device="cuda:0")
    df = DataFrame.fromRecords(rec, synth.kdd_schema(), dicts)
    nums = [c for c in synth.KDD_COLUMNS if c not in synth.KDD_CATEGORICAL + ["label", "dst_bytes"]]
    cols = dict(df._cols)
    cols["target"] = ColumnData("numeric", torch.log1p(df._column_tensor("dst_bytes").to(torch.float64)), "f64")
    df = df._with(cols=cols)
    fm = FMRegressor(labelCol="target", maxIter=20, stepSize=0.05)
    pipe = Pipeline(stages=[VectorAssembler(inputCols=nums, outputCol="raw"),
                            StandardScaler(inputCol="raw", outputCol="features", withMean=True, withStd=True), fm])
    out = pipe.fit(df).transform(df)
    ev = RegressionEvaluator(labelCol="target", metricName="rmse")
    assert math.isfinite(ev.evaluate(out))
    grid = ParamGridBuilder().addGrid(fm.factorSize, [2, 4]).addGrid(fm.regParam, [0.0, 0.01]).build()
    data = Pipeline(stages=pipe.getStages()[:2]).fit(df).transform(df).select("features", "target")
    cvm = CrossValidator(estimator=fm, estimatorParamMaps=grid, evaluator=ev, numFolds=2, seed=3).fit(data)
    want = [0.0] * len(grid)
    for train, val in fold_frames(data, 2, 3):
        for i, pm in enumerate(grid):
            want[i] += ev.evaluate(fm.fit(train, pm).transform(val))
    assert cvm.avgMetrics == [v / 2 for v in want]
