"""LinearRegression on the device: the fused least-squares / Huber kernel against the numpy restatement
(tests/linreg_oracle.py) across shapes, dtypes, modes, shifts and row offsets, canaries around its partials, chunk-order
totals that are the same bits for any batch split, the labelled Gram matrix, fits on KDD- and CICIDS-shaped data against
scikit-learn for every solver / loss / fitIntercept / standardization, the Cholesky -> quasi-Newton fallback, the
summary against the oracle, refusals, and the shim under Pipeline and CrossValidator."""
import math

import numpy as np
import pytest
import torch

import linreg_oracle as lo

pytestmark = pytest.mark.gpu

SUM_TOL = 1e-11          # relative to the largest |total|: fp64 sums of up to 20k rows in another order


def _problem(n, D, seed):
    rng = np.random.default_rng(seed)
    x = rng.normal(0.0, 1.0, (n, D)) * rng.uniform(0.2, 4.0, D) + rng.normal(0, 3, D)
    y = x @ rng.normal(0.0, 1.0, D) + rng.standard_t(3, n)
    return np.ascontiguousarray(x), y


def _totals(x, y, shift, inv, ys, yt, w, bs, eps, mode, row_offset=0):
    """the chained totals; a nonzero row_offset moves the chunk boundaries (one launch, chained here)"""
    from b200flow import dist as bdist, linreg as blr
    from b200flow._lib import call, ptr
    xt = torch.as_tensor(x).cuda()
    c = lambda a: None if a is None else torch.as_tensor(np.ascontiguousarray(a, np.float64)).cuda()   # noqa: E731
    if row_offset == 0:
        sh = bdist.Shards(xt.shape[0], 0, None, xt.device)
        return blr.loss_grad_totals(xt, c(y), c(shift), c(inv), ys, yt, c(w), c(bs), eps, mode, sh).cpu().numpy()
    D = x.shape[1]
    nc = (row_offset + x.shape[0] - 1) // 4096 - row_offset // 4096 + 1
    parts = torch.empty((nc, D + 3), dtype=torch.float64, device="cuda")
    blr.loss_grad(xt, c(y), c(shift), c(inv), ys, yt, c(w), c(bs), eps, mode, row_offset, parts)
    tot = torch.zeros(D + 3, dtype=torch.float64, device="cuda")
    call("b200flow_group_sums_chain", ptr(parts), nc, 1, D + 3, ptr(tot))
    return tot.cpu().numpy()


@pytest.mark.parametrize("n,D", [(1000, 1), (4096, 41), (9001, 119), (5000, 255), (12289, 7)])
@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("shifted", [False, True])
def test_totals_equal_the_restatement(n, D, mode, shifted):
    x, y = _problem(n, D, 11)
    rng = np.random.default_rng(3)
    inv, _ = lo.inv_std(x, 1)
    w = rng.normal(0, 0.3, D)
    shift = x.mean(0) if shifted else None
    ys, yt, b, sigma, eps = (y.mean(), 1.0 / y.std(), 0.0, 1.0, 0.0) if mode == 0 else (0.0, 1.0, 0.4, 2.5, 1.35)
    for dtype in (np.float64, np.float32):
        xd = x.astype(dtype)
        want = lo.sums(xd.astype(np.float64), y, shift, inv, ys, yt, w, b, sigma, eps, mode)
        for off in (0, 1000):
            got = _totals(xd, y, shift, inv, ys, yt, w, [b, sigma], eps, mode, off)
            assert np.max(np.abs(got - want)) <= SUM_TOL * np.max(np.abs(want)), (dtype, off)


def test_canaries_and_chunk_batches_give_the_same_bits():
    from b200flow import dist as bdist, linreg as blr, selection
    x, y = _problem(20000, 41, 12)
    xt, yt = torch.as_tensor(x).cuda(), torch.as_tensor(y).cuda()
    inv = torch.as_tensor(lo.inv_std(x, 1)[0]).cuda()
    w = torch.as_tensor(np.random.default_rng(1).normal(0, 0.3, 41)).cuda()
    bs = torch.tensor([0.2, 1.7], dtype=torch.float64, device="cuda")
    for off in (0, 1000):
        nc = (off + 20000 - 1) // 4096 - off // 4096 + 1
        buf = torch.full((nc * 44 + 128,), 777.0, dtype=torch.float64, device="cuda")
        blr.loss_grad(xt, yt, None, inv, 0.0, 1.0, w, bs, 1.35, 1, off, buf[64:64 + nc * 44].view(nc, 44))
        h = buf.cpu().numpy()
        assert np.all(h[:64] == 777.0) and np.all(h[-64:] == 777.0) and not np.any(h[64:-64] == 777.0)
    sh = bdist.Shards(20000, 0, None, xt.device)
    full = blr.loss_grad_totals(xt, yt, None, inv, 0.0, 1.0, w, bs, 1.35, 1, sh).cpu().numpy()
    old = selection.PARTIALS_BUDGET
    try:
        for budget in (44 * 8, 44 * 8 * 3):              # one and three chunks per batch
            selection.PARTIALS_BUDGET = budget
            assert np.array_equal(blr.loss_grad_totals(xt, yt, None, inv, 0.0, 1.0, w, bs, 1.35, 1, sh).cpu().numpy(), full)
    finally:
        selection.PARTIALS_BUDGET = old
    f32 = blr.loss_grad_totals(xt.float(), yt, None, inv, 0.0, 1.0, w, bs, 1.35, 1, sh)
    assert np.array_equal(f32.cpu().numpy(), blr.loss_grad_totals(xt.float().double(), yt, None, inv, 0.0, 1.0, w, bs, 1.35,
                                                                   1, sh).cpu().numpy())


def test_labelled_gram_matches_numpy_and_its_batches():
    from b200flow import dist as bdist, pca
    x, y = _problem(30000, 119, 13)
    xt, yt = torch.as_tensor(x).cuda(), torch.as_tensor(y).cuda()
    sh = bdist.Shards(30000, 0, None, xt.device)
    mx = pca.column_sums(xt, sh) / 30000
    my = float(pca.column_sums(yt.reshape(-1, 1), sh).item()) / 30000
    q = pca.centered_gram_total(xt, mx, sh, y=yt, y_mean=my).cpu().numpy()
    _, _, _, G = lo.normal_statistics(x, y)
    iu = np.triu_indices(120)
    assert np.max(np.abs(q[iu[0] + iu[1] * (iu[1] + 1) // 2] - G[iu])) <= 1e-10 * np.max(np.abs(G))
    old = pca.STAGE_BUDGET
    try:
        pca.STAGE_BUDGET = 8 * 120 * 4096 * 2            # two chunks per staged batch
        assert np.array_equal(pca.centered_gram_total(xt, mx, sh, y=yt, y_mean=my).cpu().numpy(), q)
    finally:
        pca.STAGE_BUDGET = old
    assert np.array_equal(pca.centered_gram_total(xt.float(), mx, sh, y=yt, y_mean=my).cpu().numpy(),
                          pca.centered_gram_total(xt.float().double(), mx, sh, y=yt, y_mean=my).cpu().numpy())


# ----------------------------------------------------------------------------------- fits
def _kdd(n, seed):
    """KDD-shaped: 38 numeric columns of mixed scale and three one-hot blocks (D = 119), a linear label and heavy noise"""
    rng = np.random.default_rng(seed)
    num = np.abs(rng.standard_t(3, (n, 38))) * rng.uniform(0.1, 100.0, 38)
    blocks = [np.eye(k)[rng.integers(0, k, n)] for k in (3, 70, 8)]
    x = np.concatenate([num] + blocks, 1)
    return np.ascontiguousarray(x), _label(x, rng)


def _cicids(n, seed):
    """CICIDS-shaped: 78 continuous, skewed flow statistics over scales from 0.1 to 1000"""
    rng = np.random.default_rng(seed)
    x = rng.lognormal(0.0, 0.5, (n, 78)) * 10.0 ** rng.uniform(-1, 3, 78)
    return np.ascontiguousarray(x), _label(x, rng)


def _label(x, rng):
    beta = rng.normal(0.0, 1.0, x.shape[1]) / np.maximum(x.std(0), 1e-3)
    return x @ beta + 5.0 + rng.standard_t(3, x.shape[0])


def _fit(x, y, dtype=torch.float64, **kw):
    from b200flow import linreg as blr
    return blr.linreg_fit(torch.as_tensor(x).cuda().to(dtype), torch.as_tensor(y).cuda(), blr.LinRegParams(**kw))


def _pred_close(x, fit, want_pred, tol):
    got = x @ fit.coef + fit.intercept
    return np.max(np.abs(got - want_pred)) <= tol * np.max(np.abs(want_pred))


@pytest.mark.parametrize("shape", ["kdd", "cicids"])
@pytest.mark.parametrize("fi", [True, False])
def test_squared_fits_equal_sklearn(shape, fi):
    sklm = pytest.importorskip("sklearn.linear_model")
    x, y = (_kdd if shape == "kdd" else _cicids)(20000, 5)
    if shape == "kdd":                                     # drop one column of each one-hot block: full column rank
        x = np.delete(x, [38, 41, 111], 1)
    n = x.shape[0]
    ols = sklm.LinearRegression(fit_intercept=fi).fit(x, y).predict(x)
    for st in (True, False):
        f = _fit(x, y, fit_intercept=fi, standardization=st)
        assert f.solver == "normal" and f.diag_inv_atwa is not None and _pred_close(x, f, ols, 1e-8), st
        f = _fit(x, y, fit_intercept=fi, standardization=st, solver="l-bfgs", max_iter=1000, tol=1e-15)
        assert f.solver == "l-bfgs" and _pred_close(x, f, ols, 1e-3), st
    reg = 0.05
    for ystd, solver in ((y.std(), "normal"), (y.std(ddof=1), "l-bfgs")):
        ridge = sklm.Ridge(alpha=n * reg / ystd, fit_intercept=fi, tol=1e-15, solver="cholesky").fit(x, y).predict(x)
        f = _fit(x, y, fit_intercept=fi, standardization=False, reg_param=reg, solver=solver, max_iter=1000, tol=1e-15)
        assert _pred_close(x, f, ridge, 1e-8 if solver == "normal" else 1e-3), solver


@pytest.mark.parametrize("solver", ["normal", "l-bfgs"])
def test_lasso_fits_equal_sklearn(solver):
    sklm = pytest.importorskip("sklearn.linear_model")
    x, y = _cicids(20000, 6)
    x = x[:, :20] / x[:, :20].std(0)
    reg = 0.05
    f = _fit(x, y, reg_param=reg, elastic_net_param=1.0, standardization=False, solver=solver, max_iter=2000, tol=1e-15)
    sk = sklm.Lasso(alpha=reg, tol=1e-14, max_iter=100000).fit(x, y)
    assert f.solver == ("quasi-newton" if solver == "normal" else "l-bfgs")
    assert np.max(np.abs(f.coef - sk.coef_)) <= 1e-4 * np.max(np.abs(sk.coef_)) and abs(f.intercept - sk.intercept_) <= 1e-3


@pytest.mark.parametrize("fi", [True, False])
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_huber_fits_equal_sklearn(fi, dtype):
    sklm = pytest.importorskip("sklearn.linear_model")
    x, y = _cicids(20000, 7)
    x = np.ascontiguousarray(x[:, :12] / x[:, :12].std(0))     # unit scale: scikit-learn's L-BFGS-B converges
    if dtype == torch.float32:
        x = x.astype(np.float32).astype(np.float64)
    n, reg = x.shape[0], 1e-3
    y[:200] += 1e4 * np.abs(y).max()                        # gross outliers
    f = _fit(x, y, dtype=dtype, loss="huber", reg_param=reg, standardization=False, fit_intercept=fi, max_iter=3000,
             tol=1e-15)
    sk = sklm.HuberRegressor(epsilon=1.35, alpha=n * reg / 2, fit_intercept=fi, max_iter=100000, tol=1e-12).fit(x, y)
    assert abs(f.scale - sk.scale_) <= 1e-3 * sk.scale_
    # the same optimum: the restated objective at our solution is no worse than at scikit-learn's
    std = x.std(0, ddof=1)
    obj = lambda coef, b, s: lo.huber_objective(np.concatenate([coef * std, [b, s]]), x, y, reg, 1.35, fi, False)[0]  # noqa: E731
    f_ours, f_sk = obj(f.coef, f.intercept, f.scale), obj(sk.coef_, sk.intercept_ if fi else 0.0, sk.scale_)
    assert f_ours <= f_sk * (1 + 1e-7), (f_ours, f_sk)
    assert _pred_close(x, f, sk.predict(x), 1e-2)
    fs = _fit(x, y, dtype=dtype, loss="huber", fit_intercept=fi)              # standardization: another L2 weighting
    assert fs.scale > 0 and len(fs.objective_history) == fs.iterations + 1


def test_fallback_constant_label_and_constant_columns():
    sklm = pytest.importorskip("sklearn.linear_model")
    x, y = _cicids(9000, 8)
    x = x[:, :10]
    xd = np.concatenate([x, x[:, 3:4]], 1)                  # duplicated column: Cholesky -> quasi-Newton
    f = _fit(xd, y, max_iter=2000, tol=1e-15)
    assert f.solver == "quasi-newton" and f.diag_inv_atwa is None and f.iterations == len(f.objective_history) - 1
    assert _pred_close(xd, f, sklm.LinearRegression().fit(xd, y).predict(xd), 1e-5)
    for solver in ("normal", "l-bfgs"):
        f = _fit(x, np.full(9000, 3.25), solver=solver)
        assert np.all(f.coef == 0.0) and f.intercept == 3.25 and f.objective_history == [0.0] and f.iterations == 0
        with pytest.raises(ValueError, match="standard deviation of the label is zero"):
            _fit(x, np.full(9000, 3.25), solver=solver, fit_intercept=False, reg_param=0.1)
    xc = x.copy()
    xc[:, 4] = -2.0                                         # a constant column
    want = sklm.LinearRegression().fit(np.delete(xc, 4, 1), y).predict(np.delete(xc, 4, 1))
    f = _fit(xc, y, max_iter=2000, tol=1e-15)
    assert f.solver == "quasi-newton" and f.coef[4] == 0.0 and _pred_close(xc, f, want, 1e-5)
    f = _fit(xc, y, solver="l-bfgs", max_iter=2000, tol=1e-15)
    assert f.coef[4] == 0.0 and _pred_close(xc, f, want, 1e-4)
    f = _fit(xc, y, reg_param=0.01)                         # regularised with standardization: Cholesky succeeds
    assert f.solver == "normal" and f.coef[4] == 0.0


def test_summary_equals_the_oracle():
    from b200flow import linreg as blr
    x, y = _cicids(6000, 9)
    x = x[:, :8]
    for fi in (True, False):
        f = _fit(x, y, fit_intercept=fi)
        s = blr.summarize(torch.as_tensor(x).cuda(), torch.as_tensor(y).cuda(), f, fi)
        o = lo.summary(x, y, f.coef, f.intercept, f.diag_inv_atwa, fi)
        for a, b in ((s.mse, o["mse"]), (s.rmse, o["rmse"]), (s.mae, o["mae"]), (s.r2, o["r2"]), (s.r2adj, o["r2adj"]),
                     (s.explained_variance, o["explained_variance"])):
            assert abs(a - b) <= 1e-9 * max(1.0, abs(b))
        assert s.degrees_of_freedom == o["dof"] and s.num_instances == 6000
        assert np.allclose(s.deviance_residuals, o["residual_range"], rtol=1e-9, atol=1e-9)
        assert np.max(np.abs(s.std_errors - o["se"]) / o["se"]) <= 1e-9
        assert np.max(np.abs(s.t_values - o["t"]) / np.abs(o["t"])) <= 1e-9
        assert np.max(np.abs(s.p_values - o["p"])) <= 1e-9


def test_refusals_on_the_device():
    from b200flow import _lib, linreg as blr
    p = blr.LinRegParams()
    with pytest.raises(_lib.UnsupportedParamError):
        blr.linreg_fit(torch.zeros((10, 256), dtype=torch.float64, device="cuda"), torch.zeros(10, device="cuda"), p)
    with pytest.raises(ValueError, match="at least one row"):
        blr.linreg_fit(torch.zeros((0, 3), dtype=torch.float64, device="cuda"), torch.zeros(0, device="cuda"), p)
    x = torch.ones((10, 3), dtype=torch.float64, device="cuda")
    y = torch.arange(10, dtype=torch.float64, device="cuda")
    for bad_x, bad_y in ((True, False), (False, True)):
        xb, yb = x.clone(), y.clone()
        if bad_x:
            xb[3, 1] = math.inf
        else:
            yb[4] = math.nan
        with pytest.raises(ValueError, match="finite"):
            blr.linreg_fit(xb, yb, p)


# ----------------------------------------------------------------------------------- the shim
def _frame(x, y):
    from pyspark.sql import ColumnData, DataFrame
    from b200flow import synth
    rec, dicts = synth.make_kdd(x.shape[0], 2, seed=1, device="cuda:0")
    df = DataFrame.fromRecords(rec, synth.kdd_schema(), dicts).select("duration")
    return df._with(cols={"features": ColumnData("vector", torch.as_tensor(x).cuda(), "f64"),
                          "label": ColumnData("numeric", torch.as_tensor(y).cuda(), "f64")})


def test_shim_model_summary_and_refusals():
    from pyspark.ml.feature import IllegalArgumentException
    from pyspark.ml.regression import LinearRegression, UnsupportedOperationException
    x, y = _cicids(5000, 10)
    x = x[:, :6]
    df = _frame(x, y)
    m = LinearRegression().fit(df)
    assert m.numFeatures == 6 and m.scale == 1.0 and m.hasSummary
    pred = m.transform(df)._column_tensor("prediction").cpu().numpy()
    assert np.max(np.abs(pred - (x @ m.coefficients.toArray() + m.intercept))) <= 1e-12 * np.max(np.abs(pred))
    s = m.summary
    assert s.totalIterations == 0 and s.objectiveHistory == [0.0] and len(s.coefficientStandardErrors) == 7
    assert len(s.pValues) == 7 and len(s.tValues) == 7 and s.degreesOfFreedom == 5000 - 7
    ev = m.evaluate(df)
    assert ev.r2 == s.r2 and ev.meanSquaredError == s.meanSquaredError
    res = s.residuals._column_tensor("residuals").cpu().numpy()
    assert s.devianceResiduals == [float(res.min()), float(res.max())]
    mh = LinearRegression(loss="huber", maxIter=50).fit(df)
    assert mh.scale > 0 and mh.summary.totalIterations == len(mh.summary.objectiveHistory) - 1
    with pytest.raises(UnsupportedOperationException, match="No Std. Error"):
        mh.summary.coefficientStandardErrors
    with pytest.raises(IllegalArgumentException, match="huber loss doesn't support normal solver"):
        LinearRegression(loss="huber", solver="normal").fit(df)
    with pytest.raises(IllegalArgumentException):
        LinearRegression(weightCol="w").fit(df)
    with pytest.raises(IllegalArgumentException, match="does not exist"):
        LinearRegression(labelCol="nope").fit(df)


def test_shim_pipeline_and_cross_validation():
    from pyspark.ml import Pipeline
    from pyspark.ml.evaluation import RegressionEvaluator
    from pyspark.ml.feature import StandardScaler, VectorAssembler
    from pyspark.ml.regression import LinearRegression
    from pyspark.ml.tuning import CrossValidator, ParamGridBuilder, TrainValidationSplit, fold_frames
    from pyspark.sql import ColumnData, DataFrame
    from b200flow import synth
    rec, dicts = synth.make_kdd(20000, 5, seed=7, device="cuda:0")
    df = DataFrame.fromRecords(rec, synth.kdd_schema(), dicts)
    nums = [c for c in synth.KDD_COLUMNS if c not in synth.KDD_CATEGORICAL + ["label"]]
    feats = [c for c in nums if c not in ("dst_bytes",)]
    cols = dict(df._cols)
    cols["target"] = ColumnData("numeric", df._column_tensor("dst_bytes").to(torch.float64), "f64")
    df = df._with(cols=cols)
    lr = LinearRegression(labelCol="target", maxIter=30)
    pipe = Pipeline(stages=[VectorAssembler(inputCols=feats, outputCol="raw"),
                            StandardScaler(inputCol="raw", outputCol="features"), lr])
    model = pipe.fit(df)
    out = model.transform(df)
    ev = RegressionEvaluator(labelCol="target", metricName="rmse")
    assert math.isfinite(ev.evaluate(out))
    grid = ParamGridBuilder().addGrid(lr.regParam, [0.0, 0.5]).addGrid(lr.elasticNetParam, [0.0, 1.0]).build()
    data = Pipeline(stages=pipe.getStages()[:2]).fit(df).transform(df).select("features", "target")
    cvm = CrossValidator(estimator=lr, estimatorParamMaps=grid, evaluator=ev, numFolds=2, seed=3).fit(data)
    want = [0.0] * len(grid)
    for train, val in fold_frames(data, 2, 3):
        for i, pm in enumerate(grid):
            want[i] += ev.evaluate(lr.fit(train, pm).transform(val))
    assert cvm.avgMetrics == [v / 2 for v in want]
    tvs = TrainValidationSplit(estimator=lr, estimatorParamMaps=grid, evaluator=ev, trainRatio=0.75, seed=3).fit(data)
    assert len(tvs.validationMetrics) == len(grid)
