"""GeneralizedLinearRegression on the device: the per-row kernel in every mode against the numpy restatement
(tests/glm_oracle.py) for every family / link pair, shapes, dtypes, weights, offsets and row offsets; canaries; chunk
sums that are the same bits for f32 and f64 copies; the weighted Gram matrix; fits on KDD- and CICIDS-shaped data with
Poisson, gamma and binomial labels against the restatement and scikit-learn; the quasi-Newton fallback; the summary;
linkPredictionCol; and the shim under Pipeline, CrossValidator and TrainValidationSplit."""
import math

import numpy as np
import pytest
import torch

import glm_oracle as go

pytestmark = pytest.mark.gpu

SUM_TOL = 1e-11
PAIRS = [(go.GAUSSIAN, go.IDENTITY), (go.GAUSSIAN, go.LOG), (go.GAUSSIAN, go.INVERSE), (go.BINOMIAL, go.LOGIT),
         (go.BINOMIAL, go.PROBIT), (go.BINOMIAL, go.CLOGLOG), (go.POISSON, go.LOG), (go.POISSON, go.IDENTITY),
         (go.POISSON, go.SQRT), (go.GAMMA, go.INVERSE), (go.GAMMA, go.IDENTITY), (go.GAMMA, go.LOG),
         (go.TWEEDIE, go.LOG, 1.5, 0.0), (go.TWEEDIE, go.POWER, 1.5, -0.5), (go.TWEEDIE, go.POWER, 3.0, 0.3)]


def _spec(s):
    from b200flow import glm as bg
    f, l, vp, lp = go.spec_args(s)
    return bg.Spec(f, l, vp, lp)


def _problem(n, D, spec, seed):
    """features, a coefficient vector whose eta keeps mu inside the family's domain, labels in the domain"""
    f, l = spec[0], spec[1]
    rng = np.random.default_rng(seed)
    x = np.abs(rng.normal(0.0, 1.0, (n, D))) * rng.uniform(0.2, 1.0, D)
    coef = rng.uniform(0.0, 0.3, D) / D
    b = {go.IDENTITY: 1.0, go.LOG: 0.1, go.INVERSE: 1.0, go.LOGIT: -0.2, go.PROBIT: -0.1, go.CLOGLOG: -0.5,
         go.SQRT: 1.0, go.POWER: 1.0}[l]
    if f == go.BINOMIAL:
        y = rng.uniform(0, 1, n).round(1)
    elif f in (go.POISSON, go.TWEEDIE) and not (f == go.TWEEDIE and spec[2] > 2):
        y = rng.poisson(1.5, n).astype(float)
    else:
        y = rng.gamma(2.0, 0.7, n) + 0.05
    return np.ascontiguousarray(x), y, coef, b


def _launch(x, y, w, off, coef, b, spec, mode, row_offset=0, mu_const=0.0):
    """(totals chained here, per-row outputs) of one kernel launch"""
    from b200flow import glm as bg
    from b200flow._lib import call, ptr
    c = lambda a: None if a is None else torch.as_tensor(np.ascontiguousarray(a, np.float64)).cuda()   # noqa: E731
    xt = torch.as_tensor(x).cuda()
    n, D = x.shape
    width = D + 2 if mode != 2 else 8
    k = 4 if mode == 2 else 2
    nc = (row_offset + n - 1) // 4096 - row_offset // 4096 + 1
    parts = torch.empty((nc, width), dtype=torch.float64, device="cuda") if mode != 3 else None
    out = torch.empty((n, k), dtype=torch.float64, device="cuda")
    bg.rows(xt, c(y) if mode != 3 else None, c(w), c(off), c(coef), b, mu_const, _spec(spec), mode, row_offset, out, parts)
    if mode == 3:
        return None, out.cpu().numpy()
    tot = torch.zeros(width, dtype=torch.float64, device="cuda")
    call("b200flow_group_sums_chain", ptr(parts), nc, 1, width, ptr(tot))
    return tot.cpu().numpy(), out.cpu().numpy()


def _close(got, want, tol=SUM_TOL):
    """within tol of the largest finite |total|; non-finite totals (the log of a zero weight) equal"""
    fin = np.isfinite(want)
    if not np.array_equal(fin, np.isfinite(got)) or not np.array_equal(got[~fin], want[~fin]):
        return False
    scale = np.max(np.abs(want[fin])) if fin.any() else 0.0
    return np.max(np.abs(got[fin] - want[fin]), initial=0.0) <= tol * max(scale, 1e-300)


@pytest.mark.parametrize("spec", PAIRS)
def test_rows_pass_equals_the_restatement(spec):
    for D, n in ((1, 3000), (17, 5000), (119, 9001), (255, 4500)):
        x, y, coef, b = _problem(n, D, spec, D)
        rng = np.random.default_rng(D)
        for wo in (False, True):
            w = rng.integers(0, 4, n).astype(float) if wo else None
            off = rng.uniform(-0.05, 0.05, n) if wo else None
            for dtype in (np.float64, np.float32):
                xd = x.astype(dtype)
                x64 = xd.astype(np.float64)
                for mode in (0, 1, 2, 3):
                    want_t, want_r = go.rows(x64, y, w, off, coef, b, spec, mode)
                    for ro in ((0, 1000) if dtype == np.float64 else (1000,)):
                        got_t, got_r = _launch(xd, y, w, off, coef, b, spec, mode, ro)
                        if mode != 3:
                            assert _close(got_t, want_t), (D, wo, dtype, mode, ro, got_t, want_t)
                        assert np.allclose(got_r, want_r, rtol=1e-12, atol=1e-12 * np.max(np.abs(want_r))), \
                            (D, wo, dtype, mode, ro)
                if mode == 3 and D == 17:                     # the summary's constant-mean mode
                    mc = float(np.mean(y))
                    want_t, _ = go.rows(x64, y, w, off, None, 0.0, spec, 2, mu_const=mc)
                    got_t, _ = _launch(xd, y, w, off, None, 0.0, spec, 2, 0, mu_const=mc)
                    assert _close(got_t, want_t)


def test_canaries_f32_copies_and_shard_sums_give_the_same_bits():
    from b200flow import dist as bdist, glm as bg
    spec = (go.POISSON, go.LOG)
    x, y, coef, b = _problem(20000, 41, spec, 7)
    xt, yt = torch.as_tensor(x).cuda(), torch.as_tensor(y).cuda()
    ct = torch.as_tensor(coef).cuda()
    for off in (0, 1000):
        nc = (off + 20000 - 1) // 4096 - off // 4096 + 1
        buf = torch.full((nc * 43 + 128,), 777.0, dtype=torch.float64, device="cuda")
        rbuf = torch.full((2 * 20000 + 128,), 777.0, dtype=torch.float64, device="cuda")
        bg.rows(xt, yt, None, None, ct, b, 0.0, _spec(spec), 1, off, rbuf[64:64 + 40000].view(20000, 2),
                buf[64:64 + nc * 43].view(nc, 43))
        for h in (buf.cpu().numpy(), rbuf.cpu().numpy()):
            assert np.all(h[:64] == 777.0) and np.all(h[-64:] == 777.0) and not np.any(h[64:-64] == 777.0)
    sh = bdist.Shards(20000, 0, None, xt.device)
    xf = xt.float()
    for mode in (0, 1, 2):
        a = bg.rows_total(xf, yt, None, None, ct, b, _spec(spec), mode, sh)
        c = bg.rows_total(xf.double(), yt, None, None, ct, b, _spec(spec), mode, sh)
        assert torch.equal(a[0], c[0]) and torch.equal(a[1], c[1])
    w = torch.ones(20000, dtype=torch.float64, device="cuda")
    z = torch.zeros(20000, dtype=torch.float64, device="cuda")
    for mode in (0, 1, 2):                                 # unit weights and zero offsets are the defaults' bits
        a = bg.rows_total(xt, yt, None, None, ct, b, _spec(spec), mode, sh)
        c = bg.rows_total(xt, yt, w, z, ct, b, _spec(spec), mode, sh)
        assert torch.equal(a[0], c[0]) and torch.equal(a[1], c[1])


def test_weighted_gram_matches_numpy_and_the_unweighted_path():
    from b200flow import dist as bdist, pca
    rng = np.random.default_rng(13)
    x = rng.normal(0, 1, (30000, 119)) * rng.uniform(0.2, 3, 119)
    y = rng.normal(0, 2, 30000)
    w = rng.uniform(0, 3, 30000)
    xt, yt, wt = (torch.as_tensor(a).cuda() for a in (x, y, w))
    sh = bdist.Shards(30000, 0, None, xt.device)
    mx = (w @ x) / w.sum()
    my = float((w @ y) / w.sum())
    q = pca.centered_gram_total(xt, torch.as_tensor(mx).cuda(), sh, y=yt, y_mean=my, w=wt).cpu().numpy()
    a = np.hstack([x - mx, (y - my)[:, None]])
    G = (a.T * w) @ a
    iu = np.triu_indices(120)
    assert np.max(np.abs(q[iu[0] + iu[1] * (iu[1] + 1) // 2] - G[iu])) <= 1e-10 * np.max(np.abs(G))
    ones = torch.ones(30000, dtype=torch.float64, device="cuda")
    mt = torch.as_tensor(mx).cuda()
    assert torch.equal(pca.centered_gram_total(xt, mt, sh, y=yt, y_mean=my, w=ones),
                       pca.centered_gram_total(xt, mt, sh, y=yt, y_mean=my))
    old = pca.STAGE_BUDGET
    try:
        pca.STAGE_BUDGET = 8 * 120 * 4096 * 2
        assert np.array_equal(pca.centered_gram_total(xt, mt, sh, y=yt, y_mean=my, w=wt).cpu().numpy(), q)
    finally:
        pca.STAGE_BUDGET = old


# ----------------------------------------------------------------------------------- fits
def _shaped(shape, n, seed):
    rng = np.random.default_rng(seed)
    if shape == "kdd":                     # 38 numeric columns and one-hot blocks, one column of each block dropped
        num = np.log1p(np.abs(rng.standard_t(3, (n, 38))) * rng.uniform(0.1, 100.0, 38))
        blocks = [np.eye(k)[rng.integers(0, k, n)][:, 1:] for k in (3, 12, 8)]
        x = np.concatenate([num] + blocks, 1)
    else:
        x = np.log(rng.lognormal(0.0, 0.5, (n, 30)) * 10.0 ** rng.uniform(-1, 1, 30))
    x = (x - x.mean(0)) / x.std(0)
    beta = rng.normal(0, 0.15, x.shape[1]) / math.sqrt(x.shape[1])
    return np.ascontiguousarray(x), x @ beta + 0.2, rng


def _fit(x, y, dtype=torch.float64, w=None, off=None, **kw):
    from b200flow import glm as bg
    c = lambda a: None if a is None else torch.as_tensor(a).cuda()     # noqa: E731
    return bg.glm_fit(torch.as_tensor(x).cuda().to(dtype), torch.as_tensor(y).cuda(), bg.GLMParams(**kw), weight=c(w),
                      offset=c(off))


@pytest.mark.parametrize("shape", ["kdd", "cicids"])
@pytest.mark.parametrize("family", ["poisson", "gamma", "binomial"])
def test_fits_equal_the_restatement_and_sklearn(shape, family):
    sklm = pytest.importorskip("sklearn.linear_model")
    x, eta, rng = _shaped(shape, 20000, 3)
    if family == "poisson":
        y = rng.poisson(np.exp(eta)).astype(float)
        ref = sklm.PoissonRegressor(alpha=0, tol=1e-12, max_iter=1000)
        spec = (go.POISSON, go.LOG)
    elif family == "gamma":
        y = rng.gamma(2.0, np.exp(eta) / 2.0)
        ref = sklm.GammaRegressor(alpha=0, tol=1e-12, max_iter=1000)
        spec = (go.GAMMA, go.LOG)
    else:
        y = (rng.uniform(size=x.shape[0]) < 1 / (1 + np.exp(-eta))).astype(float)
        ref = sklm.LogisticRegression(C=np.inf, tol=1e-12, max_iter=2000)
        spec = (go.BINOMIAL, go.LOGIT)
    kw = dict(family=family, link="log" if family != "binomial" else "logit", tol=1e-10, max_iter=50)
    f = _fit(x, y, **kw)
    coef, b, diag, it = go.irls(x, y, spec, tol=1e-10, max_iter=50)
    assert f.iterations == it and np.allclose(f.coef, coef, rtol=1e-8, atol=1e-10) and math.isclose(
        f.intercept, b, rel_tol=1e-8, abs_tol=1e-10)
    assert np.allclose(f.diag_inv_atwa, diag, rtol=1e-6)
    ref.fit(x, y)
    assert np.allclose(f.coef, ref.coef_.reshape(-1), rtol=1e-5, atol=1e-6)
    f32 = _fit(x.astype(np.float32), y, **kw)
    f64 = _fit(x.astype(np.float32).astype(np.float64), y, **kw)
    assert np.array_equal(f32.coef, f64.coef) and f32.intercept == f64.intercept


def test_weights_offsets_fallback_and_refusals():
    from b200flow import glm as bg
    x, eta, rng = _shaped("cicids", 8000, 4)
    y = rng.poisson(np.exp(eta)).astype(float)
    w = rng.integers(0, 3, 8000).astype(float)
    off = rng.normal(0, 0.1, 8000)
    f = _fit(x, y, w=w, off=off, family="poisson", tol=1e-10)
    coef, b, _, it = go.irls(x, y, (go.POISSON, go.LOG), w=w, off=off, tol=1e-10)
    assert f.iterations == it and np.allclose(f.coef, coef, rtol=1e-8, atol=1e-10)
    xd = np.hstack([x, x[:, :1]])                           # a duplicated column: Cholesky fails, quasi-Newton solves
    fd = _fit(xd, y, family="poisson", tol=1e-8)
    assert fd.diag_inv_atwa is None and np.all(np.isfinite(fd.coef))
    fp = _fit(x, y, family="poisson", tol=1e-10)
    pd = xd @ fd.coef + fd.intercept
    assert np.max(np.abs(pd - (x @ fp.coef + fp.intercept))) < 1e-4
    for kw, yy, match in ((dict(family="poisson"), -y, "non-negative"), (dict(family="gamma"), y, "positive"),
                          (dict(family="binomial"), y + 2, "range"), (dict(family="gaussian", link="log"), y, "positive")):
        with pytest.raises(ValueError, match=match):
            _fit(x, yy, **kw)
    with pytest.raises(ValueError, match="Weights"):
        _fit(x, y, w=-w, family="poisson")
    with pytest.raises(ValueError, match="finite"):
        yb = y.copy()
        yb[3] = np.nan
        _fit(x, yb, family="poisson")
    with pytest.raises(bg._lib.UnsupportedParamError):
        _fit(np.zeros((10, 256)), np.ones(10), family="poisson")


@pytest.mark.parametrize("case", [("gaussian", None, (go.GAUSSIAN, go.IDENTITY)), ("poisson", "log", (go.POISSON, go.LOG)),
                                  ("gamma", "inverse", (go.GAMMA, go.INVERSE)), ("binomial", "probit", (go.BINOMIAL, go.PROBIT)),
                                  ("tweedie", None, (go.TWEEDIE, go.POWER, 1.5, -0.5))])
@pytest.mark.parametrize("fi", [True, False])
@pytest.mark.parametrize("with_off", [False, True])
def test_summary_equals_the_restatement(case, fi, with_off):
    from b200flow import glm as bg
    family, link, spec = case
    x, eta, rng = _shaped("cicids", 6000, 5)
    x = np.abs(x) * 0.1
    y = rng.gamma(2.0, 1.0, 6000) + 0.5 if family != "binomial" else (rng.uniform(size=6000) < 0.4).astype(float)
    w = rng.uniform(0.5, 2.0, 6000)
    off = rng.uniform(0, 0.05, 6000) if with_off else None
    kw = dict(family=family, link=link, fit_intercept=fi, tol=1e-10)
    if family == "tweedie":
        kw["variance_power"] = 1.5
    p = bg.GLMParams(**kw)
    xt = torch.as_tensor(x).cuda()
    f = bg.glm_fit(xt, torch.as_tensor(y).cuda(), p, weight=torch.as_tensor(w).cuda(),
                   offset=None if off is None else torch.as_tensor(off).cuda())
    s = bg.summarize(xt, torch.as_tensor(y).cuda(), f, p, weight=torch.as_tensor(w).cuda(),
                     offset=None if off is None else torch.as_tensor(off).cuda())
    want = go.summary(x, y, f.coef, f.intercept, spec, w=w, off=off, fit_intercept=fi, tol=1e-10)
    for k in ("deviance", "null_deviance", "dispersion"):
        assert math.isclose(getattr(s, k), want[k], rel_tol=1e-10), k
    assert (s.aic is None) == (want["aic"] is None)
    if s.aic is not None:
        assert math.isclose(s.aic, want["aic"], rel_tol=1e-10)
    assert s.rank == want["rank"] and s.degrees_of_freedom == want["dof"] and s.num_instances == 6000
    _, res = go.rows(x, y, w, off, f.coef, f.intercept, spec, 2)
    got = s.residuals.cpu().numpy()
    assert np.allclose(got[:, 1:], res[:, 1:], rtol=1e-9, atol=1e-12)
    assert np.allclose(got[:, 0], res[:, 0], rtol=1e-9, atol=1e-7)     # sqrt of a deviance term that cancels to ~0
    mu_eta = bg.glm_predict(xt, f, None if off is None else torch.as_tensor(off).cuda())
    assert torch.equal(mu_eta, s.predictions)
    se = np.sqrt(f.diag_inv_atwa * s.dispersion)
    assert np.array_equal(s.std_errors, se) and len(s.p_values) == x.shape[1] + fi


# ----------------------------------------------------------------------------------- the shim
def _frame(x, y, extra=None):
    from pyspark.sql import ColumnData, DataFrame
    from b200flow import synth
    rec, dicts = synth.make_kdd(x.shape[0], 2, seed=1, device="cuda:0")
    df = DataFrame.fromRecords(rec, synth.kdd_schema(), dicts).select("duration")
    cols = {"features": ColumnData("vector", torch.as_tensor(x).cuda(), "f64"),
            "label": ColumnData("numeric", torch.as_tensor(y).cuda(), "f64")}
    for k, v in (extra or {}).items():
        cols[k] = ColumnData("numeric", torch.as_tensor(v).cuda(), "f64")
    return df._with(cols=cols)


def test_shim_model_summary_link_prediction_and_refusals():
    from pyspark.ml.feature import IllegalArgumentException
    from pyspark.ml.regression import GeneralizedLinearRegression, UnsupportedOperationException
    x, eta, rng = _shaped("cicids", 5000, 6)
    y = rng.poisson(np.exp(eta)).astype(float)
    df = _frame(x, y, {"w": rng.uniform(0.5, 2, 5000), "off": rng.normal(0, 0.1, 5000)})
    glr = GeneralizedLinearRegression(family="poisson", weightCol="w", offsetCol="off", linkPredictionCol="eta")
    m = glr.fit(df)
    assert m.numFeatures == 30 and m.hasSummary
    out = m.transform(df)
    s = m.summary
    mu = out._column_tensor("prediction")
    assert torch.equal(mu, s.predictions._column_tensor("prediction"))
    assert torch.equal(out._column_tensor("eta"), s.predictions._column_tensor("eta"))
    assert torch.allclose(torch.exp(out._column_tensor("eta")), mu, rtol=1e-14)
    assert s.numIterations >= 2 and s.solver == "irls" and s.rank == 31 and s.degreesOfFreedom == 5000 - 31
    assert s.residualDegreeOfFreedom == 5000 - 31 and s.residualDegreeOfFreedomNull == 4999 and s.dispersion == 1.0
    assert len(s.coefficientStandardErrors) == 31 and len(s.tValues) == 31 and len(s.pValues) == 31
    assert s.nullDeviance > s.deviance > 0 and math.isfinite(s.aic)
    for t in ("deviance", "pearson", "working", "response"):
        assert s.residuals(t)._column_tensor(t + "Residuals").shape[0] == 5000
    assert m.evaluate(df).deviance == s.deviance
    with pytest.raises(UnsupportedOperationException):
        GeneralizedLinearRegression(family="tweedie", variancePower=1.5).fit(df).summary.aic
    with pytest.raises(IllegalArgumentException, match="does not support"):
        GeneralizedLinearRegression(family="poisson", link="logit").fit(df)
    with pytest.raises(IllegalArgumentException, match="variancePower"):
        GeneralizedLinearRegression(family="tweedie", variancePower=0.5).fit(df)
    with pytest.raises(IllegalArgumentException, match="does not exist"):
        GeneralizedLinearRegression(offsetCol="nope").fit(df)


def test_shim_pipeline_and_model_selection():
    from pyspark.ml import Pipeline
    from pyspark.ml.evaluation import RegressionEvaluator
    from pyspark.ml.feature import StandardScaler, VectorAssembler
    from pyspark.ml.regression import GeneralizedLinearRegression
    from pyspark.ml.tuning import CrossValidator, ParamGridBuilder, TrainValidationSplit, fold_frames
    from pyspark.sql import ColumnData, DataFrame
    from b200flow import synth
    rec, dicts = synth.make_kdd(20000, 5, seed=7, device="cuda:0")
    df = DataFrame.fromRecords(rec, synth.kdd_schema(), dicts)
    nums = [c for c in synth.KDD_COLUMNS if c not in synth.KDD_CATEGORICAL + ["label"]]
    feats = [c for c in nums if c not in ("count",)]
    cols = dict(df._cols)
    cols["target"] = ColumnData("numeric", df._column_tensor("count").to(torch.float64), "f64")
    df = df._with(cols=cols)
    glr = GeneralizedLinearRegression(family="poisson", labelCol="target", maxIter=10)
    pipe = Pipeline(stages=[VectorAssembler(inputCols=feats, outputCol="raw"),
                            StandardScaler(inputCol="raw", outputCol="features"), glr])
    out = pipe.fit(df).transform(df)
    ev = RegressionEvaluator(labelCol="target", metricName="rmse")
    assert math.isfinite(ev.evaluate(out))
    grid = ParamGridBuilder().addGrid(glr.regParam, [0.0, 0.1]).build()
    data = Pipeline(stages=pipe.getStages()[:2]).fit(df).transform(df).select("features", "target")
    cvm = CrossValidator(estimator=glr, estimatorParamMaps=grid, evaluator=ev, numFolds=2, seed=3).fit(data)
    want = [0.0] * len(grid)
    for train, val in fold_frames(data, 2, 3):
        for i, pm in enumerate(grid):
            want[i] += ev.evaluate(glr.fit(train, pm).transform(val))
    assert cvm.avgMetrics == [v / 2 for v in want]
    tvs = TrainValidationSplit(estimator=glr, estimatorParamMaps=grid, evaluator=ev, trainRatio=0.75, seed=3).fit(data)
    assert len(tvs.validationMetrics) == len(grid)
