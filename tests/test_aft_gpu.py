"""AFTSurvivalRegression on the device: the AFT instantiation of the per-row kernel against the numpy restatement
(tests/aft_oracle.py) across D, dtypes, centring and row offsets that straddle 4096-row chunks, canaries around its
partials, chunk-order totals that are the same bits for any batch split, fits against the restatement's, recovery of
known Weibull parameters on KDD- and CICIDS-shaped data with independent censoring, a trial point that overflows e^z,
refusals, and the shim under Pipeline and CrossValidator."""
import math

import numpy as np
import pytest
import torch

import aft_oracle as ao

pytestmark = pytest.mark.gpu


def _problem(n, D, seed):
    rng = np.random.default_rng(seed)
    x = rng.normal(0.0, 1.0, (n, D)) * rng.uniform(0.2, 4.0, D) + rng.normal(0, 3, D)
    t = np.exp(rng.normal(1.0, 1.0, n))
    c = (rng.random(n) < 0.7).astype(np.float64)
    return np.ascontiguousarray(x), t, c


def _dev(a, dtype=np.float64):
    return None if a is None else torch.as_tensor(np.ascontiguousarray(a, dtype)).cuda()


def _totals(x, t, c, shift, inv, w, bs, row_offset=0):
    """the chained totals; a nonzero row_offset moves the chunk boundaries (one launch, chained here)"""
    from b200flow import aft as baft, dist as bdist
    from b200flow._lib import call, ptr
    xt = torch.as_tensor(x).cuda()
    lt, ct = _dev(np.log(t)), _dev(c, np.int32)
    if row_offset == 0:
        sh = bdist.Shards(xt.shape[0], 0, None, xt.device)
        return baft.loss_grad_totals(xt, lt, ct, _dev(shift), _dev(inv), _dev(w), _dev(bs), sh).cpu().numpy()
    D = x.shape[1]
    nc = (row_offset + x.shape[0] - 1) // 4096 - row_offset // 4096 + 1
    parts = torch.empty((nc, D + 3), dtype=torch.float64, device="cuda")
    baft.loss_grad(xt, lt, ct, _dev(shift), _dev(inv), _dev(w), _dev(bs), row_offset, parts)
    tot = torch.zeros(D + 3, dtype=torch.float64, device="cuda")
    call("b200flow_group_sums_chain", ptr(parts), nc, 1, D + 3, ptr(tot))
    return tot.cpu().numpy()


@pytest.mark.parametrize("n,D", [(1000, 1), (12289, 2), (4096, 41), (9001, 119), (5000, 255)])
@pytest.mark.parametrize("shifted", [False, True])
def test_totals_equal_the_restatement(n, D, shifted):
    x, t, c = _problem(n, D, 11)
    rng = np.random.default_rng(3)
    inv = ao.inv_std(x)
    w = rng.normal(0, 0.3 / math.sqrt(D), D)
    shift = x.mean(0) if shifted else None
    b, sigma = 0.4, 1.3
    bs = [b, sigma, math.log(sigma)]
    for dtype in (np.float64, np.float32):
        xd = x.astype(dtype)
        want = ao.sums(xd.astype(np.float64), np.log(t), c, shift, inv, w, b, sigma)
        gtol = 1e-10 * max(1.0, np.max(np.abs(want[1:])))
        for off in (0, 1000, 4095):
            got = _totals(xd, t, c, shift, inv, w, bs, off)
            assert abs(got[0] - want[0]) <= 1e-12 * abs(want[0]), (dtype, off)
            assert np.max(np.abs(got[1:] - want[1:])) <= gtol, (dtype, off)


def test_canaries_and_chunk_batches_give_the_same_bits():
    from b200flow import aft as baft, dist as bdist, selection
    x, t, c = _problem(20000, 41, 12)
    xt, lt, ct = torch.as_tensor(x).cuda(), _dev(np.log(t)), _dev(c, np.int32)
    inv = _dev(ao.inv_std(x))
    w = _dev(np.random.default_rng(1).normal(0, 0.05, 41))
    bs = _dev([0.2, 1.7, math.log(1.7)])
    for off in (0, 1000):
        nc = (off + 20000 - 1) // 4096 - off // 4096 + 1
        buf = torch.full((nc * 44 + 128,), 777.0, dtype=torch.float64, device="cuda")
        baft.loss_grad(xt, lt, ct, None, inv, w, bs, off, buf[64:64 + nc * 44].view(nc, 44))
        h = buf.cpu().numpy()
        assert np.all(h[:64] == 777.0) and np.all(h[-64:] == 777.0) and not np.any(h[64:-64] == 777.0)
    sh = bdist.Shards(20000, 0, None, xt.device)
    full = baft.loss_grad_totals(xt, lt, ct, None, inv, w, bs, sh).cpu().numpy()
    old = selection.PARTIALS_BUDGET
    try:
        for budget in (44 * 8, 44 * 8 * 3):              # one and three chunks per batch
            selection.PARTIALS_BUDGET = budget
            assert np.array_equal(baft.loss_grad_totals(xt, lt, ct, None, inv, w, bs, sh).cpu().numpy(), full)
    finally:
        selection.PARTIALS_BUDGET = old
    assert np.array_equal(baft.loss_grad_totals(xt.float(), lt, ct, None, inv, w, bs, sh).cpu().numpy(),
                          baft.loss_grad_totals(xt.float().double(), lt, ct, None, inv, w, bs, sh).cpu().numpy())


def _fit(x, t, c, dtype=torch.float64, **kw):
    from b200flow import aft as baft
    return baft.aft_fit(torch.as_tensor(x).cuda().to(dtype), torch.as_tensor(t).cuda(), torch.as_tensor(c).cuda(),
                        baft.AFTParams(**kw))


@pytest.mark.parametrize("fi", [True, False])
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_fit_equals_the_restatement(fi, dtype):
    x, t, c, _, _ = ao.weibull_data(6000, 5, 4, censor_rate=0.3)
    x = x * [1.0, 10.0, 0.1, 3.0, 1.0] + [0.0, 5.0, -1.0, 0.0, 2.0]
    if dtype == torch.float32:
        x = x.astype(np.float32).astype(np.float64)
    f = _fit(x, t, c, dtype=dtype, fit_intercept=fi, max_iter=200, tol=1e-12)
    coef, b, sigma, hist = ao.fit(x, t, c, fi=fi, max_iter=200, tol=1e-12)
    assert np.max(np.abs(f.coef - coef)) <= 1e-7 * max(1.0, np.max(np.abs(coef)))
    assert abs(f.intercept - b) <= 1e-7 * max(1.0, abs(b)) and abs(f.scale - sigma) <= 1e-7 * sigma
    assert abs(f.objective_history[-1] - hist[-1]) <= 1e-10 * abs(hist[-1])
    assert len(f.objective_history) == f.iterations + 1


def _kdd(n, seed):
    """KDD-shaped: 38 numeric columns of mixed scale and three one-hot blocks (D = 119)"""
    rng = np.random.default_rng(seed)
    num = np.abs(rng.standard_t(3, (n, 38))) * rng.uniform(0.1, 100.0, 38)
    blocks = [np.eye(k)[rng.integers(0, k, n)] for k in (3, 70, 8)]
    return np.ascontiguousarray(np.concatenate([num] + blocks, 1)), rng


def _cicids(n, seed):
    """CICIDS-shaped: 78 continuous, skewed flow statistics over scales from 0.1 to 1000"""
    rng = np.random.default_rng(seed)
    return np.ascontiguousarray(rng.lognormal(0.0, 0.5, (n, 78)) * 10.0 ** rng.uniform(-1, 3, 78)), rng


@pytest.mark.parametrize("shape", ["kdd", "cicids"])
def test_recovers_known_weibull_parameters(shape):
    """synthetic Weibull lifetimes with independent exponential censoring: the fit recovers (beta, b, sigma) within a few
    standard errors (a handful of coefficients carry signal; the rest are 0)"""
    n = 200000
    x, rng = (_kdd if shape == "kdd" else _cicids)(n, 5)
    D = x.shape[1]
    sd = x.std(0)
    beta = np.zeros(D)
    idx = [0, 3, 7, 20] if shape == "kdd" else [1, 2, 30, 60]
    beta[idx] = np.array([0.4, -0.3, 0.2, 0.5]) / sd[idx]
    b, sigma = 2.0, 0.6
    t = np.exp(x @ beta + b + sigma * np.log(rng.exponential(1.0, n)))
    cen = rng.exponential(np.median(t) * 2.0, n)
    obs, c = np.minimum(t, cen), (t <= cen).astype(np.float64)
    assert 0.1 < 1.0 - c.mean() < 0.5
    f = _fit(x, obs, c, max_iter=300, tol=1e-10)
    # a standardised coefficient's standard error is about sigma / sqrt(events); the bound allows 10 of them for the
    # largest of D deviations and the information lost to censoring
    se = sigma / math.sqrt(c.sum())
    assert np.max(np.abs((f.coef - beta) * sd)) <= 10 * se
    assert abs(f.scale - sigma) <= 10 * se
    pred = x @ f.coef + f.intercept
    assert abs(np.mean(pred - (x @ beta + b))) <= 10 * se


def test_an_overflowing_trial_point_still_converges(monkeypatch):
    """sigma = 0.3 data: L-BFGS's early trial points overshoot to a small sigma where e^z overflows; each is rejected
    (f = inf, no gradient) and the fit converges to the restatement's optimum"""
    from b200flow import aft as baft, dist as bdist
    x, t, c, _, _ = ao.weibull_data(4000, 3, 6, censor_rate=0.2, sigma=0.3)
    xt = torch.as_tensor(x).cuda()
    sh = bdist.Shards(4000, 0, None, xt.device)
    bs = _dev([0.0, math.exp(-6.0), -6.0])
    tot = baft.loss_grad_totals(xt, _dev(np.log(t)), _dev(c, np.int32), None, _dev(ao.inv_std(x)), _dev(np.zeros(3)), bs, sh)
    assert not bool(torch.isfinite(tot).all())
    seen = []
    orig = baft.loss_grad_totals

    def counting(*a):
        tot = orig(*a)
        seen.append(bool(torch.isfinite(tot).all()))
        return tot

    monkeypatch.setattr(baft, "loss_grad_totals", counting)
    f = _fit(x, t, c, max_iter=300, tol=1e-12)
    coef, b, sigma, hist = ao.fit(x, t, c, max_iter=300, tol=1e-12)
    assert not all(seen), "no trial point overflowed"
    assert math.isfinite(f.objective_history[-1]) and f.scale > 0
    assert abs(f.objective_history[-1] - hist[-1]) <= 1e-9 * abs(hist[-1])
    assert abs(f.scale - sigma) <= 1e-6 * sigma and np.max(np.abs(f.coef - coef)) <= 1e-6


def test_refusals_on_the_device():
    from b200flow import _lib, aft as baft
    p = baft.AFTParams()
    ones = torch.ones(10, dtype=torch.float64, device="cuda")
    with pytest.raises(_lib.UnsupportedParamError):
        baft.aft_fit(torch.zeros((10, 256), dtype=torch.float64, device="cuda"), ones, ones, p)
    with pytest.raises(ValueError, match="at least one row"):
        baft.aft_fit(torch.zeros((0, 3), dtype=torch.float64, device="cuda"), ones[:0], ones[:0], p)
    x = torch.randn((10, 3), dtype=torch.float64, device="cuda")
    t = torch.arange(1, 11, dtype=torch.float64, device="cuda")
    for what, val, msg in (("t", 0.0, "greater than 0"), ("t", -1.0, "greater than 0"), ("t", math.nan, "greater than 0"),
                           ("t", math.inf, "greater than 0"), ("c", 0.5, "censor must be"), ("c", math.nan, "censor must be"),
                           ("x", math.nan, "finite features")):
        xb, tb, cb = x.clone(), t.clone(), ones.clone()
        {"x": xb[3], "t": tb, "c": cb}[what][1] = val
        with pytest.raises(ValueError, match=msg):
            baft.aft_fit(xb, tb, cb, p)
    with pytest.raises(ValueError, match="one label and one censor"):
        baft.aft_fit(x, t, ones[:9], p)


# ----------------------------------------------------------------------------------- the shim
def _frame(x, t, c):
    from pyspark.sql import ColumnData, DataFrame
    from b200flow import synth
    rec, dicts = synth.make_kdd(x.shape[0], 2, seed=1, device="cuda:0")
    df = DataFrame.fromRecords(rec, synth.kdd_schema(), dicts).select("duration")
    return df._with(cols={"features": ColumnData("vector", torch.as_tensor(x).cuda(), "f64"),
                          "label": ColumnData("numeric", torch.as_tensor(t).cuda(), "f64"),
                          "censor": ColumnData("numeric", torch.as_tensor(c).cuda(), "f64")})


def test_shim_model_predict_quantiles_and_refusals():
    from pyspark.ml.feature import IllegalArgumentException
    from pyspark.ml.linalg import Vectors
    from pyspark.ml.regression import AFTSurvivalRegression
    x, t, c, _, _ = ao.weibull_data(5000, 4, 7)
    df = _frame(x, t, c)
    probs = [0.1, 0.5, 0.9]
    m = AFTSurvivalRegression(quantileProbabilities=probs, quantilesCol="quantiles").fit(df)
    coef, b, sigma, _ = ao.fit(x, t, c)
    assert m.numFeatures == 4 and abs(m.scale - sigma) <= 1e-6 * sigma and abs(m.intercept - b) <= 1e-6 * max(1, abs(b))
    assert np.max(np.abs(m.coefficients.toArray() - coef)) <= 1e-6
    out = m.transform(df)
    pred = out._column_tensor("prediction").cpu().numpy()
    want = np.exp(x @ m.coefficients.toArray() + m.intercept)
    assert np.max(np.abs(pred - want) / want) <= 1e-12
    q = out._cols["quantiles"].data.cpu().numpy()
    assert q.shape == (5000, 3)
    assert np.max(np.abs(q - ao.quantiles(x, m.coefficients.toArray(), m.intercept, m.scale, probs)) / q) <= 1e-12
    assert abs(m.predict(Vectors.dense(x[17])) - pred[17]) <= 1e-14 * pred[17]
    assert np.allclose(m.predictQuantiles(Vectors.dense(x[17])).toArray(), q[17], rtol=1e-14, atol=0)
    assert "quantiles" not in AFTSurvivalRegression().fit(df).transform(df)._cols
    from pyspark.sql import ColumnData
    half = torch.full((5000,), 0.5, dtype=torch.float64, device="cuda")
    bad = df._with(cols=dict(df._cols, censor=ColumnData("numeric", half, "f64")))
    with pytest.raises(IllegalArgumentException, match="censor must be"):
        AFTSurvivalRegression().fit(bad)
    with pytest.raises(IllegalArgumentException, match="already exists"):
        m.transform(out)


def test_shim_pipeline_and_cross_validation():
    from pyspark.ml import Pipeline
    from pyspark.ml.evaluation import RegressionEvaluator
    from pyspark.ml.feature import StandardScaler, VectorAssembler
    from pyspark.ml.regression import AFTSurvivalRegression
    from pyspark.ml.tuning import CrossValidator, ParamGridBuilder, fold_frames
    from pyspark.sql import ColumnData, DataFrame
    from b200flow import synth
    rec, dicts = synth.make_kdd(20000, 5, seed=7, device="cuda:0")
    df = DataFrame.fromRecords(rec, synth.kdd_schema(), dicts)
    nums = [c for c in synth.KDD_COLUMNS if c not in synth.KDD_CATEGORICAL + ["label", "duration"]]
    cols = dict(df._cols)
    dur = df._column_tensor("duration").to(torch.float64)
    cols["time"] = ColumnData("numeric", dur + 1.0, "f64")                    # flow duration + 1 s: positive
    cols["censor"] = ColumnData("numeric", (torch.arange(20000, device="cuda") % 4 != 0).to(torch.float64), "f64")
    df = df._with(cols=cols)
    aft = AFTSurvivalRegression(labelCol="time", maxIter=30, quantilesCol="q")
    pipe = Pipeline(stages=[VectorAssembler(inputCols=nums, outputCol="raw"),
                            StandardScaler(inputCol="raw", outputCol="features"), aft])
    out = pipe.fit(df).transform(df)
    ev = RegressionEvaluator(labelCol="time", metricName="rmse")
    assert math.isfinite(ev.evaluate(out)) and out._cols["q"].data.shape == (20000, 9)
    grid = ParamGridBuilder().addGrid(aft.fitIntercept, [True, False]).addGrid(aft.maxIter, [5, 20]).build()
    data = Pipeline(stages=pipe.getStages()[:2]).fit(df).transform(df).select("features", "time", "censor")
    cvm = CrossValidator(estimator=aft, estimatorParamMaps=grid, evaluator=ev, numFolds=2, seed=3).fit(data)
    want = [0.0] * len(grid)
    for train, val in fold_frames(data, 2, 3):
        for i, pm in enumerate(grid):
            want[i] += ev.evaluate(aft.fit(train, pm).transform(val))
    assert cvm.avgMetrics == [v / 2 for v in want]
