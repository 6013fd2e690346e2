"""LinearRegression without a GPU: params, defaults and refusals; the numpy restatement (tests/linreg_oracle.py) against
finite differences; linear.lbfgs on the restated objectives and the host normal-equation solver (b200flow.linreg
.solve_normal) against scikit-learn's optima; standard errors against the textbook formula and p values against scipy."""
import math

import numpy as np
import pytest
import torch

import linreg_oracle as lo
from b200flow import linreg as blr

sklm = pytest.importorskip("sklearn.linear_model")

COEF_TOL = 1e-6          # relative to the largest |coefficient|: both sides stop on a gradient tolerance, not exactly


def _data(n=400, D=6, seed=0, noise="normal", outliers=0):
    rng = np.random.default_rng(seed)
    x = rng.normal(0.0, 1.0, (n, D)) * rng.uniform(0.3, 5.0, D) + rng.normal(0.0, 2.0, D)
    beta = rng.normal(0.0, 2.0, D)
    e = rng.standard_t(3, n) if noise == "t" else rng.normal(0.0, 1.0, n)
    y = x @ beta + 3.0 + e
    if outliers:
        y[:outliers] += 50.0
    return np.ascontiguousarray(x), y


def _close(a, b, tol=COEF_TOL):
    a, b = np.atleast_1d(np.asarray(a, float)), np.atleast_1d(np.asarray(b, float))
    return np.max(np.abs(a - b)) <= tol * max(1.0, np.max(np.abs(b)))


def _normal(x, y, **kw):
    p = blr.LinRegParams(**kw)
    n, xb, yb, G = lo.normal_statistics(x, y)
    return blr.solve_normal(n, xb, yb, G, p)


# ----------------------------------------------------------------------------------- params and refusals
def test_defaults_match_spark():
    from pyspark.ml.regression import LinearRegression
    lr = LinearRegression()
    want = dict(maxIter=100, regParam=0.0, elasticNetParam=0.0, tol=1e-6, fitIntercept=True, standardization=True,
                solver="auto", loss="squaredError", epsilon=1.35, aggregationDepth=2, maxBlockSizeInMB=0.0, weightCol=None,
                featuresCol="features", labelCol="label", predictionCol="prediction")
    for k, v in want.items():
        assert lr.getOrDefault(k) == v, k
    assert lr.setRegParam(0.5).getRegParam() == 0.5


@pytest.mark.parametrize("kw,match", [
    (dict(loss="huber", solver="normal"), "huber loss doesn't support normal solver"),
    (dict(loss="huber", elastic_net_param=0.5), "only supports L2 regularization"),
    (dict(epsilon=1.0), "epsilon"), (dict(solver="sgd"), "solver"), (dict(loss="absolute"), "loss"),
    (dict(elastic_net_param=1.5), "elasticNetParam"), (dict(reg_param=-1.0), "regParam"), (dict(max_iter=-1), "maxIter")])
def test_refusals(kw, match):
    with pytest.raises(ValueError, match=match):
        blr.check_params(blr.LinRegParams(**kw))


def test_shim_refuses_before_touching_the_data():
    from pyspark.ml.feature import IllegalArgumentException
    from pyspark.ml.regression import LinearRegression
    for lr in (LinearRegression(loss="huber", solver="normal"), LinearRegression(loss="huber", elasticNetParam=0.1),
               LinearRegression(weightCol="w"), LinearRegression(aggregationDepth=1)):
        with pytest.raises(IllegalArgumentException):
            lr._check()


def test_solver_choice():
    assert blr.solver_for(blr.LinRegParams()) == "normal"
    assert blr.solver_for(blr.LinRegParams(solver="normal")) == "normal"
    assert blr.solver_for(blr.LinRegParams(solver="l-bfgs")) == "l-bfgs"
    assert blr.solver_for(blr.LinRegParams(loss="huber")) == "l-bfgs"


# ----------------------------------------------------------------------------------- the restatement
@pytest.mark.parametrize("fi,st", [(True, True), (False, False)])
def test_gradients_match_finite_differences(fi, st):
    x, y = _data(200, 5, 1, "t", outliers=10)
    rng = np.random.default_rng(2)
    w = rng.normal(0, 0.5, 5)
    v = np.concatenate([w, [0.7, 1.3]])
    for fun, point in ((lambda u: lo.squared_objective(u, x, y, 0.3, 0.0, fi, st), w),
                       (lambda u: lo.huber_objective(u, x, y, 0.3, 1.35, fi, st), v)):
        f, g = fun(point)
        for j in range(len(point)):
            if not fi and len(point) == 7 and j == 5:
                assert g[j] == 0.0
                continue
            h = 1e-6 * max(1.0, abs(point[j]))
            e = np.zeros_like(point)
            e[j] = h
            fd = (fun(point + e)[0] - fun(point - e)[0]) / (2 * h)
            assert abs(fd - g[j]) <= 1e-6 * max(1.0, abs(g[j])), (j, fd, g[j])


@pytest.mark.parametrize("fi", [True, False])
def test_ols_equals_sklearn_on_both_solvers(fi):
    x, y = _data(500, 6, 3)
    sk = sklm.LinearRegression(fit_intercept=fi).fit(x, y)
    coef, b, hist, it, diag, solver = _normal(x, y, fit_intercept=fi)
    assert solver == "normal" and hist == [0.0] and it == 0 and diag is not None
    assert _close(coef, sk.coef_) and _close(b, sk.intercept_)
    coef, b = lo.lbfgs_squared(x, y, fi=fi)
    assert _close(coef, sk.coef_, 1e-5) and _close(b, sk.intercept_, 1e-5)
    sc, sb, sd = lo.normal_solve_spark(x, y, fi=fi)
    assert _close(sc, sk.coef_) and _close(sb, sk.intercept_)


def test_lasso_equals_sklearn_on_both_solvers():
    """elasticNetParam = 1, standardization = false: multiplying the objective by yStd^2 (or bStd^2) gives
    (1/2n) |y - y_bar - (x - x_bar) beta|^2 + regParam |beta|_1, scikit-learn's Lasso at alpha = regParam"""
    x, y = _data(500, 6, 4)
    reg = 0.3
    sk = sklm.Lasso(alpha=reg, tol=1e-14, max_iter=100000).fit(x, y)
    coef, b, hist, it, diag, solver = _normal(x, y, reg_param=reg, elastic_net_param=1.0, standardization=False,
                                              max_iter=1000, tol=1e-14)
    assert solver == "quasi-newton" and diag is None and it == len(hist) - 1
    assert _close(coef, sk.coef_, 1e-5) and _close(b, sk.intercept_, 1e-5)
    coef, b = lo.lbfgs_squared(x, y, reg=reg, alpha=1.0, st=False, max_iter=1000)
    assert _close(coef, sk.coef_, 1e-5) and _close(b, sk.intercept_, 1e-5)


@pytest.mark.parametrize("fi", [True, False])
def test_ridge_equals_sklearn_under_the_alpha_mapping(fi):
    """elasticNetParam = 0, standardization = false: lambda_j = (regParam / yStd) / std_j^2 on w_j = beta_j std_j / yStd,
    so the penalty is 1/2 (regParam / yStd^3) |beta|^2 and the loss (1/2n yStd^2) |r|^2.  Multiplied by 2 n yStd^2 that is
    |r|^2 + (n regParam / yStd) |beta|^2: Ridge at alpha = n lambda / yStd, with the population yStd on the normal path
    and the unbiased one on the L-BFGS path."""
    x, y = _data(300, 5, 5)
    n, reg = x.shape[0], 0.2
    for ystd, fit in ((y.std(), "normal"), (y.std(ddof=1), "lbfgs")):
        sk = sklm.Ridge(alpha=n * reg / ystd, fit_intercept=fi, tol=1e-14).fit(x, y)
        if fit == "normal":
            coef, b = _normal(x, y, reg_param=reg, standardization=False, fit_intercept=fi)[:2]
        else:
            coef, b = lo.lbfgs_squared(x, y, reg=reg, fi=fi, st=False)
        assert _close(coef, sk.coef_, 1e-5) and _close(b, sk.intercept_, 1e-5), fit


@pytest.mark.parametrize("fi", [True, False])
def test_huber_equals_sklearn(fi):
    """standardization = false: (n times) the objective is scikit-learn's HuberRegressor with alpha = n lambda / 2"""
    x, y = _data(300, 4, 6, "t", outliers=15)
    n, reg, eps = x.shape[0], 0.01, 1.35
    sk = sklm.HuberRegressor(epsilon=eps, alpha=n * reg / 2, fit_intercept=fi, max_iter=100000, tol=1e-12).fit(x, y)
    coef, b, sigma = lo.lbfgs_huber(x, y, reg=reg, eps=eps, fi=fi, st=False)
    assert _close(coef, sk.coef_, 1e-4) and _close(b, sk.intercept_, 1e-4) and abs(sigma - sk.scale_) <= 1e-4 * sk.scale_


def test_standard_errors_equal_the_textbook_formula():
    x, y = _data(120, 4, 7)
    coef, b, _, _, diag, _ = _normal(x, y)
    X1 = np.concatenate([x, np.ones((x.shape[0], 1))], 1)
    res = y - X1 @ np.concatenate([coef, [b]])
    s2 = res @ res / (x.shape[0] - 5)
    want = np.sqrt(np.diag(np.linalg.inv(X1.T @ X1)) * s2)
    got = lo.summary(x, y, coef, b, diag, True)["se"]
    assert np.max(np.abs(got - want) / want) <= 1e-9
    sc, sb, sd = lo.normal_solve_spark(x, y)
    assert np.max(np.abs(sd - diag) / diag) <= 1e-9


def test_p_values_from_the_f_cdf_equal_students_t():
    from scipy import stats
    from b200flow import selection
    for t, dof in ((0.3, 5), (2.1, 17), (-4.0, 100), (8.0, 3), (0.0, 12)):
        got = 1.0 - selection.f_cdf(t * t, 1.0, float(dof))
        want = 2.0 * stats.t.sf(abs(t), dof)
        assert abs(got - want) <= 1e-12 + 1e-9 * want, (t, dof)


def test_constant_label_and_collinear_columns_on_the_host_solver():
    x, y = _data(200, 4, 8)
    coef, b, hist, it, diag, solver = _normal(x, np.full(200, 2.5))
    assert np.all(coef == 0.0) and b == 2.5 and hist == [0.0] and diag is None
    with pytest.raises(ValueError, match="standard deviation of the label is zero"):
        _normal(x, np.full(200, 2.5), fit_intercept=False, reg_param=0.1)
    xd = np.concatenate([x, x[:, 1:2]], 1)                 # a duplicated column: Cholesky -> quasi-Newton
    coef, b, hist, it, diag, solver = _normal(xd, y, max_iter=500, tol=1e-14)
    assert solver == "quasi-newton" and diag is None
    sk = sklm.LinearRegression().fit(xd, y)
    assert np.max(np.abs(xd @ coef + b - sk.predict(xd))) <= 1e-6 * np.max(np.abs(y))
    xc = x.copy()
    xc[:, 2] = 7.0                                         # a constant column without regularisation
    coef, b, hist, it, diag, solver = _normal(xc, y, max_iter=500, tol=1e-14)
    assert solver == "quasi-newton" and coef[2] == 0.0
    assert math.isfinite(b)


def test_lbfgs_rejects_a_non_positive_sigma():
    """the Huber driver's f = +inf for sigma <= 0: the line search halves until sigma > 0"""
    calls = []

    def smooth(v):
        calls.append(float(v[1]))
        if not v[1] > 0:
            return torch.tensor(math.inf, dtype=torch.float64), torch.zeros_like(v)
        return (v[0] - 1) ** 2 + v[1] + 0.1 / v[1], torch.stack([2 * (v[0] - 1), 1 - 0.1 / v[1] ** 2])

    from b200flow.linear import lbfgs
    v, hist, it = lbfgs(smooth, torch.tensor([0.0, 5.0], dtype=torch.float64), 100, 1e-14)
    assert abs(float(v[1]) - math.sqrt(0.1)) <= 1e-6 and abs(float(v[0]) - 1.0) <= 1e-6
