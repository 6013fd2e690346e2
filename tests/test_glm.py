"""GeneralizedLinearRegression without a GPU: params, validators and refusals; the restated families and links
(tests/glm_oracle.py) against finite differences and scipy; the restated IRLS against scikit-learn's GLMs and a direct
Newton solve of the score equations; weights against row replication, offsets against a shifted label; deviance, AIC,
standard errors and p values against independent formulas; and the penalised normal equations at regParam > 0."""
import math

import numpy as np
import pytest
from scipy import optimize, stats

import glm_oracle as go


def _x(n, D, seed):
    rng = np.random.default_rng(seed)
    return rng.normal(0.0, 1.0, (n, D)) * rng.uniform(0.3, 1.5, D), rng


def _pred(x, coef, b):
    return x @ coef + b


# ----------------------------------------------------------------------------------- params
def test_params_resolve_and_refusals():
    from b200flow import glm as bg
    P = bg.GLMParams
    assert bg.resolve(P()) == bg.Spec(bg.GAUSSIAN, bg.IDENTITY)
    for fam, link in bg.CANONICAL.items():
        assert bg.resolve(P(family=fam)) == bg.Spec(bg.FAMILIES.index(fam), bg.LINKS.index(link))
        for l in bg.SUPPORTED[fam]:
            bg.check_params(P(family=fam, link=l))
    assert bg.resolve(P(family="tweedie")) == bg.Spec(bg.GAUSSIAN, bg.IDENTITY)
    assert bg.resolve(P(family="tweedie", variance_power=1.0)) == bg.Spec(bg.POISSON, bg.LOG)
    assert bg.resolve(P(family="tweedie", variance_power=2.0)) == bg.Spec(bg.GAMMA, bg.INVERSE)
    assert bg.resolve(P(family="tweedie", variance_power=1.5)) == bg.Spec(bg.TWEEDIE, bg.POWER, 1.5, -0.5)
    assert bg.resolve(P(family="tweedie", variance_power=1.5, link_power=0.0)) == bg.Spec(bg.TWEEDIE, bg.LOG, 1.5, 0.0)
    assert bg.resolve(P(family="tweedie", variance_power=3.0, link_power=0.5)) == bg.Spec(bg.TWEEDIE, bg.SQRT, 3.0, 0.0)
    p = P()
    assert (p.max_iter, p.tol, p.reg_param, p.fit_intercept, p.solver) == (25, 1e-6, 0.0, True, "irls")
    for fam in bg.SUPPORTED:
        for l in bg.LINKS:
            if l not in bg.SUPPORTED[fam]:
                with pytest.raises(ValueError, match="does not support %s link function" % l):
                    bg.check_params(P(family=fam, link=l))
    for bad in (dict(family="nope"), dict(link="nope"), dict(family="tweedie", variance_power=0.5),
                dict(family="tweedie", variance_power=-1.0), dict(max_iter=-1), dict(tol=-1.0), dict(reg_param=-0.1),
                dict(solver="l-bfgs")):
        with pytest.raises(ValueError):
            bg.check_params(P(**bad))
    bg.check_params(P(family="tweedie", variance_power=1.2, link="logit"))     # link is ignored for tweedie


# ----------------------------------------------------------------------------------- families and links
@pytest.mark.parametrize("l,lp,mu", [(go.IDENTITY, 0, 0.3), (go.LOG, 0, 0.3), (go.INVERSE, 0, 0.3), (go.LOGIT, 0, 0.3),
                                     (go.PROBIT, 0, 0.3), (go.CLOGLOG, 0, 0.3), (go.SQRT, 0, 0.3), (go.POWER, -0.5, 0.7),
                                     (go.POWER, 0.0, 0.7), (go.POWER, 1.7, 0.7)])
def test_links_invert_and_differentiate(l, lp, mu):
    mus = np.array([mu, mu / 3, 0.9])
    assert np.allclose(go.unlink(l, go.link(l, mus, lp), lp), mus, rtol=1e-13, atol=0)
    h = 1e-6
    fd = (go.link(l, mus + h, lp) - go.link(l, mus - h, lp)) / (2 * h)
    assert np.allclose(go.deriv(l, mus, lp), fd, rtol=1e-7)
    if l == go.PROBIT:
        assert np.allclose(go.link(l, mus), stats.norm.ppf(mus), rtol=1e-14)
        assert np.allclose(go.deriv(l, mus), 1.0 / stats.norm.pdf(stats.norm.ppf(mus)), rtol=1e-14)


def test_families_project_initialize_and_deviance():
    from sklearn.metrics import mean_gamma_deviance, mean_poisson_deviance, mean_tweedie_deviance
    rng = np.random.default_rng(1)
    y = rng.poisson(2.0, 500).astype(float)
    mu = rng.uniform(0.5, 3.0, 500)
    w = np.ones(500)
    assert np.isclose(go.deviance(go.POISSON, y, mu, w).mean(), mean_poisson_deviance(y, mu), rtol=1e-12)
    yg = rng.gamma(2.0, 1.0, 500)
    assert np.isclose(go.deviance(go.GAMMA, yg, mu, w).mean(), mean_gamma_deviance(yg, mu), rtol=1e-12)
    for p in (1.5, 3.0):
        yy = y if p < 2 else yg
        assert np.isclose(go.deviance(go.TWEEDIE, yy, mu, w, p).mean(), mean_tweedie_deviance(yy, mu, power=p),
                          rtol=1e-10)
    assert np.isclose(go.deviance(go.GAUSSIAN, yg, mu, w).sum(), ((yg - mu) ** 2).sum())
    assert go.project(go.BINOMIAL, np.array([0.0, 1.0]))[0] == 1e-16 and go.project(go.BINOMIAL, np.array([1.0]))[0] < 1
    assert go.project(go.POISSON, np.array([np.inf]))[0] == np.finfo(float).max
    assert list(go.initialize(go.POISSON, np.array([0.0, 2.0]), None)) == [0.1, 2.0]
    assert go.initialize(go.BINOMIAL, np.array([1.0]), np.array([3.0]))[0] == 3.5 / 4.0


# ----------------------------------------------------------------------------------- fits
def _data(family, n=3000, D=4, seed=2):
    x, rng = _x(n, D, seed)
    beta = rng.normal(0, 0.4, D)
    eta = x @ beta + 0.3
    if family == go.POISSON:
        y = rng.poisson(np.exp(eta)).astype(float)
    elif family == go.GAMMA:
        y = rng.gamma(2.0, np.exp(eta) / 2.0)
    elif family == go.BINOMIAL:
        y = (rng.uniform(size=n) < 1 / (1 + np.exp(-eta))).astype(float)
    elif family == go.TWEEDIE:
        y = rng.poisson(np.exp(eta)) * rng.gamma(2.0, 0.5, n)
    else:
        y = eta + rng.normal(0, 0.5, n)
    return x, y


@pytest.mark.parametrize("case", ["gaussian", "poisson", "gamma", "tweedie", "binomial"])
def test_irls_equals_sklearn(case):
    sklm = pytest.importorskip("sklearn.linear_model")
    fam = {"gaussian": go.GAUSSIAN, "poisson": go.POISSON, "gamma": go.GAMMA, "tweedie": go.TWEEDIE,
           "binomial": go.BINOMIAL}[case]
    x, y = _data(fam)
    spec = {"gaussian": (go.GAUSSIAN, go.IDENTITY), "poisson": (go.POISSON, go.LOG), "gamma": (go.GAMMA, go.LOG),
            "tweedie": (go.TWEEDIE, go.LOG, 1.5, 0.0), "binomial": (go.BINOMIAL, go.LOGIT)}[case]
    coef, b, _, it = go.irls(x, y, spec, tol=1e-12, max_iter=100)
    ref = {"gaussian": lambda: sklm.LinearRegression(),
           "poisson": lambda: sklm.PoissonRegressor(alpha=0, tol=1e-12, max_iter=1000),
           "gamma": lambda: sklm.GammaRegressor(alpha=0, tol=1e-12, max_iter=1000),
           "tweedie": lambda: sklm.TweedieRegressor(power=1.5, link="log", alpha=0, tol=1e-12, max_iter=1000),
           "binomial": lambda: sklm.LogisticRegression(C=np.inf, tol=1e-12, max_iter=1000)}[case]().fit(x, y)
    assert np.allclose(coef, ref.coef_.reshape(-1), rtol=1e-6, atol=1e-7) and math.isclose(
        b, float(np.ravel(ref.intercept_)[0]), rel_tol=1e-6, abs_tol=1e-7), (coef, ref.coef_)
    assert (it == 1) == (case == "gaussian")


@pytest.mark.parametrize("spec", [(go.BINOMIAL, go.PROBIT), (go.BINOMIAL, go.CLOGLOG), (go.POISSON, go.SQRT),
                                  (go.GAMMA, go.INVERSE), (go.POISSON, go.IDENTITY), (go.GAUSSIAN, go.LOG)])
def test_other_links_solve_the_score_equations(spec):
    f, l = spec
    x, y = _data({go.BINOMIAL: go.BINOMIAL, go.POISSON: go.POISSON, go.GAMMA: go.GAMMA, go.GAUSSIAN: go.GAMMA}[f],
                 n=2000, D=3)
    if l in (go.INVERSE, go.IDENTITY, go.SQRT):                      # keep mu positive along the path
        x = np.abs(x) * 0.2
        y = y + (1.0 if f != go.BINOMIAL else 0.0)
    w = np.random.default_rng(5).integers(1, 4, x.shape[0]).astype(float)
    coef, b, _, _ = go.irls(x, y, spec, w=w, tol=1e-13, max_iter=200)
    xa = np.hstack([x, np.ones((x.shape[0], 1))])

    def score(v):
        mu = go.project(f, go.unlink(l, xa @ v))
        return xa.T @ (w * (y - mu) / (go.variance(f, mu) * go.deriv(l, mu)))

    v = optimize.root(score, np.concatenate([coef, [b]]) * 0.9 + 0.01, tol=1e-14).x
    assert np.allclose(np.concatenate([coef, [b]]), v, rtol=1e-7, atol=1e-9)
    assert np.max(np.abs(score(np.concatenate([coef, [b]])))) < 1e-6 * x.shape[0]


def test_weights_equal_replication_and_offsets_shift_identity_labels():
    x, y = _data(go.POISSON, n=800, D=3)
    w = np.random.default_rng(3).integers(0, 4, 800).astype(float)
    rep = np.repeat(np.arange(800), w.astype(int))
    for spec in ((go.POISSON, go.LOG), (go.GAMMA, go.LOG), (go.GAUSSIAN, go.IDENTITY)):
        yy = y + 0.5
        a = go.irls(x, yy, spec, w=w, tol=1e-13, max_iter=100)
        r = go.irls(x[rep], yy[rep], spec, tol=1e-13, max_iter=100)
        assert np.allclose(a[0], r[0], rtol=1e-9) and math.isclose(a[1], r[1], rel_tol=1e-9)
    off = np.random.default_rng(4).normal(0, 1, 800)
    for spec in ((go.GAUSSIAN, go.IDENTITY), (go.POISSON, go.IDENTITY)):
        yy = y + 3.0 + off if spec[0] == go.GAUSSIAN else y + 3.0
        o = off if spec[0] == go.GAUSSIAN else 0.1 * np.abs(off)
        a = go.irls(np.abs(x), yy, spec, off=o, tol=1e-13, max_iter=100)
        if spec[0] == go.GAUSSIAN:
            r = go.irls(np.abs(x), yy - o, spec, tol=1e-13)
            assert np.allclose(a[0], r[0], rtol=1e-10) and math.isclose(a[1], r[1], rel_tol=1e-10)
        else:                                          # identity link: mu = x.beta + b + off, so the score equations hold
            mu = np.abs(x) @ a[0] + a[1] + o
            xa = np.hstack([np.abs(x), np.ones((800, 1))])
            assert np.max(np.abs(xa.T @ ((yy - mu) / mu))) < 1e-6


# ----------------------------------------------------------------------------------- summary
def test_aic_deviance_standard_errors_and_p_values():
    for fam, spec in ((go.POISSON, (go.POISSON, go.LOG)), (go.GAMMA, (go.GAMMA, go.LOG)),
                      (go.BINOMIAL, (go.BINOMIAL, go.LOGIT)), (go.GAUSSIAN, (go.GAUSSIAN, go.IDENTITY))):
        x, y = _data(fam, n=1500, D=3)
        coef, b, diag, _ = go.irls(x, y, spec, tol=1e-12, max_iter=100)
        s = go.summary(x, y, coef, b, spec)
        mu = go.unlink(spec[1], _pred(x, coef, b))
        n, rank = x.shape[0], 4
        if fam == go.POISSON:
            ll = stats.poisson.logpmf(y, mu).sum()
        elif fam == go.BINOMIAL:
            ll = stats.binom.logpmf(y, 1, mu).sum()
        elif fam == go.GAMMA:
            d = s["deviance"] / n
            ll = stats.gamma.logpdf(y, 1 / d, scale=mu * d).sum() - 1.0
        else:
            ll = stats.norm.logpdf(y, mu, math.sqrt(s["deviance"] / n)).sum() - 1.0
        assert math.isclose(s["aic"], -2 * ll + 2 * rank, rel_tol=1e-9), fam
        assert math.isclose(s["deviance"], go.deviance(fam, y, mu, np.ones(n)).sum(), rel_tol=1e-9)
        ybar = y.mean()
        assert math.isclose(s["null_deviance"], go.deviance(fam, y, np.full(n, ybar), np.ones(n)).sum(), rel_tol=1e-12)
        W = 1.0 / (go.deriv(spec[1], mu) ** 2 * go.variance(fam, mu))
        xa = np.hstack([x, np.ones((n, 1))])
        cov = np.linalg.inv((xa.T * W) @ xa) * s["dispersion"]
        se = np.sqrt(diag * s["dispersion"])
        assert np.allclose(se, np.sqrt(np.diag(cov)), rtol=1e-6)
        if fam in (go.POISSON, go.BINOMIAL):
            assert s["dispersion"] == 1.0
        else:
            r = (y - mu) / np.sqrt(go.variance(fam, mu))
            assert math.isclose(s["dispersion"], (r * r).sum() / (n - rank), rel_tol=1e-9)
        from b200flow.selection import f_cdf
        t = np.concatenate([coef, [b]]) / se
        for v in t:
            want = 2 * stats.norm.sf(abs(v)) if fam in (go.POISSON, go.BINOMIAL) else 2 * stats.t.sf(abs(v), n - rank)
            got = 2.0 * (1.0 - 0.5 * math.erfc(-abs(v) / math.sqrt(2.0))) if fam in (go.POISSON, go.BINOMIAL) else \
                1.0 - f_cdf(v * v, 1.0, float(n - rank))
            assert math.isclose(got, want, rel_tol=1e-6, abs_tol=1e-14)


def test_regularised_fit_satisfies_its_penalised_normal_equations():
    x, y = _data(go.POISSON, n=1500, D=4)
    reg = 0.3
    coef, b, _, _ = go.irls(x, y, (go.POISSON, go.LOG), reg_param=reg, tol=1e-13, max_iter=200)
    _, zw = go.rows(x, y, None, None, coef, b, (go.POISSON, go.LOG), 1)
    z, w = zw[:, 0], zw[:, 1]
    sw = w.sum()
    xm, zm = w @ x / sw, w @ z / sw
    xc, zc = x - xm, z - zm
    sd = np.sqrt(w @ (xc * xc) / sw)
    zsd = math.sqrt(w @ (zc * zc) / sw)
    grad = (xc.T * w) @ (xc @ coef - zc) / sw + reg / zsd * sd * sd * coef
    assert np.max(np.abs(grad)) < 1e-8 and abs(zm - xm @ coef - b) < 1e-10
    plain = go.irls(x, y, (go.POISSON, go.LOG), tol=1e-13, max_iter=200)[0]
    assert np.linalg.norm(coef) < np.linalg.norm(plain)
