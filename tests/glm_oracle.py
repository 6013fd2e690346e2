"""numpy restatement of GeneralizedLinearRegression (b200flow/glm.py, csrc/glm_family.cuh, csrc/glm.cu): the families
and links, the per-row pass with the kernel's margin order, IRLS on an independent weighted least-squares solve, and the
summary.  Families / links use b200flow.glm's codes."""
import math

import numpy as np
from scipy import special

GAUSSIAN, BINOMIAL, POISSON, GAMMA, TWEEDIE = range(5)
IDENTITY, LOG, INVERSE, LOGIT, PROBIT, CLOGLOG, SQRT, POWER = range(8)
EPS, DELTA = 1e-16, 0.1
INV_SQRT_2PI = 0.3989422804014327


def link(l, mu, lp=0.0):
    with np.errstate(all="ignore"):
        return {IDENTITY: lambda: mu, LOG: lambda: np.log(mu), INVERSE: lambda: 1.0 / mu,
                LOGIT: lambda: np.log(mu / (1.0 - mu)), PROBIT: lambda: special.ndtri(mu),
                CLOGLOG: lambda: np.log(-np.log1p(-mu)), SQRT: lambda: np.sqrt(mu),
                POWER: lambda: np.log(mu) if lp == 0.0 else np.power(mu, lp)}[l]()


def unlink(l, eta, lp=0.0):
    with np.errstate(all="ignore"):
        return {IDENTITY: lambda: eta, LOG: lambda: np.exp(eta), INVERSE: lambda: 1.0 / eta,
                LOGIT: lambda: 1.0 / (1.0 + np.exp(-eta)), PROBIT: lambda: special.ndtr(eta),
                CLOGLOG: lambda: 1.0 - np.exp(-np.exp(eta)), SQRT: lambda: eta * eta,
                POWER: lambda: np.exp(eta) if lp == 0.0 else np.power(eta, 1.0 / lp)}[l]()


def deriv(l, mu, lp=0.0):
    with np.errstate(all="ignore"):
        if l == PROBIT:
            q = special.ndtri(mu)
            return 1.0 / (np.exp(-0.5 * (q * q)) * INV_SQRT_2PI)
        return {IDENTITY: lambda: np.ones_like(mu), LOG: lambda: 1.0 / mu, INVERSE: lambda: -1.0 / (mu * mu),
                LOGIT: lambda: 1.0 / (mu * (1.0 - mu)), CLOGLOG: lambda: 1.0 / ((mu - 1.0) * np.log1p(-mu)),
                SQRT: lambda: 1.0 / (2.0 * np.sqrt(mu)),
                POWER: lambda: 1.0 / mu if lp == 0.0 else lp * np.power(mu, lp - 1.0)}[l]()


def variance(f, mu, vp=0.0):
    return {GAUSSIAN: lambda: np.ones_like(mu), BINOMIAL: lambda: mu * (1.0 - mu), POISSON: lambda: mu,
            GAMMA: lambda: mu * mu, TWEEDIE: lambda: np.power(mu, vp)}[f]()


def project(f, mu):
    mu = np.asarray(mu, np.float64)
    big = np.finfo(np.float64).max
    if f == GAUSSIAN:
        return np.where(np.isinf(mu), np.where(mu > 0, big, -big), mu)
    if f == BINOMIAL:
        return np.where(mu < EPS, EPS, np.where(mu > 1.0 - EPS, 1.0 - EPS, mu))
    return np.where(mu < EPS, EPS, np.where(np.isinf(mu), big, mu))


def initialize(f, y, w):
    if f == BINOMIAL:
        return (w * y + 0.5) / (w + 1.0)
    if f in (POISSON, TWEEDIE):
        return np.where(y == 0.0, DELTA, y)
    return y


def _ylogy(y, mu):
    with np.errstate(all="ignore"):
        return np.where(y == 0.0, 0.0, y * np.log(y / mu))


def deviance(f, y, mu, w, vp=0.0):
    with np.errstate(all="ignore"):
        if f == GAUSSIAN:
            return w * (y - mu) * (y - mu)
        if f == BINOMIAL:
            return 2.0 * w * (_ylogy(y, mu) + _ylogy(1.0 - y, 1.0 - mu))
        if f == POISSON:
            return 2.0 * w * (_ylogy(y, mu) - (y - mu))
        if f == GAMMA:
            return -2.0 * w * (np.log(y / mu) - (y - mu) / mu)
        y1 = np.where(y < DELTA, DELTA, y) if 1.0 <= vp < 2.0 else y
        return 2.0 * w * (y * (np.power(y1, 1.0 - vp) - np.power(mu, 1.0 - vp)) / (1.0 - vp) -
                          (np.power(y, 2.0 - vp) - np.power(mu, 2.0 - vp)) / (2.0 - vp))


def aic_term(f, y, mu, w):
    with np.errstate(all="ignore"):
        if f == GAUSSIAN:
            return np.log(w)
        if f == BINOMIAL:
            n, k = np.floor(w + 0.5), np.floor(y * w + 0.5)
            t = special.gammaln(n + 1) - special.gammaln(k + 1) - special.gammaln(n - k + 1) + k * np.log(mu) + \
                (n - k) * np.log(1.0 - mu)
            return np.where(n == 0.0, 0.0, t)
        if f == POISSON:
            k = np.trunc(y)
            return w * (-mu + k * np.log(mu) - special.gammaln(k + 1.0))
        return np.zeros_like(y)


def margin(x, coef):
    """x . coef in the kernel's order: eight strided lane sums, combined ((p0 + p4) + (p2 + p6)) + ((p1 + p5) + (p3 + p7))"""
    n, D = x.shape
    p = np.zeros((8, n))
    for j in range(D):
        p[j % 8] = p[j % 8] + x[:, j] * coef[j]
    return ((p[0] + p[4]) + (p[2] + p[6])) + ((p[1] + p[5]) + (p[3] + p[7]))


def spec_args(spec):
    """(family, link, variance power, link power) of a (family, link[, vp[, lp]]) tuple"""
    f, l = spec[0], spec[1]
    return f, l, (spec[2] if len(spec) > 2 else 0.0), (spec[3] if len(spec) > 3 else 0.0)


def rows(x, y, w, off, coef, b, spec, mode, mu_const=None):
    """(totals, per-row outputs) of b200flow_glm_rows (mode 0 INIT, 1 REWEIGHT, 2 SUMMARY, 3 PREDICT); w / off None: 1 / 0"""
    f, l, vp, lp = spec_args(spec)
    x = np.asarray(x, np.float64)
    n, D = x.shape
    w = np.ones(n) if w is None else np.asarray(w, np.float64)
    off = np.zeros(n) if off is None else np.asarray(off, np.float64)
    with np.errstate(all="ignore"):
        if mode == 0:
            z = link(l, initialize(f, y, w), lp) - off
            return np.concatenate([[w.sum()], w @ x, [(w * z).sum()]]), np.stack([z, w], 1)
        if coef is None:
            mu = np.full(n, mu_const)
            eta = link(l, mu, lp)
        else:
            eta = (margin(x, coef) + b) + off
            mu = project(f, unlink(l, eta, lp))
        if mode == 3:
            return None, np.stack([mu, eta], 1)
        if mode == 1:
            d = deriv(l, mu, lp)
            z = (eta - off) + (y - mu) * d
            ww = w / (d * d * variance(f, mu, vp))
            return np.concatenate([[ww.sum()], ww @ x, [(ww * z).sum()]]), np.stack([z, ww], 1)
        r = y - mu
        dev = deviance(f, y, mu, w, vp)
        pr = r * np.sqrt(w) / np.sqrt(variance(f, mu, vp))
        res = np.stack([np.sign(r) * np.sqrt(np.maximum(dev, 0.0)), pr, r * deriv(l, mu, lp), r], 1)
        g = f == GAMMA
        tot = np.array([w.sum(), (w * y).sum(), dev.sum(), (pr * pr).sum(), aic_term(f, y, mu, w).sum(),
                        (w * np.log(y)).sum() if g else 0.0, (w * (y / mu)).sum() if g else 0.0,
                        (w * np.log(mu)).sum() if g else 0.0])
        return tot, res


def wls(x, z, w, fit_intercept=True, reg_param=0.0):
    """WeightedLeastSquares with standardized features and label and an L2 penalty, solved directly: (coef, intercept,
    diag of the inverse of the intercept-augmented weighted Gram matrix / sum w, intercept last)"""
    sw = w.sum()
    xm, zm = (w @ x) / sw, (w @ z) / sw
    xc, zc = x - xm, z - zm
    sd = np.sqrt((w @ (xc * xc)) / sw)
    zsd = math.sqrt((w @ (zc * zc)) / sw)
    zsd = zsd if zsd > 0 else abs(zm)
    lam = reg_param / zsd * sd * sd if reg_param else np.zeros(x.shape[1])
    if fit_intercept:
        A = (xc.T * w) @ xc / sw + np.diag(lam)
        coef = np.linalg.solve(A, (xc.T * w) @ zc / sw)
        b = zm - xm @ coef
        xa = np.hstack([x, np.ones((x.shape[0], 1))])
    else:
        A = (x.T * w) @ x / sw + np.diag(lam)
        coef = np.linalg.solve(A, (x.T * w) @ z / sw)
        b = 0.0
        xa = x
    diag = np.diag(np.linalg.inv((xa.T * w) @ xa))
    return coef, b, diag


def irls(x, y, spec, w=None, off=None, fit_intercept=True, reg_param=0.0, max_iter=25, tol=1e-6):
    """(coef, intercept, diag, iterations) of glm.py's IRLS on the restated rows pass and wls"""
    f, l = spec[0], spec[1]
    x = np.asarray(x, np.float64)
    _, zw = rows(x, y, w, off, None, 0.0, spec, 0)
    coef, b, diag = wls(x, zw[:, 0], zw[:, 1], fit_intercept, reg_param)
    if f == GAUSSIAN and l == IDENTITY:
        return coef, b, diag, 1
    it = 0
    while it < max_iter:
        _, zw = rows(x, y, w, off, coef, b, spec, 1)
        c2, b2, diag = wls(x, zw[:, 0], zw[:, 1], fit_intercept, reg_param)
        step = max(np.max(np.abs(coef - c2)), abs(b - b2))
        coef, b, it = c2, b2, it + 1
        if step < tol:
            break
    return coef, b, diag, it


def summary(x, y, coef, b, spec, w=None, off=None, fit_intercept=True, max_iter=25, tol=1e-6):
    """dict of deviance, null_deviance, dispersion and aic (None for tweedie), as glm.summarize"""
    f, l, vp, lp = spec_args(spec)
    x = np.asarray(x, np.float64)
    n, D = x.shape
    t, _ = rows(x, y, w, off, coef, b, spec, 2)
    if fit_intercept and off is None:
        null = rows(x, y, w, off, None, 0.0, spec, 2, mu_const=t[1] / t[0])[0][2]
    else:
        b0 = 0.0
        if fit_intercept:
            tt, _ = rows(x, y, w, off, None, 0.0, spec, 0)
            b0 = tt[D + 1] / tt[0]
            if not (f == GAUSSIAN and l == IDENTITY):
                for _ in range(max_iter):
                    tt, _ = rows(x, y, w, off, np.zeros(D), b0, spec, 1)
                    b1 = tt[D + 1] / tt[0]
                    step, b0 = abs(b0 - b1), b1
                    if step < tol:
                        break
        null = rows(x, y, w, off, np.zeros(D), b0, spec, 2)[0][2]
    rank = D + (1 if fit_intercept else 0)
    dof = n - rank
    disp = 1.0 if f in (BINOMIAL, POISSON) else t[3] / dof
    dev = t[2]
    if f == GAUSSIAN:
        aic = n * (math.log(dev / n * 2.0 * math.pi) + 1.0) + 2.0 - t[4]
    elif f in (BINOMIAL, POISSON):
        aic = -2.0 * t[4]
    elif f == GAMMA:
        d = dev / t[0]
        k = 1.0 / d
        aic = -2.0 * ((k - 1.0) * t[5] - t[6] / d - (math.lgamma(k) + k * math.log(d)) * t[0] - k * t[7]) + 2.0
    else:
        aic = None
    return dict(deviance=dev, null_deviance=null, dispersion=disp, aic=None if aic is None else aic + 2.0 * rank,
                rank=rank, dof=dof)
