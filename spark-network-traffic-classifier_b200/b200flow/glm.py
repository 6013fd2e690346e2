"""GeneralizedLinearRegression on the device (DESIGN.md §5o): IRLS as a loop of one per-row pass (csrc/glm.cu) and one
weighted centred Gram matrix (csrc/pca.cu) per iteration, each summed in the chunk order of dist.Shards, with
linreg.solve_normal's WeightedLeastSquares on rank 0; so every fit and summary is the same bits for any world size and
shard layout.

Spark [recalled; Spark 3 `ml/regression/GeneralizedLinearRegression.scala`, `ml/optim/IterativelyReweightedLeastSquares.scala`,
`ml/optim/WeightedLeastSquares.scala`]:

    Params: family "gaussian" (binomial, poisson, gamma, tweedie), link (the family's canonical link by default: identity,
    logit, log, inverse), variancePower 0.0 (tweedie only; 0 or >= 1), linkPower (tweedie only; default 1 - variancePower;
    0 log, 1 identity, -1 inverse, 0.5 sqrt, otherwise mu^p), fitIntercept true, maxIter 25, tol 1e-6, regParam 0.0 (L2),
    solver "irls" (the only one), aggregationDepth 2 (validated; no effect here), weightCol, offsetCol, linkPredictionCol.
    Tweedie with variancePower 0, 1 or 2 is the gaussian, poisson or gamma family.  Family / link pairs other than
    gaussian: identity, log, inverse; binomial: logit, probit, cloglog; poisson: log, identity, sqrt; gamma: inverse,
    identity, log are refused.
    Labels: binomial 0 <= y <= 1; poisson and tweedie with 1 <= p < 2 y >= 0; gamma and tweedie with p > 2 y > 0;
    gaussian with the log link y > 0, with the inverse link y != 0.  Weights finite and >= 0, not all 0.
    Families: V(mu) = 1, mu (1 - mu), mu, mu^2, mu^p.  Deviance terms: w (y - mu)^2; 2w (ylogy(y, mu) + ylogy(1 - y, 1 - mu));
    2w (ylogy(y, mu) - (y - mu)); -2w (log(y / mu) - (y - mu) / mu); tweedie 2w (y (y1^(1-p) - mu^(1-p)) / (1 - p) -
    (y^(2-p) - mu^(2-p)) / (2 - p)), y1 = max(y, 0.1) for 1 <= p < 2 (else y), with ylogy(y, mu) = 0 at y = 0 else
    y log(y / mu).  initialize: binomial (w y + 0.5) / (w + 1), poisson and tweedie y (0.1 at y = 0), others y.
    project: binomial into [eps, 1 - eps], poisson / gamma / tweedie at least eps (+inf -> the largest double), gaussian
    +-inf -> +-the largest double; eps = 1e-16.
    gaussian + identity: one WeightedLeastSquares fit (standardized features and label, elasticNet 0, regParam) on
    y - offset with the prior weights; numIterations 1.
    Otherwise IRLS: the initial model is that fit on link(initialize(y, w)) - offset; then, from (beta, b),
    eta = x . beta + b + offset, mu = project(linkInv(eta)), z = eta - offset + (y - mu) g'(mu),
    w' = w / (g'(mu)^2 V(mu)) and the WeightedLeastSquares fit on (z, w'); it stops once max |delta beta_j| and |delta b|
    are both below tol, or after maxIter iterations.  diagInvAtWA is the last fit's.
    Summary: numInstances (rows), rank = D + intercept, degreesOfFreedom = residualDegreeOfFreedom = numInstances - rank,
    residualDegreeOfFreedomNull = numInstances - intercept; deviance; nullDeviance at mu = the weighted mean of y with an
    intercept and no offset, at linkInv(offset) without an intercept, and at linkInv(b0 + offset) of an intercept-only IRLS
    fit with both; dispersion 1 for binomial and poisson, else sum w (y - mu)^2 / V(mu) / residualDegreeOfFreedom;
    aic = family term + 2 rank: gaussian n (log(deviance / n 2 pi) + 1) + 2 - sum log w; binomial -2 sum log
    Binomial(round(w), mu).pmf(round(y w)) (0 where round(w) = 0); poisson -2 sum w log Poisson(mu).pmf(trunc(y)); gamma
    -2 sum w log Gamma(shape 1 / disp, scale mu disp).pdf(y) + 2 with disp = deviance / sum w; tweedie has none.
    Residuals: response y - mu, working (y - mu) g'(mu), pearson (y - mu) sqrt(w) / sqrt(V(mu)), deviance
    sign(y - mu) sqrt(deviance term).  Standard errors sqrt(diagInvAtWA dispersion) (intercept last), t = estimate / se,
    p = 2 (1 - Phi(|t|)) for binomial and poisson, else the two-sided Student t with residualDegreeOfFreedom.

Deviations: D <= 255 (Spark: 4096).  The Gram matrix is two-pass weighted-centred where Spark sums uncentred moments.
log / exp / pow / lgamma / normcdf / normcdfinv are CUDA's, within a few ulp of the JVM's and Breeze's.  The D x D solves
run on rank 0 and are broadcast (as linreg.py).  Non-finite features, labels, weights or offsets, and a non-finite
IRLS iterate, raise ValueError.  A deviance term that rounds below zero gives a deviance residual of 0, not NaN.
"""
import math

import numpy as np
import torch

from . import _lib
from . import dist as bdist
from . import linreg, pca
from ._lib import call, ptr

MAX_D = 255
FAMILIES = ("gaussian", "binomial", "poisson", "gamma", "tweedie")
GAUSSIAN, BINOMIAL, POISSON, GAMMA, TWEEDIE = range(5)
LINKS = ("identity", "log", "inverse", "logit", "probit", "cloglog", "sqrt")
IDENTITY, LOG, INVERSE, LOGIT, PROBIT, CLOGLOG, SQRT, POWER = range(8)
INIT, REWEIGHT, SUMMARY, PREDICT = range(4)
SUPPORTED = {"gaussian": ("identity", "log", "inverse"), "binomial": ("logit", "probit", "cloglog"),
             "poisson": ("log", "identity", "sqrt"), "gamma": ("inverse", "identity", "log")}
CANONICAL = {"gaussian": "identity", "binomial": "logit", "poisson": "log", "gamma": "inverse"}
SUMMARY_WIDTH = 8
RESIDUALS = ("deviance", "pearson", "working", "response")


class GLMParams:
    __slots__ = ("family", "link", "variance_power", "link_power", "fit_intercept", "max_iter", "tol", "reg_param",
                 "solver")

    def __init__(self, family="gaussian", link=None, variance_power=0.0, link_power=None, fit_intercept=True, max_iter=25,
                 tol=1e-6, reg_param=0.0, solver="irls"):
        self.family, self.link = str(family).lower(), None if link is None else str(link).lower()
        self.variance_power = float(variance_power)
        self.link_power = None if link_power is None else float(link_power)
        self.fit_intercept, self.max_iter, self.tol = bool(fit_intercept), int(max_iter), float(tol)
        self.reg_param, self.solver = float(reg_param), str(solver).lower()


class Spec:
    """the resolved family and link: codes, tweedie's variance power and the power link's exponent"""
    __slots__ = ("family", "link", "variance_power", "link_power")

    def __init__(self, family, link, variance_power=0.0, link_power=0.0):
        self.family, self.link, self.variance_power, self.link_power = family, link, float(variance_power), float(link_power)

    def __eq__(self, o):
        return all(getattr(self, k) == getattr(o, k) for k in self.__slots__)


def check_params(p):
    """Spark's validators and refusals; raises ValueError"""
    if p.family not in FAMILIES:
        raise ValueError("family must be one of %s, got %r" % (list(FAMILIES), p.family))
    if p.link is not None and p.link not in LINKS:
        raise ValueError("link must be one of %s, got %r" % (list(LINKS), p.link))
    if not (p.variance_power == 0.0 or p.variance_power >= 1.0):
        raise ValueError("parameter variancePower given invalid value %r (must be 0 or >= 1)." % p.variance_power)
    if p.max_iter < 0:
        raise ValueError("maxIter must be >= 0, got %r" % p.max_iter)
    if not p.tol >= 0.0 or not p.reg_param >= 0.0:
        raise ValueError("tol and regParam must be >= 0, got %r and %r" % (p.tol, p.reg_param))
    if p.solver != "irls":
        raise ValueError("solver must be 'irls', got %r" % p.solver)
    if p.family != "tweedie" and p.link is not None and p.link not in SUPPORTED[p.family]:
        raise ValueError("Generalized Linear Regression with %s family does not support %s link function."
                         % (p.family, p.link))


def resolve(p):
    """Spec of valid params: tweedie with variancePower 0 / 1 / 2 is gaussian / poisson / gamma, and its linkPower 0 / 1 /
    -1 / 0.5 the log / identity / inverse / sqrt link"""
    if p.family == "tweedie":
        vp = p.variance_power
        fam = {0.0: GAUSSIAN, 1.0: POISSON, 2.0: GAMMA}.get(vp, TWEEDIE)
        lp = 1.0 - vp if p.link_power is None else p.link_power
        link = {0.0: LOG, 1.0: IDENTITY, -1.0: INVERSE, 0.5: SQRT}.get(lp, POWER)
        return Spec(fam, link, vp if fam == TWEEDIE else 0.0, lp if link == POWER else 0.0)
    link = p.link if p.link is not None else CANONICAL[p.family]
    return Spec(FAMILIES.index(p.family), LINKS.index(link))


class GLMFit:
    """coef f64 [D] (host), intercept, diag_inv_atwa ([D (+1)] host, or None after the quasi-Newton fallback), the
    number of IRLS iterations and the resolved Spec."""
    __slots__ = ("coef", "intercept", "diag_inv_atwa", "iterations", "spec")

    def __init__(self, coef, intercept, diag, iterations, spec):
        self.coef, self.intercept, self.diag_inv_atwa = coef, float(intercept), diag
        self.iterations, self.spec = int(iterations), spec


def _check_x(x):
    if not (torch.is_tensor(x) and x.is_cuda and x.dim() == 2 and x.dtype in (torch.float32, torch.float64)):
        raise _lib.B200FlowError("GeneralizedLinearRegression needs a CUDA float32 or float64 [n, D] matrix")
    if not 1 <= x.shape[1] <= MAX_D:
        raise _lib.UnsupportedParamError("GeneralizedLinearRegression supports 1 to %d features, got %d"
                                         % (MAX_D, x.shape[1]))
    return x.contiguous()


def _column(v, n, dev):
    return None if v is None else v.to(device=dev, dtype=torch.float64).reshape(-1).contiguous()


def _label_violation(spec, y):
    """the rows whose label is outside the family's domain, and its message"""
    f, l, p = spec.family, spec.link, spec.variance_power
    if f == BINOMIAL:
        return (y < 0) | (y > 1), "The response variable of Binomial family should be in range [0, 1]"
    if f == POISSON or (f == TWEEDIE and p < 2.0):
        return y < 0, "The response variable of %s family should be non-negative" % ("Poisson" if f == POISSON else
                                                                                      "Tweedie(%r)" % p)
    if f == GAMMA or f == TWEEDIE:
        return y <= 0, "The response variable of %s family should be positive" % ("Gamma" if f == GAMMA else
                                                                                  "Tweedie(%r)" % p)
    if l == LOG:
        return y <= 0, "The response variable of Gaussian family with log link should be positive"
    if l == INVERSE:
        return y == 0, "The response variable of Gaussian family with inverse link should be non-zero"
    return torch.zeros_like(y, dtype=torch.bool), ""


def prepare(x, y, spec, weight=None, offset=None, row_offset=None, group=None):
    """(x, y, weight or None, offset or None, Shards) after the checks, on every rank with one all-reduce"""
    x = _check_x(x)
    n = x.shape[0]
    grp = group if group is not None else bdist.group()
    dev = x.device
    if row_offset is None:
        row_offset, _ = bdist.global_offset(n, dev, grp)
    sh = bdist.Shards(n, row_offset, grp, dev)
    y, w, off = _column(y, n, dev), _column(weight, n, dev), _column(offset, n, dev)
    lens = any(v is not None and v.shape[0] != n for v in (y, w, off))
    out, msg = _label_violation(spec, y) if not lens else (None, "")
    false = torch.zeros((), dtype=torch.bool, device=dev)
    bad = torch.stack([torch.tensor(lens, device=dev),
                       (~torch.isfinite(x)).any(),
                       (~torch.isfinite(y)).any() if not lens else false,
                       out.any() if not lens else false,
                       ((~torch.isfinite(w)) | (w < 0)).any() if w is not None and not lens else false,
                       (~torch.isfinite(off)).any() if off is not None and not lens else false]).to(torch.int64)
    if grp is not None:
        bdist.all_reduce_(bad, grp)
    b = [int(v) for v in bad.cpu()]
    if b[0]:
        raise ValueError("GeneralizedLinearRegression needs one label, weight and offset per row")
    if sh.total == 0:
        raise ValueError("GeneralizedLinearRegression needs at least one row")
    if b[1] or b[2]:
        raise ValueError("GeneralizedLinearRegression needs finite features and labels")
    if b[3]:
        raise ValueError(msg)
    if b[4]:
        raise ValueError("Weights must be finite and non-negative")
    if b[5]:
        raise ValueError("Offsets must be finite")
    return x, y, w, off, sh


# ----------------------------------------------------------------------------------- the per-row pass
def rows(x, y, w, off, coef, intercept, mu_const, spec, mode, row_offset, rows_out, partials):
    """b200flow_glm_rows on the rows x [n, D] (f32/f64); y, w, off [n], coef [D] device f64 or None."""
    n, D = x.shape
    call("b200flow_glm_rows", ptr(x), _lib.dtype_code(x), n, x.stride(0), D, ptr(y), ptr(w), ptr(off), ptr(coef),
         float(intercept), float(mu_const), spec.family, spec.link, spec.variance_power, spec.link_power, int(mode),
         int(row_offset), ptr(rows_out), ptr(partials))


def rows_total(x, y, w, off, coef, intercept, spec, mode, sh, mu_const=0.0, per_row=True):
    """(totals [width] f64 device, per-row outputs [n, 2] (INIT / REWEIGHT) or [n, 4] (SUMMARY residuals) or None):
    the chunk sums over every rank's rows in chunk order, the same bits on every rank.  This rank's rows are one launch;
    when later ranks' leading rows complete its trailing chunk, that chunk is launched again with them (dist.chunk_tail)
    and a shard's leading rows, which belong to an earlier rank's chunk, leave their partial out."""
    n, D = x.shape
    width = D + 2 if mode != SUMMARY else SUMMARY_WIDTH
    dev = x.device
    out = torch.empty((n, 2 if mode != SUMMARY else 4), dtype=torch.float64, device=dev) if per_row or mode != SUMMARY \
        else None
    lead, o = sh.lead[sh.rank], sh.offs[sh.rank]
    t0, tail_x, _ = bdist.chunk_tail(x, None, sh)
    tail_a = None
    if sh.grp is not None and any(sh.lead):          # the same collective on every rank
        ones = torch.ones(n, dtype=torch.float64, device=dev)
        aux = torch.stack([y, w if w is not None else ones, off if off is not None else ones * 0.0], 1)
        tail_a = bdist.chunk_tail(aux, None, sh)[1]
    extra = tail_x.shape[0] > n - t0
    main = t0 if extra else n
    parts, count = [], 0
    if main > 0:
        nc = (o + main - 1) // bdist.CHUNK - o // bdist.CHUNK + 1
        p = torch.empty((nc, width), dtype=torch.float64, device=dev)
        cut = lambda t: None if t is None else t[:main]          # noqa: E731
        rows(x[:main], y[:main], cut(w), cut(off), coef, intercept, mu_const, spec, mode, o, cut(out), p)
        parts.append(p[1 if lead > 0 else 0:])
    if extra:
        tl = tail_x.shape[0]
        tout = torch.empty((tl, out.shape[1]), dtype=torch.float64, device=dev) if out is not None else None
        p = torch.empty((1, width), dtype=torch.float64, device=dev)
        a = [tail_a[:, k].contiguous() for k in range(3)]
        rows(tail_x, a[0], a[1], a[2], coef, intercept, mu_const, spec, mode, o + t0, tout, p)
        if out is not None:
            out[t0:] = tout[:n - t0]
        parts.append(p)
    count = sum(q.shape[0] for q in parts)
    allp = torch.cat(parts) if count else torch.empty((1, width), dtype=torch.float64, device=dev)
    tot = bdist.chunk_chain(allp.reshape(-1, 1, width).contiguous(), count, 1, width, sh).reshape(-1)
    return tot, out


# ----------------------------------------------------------------------------------- fitting
def _wls(x, zw, tot, p, sh):
    """WeightedLeastSquares (linreg.solve_normal) on the working response and weights zw [n, 2] and their chunk sums
    tot = [sum w, sum w x, sum w z]: (coef [D], intercept, diag or None), host, the same on every rank"""
    D, dev = x.shape[1], x.device
    t = tot.cpu().numpy()
    if not np.all(np.isfinite(t)):
        raise ValueError("GeneralizedLinearRegression: the IRLS working response or weights are not finite")
    sw = float(t[0])
    if not sw > 0.0:
        raise ValueError("Sum of weights cannot be zero.")
    xbar, zbar = t[1:D + 1] / sw, float(t[D + 1]) / sw
    z, w = zw[:, 0].contiguous(), zw[:, 1].contiguous()
    q = pca.centered_gram_total(x, torch.from_numpy(xbar).to(dev), sh, y=z, y_mean=zbar, w=w).cpu().numpy()
    W = D + 1
    iu = np.triu_indices(W)
    up = q[iu[0] + iu[1] * (iu[1] + 1) // 2]
    G = np.empty((W, W))
    G[iu] = up
    G[iu[1], iu[0]] = up
    if not np.all(np.isfinite(G)):
        raise ValueError("GeneralizedLinearRegression: the IRLS working response or weights are not finite")
    lp = linreg.LinRegParams(reg_param=p.reg_param, fit_intercept=p.fit_intercept)
    linreg.constant_label_check(sw, zbar, G, lp)          # every rank holds the same G: every rank refuses, or none

    def make():
        coef, b, _, _, diag, _ = linreg.solve_normal(sw, xbar, zbar, G, lp)
        d = np.zeros(D + 1)
        if diag is not None:
            d[:len(diag)] = diag
        return np.concatenate([coef, [b, 0 if diag is None else len(diag)], d])

    host = linreg._broadcast_host(sh, dev, 2 * D + 3, make)
    nd = int(host[D + 1])
    coef, b = host[:D].copy(), float(host[D])
    if not (np.all(np.isfinite(coef)) and math.isfinite(b)):
        raise ValueError("GeneralizedLinearRegression: the IRLS iterate is not finite")
    return coef, b, host[D + 2:D + 2 + nd].copy() if nd else None


def glm_fit(x, y, params, weight=None, offset=None, row_offset=None, group=None):
    """GeneralizedLinearRegression.fit on this rank's rows x [n, D] (f32 or f64), labels y [n], optional prior weights and
    offsets [n]; an empty shard still joins every collective.  -> GLMFit, the same bits on every rank and for any shard
    layout."""
    check_params(params)
    spec = resolve(params)
    x, y, w, off, sh = prepare(x, y, spec, weight, offset, row_offset, group)
    return _irls(x, y, w, off, spec, params, sh)


def _irls(x, y, w, off, spec, p, sh):
    dev = x.device
    tot, zw = rows_total(x, y, w, off, None, 0.0, spec, INIT, sh)
    coef, b, diag = _wls(x, zw, tot, p, sh)
    if spec.family == GAUSSIAN and spec.link == IDENTITY:
        return GLMFit(coef, b, diag, 1, spec)
    it = 0
    while it < p.max_iter:
        tot, zw = rows_total(x, y, w, off, torch.from_numpy(coef).to(dev), b, spec, REWEIGHT, sh)
        c2, b2, diag = _wls(x, zw, tot, p, sh)
        step = max(float(np.max(np.abs(coef - c2))), abs(b - b2))
        coef, b, it = c2, b2, it + 1
        if step < p.tol:
            break
    return GLMFit(coef, b, diag, it, spec)


def _intercept_only(x, y, w, off, spec, p, sh):
    """the intercept of an intercept-only IRLS fit (WeightedLeastSquares without features: the weighted mean of z)"""
    dev, D = x.device, x.shape[1]
    zero = torch.zeros(D, dtype=torch.float64, device=dev)

    def mean(tot):
        t = tot.cpu().numpy()
        if not (np.all(np.isfinite(t)) and t[0] > 0.0):
            raise ValueError("GeneralizedLinearRegression: the intercept-only IRLS iterate is not finite")
        return float(t[D + 1]) / float(t[0])

    b = mean(rows_total(x, y, w, off, None, 0.0, spec, INIT, sh)[0])
    if spec.family == GAUSSIAN and spec.link == IDENTITY:
        return b
    for _ in range(p.max_iter):
        b2 = mean(rows_total(x, y, w, off, zero, b, spec, REWEIGHT, sh)[0])
        step, b = abs(b - b2), b2
        if step < p.tol:
            break
    return b


# ----------------------------------------------------------------------------------- prediction and summary
def glm_predict(x, fit, offset=None):
    """[n, 2] f64 device: (mu, eta) of the rows x [n, D] under a fit, eta = x . coef + intercept + offset"""
    x = _check_x(x)
    if x.shape[1] != fit.coef.shape[0]:
        raise ValueError("vector size %d does not match the fitted size %d" % (x.shape[1], fit.coef.shape[0]))
    n = x.shape[0]
    off = _column(offset, n, x.device)
    if off is not None and not bool(torch.isfinite(off).all()):
        raise ValueError("Offsets must be finite")
    out = torch.empty((n, 2), dtype=torch.float64, device=x.device)
    rows(x, None, None, off, torch.from_numpy(fit.coef).to(x.device), fit.intercept, 0.0, fit.spec, PREDICT, 0, out, None)
    return out


class GLMSummary:
    """the summary numbers (host floats) and device tensors: predictions (mu, eta) [n, 2] and residuals [n, 4] in the
    order of RESIDUALS; aic None for tweedie; std_errors, t_values and p_values None after the quasi-Newton fallback."""

    def __init__(self, **kw):
        self.__dict__.update(kw)


def summarize(x, y, fit, p, weight=None, offset=None, row_offset=None, group=None):
    """GLMSummary of the rows x [n, D], labels y (this rank's shard, with optional weights and offsets) under a fit made
    with params p"""
    x, y, w, off, sh = prepare(x, y, fit.spec, weight, offset, row_offset, group)
    spec, D, dev = fit.spec, x.shape[1], x.device
    fi = p.fit_intercept
    coef = torch.from_numpy(fit.coef).to(dev)
    tot, res = rows_total(x, y, w, off, coef, fit.intercept, spec, SUMMARY, sh)
    t = tot.cpu().numpy()
    sw, dev_, pearson, aic_t = float(t[0]), float(t[2]), float(t[3]), float(t[4])
    if fi and off is None:
        null = rows_total(x, y, w, off, None, 0.0, spec, SUMMARY, sh, mu_const=float(t[1]) / sw, per_row=False)[0]
    else:
        b0 = _intercept_only(x, y, w, off, spec, p, sh) if fi else 0.0
        null = rows_total(x, y, w, off, torch.zeros(D, dtype=torch.float64, device=dev), b0, spec, SUMMARY, sh,
                          per_row=False)[0]
    n = sh.total
    rank = D + (1 if fi else 0)
    dof = n - rank
    disp = 1.0 if spec.family in (BINOMIAL, POISSON) else (pearson / dof if dof != 0 else math.nan)
    if spec.family == GAUSSIAN:
        aic = n * (math.log(dev_ / n * 2.0 * math.pi) + 1.0) + 2.0 - aic_t if dev_ > 0 else -math.inf
    elif spec.family in (BINOMIAL, POISSON):
        aic = -2.0 * aic_t
    elif spec.family == GAMMA:
        d = dev_ / sw
        k = 1.0 / d
        ll = (k - 1.0) * float(t[5]) - float(t[6]) / d - (math.lgamma(k) + k * math.log(d)) * sw - k * float(t[7])
        aic = -2.0 * ll + 2.0
    else:
        aic = None
    if aic is not None:
        aic = aic + 2.0 * rank
    out = dict(predictions=glm_predict(x, fit, off), residuals=res, num_instances=n, rank=rank, degrees_of_freedom=dof,
               residual_dof=dof, residual_dof_null=n - (1 if fi else 0), deviance=dev_,
               null_deviance=float(null[2].item()), dispersion=disp, aic=aic, std_errors=None, t_values=None,
               p_values=None)
    if fit.diag_inv_atwa is not None:
        with np.errstate(divide="ignore", invalid="ignore"):
            se = np.sqrt(fit.diag_inv_atwa * disp)
            est = np.concatenate([fit.coef, [fit.intercept]]) if fi else fit.coef
            tv = est / se
        if spec.family in (BINOMIAL, POISSON):
            pv = np.array([2.0 * (1.0 - 0.5 * math.erfc(-abs(v) / math.sqrt(2.0))) for v in tv])
        else:
            from .selection import f_cdf
            pv = np.array([1.0 - f_cdf(v * v, 1.0, float(dof)) for v in tv])
        out.update(std_errors=se, t_values=tv, p_values=pv)
    return GLMSummary(**out)
