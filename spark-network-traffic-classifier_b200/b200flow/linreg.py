"""LinearRegression on the device (DESIGN.md §5n): the normal equations from the labelled centred Gram matrix of
csrc/pca.cu, and the per-row least-squares / Huber loss and gradient of csrc/linreg.cu for the quasi-Newton paths, both
summed in the chunk order of dist.Shards, so that every fit is the same bits for any world size and shard layout.

Spark [recalled; Spark 3 `ml/regression/LinearRegression.scala`, `ml/optim/WeightedLeastSquares.scala`,
`ml/optim/NormalEquationSolver.scala`, `ml/optim/aggregator/LeastSquaresAggregator.scala`, `HuberAggregator.scala`]:

    Params: maxIter 100, regParam 0.0, elasticNetParam 0.0, tol 1e-6, fitIntercept true, standardization true, solver
    "auto" (auto / normal / l-bfgs), loss "squaredError" (or "huber"), epsilon 1.35 (> 1), aggregationDepth 2,
    maxBlockSizeInMB 0.0.  Huber with solver "normal", or with elasticNetParam > 0, is refused.
    Solver: squared loss with auto or normal takes the normal equations (D <= 4096); l-bfgs and Huber take the per-row path.

    Normal equations (WeightedLeastSquares, weights 1): population moments aBar, bBar, aStd = sqrt(aVar), bStd (/ n).
    Constant label (bStd == 0): with fitIntercept or bBar == 0 the coefficients are 0, the intercept bBar and the objective
    history [0]; otherwise regParam > 0 raises, and bStd = |bBar|.  Features are scaled by 1 / aStd (0 where aStd = 0), the
    label by 1 / bStd; effectiveRegParam = regParam / bStd, L1 = elasticNetParam of it, L2 = the rest, added to the
    diagonal of aaBar (divided by aStd_j^2 when standardization is false, 0 where aStd_j = 0).  Cholesky when
    elasticNetParam * regParam == 0; otherwise, or when Cholesky finds the matrix singular (Spark logs a warning), the
    quasi-Newton solver (OWL-QN with the L1 weights) minimises 1/2 b^T A b - ab^T b + 1/2 bbBar over the same statistics
    from [0, ..., 0, bBar].  coefficients_j = solution_j bStd / aStd_j, intercept = solution_last bStd.  diagInvAtWA: the
    diagonal of the inverse of the intercept-augmented matrix, divided by n aStd_j^2 (the intercept entry by n); the
    Cholesky path only.

    L-BFGS, squared loss: unbiased moments (the summariser's std).  A constant label takes the same early exit as above
    (regParam > 0 raises "Model cannot be regularized").  xs = (x - xBar) inv and ys = (y - yBar) / yStd with an intercept,
    neither centred without one; f(w) = (1/2n) sum (xs . w - ys)^2 + 1/2 sum_j lambda_j w_j^2 over w alone, lambda_j =
    (1 - alpha) regParam / yStd (divided by std_j^2 without standardization), the L1 weight alpha regParam / yStd (divided by
    std_j) through OWL-QN.  Starts from 0; coefficients_j = w_j yStd inv_j; intercept = yBar - coefficients . xBar.

    Huber (Owen's concomitant scale; the objective of scikit-learn's HuberRegressor): variables [w, b, sigma] from
    [0, 0, 1]; features scaled by inv and not centred, the label not scaled;
        f = (1/n) sum (sigma + H((y - xs . w - b) / sigma) sigma) + 1/2 sum_j lambda_j w_j^2,
    H(z) = z^2 for |z| <= epsilon, 2 epsilon |z| - epsilon^2 beyond; lambda_j = regParam (regParam inv_j^2 without
    standardization).  Spark runs L-BFGS-B with sigma >= tiny; here linear.lbfgs_steps runs unchanged and every trial point
    with sigma <= 0 gets f = +inf without a pass, so its backtracking rejects it.  Iterates therefore differ from Spark's;
    the objective is jointly convex for sigma > 0, so the minimiser is the same.  scale = sigma (1.0 for squared loss).

Deviations: weightCol, more than 255 features, non-finite features or labels and an empty dataset raise ValueError (the
shim's IllegalArgumentException).  The normal equations are built from a two-pass centred Gram matrix where Spark sums
uncentred moments in one pass: the same system in exact arithmetic, so the results agree to rounding.  Spark's Cholesky
(LAPACK) fails only on a non-positive pivot; here a pivot below 1e-12 of its diagonal entry also counts as singular, so
exactly collinear columns (duplicated, or constant without regularisation) take the quasi-Newton fallback reliably.  The
D x D solves run on rank 0 and are broadcast, since host BLAS differs between CPU models; the quasi-Newton optimiser state
of the per-row path lives on the device, so every rank takes the same steps (as svc.py).
"""
import math

import numpy as np
import torch

from . import _lib
from . import dist as bdist
from . import metrics, pca, selection
from .linear import lbfgs, lbfgs_steps
from ._lib import call, ptr

MAX_D = 255
HISTORY = 10
SQUARED, HUBER = 0, 1
SOLVERS = ("auto", "normal", "l-bfgs")
LOSSES = ("squarederror", "huber")
SINGULAR_PIVOT = 1e-12


class LinRegParams:
    __slots__ = ("max_iter", "reg_param", "elastic_net_param", "tol", "fit_intercept", "standardization", "solver", "loss",
                 "epsilon")

    def __init__(self, max_iter=100, reg_param=0.0, elastic_net_param=0.0, tol=1e-6, fit_intercept=True,
                 standardization=True, solver="auto", loss="squaredError", epsilon=1.35):
        self.max_iter, self.reg_param, self.elastic_net_param = int(max_iter), float(reg_param), float(elastic_net_param)
        self.tol, self.fit_intercept, self.standardization = float(tol), bool(fit_intercept), bool(standardization)
        self.solver, self.loss, self.epsilon = str(solver).lower(), str(loss).lower(), float(epsilon)


def check_params(p):
    """Spark's validators and refusals; raises ValueError"""
    if p.max_iter < 0:
        raise ValueError("maxIter must be >= 0, got %r" % p.max_iter)
    if not p.reg_param >= 0.0 or not p.tol >= 0.0:
        raise ValueError("regParam and tol must be >= 0, got %r and %r" % (p.reg_param, p.tol))
    if not 0.0 <= p.elastic_net_param <= 1.0:
        raise ValueError("elasticNetParam must be in [0, 1], got %r" % p.elastic_net_param)
    if p.solver not in SOLVERS:
        raise ValueError("solver must be one of %s, got %r" % (list(SOLVERS), p.solver))
    if p.loss not in LOSSES:
        raise ValueError("loss must be 'squaredError' or 'huber', got %r" % p.loss)
    if not p.epsilon > 1.0:
        raise ValueError("epsilon must be > 1.0, got %r" % p.epsilon)
    if p.loss == "huber" and p.solver == "normal":
        raise ValueError("LinearRegression with huber loss doesn't support normal solver, please change solver to auto "
                         "or l-bfgs.")
    if p.loss == "huber" and p.elastic_net_param > 0.0:
        raise ValueError("LinearRegression with huber loss only supports L2 regularization, but got elasticNetParam = %r."
                         % p.elastic_net_param)


def solver_for(p):
    """'normal' or 'l-bfgs': the path a fit takes"""
    return "normal" if p.loss == "squarederror" and p.solver in ("auto", "normal") else "l-bfgs"


class LinRegFit:
    """coef f64 [D] (host), intercept, scale, objective history, iterations, diag_inv_atwa ([D (+1)] host, or None) and
    the solver used ('normal', 'quasi-newton' for the normal path's fallback, or 'l-bfgs')."""
    __slots__ = ("coef", "intercept", "scale", "objective_history", "iterations", "diag_inv_atwa", "solver")

    def __init__(self, coef, intercept, scale, hist, it, diag, solver):
        self.coef, self.intercept, self.scale = coef, float(intercept), float(scale)
        self.objective_history, self.iterations, self.diag_inv_atwa, self.solver = list(hist), int(it), diag, solver


def _check_x(x):
    if not (torch.is_tensor(x) and x.is_cuda and x.dim() == 2 and x.dtype in (torch.float32, torch.float64)):
        raise _lib.B200FlowError("LinearRegression needs a CUDA float32 or float64 [n, D] matrix")
    if not 1 <= x.shape[1] <= MAX_D:
        raise _lib.UnsupportedParamError("LinearRegression supports 1 to %d features, got %d" % (MAX_D, x.shape[1]))
    return x.contiguous()


# ----------------------------------------------------------------------------------- the per-row pass
def loss_grad(x, y, shift, inv, y_shift, y_scale, w, b_sigma, eps, mode, row_offset, partials):
    """b200flow_linreg_loss_grad on the rows x [n, D] (f32/f64): partials [n_chunks, D + 3] f64 device; y f64 [n], shift
    f64 [D] or None, inv f64 [D], w f64 [D], b_sigma f64 [2] (huber) or None, all device."""
    n, D = x.shape
    call("b200flow_linreg_loss_grad", ptr(x), _lib.dtype_code(x), n, x.stride(0), D, ptr(y), ptr(shift), ptr(inv),
         float(y_shift), float(y_scale), ptr(w), ptr(b_sigma), float(eps), int(mode), int(row_offset), ptr(partials))


def loss_grad_totals(x, y, shift, inv, y_shift, y_scale, w, b_sigma, eps, mode, sh):
    """[D + 3] f64 device: the loss, gradient, b and sigma sums over every rank's rows in chunk order; the same bits on
    every rank."""
    D = x.shape[1]

    def launch(xs, _, ys, go, parts):
        loss_grad(xs, ys, shift, inv, y_shift, y_scale, w, b_sigma, eps, mode, go, parts)

    return selection.chunk_total(x, None, y, sh, 1, D + 3, launch).reshape(-1)


# ----------------------------------------------------------------------------------- fitting
def _prepare(x, y, row_offset, group):
    x = _check_x(x)
    n_local = x.shape[0]
    grp = group if group is not None else bdist.group()
    dev = x.device
    if row_offset is None:
        row_offset, _ = bdist.global_offset(n_local, dev, grp)
    sh = bdist.Shards(n_local, row_offset, grp, dev)
    y = y.to(device=dev, dtype=torch.float64).reshape(-1).contiguous()
    bad = torch.stack([(~torch.isfinite(x)).any(), (~torch.isfinite(y)).any(), torch.tensor(y.shape[0] != n_local, device=dev)])
    bad = bad.to(torch.int64)
    if grp is not None:
        bdist.all_reduce_(bad, grp)
    if int(bad[2].item()):
        raise ValueError("LinearRegression needs one label per row (a shard has %d rows and %d labels)" % (n_local, y.shape[0]))
    if sh.total == 0:
        raise ValueError("LinearRegression needs at least one row")
    if int(bad[0].item()) or int(bad[1].item()):
        raise ValueError("LinearRegression needs finite features and labels")
    return x, y, sh


def linreg_fit(x, y, params, row_offset=None, group=None):
    """LinearRegression.fit on this rank's rows x [n, D] (f32 or f64) and labels y [n]; an empty shard still joins every
    collective.  -> LinRegFit, the same bits on every rank and for any shard layout."""
    check_params(params)
    x, y, sh = _prepare(x, y, row_offset, group)
    if solver_for(params) == "normal":
        return _fit_normal(x, y, params, sh)
    return _fit_lbfgs(x, y, params, sh)


def _broadcast_host(sh, dev, size, make):
    """rank 0 computes make() -> host f64 [size] and broadcasts it; every rank returns the same host array"""
    buf = torch.empty(size, dtype=torch.float64, device=dev)
    if sh.rank == 0:
        buf.copy_(torch.from_numpy(np.asarray(make(), np.float64)))
    if sh.grp is not None:
        bdist.broadcast_(buf, 0, sh.grp)
    return buf.cpu().numpy()


def normal_statistics(x, y, sh):
    """(n, xBar [D], yBar, G [D + 1, D + 1]) (host f64): G is the centred Gram matrix of [x, y], two-pass, chunk order"""
    n, D = sh.total, x.shape[1]
    x64 = x if x.dtype == torch.float64 else x.to(torch.float64)
    mx = pca.column_sums(x64, sh) * (1.0 / n)
    my = float(pca.column_sums(y.reshape(-1, 1), sh).item()) * (1.0 / n)
    q = pca.centered_gram_total(x, mx, sh, y=y, y_mean=my).cpu().numpy()
    W = D + 1
    iu = np.triu_indices(W)
    up = q[iu[0] + iu[1] * (iu[1] + 1) // 2]
    G = np.empty((W, W))
    G[iu] = up
    G[iu[1], iu[0]] = up
    return n, mx.cpu().numpy(), my, G


def _cholesky(A):
    """lower L with A = L L^T, or None when a pivot is not positive or falls below SINGULAR_PIVOT of its diagonal entry"""
    try:
        L = np.linalg.cholesky(A)
    except np.linalg.LinAlgError:
        return None
    d = np.diag(A)
    if not np.all(np.diag(L) * np.diag(L) > SINGULAR_PIVOT * d):
        return None
    return L


def _quadratic_qn(A, ab, bb, start, max_iter, tol, l1):
    """the quasi-Newton solver of the normal equations: minimise 1/2 b^T A b - ab^T b + 1/2 bb (host torch f64)"""
    At, abt = torch.from_numpy(A), torch.from_numpy(ab)

    def smooth(v):
        Av = At @ v
        return 0.5 * (v @ Av) - abt @ v + 0.5 * bb, Av - abt

    v, hist, it = lbfgs(smooth, torch.from_numpy(start), max_iter, tol, HISTORY,
                        l1=None if l1 is None else torch.from_numpy(l1))
    return v.numpy(), hist, it


def constant_label_check(n, ybar, G, p):
    """True when the label is constant and the model is fitted without solving (coefficients 0, intercept yBar);
    ValueError when it is constant, non-zero, without an intercept and regularised"""
    if G[-1, -1] != 0.0:
        return False
    if p.fit_intercept or ybar == 0.0:
        return True
    if p.reg_param > 0.0:
        raise ValueError("The standard deviation of the label is zero. Model cannot be regularized with "
                         "standardization=true")
    return False


def solve_normal(n, xbar, ybar, G, p):
    """WeightedLeastSquares on the statistics of normal_statistics -> (coef [D], intercept, hist, iterations, diag or None,
    solver); ValueError for a constant label that cannot be fitted.  Host numpy, deterministic on one machine."""
    D = xbar.shape[0]
    fi = p.fit_intercept
    a_std = np.sqrt(np.diag(G)[:D] / n)
    raw_b_std = math.sqrt(G[D, D] / n)
    if constant_label_check(n, ybar, G, p):
        return np.zeros(D), ybar if fi else 0.0, [0.0], 0, None, "normal"
    b_std = raw_b_std if raw_b_std > 0.0 else abs(ybar)
    inv = np.where(a_std > 0, 1.0 / np.where(a_std > 0, a_std, 1.0), 0.0)
    xb, bb = xbar * inv, ybar / b_std
    cov = G[:D, :D] / n * inv[:, None] * inv[None, :]
    cxy = G[:D, D] / n * inv / b_std
    byy = G[D, D] / n / (b_std * b_std)
    eff = p.reg_param / b_std
    l1, l2 = p.elastic_net_param * eff, (1.0 - p.elastic_net_param) * eff
    lam = np.full(D, l2) if p.standardization else l2 * inv * inv
    unc = cov + np.outer(xb, xb)                                  # aaBar (scaled)
    if fi:
        A, rhs = cov + np.diag(lam), cxy
    else:
        A, rhs = unc + np.diag(lam), cxy + xb * bb
    L = _cholesky(A) if p.elastic_net_param * p.reg_param == 0.0 else None
    if L is not None:
        Li = np.linalg.solve(L, np.eye(D))
        w = Li.T @ (Li @ rhs)
        b = bb - xb @ w if fi else 0.0
        with np.errstate(divide="ignore", invalid="ignore"):
            diag = (Li * Li).sum(0) / (n * a_std * a_std)
        if fi:
            u = Li @ xb
            diag = np.concatenate([diag, [(1.0 + u @ u) / n]])
        hist, it, diag_out, solver = [0.0], 0, diag, "normal"
    else:
        if fi:                                                    # the intercept-augmented system
            Aa = np.zeros((D + 1, D + 1))
            Aa[:D, :D] = unc + np.diag(lam)
            Aa[:D, D] = Aa[D, :D] = xb
            Aa[D, D] = 1.0
            ab = np.concatenate([cxy + xb * bb, [bb]])
            start = np.concatenate([np.zeros(D), [bb]])
        else:
            Aa, ab, start = A, rhs, np.zeros(D)
        l1w = None
        if l1 != 0.0:
            l1w = np.full(D, l1) if p.standardization else l1 * inv
            if fi:
                l1w = np.concatenate([l1w, [0.0]])
        sol, hist, it = _quadratic_qn(Aa, ab, byy + bb * bb, start, p.max_iter, p.tol, l1w)
        w = sol[:D]
        b = sol[D] if fi else 0.0
        diag_out, solver = None, "quasi-newton"
    return w * b_std * inv, b * b_std if fi else 0.0, hist, it, diag_out, solver


def _fit_normal(x, y, p, sh):
    n, xbar, ybar, G = normal_statistics(x, y, sh)
    D = x.shape[1]
    H = p.max_iter + 1
    # [coef (D), intercept, iterations, history length, quasi-Newton?, diag length, diag (D + 1), history (H)]
    size = 2 * D + 6 + H

    def make():
        coef, b, hist, it, diag, solver = solve_normal(n, xbar, ybar, G, p)
        d = np.zeros(D + 1)
        if diag is not None:
            d[:len(diag)] = diag
        h = np.zeros(H)
        h[:len(hist)] = hist
        return np.concatenate([coef, [b, it, len(hist), solver == "quasi-newton", 0 if diag is None else len(diag)], d, h])

    constant_label_check(n, ybar, G, p)          # every rank holds the same G: every rank refuses, or none
    host = _broadcast_host(sh, x.device, size, make)
    it, nh, qn, nd = (int(v) for v in host[D + 1:D + 5])
    diag = host[D + 5:D + 5 + nd].copy() if nd else None
    hist = [float(v) for v in host[2 * D + 6:2 * D + 6 + nh]]
    return LinRegFit(host[:D].copy(), host[D], 1.0, hist, it, diag, "quasi-newton" if qn else "normal")


def _fit_lbfgs(x, y, p, sh):
    n, D, dev = sh.total, x.shape[1], x.device
    x64 = x if x.dtype == torch.float64 else x.to(torch.float64)
    mx = selection.group_sums_total(x64, None, 1, sh)[0] * (1.0 / n)
    my_t = selection.group_sums_total(y.reshape(-1, 1), None, 1, sh)[0] * (1.0 / n)
    my = float(my_t.item())
    t = selection.centered_moments_total(x64, None, 1, mx.contiguous(), y, my, sh).cpu().numpy().reshape(-1)
    sxx, syy = t[:D], float(t[2 * D])
    std = np.sqrt(sxx / (n - 1)) if n > 1 else np.zeros(D)
    raw_y_std = math.sqrt(syy / (n - 1)) if n > 1 else 0.0
    fi = p.fit_intercept
    if raw_y_std == 0.0:
        if fi or my == 0.0:
            return LinRegFit(np.zeros(D), my if fi else 0.0, 1.0, [0.0], 0, None, "l-bfgs")
        if p.reg_param != 0.0:
            raise ValueError("The standard deviation of the label is zero. Model cannot be regularized.")
    y_std = raw_y_std if raw_y_std > 0.0 else abs(my)
    inv_h = np.where(std > 0, 1.0 / np.where(std > 0, std, 1.0), 0.0)
    inv = torch.from_numpy(inv_h).to(dev)
    ones = torch.ones(D, dtype=torch.float64, device=dev)
    if p.loss == "huber":
        return _fit_huber(x, y, p, sh, inv)
    eff = p.reg_param / y_std
    l1, l2 = p.elastic_net_param * eff, (1.0 - p.elastic_net_param) * eff
    lam = l2 * ones if p.standardization else l2 * inv * inv
    l1w = (l1 * ones if p.standardization else l1 * inv) if l1 != 0.0 else None
    shift = mx.reshape(-1).contiguous() if fi else None
    y_shift = my if fi else 0.0

    def evaluate(v):
        tot = loss_grad_totals(x, y, shift, inv, y_shift, 1.0 / y_std, v, None, 0.0, SQUARED, sh)
        return tot[0] / (2.0 * n) + 0.5 * (lam * v * v).sum(), tot[1:D + 1] / n + lam * v

    v, hist, it = _run(evaluate, torch.zeros(D, dtype=torch.float64, device=dev), p, l1w)
    coef = v * y_std * inv
    intercept = float((my_t.reshape(-1)[0] - (coef * mx.reshape(-1)).sum()).item()) if fi else 0.0
    return LinRegFit(coef.cpu().numpy(), intercept, 1.0, hist, it, None, "l-bfgs")


def _run(evaluate, v0, p, l1w):
    """linear.lbfgs_steps driven by evaluate(v) -> (f, g); the optimiser state stays on the device"""
    steps = lbfgs_steps(v0, p.max_iter, p.tol, HISTORY, l1=l1w)
    point = next(steps)
    try:
        while True:
            point = steps.send(evaluate(point))
    except StopIteration as done:
        return done.value


def _fit_huber(x, y, p, sh, inv):
    n, D, dev = sh.total, x.shape[1], x.device
    lam = p.reg_param * (torch.ones(D, dtype=torch.float64, device=dev) if p.standardization else inv * inv)
    fi = p.fit_intercept
    zero = torch.zeros(1, dtype=torch.float64, device=dev)

    def evaluate(v):
        if not float(v[D + 1].item()) > 0.0:                # sigma <= 0: outside the domain, rejected by the line search
            return torch.tensor(math.inf, dtype=torch.float64, device=dev), torch.zeros_like(v)
        w = v[:D].contiguous()
        tot = loss_grad_totals(x, y, None, inv, 0.0, 1.0, w, v[D:].contiguous(), p.epsilon, HUBER, sh)
        f = tot[0] / n + 0.5 * (lam * w * w).sum()
        return f, torch.cat([tot[1:D + 1] / n + lam * w, tot[D + 1:D + 2] / n if fi else zero, tot[D + 2:D + 3] / n])

    v0 = torch.zeros(D + 2, dtype=torch.float64, device=dev)
    v0[D + 1] = 1.0
    v, hist, it = _run(evaluate, v0, p, None)
    coef = (v[:D] * inv).cpu().numpy()
    return LinRegFit(coef, float(v[D].item()), float(v[D + 1].item()), hist, it, None, "l-bfgs")


# ----------------------------------------------------------------------------------- prediction and summary
def weights(fit):
    """[1, D + 1] f64 host: the coefficients, then the intercept"""
    return torch.from_numpy(np.concatenate([fit.coef, [fit.intercept]])).reshape(1, -1)


def linreg_predict(x, fit):
    """[n] f64 device: x . coefficients + intercept (svc.svc_margins with one column)"""
    from .svc import svc_margins
    return svc_margins(x, weights(fit))[:, 0]


class LinRegSummary:
    """the training / evaluation summary numbers (host floats); standard errors, t and p values are None off the Cholesky
    path.  Coefficient-wise arrays carry the intercept last when the model has one."""

    def __init__(self, **kw):
        self.__dict__.update(kw)


def summarize(x, y, fit, fit_intercept, group=None):
    """LinRegSummary of the rows x [n, D], labels y [n] (this rank's shard) under a fit: regression_metrics with
    through_origin = not fit_intercept, r2adj, the residual range (exact MIN / MAX all-reduces), degrees of freedom and,
    with diag_inv_atwa, the coefficient standard errors, t values and two-sided p values."""
    x = _check_x(x)
    grp = group if group is not None else bdist.group()
    y = y.to(device=x.device, dtype=torch.float64).reshape(-1).contiguous()
    pred = linreg_predict(x, fit)
    res = y - pred
    m = metrics.regression_metrics(y, pred, grp, through_origin=not fit_intercept)
    n = torch.tensor([x.shape[0]], dtype=torch.int64, device=x.device)
    ext = torch.stack([res.min() if res.shape[0] else torch.tensor(math.inf, dtype=torch.float64, device=x.device),
                       -res.max() if res.shape[0] else torch.tensor(math.inf, dtype=torch.float64, device=x.device)])
    if grp is not None:
        import torch.distributed as dist
        bdist.all_reduce_(n, grp)
        bdist.all_reduce_(ext, grp, op=dist.ReduceOp.MIN)
    n = int(n.item())
    D = x.shape[1]
    i = 1 if fit_intercept else 0
    dof = n - D - i
    e = ext.cpu().numpy()
    out = dict(predictions=pred, residuals=res, num_instances=n, degrees_of_freedom=dof, mse=m["mse"], rmse=m["rmse"],
               mae=m["mae"], explained_variance=m["var"], r2=m["r2"], deviance_residuals=[float(e[0]), float(-e[1])],
               std_errors=None, t_values=None, p_values=None)
    with np.errstate(divide="ignore", invalid="ignore"):
        out["r2adj"] = float(1.0 - (1.0 - m["r2"]) * (n - i) / (n - D - i)) if n - D - i != 0 else math.nan
        if fit.diag_inv_atwa is not None:
            sigma2 = m["mse"] * n / dof if dof > 0 else math.nan
            se = np.sqrt(fit.diag_inv_atwa * sigma2)
            est = np.concatenate([fit.coef, [fit.intercept]]) if fit_intercept else fit.coef
            tv = est / se
            out.update(std_errors=se, t_values=tv,
                       p_values=np.array([1.0 - selection.f_cdf(t * t, 1.0, float(dof)) for t in tv]))
    return LinRegSummary(**out)
