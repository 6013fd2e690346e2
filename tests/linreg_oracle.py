"""numpy restatement of LinearRegression (b200flow/linreg.py's docstring): the kernel's per-row sums, the three objectives
the optimiser sees (normal equations, L-BFGS squared loss, Huber), the normal-path statistics and the summary formulas."""
import math

import numpy as np
import torch

from b200flow.linear import lbfgs


def inv_std(x, ddof):
    s = x.std(0, ddof=ddof) if x.shape[0] > ddof else np.zeros(x.shape[1])
    return np.where(s > 0, 1.0 / np.where(s > 0, s, 1.0), 0.0), s


def sums(x, y, shift, inv, y_shift, y_scale, w, b, sigma, eps, mode):
    """[D + 3]: what b200flow_linreg_loss_grad totals over the rows (mode 0 squared, 1 huber)"""
    xs = ((x - shift) if shift is not None else x) * inv
    m = xs @ w
    if mode == 0:
        d = m - (y - y_shift) * y_scale
        return np.concatenate([[np.sum(d * d)], d @ xs, [d.sum(), 0.0]])
    z = (y - m - b) / sigma
    inner = np.abs(z) <= eps
    loss = np.where(inner, sigma + z * z * sigma, sigma + (2 * eps * np.abs(z) - eps * eps) * sigma)
    a = np.where(inner, -2.0 * z, -2.0 * eps * np.sign(z))
    s = np.where(inner, 1.0 - z * z, 1.0 - eps * eps)
    return np.concatenate([[loss.sum()], a @ xs, [a.sum(), s.sum()]])


def squared_objective(w, x, y, reg, alpha, fi, st):
    """(f, g) of the L-BFGS squared-loss objective over w (scaled space), L2 part only (L1 goes to OWL-QN); unbiased
    moments.  -> also the L1 weights and the back-transform (coef, intercept) of a solution"""
    n, D = x.shape
    inv, _ = inv_std(x, 1)
    ystd = y.std(ddof=1)
    mx, my = x.mean(0), y.mean()
    t = sums(x, y, mx if fi else None, inv, my if fi else 0.0, 1.0 / ystd, w, 0.0, 1.0, 0.0, 0)
    eff = reg / ystd
    lam = (1 - alpha) * eff * (np.ones(D) if st else inv * inv)
    return t[0] / (2 * n) + 0.5 * np.sum(lam * w * w), t[1:D + 1] / n + lam * w


def squared_l1(x, y, reg, alpha, st):
    inv, _ = inv_std(x, 1)
    return alpha * reg / y.std(ddof=1) * (np.ones(x.shape[1]) if st else inv)


def huber_objective(v, x, y, reg, eps, fi, st):
    """(f, g) of the Huber objective over [w, b, sigma]"""
    n, D = x.shape
    inv, _ = inv_std(x, 1)
    w, b, sigma = v[:D], v[D], v[D + 1]
    t = sums(x, y, None, inv, 0.0, 1.0, w, b, sigma, eps, 1)
    lam = reg * (np.ones(D) if st else inv * inv)
    g = np.concatenate([t[1:D + 1] / n + lam * w, [t[D + 1] / n if fi else 0.0, t[D + 2] / n]])
    return t[0] / n + 0.5 * np.sum(lam * w * w), g


def _torch_smooth(fun):
    def smooth(v):
        f, g = fun(v.numpy())
        return torch.tensor(f, dtype=torch.float64), torch.from_numpy(np.asarray(g, np.float64))
    return smooth


def lbfgs_squared(x, y, reg=0.0, alpha=0.0, fi=True, st=True, max_iter=500, tol=1e-14):
    """linear.lbfgs on the restated squared objective -> (coef, intercept)"""
    D = x.shape[1]
    inv, _ = inv_std(x, 1)
    l1 = squared_l1(x, y, reg, alpha, st) if alpha * reg > 0 else None
    v, _, _ = lbfgs(_torch_smooth(lambda w: squared_objective(w, x, y, reg, alpha, fi, st)), torch.zeros(D, dtype=torch.float64),
                    max_iter, tol, 10, l1=None if l1 is None else torch.from_numpy(l1))
    coef = v.numpy() * y.std(ddof=1) * inv
    return coef, (y.mean() - coef @ x.mean(0)) if fi else 0.0


def lbfgs_huber(x, y, reg=0.0, eps=1.35, fi=True, st=True, max_iter=2000, tol=1e-15):
    """linear.lbfgs on the restated Huber objective (f = inf where sigma <= 0) -> (coef, intercept, sigma)"""
    D = x.shape[1]
    inv, _ = inv_std(x, 1)

    def fun(v):
        if not v[D + 1] > 0:
            return math.inf, np.zeros_like(v)
        return huber_objective(v, x, y, reg, eps, fi, st)

    v0 = np.zeros(D + 2)
    v0[D + 1] = 1.0
    v, _, _ = lbfgs(_torch_smooth(fun), torch.from_numpy(v0), max_iter, tol, 10)
    v = v.numpy()
    return v[:D] * inv, v[D], v[D + 1]


def normal_statistics(x, y):
    """(n, xBar, yBar, G): the two-pass centred Gram matrix of [x, y]"""
    xy = np.concatenate([x, y[:, None]], 1)
    c = xy - xy.mean(0)
    return x.shape[0], x.mean(0), y.mean(), c.T @ c


def normal_solve_spark(x, y, reg=0.0, fi=True, st=True):
    """WeightedLeastSquares' Cholesky path as Spark writes it: the one-pass uncentred scaled moments and the
    intercept-augmented system (elasticNetParam = 0) -> (coef, intercept, diagInvAtWA)"""
    n, D = x.shape
    a_std, b_std = x.std(0), y.std()
    inv = np.where(a_std > 0, 1.0 / np.where(a_std > 0, a_std, 1.0), 0.0)
    xs, ys = x * inv, y / b_std
    aa, ab = xs.T @ xs / n, xs.T @ ys / n
    lam = reg / b_std * (np.ones(D) if st else inv * inv)
    aa = aa + np.diag(lam)
    if fi:
        xb = xs.mean(0)
        aa = np.block([[aa, xb[:, None]], [xb[None, :], np.ones((1, 1))]])
        ab = np.concatenate([ab, [ys.mean()]])
    sol = np.linalg.solve(aa, ab)
    inv_diag = np.diag(np.linalg.inv(aa))
    mult = np.concatenate([a_std * a_std, [1.0]]) if fi else a_std * a_std
    return sol[:D] * b_std * inv, (sol[D] * b_std if fi else 0.0), inv_diag / (n * mult)


def summary(x, y, coef, intercept, diag, fi):
    """the summary numbers: residuals, mse, r2 (through the origin without an intercept), r2adj, dof, standard errors,
    t values and p values (Student's t, two-sided), the intercept last"""
    from scipy import stats
    n, D = x.shape
    pred = x @ coef + intercept
    res = y - pred
    mse = np.mean(res * res)
    i = 1 if fi else 0
    den = np.sum((y - y.mean()) ** 2) if fi else np.sum(y * y)
    r2 = 1.0 - np.sum(res * res) / den
    dof = n - D - i
    out = dict(mse=mse, rmse=math.sqrt(mse), mae=np.mean(np.abs(res)), r2=r2, r2adj=1 - (1 - r2) * (n - i) / (n - D - i),
               dof=dof, residual_range=(res.min(), res.max()),
               explained_variance=np.mean((pred - y.mean()) ** 2))
    if diag is not None:
        se = np.sqrt(diag * np.sum(res * res) / dof)
        est = np.concatenate([coef, [intercept]]) if fi else coef
        tv = est / se
        out.update(se=se, t=tv, p=2.0 * stats.t.sf(np.abs(tv), dof))
    return out
