"""numpy restatement of LinearSVC (b200flow/svc.py, DESIGN.md §5j): the scaling, the hinge + L2 objective and its
subgradient, and an independent solver of the same problem written as a quadratic programme.

    xs = x inv, inv_j = 1 / std_j (unbiased; 0 where std_j == 0); y' = 2 label - 1; m = beta . xs + b;
    f(beta, b) = (1/n) sum max(0, 1 - y' m) + 1/2 sum lambda_j beta_j^2, lambda_j = regParam (standardization) or
    regParam inv_j^2; a row adds -y' [xs, 1] to the subgradient iff 1 - y' m > 0.
The QP: min (1/n) sum xi + 1/2 sum lambda_j beta_j^2 subject to xi_i >= 1 - y'_i (beta . xs_i + b) and xi >= 0."""
import numpy as np
from scipy.optimize import minimize


def inv_std(x):
    x = np.asarray(x, np.float64)
    std = x.std(0, ddof=1) if x.shape[0] > 1 else np.zeros(x.shape[1])
    return np.where(std > 0, 1.0 / np.where(std > 0, std, 1.0), 0.0)


def penalty(x, reg, standardization):
    inv = inv_std(x)
    return reg * (np.ones(x.shape[1]) if standardization else inv * inv)


def sums(w, xs, yp):
    """(hinge loss sum, subgradient sums [D + 1]) at w = [beta, b] over the scaled rows xs with signs yp"""
    m = xs @ w[:-1] + w[-1]
    h = 1.0 - yp * m
    act = h > 0
    g = np.concatenate([-(yp[act] @ xs[act]), [-yp[act].sum()]])
    return h[act].sum(), g


def objective(w, x, label, reg, standardization=True, fit_intercept=True):
    """(f, g) at w = [beta (scaled space), b]"""
    x = np.asarray(x, np.float64)
    n, D = x.shape
    xs = x * inv_std(x)
    yp = 2.0 * np.asarray(label, np.float64) - 1.0
    lam = penalty(x, reg, standardization)
    loss, g = sums(w, xs, yp)
    beta = w[:D]
    g = g / n
    g[:D] += lam * beta
    if not fit_intercept:
        g[D] = 0.0
    return loss / n + 0.5 * np.sum(lam * beta * beta), g


def qp_solve(x, label, reg, standardization=True, fit_intercept=True):
    """the minimiser of f by SLSQP on the QP in (beta, b, xi) -> (w = [beta, b] in the scaled space, f(w))"""
    x = np.asarray(x, np.float64)
    n, D = x.shape
    xs = x * inv_std(x)
    yp = 2.0 * np.asarray(label, np.float64) - 1.0
    lam = penalty(x, reg, standardization)
    nb = D + 1

    def fun(z):
        beta = z[:D]
        return z[nb:].sum() / n + 0.5 * np.sum(lam * beta * beta)

    def jac(z):
        g = np.zeros_like(z)
        g[:D] = lam * z[:D]
        g[nb:] = 1.0 / n
        return g

    # xi_i + y'_i (beta . xs_i + b) - 1 >= 0
    A = np.zeros((n, nb + n))
    A[:, :D] = yp[:, None] * xs
    A[:, D] = yp if fit_intercept else 0.0
    A[:, nb:] = np.eye(n)
    cons = [{"type": "ineq", "fun": lambda z: A @ z - 1.0, "jac": lambda z: A}]
    bounds = [(None, None)] * D + [(None, None) if fit_intercept else (0.0, 0.0)] + [(0.0, None)] * n
    z0 = np.concatenate([np.zeros(nb), np.full(n, 1.0)])
    res = minimize(fun, z0, jac=jac, bounds=bounds, constraints=cons, method="SLSQP",
                   options={"maxiter": 2000, "ftol": 1e-15})
    w = res.x[:nb].copy()
    if not fit_intercept:
        w[D] = 0.0
    return w, objective(w, x, label, reg, standardization, fit_intercept)[0]


def blobs(n, D, gap, seed, constant=None):
    """two Gaussian classes whose means are `gap` apart along every axis; labels 0 / 1 (float); column `constant` fixed"""
    rng = np.random.default_rng(seed)
    y = (rng.random(n) < 0.4).astype(np.float64)
    x = rng.normal(0.0, 1.0, (n, D)) * rng.uniform(0.5, 3.0, D) + np.outer(y, np.full(D, gap)) + rng.normal(0, 2, D)
    if constant is not None:
        x[:, constant] = 3.25
    return np.ascontiguousarray(x), y
