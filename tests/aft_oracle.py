"""numpy restatement of AFTSurvivalRegression (b200flow/aft.py's docstring): the kernel's per-row sums, the objective
the optimiser sees, the full fit (standardisation, centring, unscaling) and the quantiles."""
import math

import numpy as np
import torch

from b200flow.linear import lbfgs


def inv_std(x):
    s = x.std(0, ddof=1) if x.shape[0] > 1 else np.zeros(x.shape[1])
    return np.where(s > 0, 1.0 / np.where(s > 0, s, 1.0), 0.0)


def sums(x, log_t, censor, shift, inv, w, b, sigma):
    """[D + 3]: what b200flow_aft_loss_grad totals over the rows"""
    xs = ((x - shift) if shift is not None else x) * inv
    z = (log_t - xs @ w - b) / sigma
    ez = np.exp(z)
    d = np.asarray(censor, np.float64)
    loss = d * math.log(sigma) - d * z + ez
    a = (d - ez) / sigma
    s = d + (d - ez) * z
    return np.concatenate([[loss.sum()], a @ xs, [a.sum(), s.sum()]])


def objective(v, x, t, censor, fi):
    """(f, g) over v = [beta (D), b, log sigma] in the standardised space"""
    n, D = x.shape
    inv = inv_std(x)
    with np.errstate(over="ignore", invalid="ignore"):
        tot = sums(x, np.log(t), censor, x.mean(0) if fi else None, inv, v[:D], v[D], math.exp(v[D + 1]))
    if not np.all(np.isfinite(tot)):
        return math.inf, np.zeros_like(v)
    return tot[0] / n, np.concatenate([tot[1:D + 1] / n, [tot[D + 1] / n if fi else 0.0, tot[D + 2] / n]])


def fit(x, t, censor, fi=True, max_iter=100, tol=1e-6):
    """linear.lbfgs on the restated objective -> (coef, intercept, scale, objective history)"""
    D = x.shape[1]

    def smooth(v):
        f, g = objective(v.numpy(), x, t, censor, fi)
        return torch.tensor(f, dtype=torch.float64), torch.from_numpy(np.asarray(g, np.float64))

    v, hist, _ = lbfgs(smooth, torch.zeros(D + 2, dtype=torch.float64), max_iter, tol, 10)
    v = v.numpy()
    coef = v[:D] * inv_std(x)
    return coef, (v[D] - coef @ x.mean(0)) if fi else v[D], math.exp(v[D + 1]), hist


def quantiles(x, coef, intercept, scale, probs):
    """[n, P]: lambda (-log(1 - p))^scale, lambda = exp(x . coef + intercept)"""
    lam = np.exp(x @ coef + intercept)
    return lam[:, None] * np.array([(-math.log1p(-p)) ** scale for p in probs])[None, :]


def weibull_data(n, D, seed, censor_rate=0.3, sigma=0.7, scale_x=1.0):
    """lifetimes log t = x . beta + b + sigma log E (E ~ Exp(1): Weibull with shape 1 / sigma), right-censored at an
    independent exponential time.  -> (x, observed time, censor, beta, b)"""
    rng = np.random.default_rng(seed)
    x = rng.normal(0.0, 1.0, (n, D)) * scale_x
    beta = rng.normal(0.0, 0.5, D)
    b = 1.5
    t_event = np.exp(x @ beta + b + sigma * np.log(rng.exponential(1.0, n)))
    if censor_rate > 0:
        c_time = rng.exponential(np.median(t_event) / censor_rate, n)
        obs = np.minimum(t_event, c_time)
        censor = (t_event <= c_time).astype(np.float64)
    else:
        obs, censor = t_event, np.ones(n)
    return x, obs, censor, beta, b
