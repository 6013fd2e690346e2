"""numpy restatement of FMRegressor (b200flow/fm.py, DESIGN.md §5r): FMClassifier's restatement (tests/fm_oracle.py) with
MSEFactorizationMachinesGradient's squared error, loss (r - y)^2 and multiplier g = 2 (r - y), in runMiniBatchSGD's loop."""
import numpy as np

import fm_oracle as fo


def sums(w, X, y, D, k, fit_linear=True, fit_intercept=True):
    """(loss sum, gradient sum in w's layout) over the rows X with labels y"""
    V, _, _ = fo.split(w, D, k, fit_linear, fit_intercept)
    r = fo.raw(w, X, D, k, fit_linear, fit_intercept)
    d = r - y
    g = 2.0 * d
    s = X @ V
    gv = (X * g[:, None]).T @ s - V * ((X * X).T @ g)[:, None]
    parts = [gv.reshape(-1)]
    if fit_linear:
        parts.append(X.T @ g)
    if fit_intercept:
        parts.append([g.sum()])
    return np.sum(d * d), np.concatenate(parts)


def fit(X, y, k=8, fit_linear=True, fit_intercept=True, reg=0.0, fraction=1.0, init_std=0.01, max_iter=100, step=1.0,
        tol=1e-6, solver="adamW", seed=0):
    """runMiniBatchSGD -> (w, loss history, updates made)"""
    X = np.asarray(X, np.float64)
    y = np.asarray(y, np.float64)
    n, D = X.shape
    w = fo.init_coefficients(D, k, fit_linear, fit_intercept, init_std, seed)
    upd = (fo.AdamW if solver == "adamW" else fo.GD)(w.shape[0])
    n0 = np.sqrt(np.sum(w * w))
    reg_val = 0.5 * reg * n0 * n0
    hist, prev = [], None
    for it in range(1, max_iter + 1):
        keep = fo.batch_mask(n, fraction, it)
        nb = int(keep.sum())
        if nb == 0:
            continue
        loss, g = sums(w, X[keep], y[keep], D, k, fit_linear, fit_intercept)
        hist.append(loss / nb + reg_val)
        w_old = w
        w, reg_val = upd(w, g / nb, step, it, reg)
        if prev is not None and np.sqrt(np.sum((w - w_old) ** 2)) < tol * max(np.sqrt(np.sum(w * w)), 1.0):
            return w, hist, len(hist)
        prev = w_old
    return w, hist, len(hist)


def doctest_data():
    """the PySpark FMRegressor doctest: (2.0, [2.0]), (1.0, [1.0]), (0.0, [0.0]); factorSize 2, seed 16"""
    return np.array([[2.0], [1.0], [0.0]]), np.array([2.0, 1.0, 0.0])


DOCTEST = {"intercept": -0.0032501766849261557, "x": [-2.0, 0.5, 1.0, 4.0],
           "prediction": [-1.9989237712341565, 0.4956682219523814, 0.994586620589689, 3.9880970124135344]}
