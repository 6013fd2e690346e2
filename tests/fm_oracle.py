"""numpy restatement of FMClassifier (b200flow/fm.py, DESIGN.md §5k) in Spark's loop order: java.util.Random and the
factor init, the per-row raw value, loss and gradient (FactorizationMachinesAggregator), the gd and adamW updaters, and
mllib's runMiniBatchSGD with this project's FMMB batch draw.

Coefficients w = [V (D x k, row-major), lin (D) if fit_linear, b if fit_intercept]."""
import math

import numpy as np

from b200flow.kmeans import philox

PURPOSE_FMMB = 0x464D4D42


class JavaRandom:
    """java.util.Random(seed): the 48-bit LCG, nextDouble and the polar nextGaussian"""

    def __init__(self, seed):
        self.seed = (seed ^ 0x5DEECE66D) & ((1 << 48) - 1)
        self.cached = None

    def next(self, bits):
        self.seed = (self.seed * 0x5DEECE66D + 0xB) & ((1 << 48) - 1)
        r = self.seed >> (48 - bits)
        return r - (1 << 32) if r & (1 << 31) else r

    def next_double(self):
        return ((self.next(26) << 27) + self.next(27)) * 2.0 ** -53

    def next_gaussian(self):
        if self.cached is not None:
            g, self.cached = self.cached, None
            return g
        while True:
            v1, v2 = 2 * self.next_double() - 1, 2 * self.next_double() - 1
            s = v1 * v1 + v2 * v2
            if s < 1 and s != 0:
                break
        mult = math.sqrt(-2 * math.log(s) / s)
        self.cached = v2 * mult
        return v1 * mult


def init_coefficients(D, k, fit_linear, fit_intercept, init_std, seed):
    rnd = JavaRandom(seed)
    v = [rnd.next_gaussian() * init_std for _ in range(D * k)]
    return np.array(v + [0.0] * (D if fit_linear else 0) + [0.0] * (1 if fit_intercept else 0), np.float64)


def split(w, D, k, fit_linear, fit_intercept):
    V = w[:D * k].reshape(D, k)
    lin = w[D * k:D * k + D] if fit_linear else np.zeros(D)
    b = w[-1] if fit_intercept else 0.0
    return V, lin, b


def raw(w, X, D, k, fit_linear=True, fit_intercept=True):
    """r per row of X, Spark's getRawPrediction order"""
    V, lin, b = split(w, D, k, fit_linear, fit_intercept)
    r = np.full(X.shape[0], float(b)) + X @ lin
    for f in range(k):
        vx = X * V[:, f]
        r = r + 0.5 * (vx.sum(1) ** 2 - (vx * vx).sum(1))
    return r


def log1p_exp(v):
    return np.where(v > 0, v + np.log1p(np.exp(-np.abs(v))), np.log1p(np.exp(np.minimum(v, 0))))


def sums(w, X, y, D, k, fit_linear=True, fit_intercept=True):
    """(loss sum, gradient sum in w's layout) over the rows X with 0/1 labels y"""
    V, _, _ = split(w, D, k, fit_linear, fit_intercept)
    r = raw(w, X, D, k, fit_linear, fit_intercept)
    g = 1.0 / (1.0 + np.exp(-r)) - y
    loss = np.where(y > 0, log1p_exp(-r), log1p_exp(r)).sum()
    s = X @ V                                             # [n, k]
    gv = (X * g[:, None]).T @ s - V * ((X * X).T @ g)[:, None]
    parts = [gv.reshape(-1)]
    if fit_linear:
        parts.append(X.T @ g)
    if fit_intercept:
        parts.append([g.sum()])
    return loss, np.concatenate(parts)


def batch_mask(n, fraction, it, row_offset=0):
    """rows in iteration it's mini-batch: Philox(FMMB, key seed 42 + it, counter global row) word 0 < floor(fraction 2^32)"""
    if fraction >= 1.0:
        return np.ones(n, bool)
    thr = math.floor(fraction * 2.0 ** 32)
    return np.array([philox(42 + it, PURPOSE_FMMB, r, r >> 32)[0] < thr for r in range(row_offset, row_offset + n)], bool)


class GD:
    def __init__(self, size):
        pass

    def __call__(self, w, g, step, it, reg):
        eta = step / math.sqrt(it)
        w = w * (1.0 - eta * reg) + (-eta) * g
        n = np.sqrt(np.sum(w * w))
        return w, 0.5 * reg * n * n


class AdamW:
    b1, b2, eps = 0.9, 0.999, 1e-8

    def __init__(self, size):
        self.m, self.v = np.zeros(size), np.zeros(size)
        self.b1t = self.b2t = 1.0

    def __call__(self, w, g, step, it, reg):
        if step > 0:
            self.m = self.m * self.b1 + (1 - self.b1) * g
            self.v = self.v * self.b2 + (1 - self.b2) * (g * g)
            self.b1t *= self.b1
            self.b2t *= self.b2
            m_hat = self.m / (1 - self.b1t)
            v_hat = self.v / (1 - self.b2t)
            w = w - (step * m_hat / (np.sqrt(v_hat) + self.eps) + reg * w)
        n = np.sqrt(np.sum(w * w))
        return w, 0.5 * reg * n * n


def fit(X, y, k=8, fit_linear=True, fit_intercept=True, reg=0.0, fraction=1.0, init_std=0.01, max_iter=100, step=1.0,
        tol=1e-6, solver="adamW", seed=0, w0=None):
    """runMiniBatchSGD -> (w, loss history, updates made)"""
    X = np.asarray(X, np.float64)
    y = np.asarray(y, np.float64)
    n, D = X.shape
    w = init_coefficients(D, k, fit_linear, fit_intercept, init_std, seed) if w0 is None else np.array(w0, np.float64)
    upd = (AdamW if solver == "adamW" else GD)(w.shape[0])
    n0 = np.sqrt(np.sum(w * w))
    reg_val = 0.5 * reg * n0 * n0
    hist, prev = [], None
    for it in range(1, max_iter + 1):
        keep = batch_mask(n, fraction, it)
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
    """the PySpark FMClassifier doctest: (label 1, x = [1.0]), (label 0, x = [0.0]); factorSize 2, seed 11"""
    return np.array([[1.0], [0.0]]), np.array([1.0, 0.0])


DOCTEST = {"intercept": -7.316665276826291, "linear": [14.8232], "factors": [0.0163, -0.0051],
           "x": [-1.0, 0.5, 1.0, 2.0],
           "probability": [[0.9999999997574736, 2.425264676902229e-10], [0.47627851732981163, 0.5237214826701884],
                           [5.491554426243495e-4, 0.9994508445573757], [2.005766663870645e-10, 0.9999999997994233]]}
