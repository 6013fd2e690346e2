"""numpy restatement of b200flow/naive_bayes.py: b200flow_nb_moments' per-chunk class sums (each a sequential sum in row order
from +0.0, as np.cumsum is) and their chunk-order totals, the four fits in the loop order the module docstring states, and
b200flow_nb_raw's scores as scalar fp64 sums in feature order."""
import numpy as np

from selection_oracle import chain, chunks

MODEL_TYPES = ("multinomial", "complement", "bernoulli", "gaussian")


def _seq_rows(v):
    """v [m, W] -> [W]: the sequential sum of every column over the rows from +0.0."""
    acc = np.zeros(v.shape[1])
    for r in v:
        acc = acc + r
    return acc


def _seq(values):
    acc = 0.0
    for v in values:
        acc = acc + float(v)
    return acc


def label_ids(y, C):
    y = np.asarray(y, np.float64)
    ok = (y >= 0) & (y < C) & (y == np.floor(y))
    return np.where(ok, y, -1).astype(np.int64)


def moment_partials(x, ids, w, C, centers, row_offset):
    """[n_chunks, C, D + 1] (centers None) or [n_chunks, C + 1, D] of b200flow_nb_moments."""
    x = np.asarray(x, np.float64)
    n, D = x.shape
    w = np.ones(n) if w is None else np.asarray(w, np.float64)
    cl = chunks(n, row_offset)
    out = np.zeros((len(cl), C if centers is None else C + 1, D + 1 if centers is None else D))
    for k, (lo, hi) in enumerate(cl):
        xs, gs, ws = x[lo:hi], ids[lo:hi], w[lo:hi]
        for c in range(C):
            m = gs == c
            if centers is None:
                out[k, c, :D] = _seq_rows(ws[m][:, None] * xs[m])
                out[k, c, D] = _seq(ws[m])
            else:
                d = xs[m] - centers[c]
                out[k, c] = _seq_rows(ws[m][:, None] * (d * d))
        if centers is not None:
            m = (gs >= 0) & (gs < C)
            e = xs[m] - centers[C]
            out[k, C] = _seq_rows(ws[m][:, None] * (e * e))
    return out


class Fit:
    def __init__(self, **kw):
        self.__dict__.update(kw)


def fit(x, y, C, model_type, smoothing=1.0, w=None):
    """-> Fit with pi, theta, sigma, present and the score coefficients a, b, c0, c1 of b200flow_nb_raw."""
    x = np.asarray(x, np.float64)
    D = x.shape[1]
    ids = label_ids(y, C)
    tot = chain(moment_partials(x, ids, w, C, None, 0))
    S, Wc = tot[:, :D], tot[:, D]
    N = _seq(Wc)
    present = Wc > 0.0
    L = int(present.sum())
    lam = float(smoothing)
    col = np.array([_seq(S[:, j]) for j in range(D)])           # sum over the classes in class order
    with np.errstate(divide="ignore", invalid="ignore"):
        if model_type == "gaussian":
            pi = np.log(Wc) - np.log(N)
            theta = np.where(present[:, None], S / Wc[:, None], 0.0)
            centers = np.concatenate([theta, (col / N)[None, :]])
            q = chain(moment_partials(x, ids, w, C, centers, 0))
            eps = 1e-9 * max(q[C] / N)
            sigma = np.where(present[:, None], eps + q[:C] / Wc[:, None], 0.0)
        else:
            pi = np.log(Wc + lam) - np.log(N + L * lam)
            if model_type == "complement":
                comp = col[None, :] - S
                theta = -(np.log(comp + lam) - np.log(np.array([_seq(r) for r in comp]) + D * lam)[:, None])
            elif model_type == "bernoulli":
                theta = np.log(S + lam) - np.log(Wc + 2.0 * lam)[:, None]
            else:
                theta = np.log(S + lam) - np.log(np.array([_seq(r) for r in S]) + D * lam)[:, None]
            theta = np.where(present[:, None], theta, 0.0)
            sigma = np.zeros((0, 0))
    pi = np.where(present, pi, -np.inf)
    a, b, c0, c1 = theta, None, np.zeros(C), None
    if model_type == "gaussian":
        b, c0 = sigma, pi
        c1 = np.array([_seq(np.log(sigma[c])) if present[c] else 0.0 for c in range(C)])
    elif model_type == "bernoulli":
        with np.errstate(divide="ignore", invalid="ignore"):
            l1 = np.log1p(-np.exp(theta))
        a = theta - l1
        c0 = pi + np.array([_seq(r) for r in l1])
    return Fit(model_type=model_type, pi=pi, theta=theta, sigma=sigma, present=present, a=a, b=b, c0=c0, c1=c1)


def raw_sums(f, x):
    """[n, C]: b200flow_nb_raw's values before any normalisation (model 0 for gaussian, 1 otherwise)."""
    x = np.asarray(x, np.float64)
    n, D = x.shape
    acc = np.zeros((n, len(f.present)))
    with np.errstate(divide="ignore", invalid="ignore"):          # an absent class's zero rows; masked below
        for j in range(D):
            if f.model_type == "gaussian":
                d = x[:, j:j + 1] - f.a[None, :, j]
                acc = acc + (d * d) / f.b[None, :, j]
            else:
                acc = acc + x[:, j:j + 1] * f.a[None, :, j]
        out = f.c0 - (acc + f.c1) / 2.0 if f.model_type == "gaussian" else acc + f.c0
    return np.where(f.present[None, :], out, -np.inf)


def raw(f, x):
    """rawPrediction: raw_sums, and for complement z - logsumexp(z) over the present classes."""
    if f.model_type == "multinomial":
        return np.asarray(x, np.float64) @ f.theta.T + f.pi
    z = raw_sums(f, x)
    if f.model_type != "complement":
        return z
    zp = z[:, f.present]
    m = zp.max(1, keepdims=True)
    lse = m + np.log(np.exp(zp - m).sum(1, keepdims=True))
    return np.where(f.present[None, :], z - lse, -np.inf)


def probability(r):
    e = np.exp(r - r.max(1, keepdims=True))
    return e / e.sum(1, keepdims=True)
