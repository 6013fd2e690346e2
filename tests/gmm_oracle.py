"""numpy fp64 restatement of GaussianMixture (DESIGN.md §5g): the GMMS sample and initRandom, the density constants from
numpy's eigh, the log-space E-step with q summed in feature order, the raw-moment sums, Spark's M-step and the EM loop.
Written from the formulas, independently of csrc/gmm.cu and b200flow/gmm.py."""
import math

import numpy as np

PURPOSE_GMMS = 0x474D4D53
EPSILON = 2.220446049250313e-16
_M32 = 0xFFFFFFFF


def philox(seed, purpose, c0, c1=0, c2=0, c3=0):
    k0, k1 = (int(seed) & _M32) ^ purpose, (int(seed) >> 32) & _M32
    c = [c0 & _M32, c1 & _M32, c2 & _M32, c3 & _M32]
    for _ in range(10):
        p0, p1 = 0xD2511F53 * c[0], 0xCD9E8D57 * c[2]
        c = [(p1 >> 32) ^ c[1] ^ k0, p1 & _M32, (p0 >> 32) ^ c[3] ^ k1, p0 & _M32]
        k0, k1 = (k0 + 0x9E3779B9) & _M32, (k1 + 0xBB67AE85) & _M32
    return c


def sample_rows(seed, k, N):
    out = []
    for j in range(5 * k):
        w = philox(seed, PURPOSE_GMMS, j, j >> 32)
        u = float((w[0] << 21) | (w[1] >> 11)) * 2.0 ** -53
        out.append(min(math.floor(u * N), N - 1))
    return np.array(out)


def init(x, k, seed):
    """(weights, means, covariances) of initRandom with numSamples = 5."""
    s = x[sample_rows(seed, k, x.shape[0])]
    D = x.shape[1]
    means, covs = np.zeros((k, D)), np.zeros((k, D, D))
    for i in range(k):
        m = np.zeros(D)
        for r in s[5 * i:5 * i + 5]:
            m = m + r
        m = m * (1.0 / 5)
        ss = np.zeros(D)
        for r in s[5 * i:5 * i + 5]:
            ss = ss + (r - m) * (r - m)
        means[i] = m
        covs[i] = np.diag(ss * (1.0 / 5))
    return np.full(k, 1.0 / k), means, covs


def constants(cov):
    """(root R [D, D], u) of one covariance."""
    D = cov.shape[0]
    d, U = np.linalg.eigh(cov)
    keep = d > EPSILON * d.max() * D if d.max() > 0 else np.zeros(D, bool)
    R = np.zeros((D, D))
    for o in np.nonzero(keep)[0]:
        R[o] = math.sqrt(1.0 / d[o]) * U[:, o]
    logdet = 0.0
    for v in d[keep]:
        logdet = logdet + math.log(v)
    return R, -0.5 * (D * math.log(2.0 * math.pi) + logdet)


def q_form(x, mean, R):
    """||R (x - mean)||^2 per row, the squares added in feature order from +0.0."""
    y = (x - mean) @ R.T
    q = np.zeros(x.shape[0])
    for j in range(y.shape[1]):
        q = q + y[:, j] * y[:, j]
    return q


def logpdf(x, mean, cov):
    R, u = constants(cov)
    return u - 0.5 * q_form(x, mean, R)


def estep(x, weights, means, covs):
    """(responsibilities [n, k], lse [n]) in log space."""
    k = weights.shape[0]
    s = np.empty((x.shape[0], k))
    for i in range(k):
        R, u = constants(covs[i])
        s[:, i] = (math.log(weights[i]) + u) - 0.5 * q_form(x, means[i], R)
    t = np.logaddexp(math.log(EPSILON), s)
    m = t.max(1)
    lse = m + np.log(np.exp(t - m[:, None]).sum(1))
    return np.exp(t - lse[:, None]), lse


def em_step(x, weights, means, covs):
    """(LL, weights, means, covariances): the sums with the given parameters and Spark's update."""
    r, lse = estep(x, weights, means, covs)
    k, D = weights.shape[0], x.shape[1]
    W = r.sum(0)
    S = r.T @ x
    nw, nm, nc = np.empty(k), np.empty((k, D)), np.empty((k, D, D))
    sw = 0.0
    for v in W:
        sw = sw + v
    for i in range(k):
        Q = (x * r[:, i:i + 1]).T @ x
        m = S[i] * (1.0 / W[i])
        nm[i] = m
        nc[i] = (Q + m[:, None] * ((-W[i]) * m[None, :])) * (1.0 / W[i])
        nc[i] = np.triu(nc[i]) + np.triu(nc[i], 1).T
        nw[i] = W[i] / sw
    return float(lse.sum()), nw, nm, nc


def fit(x, k, max_iter=100, tol=0.01, seed=0):
    """(weights, means, covariances, logLikelihood, numIter)."""
    w, m, c = init(x, k, seed)
    ll, prev, it = -1.7976931348623157e308, 0.0, 0
    while it < max_iter and abs(ll - prev) > tol:
        L, w, m, c = em_step(x, w, m, c)
        prev, ll = ll, L
        it += 1
    return w, m, c, ll, it


def predict(x, weights, means, covs):
    r, _ = estep(x, weights, means, covs)
    return r, r.argmax(1).astype(np.int32)
