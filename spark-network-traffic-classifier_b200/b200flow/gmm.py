"""GaussianMixture (full covariance, EM) on the device (DESIGN.md §5g): the E-step and the responsibility-weighted moments
from csrc/gmm.cu's fp64 tensor-core kernels, summed in the chunk order of dist.Shards; the eigendecompositions, the
parameter updates and the stop test on the host from the chained totals.

Spark [recalled; Spark 3 `ml/clustering/GaussianMixture.scala`, `ml/stat/distribution/MultivariateGaussian.scala`]:

    initRandom, numSamples = 5: takeSample(withReplacement = true, 5k rows); component i takes samples [5i, 5i + 5): its
    mean is their sum in sample order times 1.0/5, its covariance the diagonal of the sum of (x - mean)^2 times 1.0/5, its
    weight 1.0/k.  Here sample j is global row min(floor(u N), N - 1), u the 53-bit uniform of Philox(seed, 'GMMS',
    (j_lo, j_hi, 0, 0)) (DESIGN §5), not XORShiftRandom.
    calculateCovarianceConstants: Sigma = U diag(d) U^T (eigSym), tol = EPSILON max(d) D with EPSILON = 2^-52 (MLUtils);
    root R = diag(1/sqrt(d)) U^T with zero rows where d <= tol; u = -0.5 (D log(2 pi) + sum of log d over the kept d)
    (D, not the rank); logpdf(x) = u - 0.5 ||R (x - mu)||^2.
    ExpectationAggregator: p_i = EPSILON + w_i pdf_i(x), LL += log(sum p), r_i = p_i / sum p; the sums W_i = sum r_i,
    S_i = sum r_i x and Q_i = sum r_i x x^T (raw moments, packed upper).
    updateWeightsAndGaussians: mu = S (1/W); Sigma = Q then BLAS.spr(-W, mu, .) then scal(1/W); w = W / sum W.
    Loop: ll = Double.MinValue, llPrev = 0.0; while iter < maxIter and |ll - llPrev| > tol: sums with the current
    parameters, update, llPrev = ll, ll = LL, iter += 1.

Deviations: the E-step is computed in log space, t_i = logaddexp(log EPSILON, log w_i + logpdf_i), r_i = exp(t_i - lse(t)),
LL += lse(t) (equal in exact arithmetic; Spark's exp(logpdf) can overflow to inf / NaN, this cannot); the eigendecomposition
is numpy's eigh on rank 0 (broadcast), not Breeze's; a non-finite updated parameter raises ValueError instead of being
carried into the next iteration; D <= 256 and k <= 64.

Every chunk's partial row [LL, then per component W, S, Q] depends only on the chunk's rows; the partials are added in
chunk order and passed rank to rank (dist.chunk_tail / chunk_chain).  So the model is the same bits for any world size.
"""
import math

import numpy as np
import torch

from . import _lib
from . import dist as bdist
from .kmeans import philox, uniform
from ._lib import call, ptr

PURPOSE_GMMS = 0x474D4D53
EPSILON = 2.220446049250313e-16
DOUBLE_MIN = -1.7976931348623157e308
NUM_SAMPLES = 5
MAX_D, MAX_K = 256, 64
# device memory for one batch of chunks: their partial rows and responsibilities.  At k = 23, D = 119 a partial row is
# 1.3 MB, so the 897 chunks of 3.67 M rows are summed in batches rather than held at once.
PARTIALS_BUDGET = 256 << 20


def width(k, D):
    """length of a partial row: LL, then per component W, S [D], Q packed upper [D(D+1)/2]."""
    return 1 + k * (1 + D + D * (D + 1) // 2)


def sample_rows(seed, k, N):
    """the 5k global rows of initRandom's sample with replacement (GMMS draws)."""
    out = []
    for j in range(NUM_SAMPLES * k):
        w = philox(seed, PURPOSE_GMMS, j, j >> 32)
        out.append(min(int(math.floor(uniform(w[0], w[1]) * N)), N - 1))
    return out


def init_params(samples, k):
    """(weights [k], means [k, D], covariances [k, D, D]) of initRandom from the sampled rows [5k, D] (host f64)."""
    D = samples.shape[1]
    means, covs = np.empty((k, D)), np.zeros((k, D, D))
    for i in range(k):
        sl = samples[NUM_SAMPLES * i:NUM_SAMPLES * (i + 1)]
        acc = np.zeros(D)
        for r in sl:
            acc = acc + r
        mean = acc * (1.0 / NUM_SAMPLES)
        ss = np.zeros(D)
        for r in sl:
            d = r - mean
            ss = ss + d * d
        means[i] = mean
        covs[i][np.arange(D), np.arange(D)] = ss * (1.0 / NUM_SAMPLES)
    return np.full(k, 1.0 / k), means, covs


def density_constants(covs):
    """(roots [k, D, D], u [k]) of calculateCovarianceConstants for covariances [k, D, D] (host f64)."""
    k, D = covs.shape[0], covs.shape[1]
    roots, u = np.zeros((k, D, D)), np.empty(k)
    for i in range(k):
        d, U = np.linalg.eigh(covs[i])
        mx = float(d.max())
        keep = d > (EPSILON * mx) * D if mx > 0 else np.zeros(D, bool)
        logdet = 0.0
        for v in d[keep]:
            logdet = logdet + math.log(v)
        roots[i][keep] = np.sqrt(1.0 / d[keep])[:, None] * U[:, keep].T
        u[i] = -0.5 * (D * math.log(2.0 * math.pi) + logdet)
    return roots, u


def m_step(tot, k, D):
    """(weights, means, covariances) from the chained totals [width(k, D)]; ValueError naming a component whose updated
    parameters are not finite."""
    per = 1 + D + D * (D + 1) // 2
    iu = np.triu_indices(D)
    pos = iu[0] + iu[1] * (iu[1] + 1) // 2              # (a, b), a <= b, in packed-upper order
    Ws = [np.float64(tot[1 + i * per]) for i in range(k)]
    sw = np.float64(0.0)
    for v in Ws:
        sw = sw + v
    weights, means, covs = np.empty(k), np.empty((k, D)), np.empty((k, D, D))
    for i in range(k):
        b = 1 + i * per
        W = Ws[i]
        with np.errstate(all="ignore"):             # a vanished component is reported below
            mean = tot[b + 1:b + 1 + D] * (1.0 / W)
            Q = tot[b + 1 + D:b + per][pos]
            up = (Q + mean[iu[0]] * ((-W) * mean[iu[1]])) * (1.0 / W)
            weights[i] = W / sw
        cov = np.empty((D, D))
        cov[iu] = up
        cov[iu[1], iu[0]] = up
        means[i], covs[i] = mean, cov
        if not (math.isfinite(weights[i]) and np.isfinite(mean).all() and np.isfinite(cov).all()):
            raise ValueError("GaussianMixture: component %d has non-finite parameters after an EM step (weight sum %r); "
                             "its responsibilities vanished or the data overflow" % (i, float(W)))
    return weights, means, covs


def check_shape(D, k):
    if int(k) != k or int(k) < 2:
        raise ValueError("k must be an integer > 1, got %r" % (k,))
    if int(k) > MAX_K:
        raise _lib.UnsupportedParamError("GaussianMixture supports k <= %d, got %d" % (MAX_K, k))
    if not 1 <= D <= MAX_D:
        raise _lib.UnsupportedParamError("GaussianMixture supports 1 to %d features, got %d" % (MAX_D, D))
    return int(k)


def _check_x(x):
    if not (torch.is_tensor(x) and x.is_cuda and x.dim() == 2 and x.dtype == torch.float64):
        raise _lib.B200FlowError("GaussianMixture needs a CUDA float64 [n, D] matrix")
    return x.contiguous()


def estep(x, means, roots, log_consts, row_offset=0, resp=None, pred=None, partials=None):
    """b200flow_gmm_estep on the rows x [n, D]: means, roots, log_consts device f64."""
    n, D = x.shape
    call("b200flow_gmm_estep", ptr(x), n, D, D, means.shape[0], ptr(means), ptr(roots), ptr(log_consts), row_offset,
         ptr(resp), ptr(pred), ptr(partials))


def moments(x, resp, row_offset, partials):
    n, D = x.shape
    call("b200flow_gmm_moments", ptr(x), n, D, D, resp.shape[1], ptr(resp), row_offset, ptr(partials))


def em_sums(x, means, roots, log_consts, sh):
    """[width(k, D)] f64 device: LL and the sums W, S, Q over every rank's rows in chunk order; the same bits on every rank.
    The chunks are computed in batches of at most PARTIALS_BUDGET bytes of partials and responsibilities."""
    D, k = x.shape[1], means.shape[0]
    P = width(k, D)
    lead, off = sh.lead[sh.rank], sh.offs[sh.rank]
    t0, tail_x, _ = bdist.chunk_tail(x, None, sh)
    nb = max(1, PARTIALS_BUDGET // (8 * (P + bdist.CHUNK * k)))
    pieces = [(x[s:min(s + nb * bdist.CHUNK, t0)], off + s) for s in range(lead, t0, nb * bdist.CHUNK)]
    if tail_x.shape[0]:
        pieces.append((tail_x.contiguous(), off + t0))

    def run(xs, go):
        nc = (xs.shape[0] + bdist.CHUNK - 1) // bdist.CHUNK
        parts = torch.empty((nc, P), dtype=torch.float64, device=x.device)
        resp = torch.empty((xs.shape[0], k), dtype=torch.float64, device=x.device)
        estep(xs, means, roots, log_consts, go, resp=resp, partials=parts)
        moments(xs, resp, go, parts)
        return parts, nc

    if not pieces:
        return bdist.chunk_chain(torch.empty((1, P), dtype=torch.float64, device=x.device), 0, 1, P, sh).reshape(-1)
    first, nc = run(*pieces[0])
    return bdist.chunk_chain(first, nc, 1, P, sh, more=(run(*p) for p in pieces[1:])).reshape(-1)


def _constants(covs, weights, sh, device):
    """(roots [k, D, D] device, log w + u [k] device): the eigendecompositions on rank 0, broadcast to the others."""
    k, D = covs.shape[0], covs.shape[1]
    buf = torch.empty(k * D * D + k, dtype=torch.float64, device=device)
    if sh.rank == 0:
        roots, u = density_constants(covs)
        buf.copy_(torch.from_numpy(np.concatenate([roots.ravel(), u])))
    if sh.grp is not None:
        bdist.broadcast_(buf, 0, sh.grp)
    u = buf[k * D * D:].cpu().numpy()
    c = np.array([math.log(w) + v for w, v in zip(weights, u)])
    return buf[:k * D * D].reshape(k, D, D).contiguous(), torch.from_numpy(c).to(device), u


def _sample(x, seed, k, sh):
    """the sampled rows [5k, D] as a host array, each fetched from the rank that holds it."""
    idx = np.array(sample_rows(seed, k, sh.total), dtype=np.int64)
    if sh.grp is None:
        return x[torch.from_numpy(idx).to(x.device)].cpu().numpy()
    off, n = sh.offs[sh.rank], x.shape[0]
    have = (idx >= off) & (idx < off + n)
    buf = torch.zeros((idx.shape[0], x.shape[1]), dtype=torch.float64, device=x.device)
    if have.any():
        buf[torch.from_numpy(np.nonzero(have)[0]).to(x.device)] = x[torch.from_numpy(idx[have] - off).to(x.device)]
    parts = bdist.all_gather_list(buf, sh.grp)
    flags = bdist.all_gather_list(torch.from_numpy(have.astype(np.int64)).to(x.device), sh.grp)
    out = np.zeros((idx.shape[0], x.shape[1]))
    for p, f in zip(parts, flags):
        m = f.cpu().numpy().astype(bool)
        out[m] = p.cpu().numpy()[m]
    return out


class GMMFit:
    """weights [k], means [k, D], covariances [k, D, D] (host f64); roots (device) and log_consts (device, log w + u) of
    the final parameters; log_likelihood and num_iter; cluster_sizes and the local rows' prob / pred under the final model."""

    def __init__(self, weights, means, covariances, roots, log_consts, log_likelihood, num_iter):
        self.weights, self.means, self.covariances = weights, means, covariances
        self.roots, self.log_consts = roots, log_consts
        self.log_likelihood, self.num_iter = log_likelihood, num_iter
        self.cluster_sizes = self.prob = self.pred = None


def gmm_fit(x, k, max_iter=100, tol=0.01, seed=0, row_offset=None, group=None):
    """GaussianMixture.fit on this rank's rows x [n, D] f64 (row_offset = its first global row, default from
    dist.global_offset).  An empty shard still joins every collective.  -> GMMFit."""
    x = _check_x(x)
    D = x.shape[1]
    k = check_shape(D, k)
    max_iter = int(max_iter)
    if max_iter < 0 or not tol >= 0:
        raise ValueError("maxIter must be >= 0 and tol >= 0")
    grp = group if group is not None else bdist.group()
    dev = x.device
    if row_offset is None:
        row_offset, _ = bdist.global_offset(x.shape[0], dev, grp)
    sh = bdist.Shards(x.shape[0], row_offset, grp, dev)
    bad = (~torch.isfinite(x)).any().to(torch.int64).reshape(1)
    if grp is not None:
        bdist.all_reduce_(bad, grp)
    if sh.total == 0 or int(bad.item()):
        raise ValueError("GaussianMixture needs at least one row and finite features")
    weights, means, covs = init_params(_sample(x, seed, k, sh), k)
    ll, ll_prev, it = DOUBLE_MIN, 0.0, 0
    while it < max_iter and abs(ll - ll_prev) > tol:
        roots, c, _ = _constants(covs, weights, sh, dev)
        tot = em_sums(x, torch.from_numpy(means).to(dev), roots, c, sh).cpu().numpy()
        weights, means, covs = m_step(tot, k, D)
        ll_prev, ll = ll, float(tot[0])
        it += 1
    roots, c, _ = _constants(covs, weights, sh, dev)
    fit = GMMFit(weights, means, covs, roots, c, ll, it)
    fit.prob, fit.pred = gmm_predict(x, fit)
    sizes = torch.bincount(fit.pred.to(torch.int64), minlength=k)
    if grp is not None:
        bdist.all_reduce_(sizes, grp)
    fit.cluster_sizes = sizes.cpu().numpy()
    return fit


def gmm_predict(x, fit):
    """(probability f64 [n, k], prediction int32 [n]) of the rows x [n, D] f64 under a GMMFit; non-finite features raise."""
    x = _check_x(x)
    n, D = x.shape
    k = fit.means.shape[0]
    if D != fit.means.shape[1]:
        raise ValueError("the model has %d features, the rows have %d" % (fit.means.shape[1], D))
    if n and not bool(torch.isfinite(x).all().item()):
        raise ValueError("GaussianMixture needs finite features")
    prob = torch.empty((n, k), dtype=torch.float64, device=x.device)
    pred = torch.empty(n, dtype=torch.int32, device=x.device)
    mu = torch.from_numpy(fit.means).to(x.device)
    estep(x, mu, fit.roots.to(x.device), fit.log_consts.to(x.device), 0, resp=prob, pred=pred)
    return prob, pred
