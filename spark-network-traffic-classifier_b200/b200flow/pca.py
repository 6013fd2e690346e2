"""PCA and Pearson correlation on the device (DESIGN.md §5h): the column sums from the grouped-sum kernel, the centred Gram
matrix and the projection from csrc/pca.cu's fp64 tensor-core kernels, summed in the chunk order of dist.Shards; the
eigendecomposition on the host from the chained totals.

Spark [recalled; Spark 3 `mllib/feature/PCA.scala`, `mllib/linalg/distributed/RowMatrix.scala`, `ml/feature/PCA.scala`,
`ml/stat/Correlation.scala`]:

    PCA.fit(k): D = vector size; require 1 <= k <= D ("source vector size D must be no less than k") and more than one row
    ("Cannot compute the covariance of a RowMatrix with <= 1 row").
    computeCovariance: mean = (sum of the rows) (1.0 / n); computeDenseVectorCovariance subtracts the mean from every row
    before BLAS.spr, Q_ab = sum (x_a - mean_a)(x_b - mean_b) for a <= b (two passes, not sum x x^T - n mean mean^T);
    C = Q (1.0 / (n - 1)), mirrored.
    computePrincipalComponentsAndExplainedVariance: (u, s) of the SVD of C; pc = the first k columns of u;
    explainedVariance = the first k of s / sum(s).  All features constant: sum(s) = 0 and the ratios are NaN.
    PCAModel.transform: y = pc^T x.  The mean is not subtracted.
    Correlation.corr(method = "pearson"): r_ab = C_ab / (sqrt(C_aa) sqrt(C_bb)); 1.0 on the diagonal; NaN (with a warning)
    wherever either variance is 0, the diagonal included.

Deviations: the mean is the chained chunk-order sum (b200flow_group_sums) times 1.0/n, not the online summariser's running
mean; the SVD of the symmetric C is numpy's eigh on rank 0 (broadcast), s = |eigenvalue|, ordered by s descending (stable
on eigh's output reversed); LAPACK's column signs are not reproducible, so each column of pc is multiplied by +-1 so that
its entry of largest magnitude is positive (the lowest index decides between equal magnitudes); non-finite features raise
ValueError; D <= 256.

Every chunk's partial (the column sums, then the packed upper Q) depends only on the chunk's rows; the partials are added
in chunk order and passed rank to rank (dist.chunk_tail / chunk_chain).  So the model is the same bits for any world size.
"""
import numpy as np
import torch

from . import _lib
from . import dist as bdist
from .kmeans import grouped_sum
from ._lib import call, ptr

MAX_D = 256
# device memory for one batch of chunks' partial rows.  At D = 256 a partial row is 263 KB, so the 897 chunks of 3.67 M rows
# (236 MB) are summed in batches rather than held at once.
PARTIALS_BUDGET = 64 << 20
# device memory for one staged [x, y] batch of the labelled Gram matrix (LinearRegression's normal equations)
STAGE_BUDGET = 256 << 20


class PCAFit:
    """pc [D, k], explained_variance [k], mean [D], cov [D, D] (host f64)."""

    def __init__(self, pc, explained_variance, mean, cov):
        self.pc, self.explained_variance, self.mean, self.cov = pc, explained_variance, mean, cov


def components(cov, k):
    """(pc [D, k], explainedVariance [k]) of a covariance matrix [D, D] (host f64): eigh, s = |d| descending, the sign
    rule, s / sum(s) with the sum over all D values in that order from +0.0."""
    d, U = np.linalg.eigh(cov)
    s, U = np.abs(d)[::-1], U[:, ::-1]
    order = np.argsort(-s, kind="stable")
    s, U = s[order], U[:, order]
    total = np.float64(0.0)
    for v in s:
        total = total + v
    pc = np.ascontiguousarray(U[:, :k])
    for j in range(k):
        if pc[np.argmax(np.abs(pc[:, j])), j] < 0:                  # argmax: the lowest index of equal magnitudes
            pc[:, j] = -pc[:, j]
    with np.errstate(invalid="ignore", divide="ignore"):            # all features constant: 0 / 0 = NaN, as in Spark
        return pc, s[:k] / total


def check_k(D, k):
    if k is None or int(k) != k or not 1 <= int(k) <= D:
        raise ValueError("source vector size %d must be no less than k = %r, and k must be an integer >= 1" % (D, k))
    return int(k)


def _check_x(x):
    if not (torch.is_tensor(x) and x.is_cuda and x.dim() == 2 and x.dtype == torch.float64):
        raise _lib.B200FlowError("PCA needs a CUDA float64 [n, D] matrix")
    if not 1 <= x.shape[1] <= MAX_D:
        raise _lib.UnsupportedParamError("PCA supports 1 to %d features, got %d" % (MAX_D, x.shape[1]))
    return x.contiguous()


def centered_gram(x, shift, row_offset, partials):
    """b200flow_centered_gram on the rows x [n, D]: shift device f64 [D] or None."""
    n, D = x.shape
    call("b200flow_centered_gram", ptr(x), n, D, D, ptr(shift), row_offset, ptr(partials))


def project(x, pc):
    """x [n, D] pc [D, k] (device f64) by b200flow_pca_project."""
    n, D = x.shape
    out = torch.empty((n, pc.shape[1]), dtype=torch.float64, device=x.device)
    call("b200flow_pca_project", ptr(x), n, D, D, ptr(pc), pc.shape[1], ptr(out))
    return out


def column_sums(x, sh):
    """[D] f64 device: the sum of every rank's rows in chunk order; the same bits on every rank."""
    return grouped_sum(x, None, 1, sh)[0].reshape(-1)


def weighted_centered_gram(x, shift, w, row_offset, partials):
    """b200flow_weighted_centered_gram on the rows x [n, D] with row weights w [n] (device f64): shift device f64 [D]."""
    n, D = x.shape
    call("b200flow_weighted_centered_gram", ptr(x), n, D, D, ptr(shift), ptr(w), row_offset, ptr(partials))


def centered_gram_total(x, mean, sh, y=None, y_mean=None, w=None):
    """[D(D+1)/2] f64 device: the packed upper triangle of sum (x - mean)(x - mean)^T over every rank's rows in chunk
    order (mean device f64 [D] or None); the same bits on every rank.  The chunks are computed in batches of at most
    PARTIALS_BUDGET bytes of partial rows.  With a label y [n] f64 (and y_mean, a float), the Gram matrix is that of the
    rows [x, y] shifted by [mean, y_mean], [(D+1)(D+2)/2]: each batch is staged as an f64 [rows, D + 1] matrix of at most
    STAGE_BUDGET bytes (x may then be f32).  With a row weight w [n] f64 as well, it is sum w (a - shift)(a - shift)^T over
    those rows (GeneralizedLinearRegression's IRLS); w travels with y."""
    if y is not None:
        return _labelled_gram_total(x, mean, y, y_mean, sh, w)
    D = x.shape[1]
    P = D * (D + 1) // 2
    lead, off = sh.lead[sh.rank], sh.offs[sh.rank]
    t0, tail_x, _ = bdist.chunk_tail(x, None, sh)
    nb = max(1, PARTIALS_BUDGET // (8 * P))
    pieces = [(x[s:min(s + nb * bdist.CHUNK, t0)], off + s) for s in range(lead, t0, nb * bdist.CHUNK)]
    if tail_x.shape[0]:
        pieces.append((tail_x.contiguous(), off + t0))

    def run(xs, go):
        nc = (xs.shape[0] + bdist.CHUNK - 1) // bdist.CHUNK
        parts = torch.empty((nc, P), dtype=torch.float64, device=x.device)
        centered_gram(xs, mean, go, parts)
        return parts, nc

    if not pieces:
        return bdist.chunk_chain(torch.empty((1, P), dtype=torch.float64, device=x.device), 0, 1, P, sh).reshape(-1)
    first, nc = run(*pieces[0])
    return bdist.chunk_chain(first, nc, 1, P, sh, more=(run(*p) for p in pieces[1:])).reshape(-1)


def stage_rows(D):
    """rows of one staged [x, y] batch of _labelled_gram_total: whole chunks within STAGE_BUDGET and PARTIALS_BUDGET"""
    P = (D + 1) * (D + 2) // 2
    nb = max(1, min(PARTIALS_BUDGET // (8 * P), STAGE_BUDGET // (8 * (D + 1) * bdist.CHUNK)))
    return nb * bdist.CHUNK


def _labelled_gram_total(x, mean, y, y_mean, sh, w=None):
    """centered_gram_total of the rows [x, y] shifted by [mean, y_mean] (weighted by w when given), staged batch by batch"""
    D = x.shape[1]
    W = D + 1
    P = W * (W + 1) // 2
    lead, off = sh.lead[sh.rank], sh.offs[sh.rank]
    t0, tail_x, _ = bdist.chunk_tail(x, None, sh)
    tail_y = bdist.chunk_tail(y.reshape(-1, 1), None, sh)[1].reshape(-1)
    tail_w = bdist.chunk_tail(w.reshape(-1, 1), None, sh)[1].reshape(-1).contiguous() if w is not None else None
    step = stage_rows(D)
    cut = lambda t, s: t[s:min(s + step, t0)] if t is not None else None          # noqa: E731
    pieces = [(x[s:min(s + step, t0)], y[s:min(s + step, t0)], cut(w, s), off + s) for s in range(lead, t0, step)]
    if tail_x.shape[0]:
        pieces.append((tail_x, tail_y, tail_w, off + t0))
    shift = torch.cat([mean.to(torch.float64).reshape(-1),
                       torch.tensor([float(y_mean)], dtype=torch.float64, device=x.device)]).contiguous()

    def run(xs, ys, ws, go):
        xy = torch.empty((xs.shape[0], W), dtype=torch.float64, device=x.device)
        xy[:, :D] = xs
        xy[:, D] = ys
        nc = (go + xs.shape[0] - 1) // bdist.CHUNK - go // bdist.CHUNK + 1
        parts = torch.empty((nc, P), dtype=torch.float64, device=x.device)
        if ws is None:
            centered_gram(xy, shift, go, parts)
        else:
            weighted_centered_gram(xy, shift, ws, go, parts)
        return parts, nc

    if not pieces:
        return bdist.chunk_chain(torch.empty((1, P), dtype=torch.float64, device=x.device), 0, 1, P, sh).reshape(-1)
    first, nc = run(*pieces[0])
    return bdist.chunk_chain(first, nc, 1, P, sh, more=(run(*p) for p in pieces[1:])).reshape(-1)


def _moments(x, row_offset, group, what):
    """(Shards, mean [D], covariance [D, D]) (host f64) of every rank's rows; an empty shard still joins every collective."""
    grp = group if group is not None else bdist.group()
    dev = x.device
    if row_offset is None:
        row_offset, _ = bdist.global_offset(x.shape[0], dev, grp)
    sh = bdist.Shards(x.shape[0], row_offset, grp, dev)
    bad = (~torch.isfinite(x)).any().to(torch.int64).reshape(1)
    if grp is not None:
        bdist.all_reduce_(bad, grp)
    if int(bad.item()):
        raise ValueError("%s needs finite features" % what)
    n, D = sh.total, x.shape[1]
    if n <= 1:
        raise ValueError("Cannot compute the covariance of a RowMatrix with <= 1 row.")
    mean = column_sums(x, sh).cpu().numpy() * (1.0 / n)
    q = centered_gram_total(x, torch.from_numpy(mean).to(dev), sh).cpu().numpy()
    iu = np.triu_indices(D)
    up = q[iu[0] + iu[1] * (iu[1] + 1) // 2] * (1.0 / (n - 1))
    cov = np.empty((D, D))
    cov[iu] = up
    cov[iu[1], iu[0]] = up
    return sh, mean, cov


def pca_fit(x, k, row_offset=None, group=None):
    """PCA.fit on this rank's rows x [n, D] f64 (row_offset = its first global row, default from dist.global_offset).
    An empty shard still joins every collective.  -> PCAFit."""
    x = _check_x(x)
    D = x.shape[1]
    k = check_k(D, k)
    sh, mean, cov = _moments(x, row_offset, group, "PCA")
    buf = torch.empty(D * k + k, dtype=torch.float64, device=x.device)
    if sh.rank == 0:                                                # rank 0's eigendecomposition, broadcast to the others
        pc, ev = components(cov, k)
        buf.copy_(torch.from_numpy(np.concatenate([pc.ravel(), ev])))
    if sh.grp is not None:
        bdist.broadcast_(buf, 0, sh.grp)
    host = buf.cpu().numpy()
    return PCAFit(host[:D * k].reshape(D, k).copy(), host[D * k:].copy(), mean, cov)


def pca_transform(x, fit):
    """[n, k] f64 device: pc^T x of the rows x [n, D] f64 under a PCAFit (the mean is not subtracted, as in Spark)."""
    x = _check_x(x)
    if x.shape[1] != fit.pc.shape[0]:
        raise ValueError("vector size %d does not match the fitted size %d" % (x.shape[1], fit.pc.shape[0]))
    return project(x, torch.from_numpy(np.ascontiguousarray(fit.pc)).to(x.device))


def correlation(cov):
    """Pearson's r [D, D] from a covariance matrix (host f64): NaN wherever either variance is 0."""
    sd = np.sqrt(np.diag(cov))
    with np.errstate(invalid="ignore", divide="ignore"):
        r = cov / (sd[:, None] * sd[None, :])
    D = cov.shape[0]
    r[np.arange(D), np.arange(D)] = 1.0
    zero = sd == 0
    r[zero, :] = np.nan
    r[:, zero] = np.nan
    return r


def pearson(x, row_offset=None, group=None):
    """the Pearson correlation matrix [D, D] (host f64) of every rank's rows x [n, D] f64, identical for any world size."""
    x = _check_x(x)
    return correlation(_moments(x, row_offset, group, "Correlation")[2])
