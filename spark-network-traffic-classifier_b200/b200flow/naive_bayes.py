"""NaiveBayes on the device (DESIGN.md §5u): the class statistics from csrc/naive_bayes.cu's b200flow_nb_moments, summed in
the chunk order of dist.Shards, the model on the host from totals that are the same bits on every rank, and the scores
from b200flow_nb_raw, one fixed-order sum per (row, class).

Spark [recalled; Spark 3 `ml/classification/NaiveBayes.scala`]:  w is the row weight (1.0 without weightCol),
W_c = sum w over the rows of class c, N = sum_c W_c, S_cj = sum w x_j over the rows of class c, lambda = smoothing, D features,
C classes; a class is present iff W_c > 0, and L is the number of present classes.  An absent class gets pi = -inf and
raw = -inf (never predicted, probability 0) and zero theta and sigma rows.
    multinomial: pi_c = log(W_c + lambda) - log(N + L lambda), theta_cj = log(S_cj + lambda) - log(sum_j S_cj + D lambda),
        raw = pi + theta x; features >= 0.
    complement: pi as multinomial; comp_cj = (sum_c' S_c'j) - S_cj (classes in order), theta_cj = -(log(comp_cj + lambda)
        - log(sum_j comp_cj + D lambda)); raw = z - logsumexp(z) over the present classes, z_c = sum_j x_j theta_cj (pi is
        not used); features >= 0.
    bernoulli: pi as multinomial; theta_cj = log(S_cj + lambda) - log(W_c + 2 lambda); raw_c = sum_j x_j (theta_cj -
        log1p(-exp theta_cj)) + (pi_c + sum_j log1p(-exp theta_cj)); features exactly 0 or 1, at fit and at transform.
    gaussian: smoothing is ignored; pi_c = log(W_c) - log(N), theta_cj = S_cj / W_c, sigma_cj = eps + Q_cj / W_c with
        Q_cj = sum w (x_j - theta_cj)^2 over class c, eps = 1e-9 max_j (G_j / N), G_j = sum w (x_j - mu_j)^2 over every row,
        mu_j = (sum_c S_cj) / N; raw_c = pi_c - (sum_j d d / sigma_cj + sum_j log sigma_cj) / 2, d = x_j - theta_cj (the 2 pi
        constant left out).
    probability = softmax(raw), prediction = argmax(raw).

Order of the arithmetic (what makes the result the same bits for any world size): every sum over rows is a chunk-order
total of b200flow_nb_moments' partials; on the host every sum over classes or features runs sequentially in index order from
+0.0 (N, L lambda, sum_j S_cj, sum_c S_cj, the bernoulli bias, logVarSum, max_j), and the rest is elementwise numpy.

Deviations: the gaussian variances are two-pass centred sums, not Spark's sum w x^2 / W - m^2 (the same in exact
arithmetic; a feature near 1e9 keeps a small variance); non-finite features, and weights that are negative or not finite,
are refused at fit; a gaussian fit on features that are all constant (eps = 0, sigma = 0) raises instead of producing a NaN
model; a fit with a total weight of 0 raises; D <= 256 and C <= 256.
"""
import numpy as np
import torch

from . import _lib
from . import dist as bdist
from . import selection as bsel
from ._lib import call, ptr

MAX_D = 256
MAX_C = 256
MODEL_TYPES = ("multinomial", "complement", "bernoulli", "gaussian")
_RAW_GAUSSIAN, _RAW_LINEAR, _RAW_NORMALISED = 0, 1, 2


class NBFit:
    """pi [C], theta [C, D], sigma [C, D] (gaussian) or [0, 0], present bool [C] (device f64 / bool), and the score
    coefficients of b200flow_nb_raw (device)."""
    __slots__ = ("model_type", "pi", "theta", "sigma", "present", "_a", "_b", "_c0", "_c1", "_present_u8")

    def __init__(self, model_type, pi, theta, sigma, present, a, b, c0, c1):
        self.model_type, self.pi, self.theta, self.sigma, self.present = model_type, pi, theta, sigma, present
        self._a, self._b, self._c0, self._c1 = a, b, c0, c1
        self._present_u8 = present.to(torch.uint8)


def _check_x(x, what):
    if not (torch.is_tensor(x) and x.is_cuda and x.dim() == 2 and x.dtype in (torch.float32, torch.float64)):
        raise _lib.B200FlowError("%s needs a CUDA float32 or float64 [n, D] matrix" % what)
    if not 1 <= x.shape[1] <= MAX_D:
        raise _lib.UnsupportedParamError("%s supports 1 to %d features, got %d" % (what, MAX_D, x.shape[1]))
    return x if x.shape[1] == 1 or x.stride(1) == 1 else x.contiguous()


def _rows(x):
    """(pointer, dtype code, ld) of a row-major matrix whose rows may be strided."""
    if not x.is_cuda:
        raise _lib.B200FlowError("b200flow kernels need CUDA tensors (got %s); there is no CPU fallback" % x.device)
    return x.data_ptr(), _lib.dtype_code(x), max(int(x.stride(0)), x.shape[1]) if x.shape[0] > 1 else x.shape[1]


def _seq(a, axis):
    """the sequential sum along axis from +0.0 (np.cumsum adds in index order)."""
    a = np.asarray(a, np.float64)
    if a.shape[axis] == 0:
        return np.zeros(np.delete(a.shape, axis))
    return np.take(np.cumsum(a, axis=axis), -1, axis=axis)


def _moments_total(x, ids, w, C, centers, sh, bad):
    """[C, D + 1] (centers None) or [C + 1, D] f64 device: b200flow_nb_moments' chunk-order totals over every rank's rows."""
    D = x.shape[1]
    G, width = (C, D + 1) if centers is None else (C + 1, D)

    def launch(xs, i_s, ws, go, parts):
        p, code, ld = _rows(xs)
        call("b200flow_nb_moments", p, code, xs.shape[0], D, ld, ptr(i_s), ptr(ws), C, ptr(centers), go, ptr(parts), ptr(bad))

    return bsel.chunk_total(x, ids, w, sh, G, width, launch)


def nb_fit(x, y, num_classes, model_type="multinomial", smoothing=1.0, weights=None, row_offset=None, group=None):
    """this rank's rows x [n, D] (f32 or f64), labels y [n] (class indices as floats or integers), weights [n] or None ->
    NBFit; identical for any world size.  row_offset: the rank's first global row (default from dist.global_offset);
    group: the process group the rows are sharded over (default dist.group())."""
    if model_type not in MODEL_TYPES:
        raise ValueError("NaiveBayes modelType must be one of %s, got %r" % (", ".join(MODEL_TYPES), model_type))
    x = _check_x(x, "NaiveBayes")
    n, D = x.shape
    C = int(num_classes)
    if not 1 <= C <= MAX_C:
        raise _lib.UnsupportedParamError("NaiveBayes supports 1 to %d classes, got %d" % (MAX_C, C))
    dev = x.device
    grp = group if group is not None else bdist.group()
    if row_offset is None:
        row_offset, _ = bdist.global_offset(n, dev, grp)
    sh = bdist.Shards(n, row_offset, grp, dev)
    yf = y.to(dev, torch.float64)
    ids = torch.where((yf >= 0) & (yf < C) & (yf == torch.floor(yf)), yf, torch.full_like(yf, -1.0)).to(torch.int32).contiguous()
    w = weights.to(dev, torch.float64).contiguous() if weights is not None else None
    bad = torch.zeros(5, dtype=torch.int64, device=dev)
    tot = _moments_total(x, ids, w, C, None, sh, bad).cpu().numpy()
    if grp is not None:
        bdist.all_reduce_(bad, grp)
    nonfinite, negative, not_binary, bad_w, bad_l = (int(v) for v in bad.cpu())
    if bad_l:
        raise ValueError("NaiveBayes was given %d labels that are not integers in [0, %d)" % (bad_l, C))
    if bad_w:
        raise ValueError("NaiveBayes weights must be finite and nonnegative; found %d that are not" % bad_w)
    if nonfinite:
        raise ValueError("NaiveBayes requires finite feature values but found %d that are not" % nonfinite)
    if negative and model_type in ("multinomial", "complement"):
        raise ValueError("requirement failed: Naive Bayes requires nonnegative feature values but found a negative value.")
    if not_binary and model_type == "bernoulli":
        raise ValueError("requirement failed: Bernoulli naive Bayes requires 0 or 1 feature values but found a value that "
                         "is neither.")
    S, Wc = tot[:, :D], tot[:, D]
    N = float(_seq(Wc, 0))
    if not N > 0.0:
        raise ValueError("NaiveBayes needs a positive total weight, got %r" % N)
    present = Wc > 0.0
    L = int(present.sum())
    lam = float(smoothing)
    with np.errstate(divide="ignore", invalid="ignore"):
        if model_type == "gaussian":
            pi = np.log(Wc) - np.log(N)
            theta = S / Wc[:, None]
            theta[~present] = 0.0
            mu = _seq(S, 0) / N
            centers = torch.from_numpy(np.concatenate([theta, mu[None, :]])).to(dev)
            q = _moments_total(x, ids, w, C, centers, sh, None).cpu().numpy()
            eps = 1e-9 * np.max(q[C] / N)
            if not eps > 0.0:
                raise ValueError("requirement failed: gaussian NaiveBayes needs a feature that is not constant over the "
                                 "training rows (every variance is 0).")
            sigma = eps + q[:C] / Wc[:, None]
            sigma[~present] = 0.0
        else:
            pi = np.log(Wc + lam) - np.log(N + L * lam)
            if model_type == "complement":
                comp = _seq(S, 0)[None, :] - S
                theta = -(np.log(comp + lam) - np.log(_seq(comp, 1) + D * lam)[:, None])
            elif model_type == "bernoulli":
                theta = np.log(S + lam) - np.log(Wc + 2.0 * lam)[:, None]
            else:
                theta = np.log(S + lam) - np.log(_seq(S, 1) + D * lam)[:, None]
            theta[~present] = 0.0
            sigma = np.zeros((0, 0))
    pi[~present] = -np.inf
    a, b, c0, c1 = theta, None, np.zeros(C), None
    if model_type == "gaussian":
        b, c0, c1 = sigma, pi, _seq(np.log(np.where(present[:, None], sigma, 1.0)), 1)
    elif model_type == "bernoulli":
        with np.errstate(divide="ignore", invalid="ignore"):
            l1 = np.log1p(-np.exp(theta))
            a, c0 = theta - l1, pi + _seq(l1, 1)
    put = lambda v: None if v is None else torch.from_numpy(np.ascontiguousarray(v, np.float64)).to(dev)   # noqa: E731
    return NBFit(model_type, put(pi), put(theta), put(sigma), torch.from_numpy(present).to(dev), put(a), put(b), put(c0), put(c1))


def nb_raw(fit, x):
    """rawPrediction [n, C] f64 of the rows x [n, D] (f32 or f64) under a complement, bernoulli or gaussian fit (a
    multinomial fit scores with b200flow.linear.nb_raw).  A bernoulli fit raises on a value that is not 0 or 1."""
    if fit.model_type not in ("complement", "bernoulli", "gaussian"):
        raise ValueError("nb_raw scores complement, bernoulli and gaussian fits, got %r" % (fit.model_type,))
    x = _check_x(x, "NaiveBayesModel")
    n, D = x.shape
    C = fit.present.shape[0]
    if D != fit.theta.shape[1]:
        raise ValueError("NaiveBayesModel was fit on %d features, got %d" % (fit.theta.shape[1], D))
    raw = torch.empty((n, C), dtype=torch.float64, device=x.device)
    if n == 0:
        return raw
    bad = torch.zeros(1, dtype=torch.int64, device=x.device) if fit.model_type == "bernoulli" else None
    model = {"gaussian": _RAW_GAUSSIAN, "bernoulli": _RAW_LINEAR, "complement": _RAW_NORMALISED}[fit.model_type]
    p, code, ld = _rows(x)
    call("b200flow_nb_raw", p, code, n, D, ld, model, ptr(fit._a), ptr(fit._b), ptr(fit._c0), ptr(fit._c1),
         ptr(fit._present_u8), C, ptr(raw), ptr(bad))
    if bad is not None and int(bad.item()):
        raise ValueError("requirement failed: Bernoulli naive Bayes requires 0 or 1 feature values but found a value that "
                         "is neither.")
    return raw
