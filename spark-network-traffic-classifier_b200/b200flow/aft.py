"""AFTSurvivalRegression on the device (DESIGN.md §5q): the Weibull accelerated-failure-time model, fitted by L-BFGS on
the per-row loss and gradient of csrc/linreg.cu's AFT instantiation, summed in the chunk order of dist.Shards, so that
every fit is the same bits for any world size and shard layout.

Spark [recalled; Spark 3 `ml/regression/AFTSurvivalRegression.scala`, `ml/optim/aggregator/AFTAggregator.scala`]:

    Params: censorCol "censor", quantileProbabilities [0.01, 0.05, 0.1, 0.25, 0.5, 0.75, 0.9, 0.95, 0.99] (non-empty, each
    strictly inside (0, 1)), quantilesCol unset, fitIntercept true, maxIter 100 (>= 0), tol 1e-6 (>= 0), aggregationDepth 2
    (>= 2), maxBlockSizeInMB 0.0 (>= 0).  The label is a positive lifetime t; the censor is 1.0 when the event was observed
    and 0.0 when the row is censored (any other value raises).

    Features are standardised by the summariser's unbiased std: inv_j = 1 / std_j, 0 where std_j = 0.  With fitIntercept
    xs = (x - mean) inv (Spark applies the same centring through its scaledMean offset; equal up to rounding), without it
    xs = x inv and the intercept's gradient is 0.  The variables v = [beta (D), b, log sigma] start from 0.  Per row, with
    y = log t and delta the censor,
        z = (y - xs . beta - b) / sigma,   loss = delta log sigma - delta z + e^z,
        d/dbeta_j = a xs_j, d/db = a with a = (delta - e^z) / sigma,   d/dlog sigma = delta + (delta - e^z) z,
    f and g are the sums over n (RDDLossFunction divides by the weight sum, here the row count).  Breeze L-BFGS with
    history 10 (linear.lbfgs_steps), no regularisation.

    Model: coefficients_j = beta_j inv_j, intercept = b - coefficients . mean (b alone without an intercept), scale =
    exp(log sigma).  predict(x) = exp(x . coefficients + intercept); predictQuantiles(x) = lambda exp(log(-log1p(-p)) scale)
    for each p of quantileProbabilities, lambda = predict(x).

Deviations: a trial point whose loss or gradient total is not finite (e^z overflows at a small sigma) gets f = +inf and a
zero gradient without a further pass, so the line search backtracks from it; Spark would hand the non-finite value to
Breeze.  More than 255 features, non-finite features, and an empty dataset raise ValueError (the shim's
IllegalArgumentException).  The optimiser state lives on the device, so every rank takes the same steps (as linreg.py).
"""
import math

import torch

from . import _lib
from . import dist as bdist
from . import selection
from .linear import lbfgs_steps
from ._lib import call, ptr

MAX_D = 255
HISTORY = 10
QUANTILES = (0.01, 0.05, 0.1, 0.25, 0.5, 0.75, 0.9, 0.95, 0.99)


class AFTParams:
    __slots__ = ("max_iter", "tol", "fit_intercept", "quantile_probabilities")

    def __init__(self, max_iter=100, tol=1e-6, fit_intercept=True, quantile_probabilities=QUANTILES):
        self.max_iter, self.tol, self.fit_intercept = int(max_iter), float(tol), bool(fit_intercept)
        self.quantile_probabilities = [float(p) for p in quantile_probabilities]


def check_quantiles(probs):
    """Spark's quantileProbabilities validator; raises ValueError"""
    probs = list(probs)
    if not probs or not all(0.0 < float(p) < 1.0 for p in probs):
        raise ValueError("quantileProbabilities must be a non-empty array of values in (0, 1), got %r" % (probs,))


def check_params(p):
    """Spark's validators; raises ValueError"""
    if p.max_iter < 0:
        raise ValueError("maxIter must be >= 0, got %r" % p.max_iter)
    if not p.tol >= 0.0:
        raise ValueError("tol must be >= 0, got %r" % p.tol)
    check_quantiles(p.quantile_probabilities)


class AFTFit:
    """coef f64 [D] (host), intercept, scale, objective history and iterations"""
    __slots__ = ("coef", "intercept", "scale", "objective_history", "iterations")

    def __init__(self, coef, intercept, scale, hist, it):
        self.coef, self.intercept, self.scale = coef, float(intercept), float(scale)
        self.objective_history, self.iterations = list(hist), int(it)


def _check_x(x):
    if not (torch.is_tensor(x) and x.is_cuda and x.dim() == 2 and x.dtype in (torch.float32, torch.float64)):
        raise _lib.B200FlowError("AFTSurvivalRegression needs a CUDA float32 or float64 [n, D] matrix")
    if not 1 <= x.shape[1] <= MAX_D:
        raise _lib.UnsupportedParamError("AFTSurvivalRegression supports 1 to %d features, got %d" % (MAX_D, x.shape[1]))
    return x.contiguous()


# ----------------------------------------------------------------------------------- the per-row pass
def loss_grad(x, log_t, censor, shift, inv, w, b_sigma, row_offset, partials):
    """b200flow_aft_loss_grad on the rows x [n, D] (f32/f64): partials [n_chunks, D + 3] f64 device; log_t f64 [n], censor
    int32 [n] (1 observed, 0 censored), shift f64 [D] or None, inv f64 [D], w f64 [D], b_sigma f64 [3] = [b, sigma,
    log sigma], all device."""
    n, D = x.shape
    call("b200flow_aft_loss_grad", ptr(x), _lib.dtype_code(x), n, x.stride(0), D, ptr(log_t), ptr(censor), ptr(shift),
         ptr(inv), ptr(w), ptr(b_sigma), int(row_offset), ptr(partials))


def loss_grad_totals(x, log_t, censor, shift, inv, w, b_sigma, sh):
    """[D + 3] f64 device: the loss, gradient, b and log-sigma sums over every rank's rows in chunk order; the same bits on
    every rank.  The censor travels with the rows as chunk_total's int32 row ids."""
    D = x.shape[1]

    def launch(xs, cs, ys, go, parts):
        loss_grad(xs, ys, cs, shift, inv, w, b_sigma, go, parts)

    return selection.chunk_total(x, censor, log_t, sh, 1, D + 3, launch).reshape(-1)


# ----------------------------------------------------------------------------------- fitting
def _prepare(x, label, censor, row_offset, group):
    x = _check_x(x)
    n_local = x.shape[0]
    grp = group if group is not None else bdist.group()
    dev = x.device
    if row_offset is None:
        row_offset, _ = bdist.global_offset(n_local, dev, grp)
    sh = bdist.Shards(n_local, row_offset, grp, dev)
    t = label.to(device=dev, dtype=torch.float64).reshape(-1).contiguous()
    c = censor.to(device=dev, dtype=torch.float64).reshape(-1).contiguous()
    one = torch.tensor(True, device=dev)
    shape_bad = one if (t.shape[0] != n_local or c.shape[0] != n_local) else ~one
    bad = torch.stack([shape_bad, (~torch.isfinite(x)).any(), (~(torch.isfinite(t) & (t > 0.0))).any() if n_local else ~one,
                       (~((c == 0.0) | (c == 1.0))).any() if n_local else ~one]).to(torch.int64)
    if grp is not None:
        bdist.all_reduce_(bad, grp)
    if int(bad[0].item()):
        raise ValueError("AFTSurvivalRegression needs one label and one censor per row (a shard has %d rows, %d labels and "
                         "%d censors)" % (n_local, t.shape[0], c.shape[0]))
    if sh.total == 0:
        raise ValueError("AFTSurvivalRegression needs at least one row")
    if int(bad[1].item()):
        raise ValueError("AFTSurvivalRegression needs finite features")
    if int(bad[2].item()):
        raise ValueError("The lifetime or label should be greater than 0 (and finite).")
    if int(bad[3].item()):
        raise ValueError("censor must be 1.0 or 0.0")
    return x, torch.log(t), c.to(torch.int32).contiguous(), sh


def aft_fit(x, label, censor, params, row_offset=None, group=None):
    """AFTSurvivalRegression.fit on this rank's rows x [n, D] (f32 or f64), lifetimes label [n] and censors [n]; an empty
    shard still joins every collective.  -> AFTFit, the same bits on every rank and for any shard layout."""
    check_params(params)
    x, log_t, cens, sh = _prepare(x, label, censor, row_offset, group)
    n, D, dev = sh.total, x.shape[1], x.device
    x64 = x if x.dtype == torch.float64 else x.to(torch.float64)
    mx = selection.group_sums_total(x64, None, 1, sh)[0] * (1.0 / n)
    # the centred moments kernel with log t as its label column; only the feature sums of squares are used
    t = selection.centered_moments_total(x64, None, 1, mx.contiguous(), log_t, 0.0, sh).reshape(-1)
    std = torch.sqrt(t[:D] / (n - 1)) if n > 1 else torch.zeros(D, dtype=torch.float64, device=dev)
    inv = torch.where(std > 0, 1.0 / torch.where(std > 0, std, torch.ones_like(std)), torch.zeros_like(std)).contiguous()
    fi = params.fit_intercept
    shift = mx.reshape(-1).contiguous() if fi else None
    zero = torch.zeros(1, dtype=torch.float64, device=dev)

    def evaluate(v):
        bs = torch.stack([v[D], torch.exp(v[D + 1]), v[D + 1]]).contiguous()
        tot = loss_grad_totals(x, log_t, cens, shift, inv, v[:D].contiguous(), bs, sh)
        if not bool(torch.isfinite(tot).all().item()):     # e^z overflowed: rejected by the line search
            return torch.tensor(math.inf, dtype=torch.float64, device=dev), torch.zeros_like(v)
        return tot[0] / n, torch.cat([tot[1:D + 1] / n, tot[D + 1:D + 2] / n if fi else zero, tot[D + 2:D + 3] / n])

    steps = lbfgs_steps(torch.zeros(D + 2, dtype=torch.float64, device=dev), params.max_iter, params.tol, HISTORY)
    point = next(steps)
    try:
        while True:
            point = steps.send(evaluate(point))
    except StopIteration as done:
        v, hist, it = done.value
    coef = v[:D] * inv
    b = v[D] - (coef * mx.reshape(-1)).sum() if fi else v[D]
    return AFTFit(coef.cpu().numpy(), float(b.item()), float(torch.exp(v[D + 1]).item()), hist, it)


# ----------------------------------------------------------------------------------- prediction
def aft_predict(x, fit):
    """[n] f64 device: exp(x . coefficients + intercept) (svc.svc_margins with one column, then exp)"""
    from .linreg import weights
    from .svc import svc_margins
    return torch.exp(svc_margins(x, weights(fit))[:, 0])


def quantile_factors(probs, scale):
    """[P] f64 host floats: exp(log(-log1p(-p)) scale), the factor of each quantile of the Weibull lifetime"""
    return [math.exp(math.log(-math.log1p(-float(p))) * scale) for p in probs]


def aft_predict_quantiles(x, fit, probs, lam=None):
    """[n, P] f64 device: lambda exp(log(-log1p(-p)) scale) for each p, lambda = aft_predict(x, fit) unless given"""
    lam = aft_predict(x, fit) if lam is None else lam
    q = torch.tensor(quantile_factors(probs, fit.scale), dtype=torch.float64, device=lam.device)
    return lam[:, None] * q[None, :]
