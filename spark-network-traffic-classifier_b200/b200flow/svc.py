"""LinearSVC and OneVsRest(LinearSVC) on the device (DESIGN.md §5j): the hinge loss and its subgradient from csrc/svc.cu's
fused fp64 tensor-core kernel, summed in the chunk order of dist.Shards, and the OWL-QN of linear.lbfgs_steps with an L1
weight of zero, one optimiser per class column, all of them advanced together.

Spark [recalled; Spark 3 `ml/classification/LinearSVC.scala`, `ml/optim/aggregator/HingeAggregator.scala`,
`HingeBlockAggregator.scala`]:

    Binary only: numClasses (label metadata, else max label + 1) must be 2.  Features are scaled by inv_j = 1 / std_j
    (the unbiased std; 0 where std_j == 0), xs = x inv, and not centred.  With y' = 2 label - 1 and m = beta . xs + b,
        f(beta, b) = (1/n) sum_i max(0, 1 - y'_i m_i) + 1/2 sum_j lambda_j beta_j^2,
    lambda_j = regParam with standardization, regParam inv_j^2 without; the intercept is not penalised, and stays 0 with
    its gradient zeroed when fitIntercept is false.  A row adds -y' [xs, 1] to the subgradient iff 1 - y' m > 0, so a row
    at margin exactly 1 adds neither loss nor gradient.  Breeze OWLQN with an L1 weight of 0, 10 corrections, from 0, at
    most maxIter iterations, the relative-decrease tol stop.  coefficients = beta inv, intercept = b.

Centring is left out as Spark leaves it out: with an intercept, centring the features only moves the intercept
(beta . (x - mu) + b = beta . x + (b - beta . mu)), so the minimising coefficients are the same.

One code path serves both estimators: the standalone LinearSVC is svc_fit_classes(positives=[1]), OneVsRest(LinearSVC) is
positives=range(K).  Each round the driver collects the pending trial point of every unfinished class, evaluates them in
ONE kernel pass over the rows and hands each class its own (f, g).  A column's partial does not depend on the other
columns of the launch (csrc/svc.cu), and the objective is assembled per class in one fixed order, so every
class takes exactly the steps of its standalone fit, and the models are the same bits for any world size.  The optimiser
state is kept on the device rather than the host: host reductions and BLAS calls pick their vector width by CPU model, so
host arithmetic can differ between machines, and ranks whose optimisers disagree would stop after different rounds.
"""
import numpy as np
import torch

from . import _lib
from . import dist as bdist
from . import selection
from .linear import lbfgs_steps
from ._lib import call, ptr

MAX_D = 255
HISTORY = 10


class SVCParams:
    __slots__ = ("max_iter", "reg_param", "tol", "fit_intercept", "standardization")

    def __init__(self, max_iter=100, reg_param=0.0, tol=1e-6, fit_intercept=True, standardization=True):
        self.max_iter, self.reg_param, self.tol = int(max_iter), float(reg_param), float(tol)
        self.fit_intercept, self.standardization = bool(fit_intercept), bool(standardization)


class SVCFit:
    __slots__ = ("coef", "intercept", "objective_history", "iterations")

    def __init__(self, coef, intercept, hist, it):
        self.coef, self.intercept, self.objective_history, self.iterations = coef, intercept, hist, it


def _check_x(x):
    if not (torch.is_tensor(x) and x.is_cuda and x.dim() == 2 and x.dtype in (torch.float32, torch.float64)):
        raise _lib.B200FlowError("LinearSVC needs a CUDA float32 or float64 [n, D] matrix")
    if not 1 <= x.shape[1] <= MAX_D:
        raise _lib.UnsupportedParamError("LinearSVC supports 1 to %d features, got %d" % (MAX_D, x.shape[1]))
    return x.contiguous()


def loss_grad(x, labels, positives, inv_std, weights, row_offset, partials):
    """b200flow_svc_loss_grad on the rows x [n, D] (f32/f64): partials [n_chunks, K, D + 2] f64 device; labels int32 [n],
    positives int32 [K], inv_std f64 [D] and weights f64 [K, D + 1], all device."""
    n, D = x.shape
    call("b200flow_svc_loss_grad", ptr(x), _lib.dtype_code(x), n, x.stride(0), D, ptr(labels), ptr(positives),
         int(positives.shape[0]), ptr(inv_std), ptr(weights), int(row_offset), ptr(partials))


def loss_grad_totals(x, labels, positives, inv_std, weights, sh):
    """[K, D + 2] f64 device: per class column, the hinge loss sum (slot 0) and subgradient sums over every rank's rows, in
    chunk order; the same bits on every rank."""
    K, D = int(positives.shape[0]), x.shape[1]

    def launch(xs, ids, _, go, parts):
        loss_grad(xs, ids, positives, inv_std, weights, go, parts)

    return selection.chunk_total(x, labels, None, sh, K, D + 2, launch)


def svc_margins(x, weights):
    """raw [n, K] f64 device: [x, 1] . weights[k] for weights [K, D + 1] f64 (original scale), one launch over K columns."""
    x = _check_x(x)
    n, D = x.shape
    w = weights.to(device=x.device, dtype=torch.float64).contiguous()
    if w.dim() != 2 or w.shape[1] != D + 1:
        raise ValueError("the model has %d features, the input %d" % (w.shape[1] - 1, D))
    K = w.shape[0]
    raw = torch.empty((max(n, 1), K), dtype=torch.float64, device=x.device)
    call("b200flow_svc_margins", ptr(x), _lib.dtype_code(x), n, x.stride(0), D, K, ptr(w), ptr(raw))
    return raw[:n]


def _objective(t, v, lam, n, D, fit_intercept):
    """(f, g) of one class from its totals t [D + 2] (device): loss / n + 1/2 sum lambda_j beta_j^2, in this order."""
    beta = v[:D]
    f = t[0] / n + 0.5 * (lam * beta * beta).sum()
    gi = t[D + 1:] / n if fit_intercept else torch.zeros(1, dtype=torch.float64, device=t.device)
    return f, torch.cat([t[1:D + 1] / n + lam * beta, gi])


def svc_fit_classes(x, labels, positives, params, row_offset=None, group=None):
    """LinearSVC fits of this rank's rows x [n, D] (f32 or f64) for each positive label: fit k treats label ==
    positives[k] as the positive class.  Labels must be integers in [0, max(2, max(positives) + 1)).  An empty shard still
    joins every collective.  -> [SVCFit(coef f64 [D] host, intercept float, objective history, iterations)] per class."""
    x = _check_x(x)
    n_local, D = x.shape
    positives = [int(p) for p in positives]
    K = len(positives)
    if K < 1:
        raise ValueError("LinearSVC needs at least one class to fit")
    n_labels = max(2, max(positives) + 1)
    _lib.svc_config(D, K)
    grp = group if group is not None else bdist.group()
    dev = x.device
    if row_offset is None:
        row_offset, _ = bdist.global_offset(n_local, dev, grp)
    sh = bdist.Shards(n_local, row_offset, grp, dev)
    yf = labels.to(device=dev, dtype=torch.float64).reshape(-1)
    yi = yf.to(torch.int32).contiguous()
    bad = torch.stack([((yf < 0) | (yf >= n_labels) | (yf != torch.floor(yf))).any(), (~torch.isfinite(x)).any(),
                       torch.tensor(yf.shape[0] != n_local, device=dev)])
    bad = bad.to(torch.int64)
    if grp is not None:
        bdist.all_reduce_(bad, grp)
    if int(bad[2].item()):                                  # the kernel reads one label per row
        raise ValueError("LinearSVC needs one label per row (a shard has %d rows and %d labels)" % (n_local, yf.shape[0]))
    if sh.total == 0:
        raise ValueError("LinearSVC needs at least one row")
    if int(bad[0].item()):
        raise ValueError("Classifier was given dataset with invalid label. Labels must be integers in [0, %d)." % n_labels)
    if int(bad[1].item()):
        raise ValueError("LinearSVC needs finite features")
    n = sh.total
    std = np.sqrt(selection.variances(x.to(torch.float64), row_offset, grp))
    inv = torch.from_numpy(np.where(std > 0, 1.0 / np.where(std > 0, std, 1.0), 0.0))
    inv_dev = inv.to(dev)
    lam = params.reg_param * (torch.ones(D, dtype=torch.float64, device=dev) if params.standardization else inv_dev * inv_dev)
    pos_dev = torch.tensor(positives, dtype=torch.int32, device=dev)

    # the optimiser state lives on the device: its arithmetic is then the GPU's, the same on every rank whatever host CPU
    # (and so whatever vectorised CPU reduction or BLAS path) the rank runs on
    zeros = torch.zeros(D + 1, dtype=torch.float64, device=dev)
    steps = [lbfgs_steps(zeros.clone(), params.max_iter, params.tol, HISTORY, l1=zeros) for _ in range(K)]
    pending = {k: next(s) for k, s in enumerate(steps)}
    done = [None] * K
    while pending:
        ks = sorted(pending)
        w = torch.stack([pending[k] for k in ks])
        sel = pos_dev if len(ks) == K else pos_dev[torch.tensor(ks, device=dev)].contiguous()
        tot = loss_grad_totals(x, yi, sel, inv_dev, w, sh)
        for i, k in enumerate(ks):
            fg = _objective(tot[i], pending[k], lam, n, D, params.fit_intercept)
            try:
                pending[k] = steps[k].send(fg)
            except StopIteration as stop:
                done[k] = stop.value
                del pending[k]
    fits = []
    for v, hist, it in done:
        fits.append(SVCFit((v[:D] * inv_dev).cpu().numpy(), float(v[D].item()), hist, it))
    return fits
