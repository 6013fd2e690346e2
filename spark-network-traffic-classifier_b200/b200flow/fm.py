"""FMClassifier, OneVsRest(FMClassifier) and FMRegressor on the device (DESIGN.md §5k, §5r): the logistic (classifier)
or squared-error (regressor) factorization-machine loss and its gradient from csrc/fm.cu's fused fp64 tensor-core kernel,
summed in the chunk order of dist.Shards, and mllib's mini-batch gradient descent with the gd or adamW updater, one
optimiser per class column, all of them advanced together.

Spark [recalled; Spark 3 `ml/regression/FMRegressor.scala` (trait FactorizationMachines), `FMClassifier.scala`, mllib
`GradientDescent.runMiniBatchSGD`]:

    Binary only.  Coefficients [V (D x k, row-major), w (D) if fitLinear, b if fitIntercept], V drawn as
    java.util.Random(seed).nextGaussian() * initStd in Array.fill order, w and b zero.  Per row
        r = b + sum_i w_i x_i + 1/2 sum_f [(sum_i v_if x_i)^2 - sum_i (v_if x_i)^2],  g = sigmoid(r) - y,
        loss = log1pExp(-r) if y > 0 else log1pExp(r),
        dv_if = g (x_i s_f - v_if x_i^2), dw_i = g x_i, db = g.
    regVal_0 = 1/2 regParam |w_0|^2; for i = 1..maxIter, over the rows drawn with fraction miniBatchFraction: if the
    batch is not empty, history += lossSum / batchSize + regVal, then the updater takes gradSum / batchSize; stop when
    |w_i - w_{i-1}| < tol max(|w_i|, 1), from the second update on.
    FMRegressor (MSEFactorizationMachinesGradient): the same loop on one column, with the label y used as it is,
    g = 2 (r - y) and loss = (r - y)^2; the prediction is r.
    gd (SquaredL2Updater): eta = stepSize / sqrt(i), w <- w (1 - eta regParam) - eta g.
    adamW (AdamWUpdater): m = b1 m + (1 - b1) g, v = b2 v + (1 - b2) g^2, b1^t *= b1, b2^t *= b2,
    w -= stepSize m_hat / (sqrt(v_hat) + eps) + regParam w.  Both return regVal = 1/2 regParam |w|^2.

Spark samples each iteration's batch with `data.sample(false, fraction, 42 + i)`, which cannot be reproduced; here a row
is in the batch iff its Philox draw (purpose FMMB, key seed 42 + i, counter the global row) is below floor(fraction 2^32).
The draw depends neither on the class nor on the estimator seed, so the classes of a OneVsRest fit share each batch.

One code path serves both classifier estimators: the standalone FMClassifier is fm_fit_classes(positives=[1]), OneVsRest
(FMClassifier) is positives=range(K); FMRegressor (fm_regression_fit) runs the same optimiser loop (_minibatch_sgd) on
the squared-error totals.  Each iteration makes ONE kernel pass over the classes still running.  A column's
partial does not depend on the other columns of the launch (csrc/fm.cu); the updates are elementwise, and every reduction
(|w|, |w - w_prev|) is taken per class on a fresh tensor of the standalone fit's shape, so every class takes exactly the
steps of its standalone fit.  The optimiser state is f64 on the device: host reductions pick their vector width by CPU
model, and ranks whose optimisers disagreed would stop after different iterations.
"""
import math

import numpy as np
import torch

from . import _lib
from . import dist as bdist
from . import selection
from ._lib import call, ptr

MAX_D = 255
SOLVERS = ("gd", "adamW")
BETA1, BETA2, EPSILON = 0.9, 0.999, 1e-8


class FMParams:
    __slots__ = ("factor_size", "fit_intercept", "fit_linear", "reg_param", "mini_batch_fraction", "init_std", "max_iter",
                 "step_size", "tol", "solver", "seed")

    def __init__(self, factor_size=8, fit_intercept=True, fit_linear=True, reg_param=0.0, mini_batch_fraction=1.0,
                 init_std=0.01, max_iter=100, step_size=1.0, tol=1e-6, solver="adamW", seed=0):
        self.factor_size, self.fit_intercept, self.fit_linear = int(factor_size), bool(fit_intercept), bool(fit_linear)
        self.reg_param, self.mini_batch_fraction, self.init_std = float(reg_param), float(mini_batch_fraction), float(init_std)
        self.max_iter, self.step_size, self.tol = int(max_iter), float(step_size), float(tol)
        self.solver, self.seed = str(solver), int(seed)


class FMFit:
    __slots__ = ("factors", "linear", "intercept", "objective_history", "iterations")

    def __init__(self, factors, linear, intercept, hist, it):
        self.factors, self.linear, self.intercept = factors, linear, intercept
        self.objective_history, self.iterations = hist, it


class JavaRandom:
    """java.util.Random: the 48-bit LCG, nextDouble and the polar-method nextGaussian with its cached second value.  Scalar
    Python arithmetic only, so that every host computes the same bits (math.log stands in for StrictMath.log)."""
    _MULT, _MASK = 0x5DEECE66D, (1 << 48) - 1

    def __init__(self, seed):
        self._seed = (int(seed) ^ self._MULT) & self._MASK
        self._next_gaussian = None

    def next_bits(self, bits):
        self._seed = (self._seed * self._MULT + 0xB) & self._MASK
        v = self._seed >> (48 - bits)
        return v - (1 << 32) if v >= 1 << 31 else v

    def next_double(self):
        return ((self.next_bits(26) << 27) + self.next_bits(27)) * 2.0 ** -53

    def next_gaussian(self):
        if self._next_gaussian is not None:
            v, self._next_gaussian = self._next_gaussian, None
            return v
        while True:
            v1 = 2 * self.next_double() - 1
            v2 = 2 * self.next_double() - 1
            s = v1 * v1 + v2 * v2
            if 0 < s < 1:
                break
        mult = math.sqrt(-2 * math.log(s) / s)
        self._next_gaussian = v2 * mult
        return v1 * mult


def init_factors(D, factor_size, init_std, seed):
    """V [D, factor_size] f64 host: Spark's Array.fill(D * k)(rnd.nextGaussian() * initStd), row-major"""
    rnd = JavaRandom(seed)
    return np.array([rnd.next_gaussian() * init_std for _ in range(D * factor_size)], np.float64).reshape(D, factor_size)


def _check_x(x):
    if not (torch.is_tensor(x) and x.is_cuda and x.dim() == 2 and x.dtype in (torch.float32, torch.float64)):
        raise _lib.B200FlowError("FMClassifier needs a CUDA float32 or float64 [n, D] matrix")
    if not 1 <= x.shape[1] <= MAX_D:
        raise _lib.UnsupportedParamError("FMClassifier supports 1 to %d features, got %d" % (MAX_D, x.shape[1]))
    return x.contiguous()


def loss_grad(x, labels, positives, weights, factor_size, fraction, batch_seed, row_offset, partials):
    """b200flow_fm_loss_grad on the rows x [n, D] (f32/f64): partials [n_chunks, K, D (k + 1) + D + 3] f64 device; labels
    int32 [n], positives int32 [K] and weights f64 [K, D (k + 1) + 1], all device."""
    n, D = x.shape
    call("b200flow_fm_loss_grad", ptr(x), _lib.dtype_code(x), n, x.stride(0), D, int(factor_size), ptr(labels), ptr(positives),
         int(positives.shape[0]), ptr(weights), float(fraction), int(batch_seed), int(row_offset), ptr(partials))


def fm_loss_grad_totals(x, labels, positives, weights, factor_size, fraction, batch_seed, sh):
    """[K, D (k + 1) + D + 3] f64 device: per class column, the loss sum, the batch row count and the gradient sums of
    b200flow_fm_loss_grad over every rank's rows, in chunk order; the same bits on every rank."""
    K, D = int(positives.shape[0]), x.shape[1]

    def launch(xs, ids, _, go, parts):
        loss_grad(xs, ids, positives, weights, factor_size, fraction, batch_seed, go, parts)

    return selection.chunk_total(x, labels, None, sh, K, D * (factor_size + 1) + D + 3, launch)


def fm_raw(x, weights, factor_size):
    """raw [n, K] f64 device: r of every row under weights [K, D (k + 1) + 1] f64 ([V | w | b] per class), one launch over
    the K columns."""
    x = _check_x(x)
    n, D = x.shape
    w = weights.to(device=x.device, dtype=torch.float64).contiguous()
    if w.dim() != 2 or w.shape[1] != D * (factor_size + 1) + 1:
        raise ValueError("the model has %d features, the input %d" % ((w.shape[1] - 1) // (factor_size + 1), D))
    K = w.shape[0]
    raw = torch.empty((max(n, 1), K), dtype=torch.float64, device=x.device)
    call("b200flow_fm_raw", ptr(x), _lib.dtype_code(x), n, x.stride(0), D, int(factor_size), K, ptr(w), ptr(raw))
    return raw[:n]


def regression_loss_grad(x, y, weights, factor_size, fraction, batch_seed, row_offset, partials):
    """b200flow_fm_regression_loss_grad on the rows x [n, D] (f32/f64): partials [n_chunks, 1, D (k + 1) + D + 3] f64
    device; labels y f64 [n] and weights f64 [1, D (k + 1) + 1], device."""
    n, D = x.shape
    call("b200flow_fm_regression_loss_grad", ptr(x), _lib.dtype_code(x), n, x.stride(0), D, int(factor_size), ptr(y),
         ptr(weights), float(fraction), int(batch_seed), int(row_offset), ptr(partials))


def fm_regression_loss_grad_totals(x, y, weights, factor_size, fraction, batch_seed, sh):
    """[1, D (k + 1) + D + 3] f64 device: b200flow_fm_regression_loss_grad's sums over every rank's rows, in chunk order;
    the same bits on every rank."""
    D = x.shape[1]

    def launch(xs, _, ys, go, parts):
        regression_loss_grad(xs, ys, weights, factor_size, fraction, batch_seed, go, parts)

    return selection.chunk_total(x, None, y, sh, 1, D * (factor_size + 1) + D + 3, launch)


def _norm(v):
    """|v| of one class's coefficients on a fresh tensor, so that the reduction is the standalone fit's whatever row of a
    class batch v came from"""
    return torch.linalg.vector_norm(v.clone())


def fm_fit_classes(x, labels, positives, params, row_offset=None, group=None):
    """FMClassifier fits of this rank's rows x [n, D] (f32 or f64) for each positive label: fit k treats label ==
    positives[k] as label 1 and every other label as 0.  Labels must be integers in [0, max(2, max(positives) + 1)).  An
    empty shard still joins every collective.  -> [FMFit(factors f64 [D, k], linear f64 [D], intercept float, objective
    history, iterations)] per class."""
    x = _check_x(x)
    n_local, D = x.shape
    positives = [int(p) for p in positives]
    K = len(positives)
    if K < 1:
        raise ValueError("FMClassifier needs at least one class to fit")
    if params.solver not in SOLVERS:
        raise ValueError("solver must be 'gd' or 'adamW', got %r" % (params.solver,))
    kf = params.factor_size
    n_labels = max(2, max(positives) + 1)
    _lib.fm_config(D, kf, K)
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
        raise ValueError("FMClassifier needs one label per row (a shard has %d rows and %d labels)" % (n_local, yf.shape[0]))
    if sh.total == 0:
        raise ValueError("FMClassifier needs at least one row")
    if int(bad[0].item()):
        raise ValueError("Classifier was given dataset with invalid label. Labels must be integers in [0, %d)." % n_labels)
    if int(bad[1].item()):
        raise ValueError("FMClassifier needs finite features")
    pos_dev = torch.tensor(positives, dtype=torch.int32, device=dev)

    def totals(wk, ia, act, it):
        sel = pos_dev if len(act) == K else pos_dev[ia].contiguous()
        return fm_loss_grad_totals(x, yi, sel, wk, kf, params.mini_batch_fraction, 42 + it, sh)

    return _minibatch_sgd(K, D, params, dev, totals)


def fm_regression_fit(x, labels, params, row_offset=None, group=None):
    """FMRegressor fit of this rank's rows x [n, D] (f32 or f64) and finite labels [n].  An empty shard still joins every
    collective.  -> FMFit(factors f64 [D, k], linear f64 [D], intercept float, objective history, iterations)."""
    x = _check_x(x)
    n_local, D = x.shape
    if params.solver not in SOLVERS:
        raise ValueError("solver must be 'gd' or 'adamW', got %r" % (params.solver,))
    kf = params.factor_size
    _lib.fm_config(D, kf, 1)
    grp = group if group is not None else bdist.group()
    dev = x.device
    if row_offset is None:
        row_offset, _ = bdist.global_offset(n_local, dev, grp)
    sh = bdist.Shards(n_local, row_offset, grp, dev)
    y = labels.to(device=dev, dtype=torch.float64).reshape(-1).contiguous()
    bad = torch.stack([(~torch.isfinite(y)).any(), (~torch.isfinite(x)).any(), torch.tensor(y.shape[0] != n_local, device=dev)])
    bad = bad.to(torch.int64)
    if grp is not None:
        bdist.all_reduce_(bad, grp)
    if int(bad[2].item()):                                  # the kernel reads one label per row
        raise ValueError("FMRegressor needs one label per row (a shard has %d rows and %d labels)" % (n_local, y.shape[0]))
    if sh.total == 0:
        raise ValueError("FMRegressor needs at least one row")
    if int(bad[0].item()):
        raise ValueError("FMRegressor needs finite labels")
    if int(bad[1].item()):
        raise ValueError("FMRegressor needs finite features")

    def totals(wk, ia, act, it):
        return fm_regression_loss_grad_totals(x, y, wk, kf, params.mini_batch_fraction, 42 + it, sh)

    return _minibatch_sgd(1, D, params, dev, totals)[0]


def _minibatch_sgd(K, D, params, dev, totals):
    """runMiniBatchSGD for K columns in lockstep: totals(wk [len(act), D (k + 1) + 1] kernel weights, ia (device indices of
    the active columns), act (their list), iteration) -> the kernel layout's sums [len(act), D (k + 1) + D + 3] of the
    active columns.  -> [FMFit] per column."""
    kf = params.factor_size
    # the coefficients in Spark's layout [V | w if fitLinear | b if fitIntercept], one row per class, f64 on the device
    nv = D * kf
    P = nv + (D if params.fit_linear else 0) + (1 if params.fit_intercept else 0)
    v0 = torch.from_numpy(init_factors(D, kf, params.init_std, params.seed).reshape(-1))
    coef = torch.zeros((K, P), dtype=torch.float64, device=dev)
    coef[:, :nv] = v0.to(dev)
    m = torch.zeros_like(coef)
    v = torch.zeros_like(coef)
    b1t = b2t = 1.0
    reg = params.reg_param
    half_reg = torch.tensor(0.5 * reg, dtype=torch.float64, device=dev)

    def reg_val(nrm):
        return half_reg * nrm * nrm

    reg_vals = torch.stack([reg_val(_norm(coef[k])) for k in range(K)])
    hist = [[] for _ in range(K)]
    updates = [0] * K
    done = [False] * K
    for it in range(1, params.max_iter + 1):
        act = [k for k in range(K) if not done[k]]
        if not act:
            break
        ia = torch.tensor(act, device=dev)
        cur = coef if len(act) == K else coef[ia]
        wk = torch.zeros((len(act), D * (kf + 1) + 1), dtype=torch.float64, device=dev)
        wk[:, :nv] = cur[:, :nv]
        if params.fit_linear:
            wk[:, nv:nv + D] = cur[:, nv:nv + D]
        if params.fit_intercept:
            wk[:, -1] = cur[:, -1]
        tot = totals(wk, ia, act, it)
        batch = float(tot[0, 1].item())
        if batch == 0.0:                                    # an empty batch: no update, the iteration still counts
            continue
        nb = tot[:, 1:2]
        gv = tot[:, 2:2 + nv] - cur[:, :nv] * tot[:, 3 + nv + D:3 + nv + 2 * D].repeat_interleave(kf, dim=1)
        parts = [gv]
        if params.fit_linear:
            parts.append(tot[:, 2 + nv:2 + nv + D])
        if params.fit_intercept:
            parts.append(tot[:, 2 + nv + D:3 + nv + D])
        g = torch.cat(parts, 1) / nb
        hist_vals = tot[:, 0] / nb[:, 0] + (reg_vals if len(act) == K else reg_vals[ia])
        if params.solver == "gd":
            eta = params.step_size / math.sqrt(it)
            new = cur * (1.0 - eta * reg) + (-eta) * g
        else:
            ma = (m if len(act) == K else m[ia]) * BETA1 + (1 - BETA1) * g
            va = (v if len(act) == K else v[ia]) * BETA2 + (1 - BETA2) * (g * g)
            b1t *= BETA1
            b2t *= BETA2
            m_hat = ma / torch.tensor(1 - b1t, dtype=torch.float64, device=dev)
            v_hat = va / torch.tensor(1 - b2t, dtype=torch.float64, device=dev)
            new = cur - (params.step_size * m_hat / (torch.sqrt(v_hat) + EPSILON) + reg * cur)
            m[ia], v[ia] = ma, va
        diff = new - cur
        nrm = torch.stack([_norm(new[i]) for i in range(len(act))])
        dn = torch.stack([_norm(diff[i]) for i in range(len(act))])
        conv = dn < params.tol * torch.clamp(nrm, min=1.0)
        reg_vals[ia] = reg_val(nrm)
        coef[ia] = new
        hv, cv = hist_vals.cpu().numpy(), conv.cpu().numpy()
        for i, k in enumerate(act):
            hist[k].append(float(hv[i]))
            updates[k] += 1
            done[k] = updates[k] >= 2 and bool(cv[i])
    c = coef.cpu().numpy()
    fits = []
    for k in range(K):
        lin = c[k, nv:nv + D].copy() if params.fit_linear else np.zeros(D)
        b = float(c[k, -1]) if params.fit_intercept else 0.0
        fits.append(FMFit(c[k, :nv].reshape(D, kf).copy(), lin, b, hist[k], len(hist[k])))
    return fits
