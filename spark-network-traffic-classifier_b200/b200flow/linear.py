"""The two non-tree classifiers the reference scripts also fit (SURVEY.md 8f-4; kdd99.py:57-58,67 and cicids17.py:61-62,71):
multinomial naive Bayes and elastic-net logistic regression, with MLlib's statistics and objective.  Plain torch (fp64) on the
tensors' own device: they are not roofline targets — the contraction is one [C x n] x [n x D] product — but their numbers are
checked against oracle/linear.py and scikit-learn (tests/test_linear_models.py).

MLlib [recalled; Spark 2.4 `ml/classification/NaiveBayes.scala`, `ml/classification/LogisticRegression.scala`,
`ml/optim/aggregator/LogisticAggregator.scala`, breeze `optimize/OWLQN.scala`]:

NaiveBayes (multinomial): per label present in the data n_c = #rows, s_cj = sum of feature j; L = #labels PRESENT;
    pi_c = log(n_c + lambda) - log(N + L lambda);  theta_cj = log(s_cj + lambda) - log(sum_j s_cj + D lambda);
    raw(x) = pi + theta x;  probability = softmax(raw);  negative feature values are rejected.
    Labels absent from the training rows get pi = -inf here (never predicted, probability 0); MLlib would emit a model with L
    rows and report the ROW index as the prediction — the same numbers whenever every label is present.

LogisticRegression (standardization=True): features are scaled by 1 / (unbiased std) (std 0 -> the feature is dropped), not
    centred; minimise over (B, b)
        (1/n) sum_i [ logsumexp(B xs_i + b) - (B xs_i + b)_{y_i} ]  +  regParam * ( alpha * |B|_1 + (1 - alpha)/2 * |B|_2^2 )
    (intercepts unpenalised) with OWL-QN (L-BFGS, 10 corrections) started from B = 0, b_k = log(count_k + 1) centred; at most
    maxIter iterations, stop when the relative decrease falls under tol.  Afterwards B is mapped back to the original feature
    scale and the multinomial intercepts are centred.  numClasses == 2 with family auto/binomial: one coefficient row, the
    margin of class 1 (pivot class 0).
    Breeze's exact line-search constants are not reproducible from memory: iterates are NOT MLlib's iterate for iterate; the
    objective is strictly convex in B once regParam * (1 - alpha) > 0, and what is tested is that the same minimiser is reached.
"""
import math

import torch

from . import dist as bdist


def _allsum(t, group):
    """rows are sharded over ranks (one process per GPU): every statistic below is a sum over rows, reduced over the ranks, so
    that each rank takes the same optimiser steps on the same numbers.  fp64 sums in rank order: equal on every rank; they differ
    from the single-process value only by the association of the partial sums."""
    return bdist.all_reduce_sum_(t, group) if group is not None else t


class NaiveBayesFit:
    __slots__ = ("pi", "theta", "present")

    def __init__(self, pi, theta, present):
        self.pi, self.theta, self.present = pi, theta, present


def nb_fit(x, y, num_classes, smoothing=1.0, group=None):
    """x [n, D] (any float dtype, >= 0), y [n] class indices -> NaiveBayesFit with pi [C], theta [C, D] (fp64).
    group: torch.distributed group over which the rows are sharded (None: single process)."""
    x = x.to(torch.float64)
    neg = _allsum((x < 0).any().to(torch.int64).reshape(1), group)
    if int(neg.item()):
        raise ValueError("requirement failed: Naive Bayes requires nonnegative feature values but found a negative value.")
    C, D = int(num_classes), x.shape[1]
    yl = y.to(torch.int64)
    n_c = _allsum(torch.bincount(yl, minlength=C).to(torch.float64), group)
    s = _allsum(torch.zeros((C, D), dtype=torch.float64, device=x.device).index_add_(0, yl, x), group)
    present = n_c > 0
    L = int(present.sum().item())
    lam = float(smoothing)
    pi = torch.log(n_c + lam) - math.log(float(n_c.sum().item()) + L * lam)
    theta = torch.log(s + lam) - torch.log(s.sum(1, keepdim=True) + D * lam)
    pi = torch.where(present, pi, torch.full_like(pi, float("-inf")))
    theta = torch.where(present[:, None], theta, torch.zeros_like(theta))
    return NaiveBayesFit(pi, theta, present)


def nb_raw(fit, x):
    return x.to(torch.float64) @ fit.theta.t() + fit.pi


# ----------------------------------------------------------------------------------------- logistic regression (OWL-QN)
class LogisticFit:
    __slots__ = ("coef", "intercept", "objective_history", "iterations", "binomial")

    def __init__(self, coef, intercept, hist, it, binomial):
        self.coef, self.intercept, self.objective_history, self.iterations, self.binomial = coef, intercept, hist, it, binomial


def _margins(xs, B, b, binomial):
    z = xs @ B.t() + b
    return torch.cat([torch.zeros_like(z), z], 1) if binomial else z


def lr_loss_grad(xs, y1h, B, b, l2, binomial, fit_intercept=True, n_total=None, group=None):
    """smooth part: mean multinomial log-loss + sum_j l2_j/2 |B_j|^2 (l2: scalar or one weight per feature) and its gradient.
    With a group: xs / y1h are this rank's rows, n_total the global row count; loss and gradient sums are all-reduced."""
    n = xs.shape[0] if n_total is None else n_total
    z = _margins(xs, B, b, binomial)
    lse = torch.logsumexp(z, 1)
    R = torch.softmax(z, 1) - y1h                                     # [n, C]
    if binomial:
        R = R[:, 1:]
    packed = torch.cat([(lse - (z * y1h).sum(1)).sum().reshape(1), (R.t() @ xs).reshape(-1), R.sum(0)])
    packed = _allsum(packed, group) / n
    K, D = B.shape
    loss = packed[0] + 0.5 * (l2 * B * B).sum()
    gB = packed[1:1 + K * D].view(K, D) + l2 * B
    gb = packed[1 + K * D:] if fit_intercept else torch.zeros_like(b)
    return loss, gB, gb


def _pseudo_gradient(x, g, c):
    """Andrew & Gao (2007) eq. 4: the steepest-descent subgradient of f + c|x|_1."""
    right, left = g + c, g - c
    at0 = torch.where(right < 0, right, torch.where(left > 0, left, torch.zeros_like(g)))
    return torch.where(x > 0, right, torch.where(x < 0, left, at0))


def lbfgs_steps(v, max_iter, tol, history=10, l1=None):
    """lbfgs as a generator: it yields every point at which it needs the smooth part, receives (f, gradient) for that point
    through send(), and returns (v, objective history, iterations).  So several problems can advance in lockstep, their
    evaluations batched by the caller, each taking exactly the steps of its own lbfgs run."""
    def full(v, f):
        return f if l1 is None else f + (l1 * v.abs()).sum()

    f, g = yield v
    F = float(full(v, f).item())
    hist = [F]
    S, Y, RHO = [], [], []
    it = 0
    while it < int(max_iter):
        pg = g if l1 is None else _pseudo_gradient(v, g, l1)
        if float(pg.norm().item()) <= 1e-14:
            break
        q = pg.clone()                                                 # two-loop recursion on the pseudo-gradient
        al = []
        for s_, y_, r_ in zip(reversed(S), reversed(Y), reversed(RHO)):
            a = r_ * (s_ @ q)
            al.append(a)
            q -= a * y_
        if S:
            q *= (S[-1] @ Y[-1]) / (Y[-1] @ Y[-1])
        for (s_, y_, r_), a in zip(zip(S, Y, RHO), reversed(al)):
            q += (a - r_ * (y_ @ q)) * s_
        d = -q
        if l1 is not None:
            d = torch.where(d * pg < 0, d, torch.zeros_like(d))        # keep only components that descend along -pg
            if not bool((d != 0).any()):
                d = -pg
            orth = torch.where(v != 0, torch.sign(v), torch.sign(-pg)) # the orthant the step must stay in
        dir_deriv = float((pg @ d).item())
        step = 1.0 if S else min(1.0, 1.0 / max(float(pg.norm().item()), 1e-300))
        ok = False
        for _ in range(40):
            vn = v + step * d
            if l1 is not None:
                vn = torch.where(vn * orth < 0, torch.zeros_like(vn), vn)  # projection onto the orthant
            fn, gn = yield vn
            Fn = float(full(vn, fn).item())
            if Fn <= F + 1e-4 * float((pg @ (vn - v)).item()):
                ok = True
                break
            step *= 0.5
        if not ok or dir_deriv >= 0 and not S:
            break
        s_, y_ = vn - v, gn - g
        sy = float((s_ @ y_).item())
        if sy > 1e-300:
            S.append(s_); Y.append(y_); RHO.append(1.0 / sy)
            if len(S) > history:
                S.pop(0); Y.pop(0); RHO.pop(0)
        v, g, f = vn, gn, fn
        it += 1
        hist.append(Fn)
        improved = (F - Fn) / max(abs(Fn), abs(F), 1e-300)
        F = Fn
        if improved <= tol and it > 1:
            break
    return v, hist, it


def lbfgs(smooth, v, max_iter, tol, history=10, l1=None):
    """minimise smooth(v) -> (f, gradient) from v: L-BFGS with `history` corrections, backtracking (Armijo 1e-4, halving,
    at most 40 trials), stopping after max_iter iterations or once the relative decrease (F - Fn) / max(|Fn|, |F|) falls
    to tol after the first iteration.  l1 (one weight per variable) makes it OWL-QN for f + sum l1 |v|: the direction
    is kept to the components that descend along the pseudo-gradient and the steps are projected onto the orthant; None
    is plain L-BFGS (Breeze LBFGS, what Spark runs without an L1 term).  -> (v, objective history, iterations)."""
    steps = lbfgs_steps(v, max_iter, tol, history, l1)
    point = next(steps)
    try:
        while True:
            point = steps.send(smooth(point))
    except StopIteration as done:
        return done.value


def lr_fit(x, y, num_classes, max_iter=100, reg_param=0.0, elastic_net=0.0, tol=1e-6, fit_intercept=True, standardization=True,
           family="auto", history=10, group=None):
    x = x.to(torch.float64)
    n_local, D = x.shape
    C = int(num_classes)
    binomial = family == "binomial" or (family == "auto" and C <= 2)
    if binomial and C > 2:
        raise ValueError("Binomial family only supports 1 or 2 outcome classes but found %d." % C)
    if group is None:
        n = n_local
        std = x.std(0, unbiased=True) if n > 1 else torch.zeros(D, dtype=torch.float64, device=x.device)
    else:                                                               # two passes over the shards: global mean, then squared deviations
        head = _allsum(torch.cat([torch.tensor([float(n_local)], dtype=torch.float64, device=x.device), x.sum(0)]), group)
        n = int(round(head[0].item()))
        mean = head[1:] / max(n, 1)
        ss = _allsum(((x - mean) ** 2).sum(0), group)
        std = torch.sqrt(ss / (n - 1)) if n > 1 else torch.zeros(D, dtype=torch.float64, device=x.device)
    inv = torch.where(std > 0, 1.0 / std, torch.zeros_like(std))
    xs = x * inv                                                        # std 0 -> column of zeros -> coefficient stays 0
    yl = y.to(torch.int64)
    Cm = max(C, 2) if binomial else C
    y1h = torch.nn.functional.one_hot(yl, Cm).to(torch.float64)
    l1, l2 = reg_param * elastic_net, reg_param * (1.0 - elastic_net)
    ones = torch.ones(D, dtype=torch.float64, device=x.device)
    # standardization=False: MLlib still optimises in the scaled space but penalises the ORIGINAL-scale coefficients B / std
    l1w_row, l2w_row = (l1 * ones, l2 * ones) if standardization else (l1 * inv, l2 * inv * inv)
    K = 1 if binomial else C
    counts = _allsum(torch.bincount(yl, minlength=Cm).to(torch.float64), group)
    B = torch.zeros((K, D), dtype=torch.float64, device=x.device)
    if not fit_intercept:
        b = torch.zeros(K, dtype=torch.float64, device=x.device)
    elif binomial:
        b = torch.log(counts[1:2] / counts[0:1]) if bool((counts[:2] > 0).all()) else torch.zeros(1, dtype=torch.float64, device=x.device)
    else:
        b = torch.log1p(counts)
        b = b - b.mean()
    cw = torch.cat([l1w_row.repeat(K), torch.zeros(K, dtype=torch.float64, device=x.device)])      # l1 weight per variable

    def unpack(v):
        return v[:K * D].view(K, D), v[K * D:]

    def smooth(v):
        Bv, bv = unpack(v)
        f, gB, gb = lr_loss_grad(xs, y1h, Bv, bv, l2w_row, binomial, fit_intercept, n, group)
        return f, torch.cat([gB.reshape(-1), gb])

    v, hist, it = lbfgs(smooth, torch.cat([B.reshape(-1), b]), max_iter, tol, history, l1=cw)
    B, b = unpack(v)
    coef = B * inv                                                      # back to the original feature scale
    if fit_intercept and not binomial:
        b = b - b.mean()
    return LogisticFit(coef.contiguous(), b.contiguous(), hist, it, binomial)


def lr_raw(fit, x):
    """rawPrediction: the margins (binomial: [-m, m] like MLlib's BinaryLogisticRegression)."""
    z = x.to(torch.float64) @ fit.coef.t() + fit.intercept
    return torch.cat([-z, z], 1) if fit.binomial else z


def lr_probability(fit, raw):
    """probability: softmax of the margins; binomial: [1 - sigmoid(m), sigmoid(m)]."""
    if fit.binomial:
        p1 = torch.sigmoid(raw[:, 1:2])
        return torch.cat([1.0 - p1, p1], 1)
    return torch.softmax(raw, 1)
