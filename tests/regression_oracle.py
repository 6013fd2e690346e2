"""Sequential numpy restatement of DecisionTreeRegressor / RandomForestRegressor as b200flow trains them (DESIGN.md §5l) and
of RegressionEvaluator's exact sums.  findSplits, binning, the Poisson bag weights and the feature subsets come from the C
oracle (oracle/); each tree is tests/gbt_oracle.py's grow_tree on the label grid; leaf values, leaf variances and the
evaluator's fixed-point sums are restated operation for operation, so the device results must equal these bit for bit.
Rows are not de-duplicated: the histograms are exact integer sums, so merging equal records cannot change a tree."""
import math

import numpy as np

import gbt_oracle as go
import oracle

E_MIN, E_MAX = -300, 300


def resolve_strategy(strategy, num_trees):
    s = str(strategy)
    return ("all" if int(num_trees) == 1 else "onethird") if s == "auto" else s


def label_grid(max_abs, w_max):
    """(E, S, S2): max |y| <= 2^E, S = S2 = 61 - ceil(log2 w_max)"""
    lg = int(math.ceil(math.log2(max(int(w_max), 2))))
    if not max_abs > 0.0:
        E = 0
    else:
        mnt, e = math.frexp(float(max_abs))
        E = e - 1 if mnt == 0.5 else e
    if E > E_MAX:
        raise ValueError("label beyond 2^%d" % E_MAX)
    return max(E, E_MIN), 61 - lg, 61 - lg


def to_grid(y, E, S, S2):
    ys = np.ldexp(np.asarray(y, np.float64), -E)
    q = np.rint(ys * 2.0 ** S).astype(np.int64)
    yh = q.astype(np.float64) * 2.0 ** -S
    return q, np.rint(yh * yh * 2.0 ** S2).astype(np.int64)


def fit(x, y, arity, num_trees=20, max_depth=5, max_bins=32, min_inst=1, min_gain=0.0, subsampling_rate=1.0, strategy="auto",
        seed=0, bootstrap=True):
    """end to end on a dense matrix: -> dict(trees, T, E, S, S2, thresholds, n_thr, max_bins, ...)"""
    x = np.ascontiguousarray(x, np.float64)
    y = np.asarray(y, np.float64)
    n, F = x.shape
    T = int(num_trees)
    arity = np.asarray(arity, np.int32)
    if not np.isfinite(y).all():
        raise ValueError("a label is NaN or infinite")
    mpb, kind, m = oracle.build_metadata(n, F, 2, arity, max_bins, T, resolve_strategy(strategy, T))
    frac = min(1.0, max(mpb * mpb, 10000) / n) if (arity == 0).any() else 1.0
    thr, n_thr, _ = oracle.find_splits(x, seed, int(frac * 4294967296.0), arity, mpb)
    tp, bad = oracle.bin_rows(x, thr, n_thr, arity, mpb)
    assert bad == 0
    bins = tp[:, :F]
    feat_bins = np.where(arity > 0, arity, n_thr + 1).astype(np.int32)
    if bootstrap and T > 1:
        W = oracle.bag_weights(seed, T, n, oracle.poisson_cdf_table(subsampling_rate)).astype(np.int64)
    else:
        W = np.ones((T, n), np.int64)
    E, S, S2 = label_grid(float(np.abs(y).max()) if n else 0.0, int(W.sum(1).max()) if n else 0)
    q, q2 = to_grid(y, E, S, S2)
    Sk, S2k = S - E, S2 - 2 * E
    trees = []
    for t in range(T):
        nodes = go.grow_tree(t, bins, W[t], q, q2, feat_bins, kind, m, max_depth, min_inst, min_gain, seed, Sk, S2k)
        for nd in nodes.values():
            st = nd["stats"]
            nd["payload"] = go.leaf_value(nd, 1.0, Sk)
            nd["variance"] = float(go.variance(st[0], st[1], st[2], Sk, S2k))
        trees.append(nodes)
    return dict(trees=trees, T=T, E=E, S=S, S2=S2, thresholds=thr, n_thr=n_thr, max_bins=mpb, feat_bins=feat_bins,
                feat_kind=kind, m=m, arity=arity)


def predict(model, bins):
    """-> (prediction, leaf variance of tree 0): Σ over the trees in tree order from +0.0, / T"""
    s = np.zeros(bins.shape[0])
    var = None
    for t, nodes in enumerate(model["trees"]):
        leaf = go.walk(nodes, bins)
        s = s + np.array([nodes[int(i)]["payload"] for i in leaf])
        if t == 0:
            var = 0.0 + np.array([nodes[int(i)]["variance"] for i in leaf])
    return (s if model["T"] == 1 else s / float(model["T"])), var


def predict_x(model, x):
    tp, _ = oracle.bin_rows(np.ascontiguousarray(x, np.float64), model["thresholds"], model["n_thr"], model["arity"],
                            model["max_bins"])
    return predict(model, tp[:, :x.shape[1]])


def export(model):
    """canonical arrays ordered by (tree, node id), as RegressionModel.export gives them"""
    return go.export(dict(trees=model["trees"]))


def feature_importances(model, F):
    imp = np.zeros(F)
    for nodes in model["trees"]:
        v = np.zeros(F)
        for nd in nodes.values():
            if not nd["leaf"]:
                v[nd["feat"]] += nd["gain"] * float(nd["stats"][0])
        if v.sum() > 0:
            imp += v / v.sum()
    return imp / imp.sum() if imp.sum() > 0 else imp


# ------------------------------------------------------------------ RegressionEvaluator
def fixed_shift(max_abs, n):
    if not max_abs > 0.0:
        return 0
    mnt, e = math.frexp(max_abs)
    E = e - 1 if mnt == 0.5 else e
    return 126 - int(math.ceil(math.log2(max(n, 2)))) - E


def exact_sum(t, n):
    """the double nearest to the exact sum of rint(t 2^sh) / 2^sh, by Python ints"""
    t = np.asarray(t, np.float64)
    sh = fixed_shift(float(np.abs(t).max()) if t.size else 0.0, n)
    v = np.rint(np.ldexp(t, sh))
    total = sum(int(a) for a in v.tolist())
    if total == 0:
        return 0.0
    return total / (1 << sh) if sh >= 0 else float(total * (1 << -sh))


def metrics(label, pred, through_origin=False):
    y, p = np.asarray(label, np.float64), np.asarray(pred, np.float64)
    n = y.shape[0]
    nan = float("nan")
    out_nan = dict(mse=nan, rmse=nan, mae=nan, var=nan, r2=nan)
    if n == 0:
        return out_nan
    with np.errstate(all="ignore"):
        d = y - p
        t0 = [y, y * y, d * d, np.abs(d)]
    if not (np.isfinite(y).all() and np.isfinite(p).all() and all(np.isfinite(t).all() for t in t0)):
        return out_nan
    sy, syy, sserr, sabs = (exact_sum(t, n) for t in t0)
    mean = sy / n
    with np.errstate(all="ignore"):
        a, b = y - mean, p - mean
        t1 = [a * a, b * b]
    if not all(np.isfinite(t).all() for t in t1):
        return out_nan
    sstot, ssreg = (exact_sum(t, n) for t in t1)
    mse = sserr / n
    den = syy if through_origin else sstot
    r2 = (1.0 - sserr / den) if den != 0.0 else (nan if sserr == 0.0 else -math.inf)
    return dict(mse=mse, rmse=math.sqrt(mse), mae=sabs / n, var=ssreg / n, r2=r2)
