"""Sequential numpy restatement of GBTRegressor as b200flow trains it (DESIGN.md §5m): Spark 3's GradientBoostedTrees.boost
with SquaredError or AbsoluteError over regression trees, each iteration's residuals on a grid whose exponent comes from that
iteration's max |r|.  findSplits, binning, the Bernoulli subsample draws and the feature subsets come from the C oracle
(oracle/); each tree is tests/gbt_oracle.py's grow_tree; the grid is tests/regression_oracle.py's; residuals, E_m, payloads
and margins are restated operation for operation, so the device model must equal this bit for bit.  Rows are not
de-duplicated: the histograms are exact integer sums, so merging equal records cannot change a tree."""
import numpy as np

import gbt_oracle as go
import oracle
import regression_oracle as ro


def residual_exponent(max_abs):
    """E_m from max |r|: label_grid's rule; beyond 2^300 refused"""
    if max_abs > 2.0 ** ro.E_MAX:
        raise ValueError("residual beyond 2^%d" % ro.E_MAX)
    return ro.label_grid(max_abs, 2)[0]


def residual(y, Fm, loss):
    """-loss.gradient(F, y); a NaN residual becomes 0"""
    with np.errstate(all="ignore"):
        d = y - Fm
        r = 2.0 * d if loss == "squared" else np.where(d < 0.0, -1.0, 1.0)
    return np.where(np.isnan(r), 0.0, r)


def boost(bins, y, W, feat_bins, feat_kind, m, max_iter, step_size, max_depth, min_inst, min_gain, seed, loss, n_global):
    """-> (trees, tree weights, E sequence, S, S2, training margin) on binned rows with f64 labels y"""
    n = bins.shape[0]
    E, S, S2 = ro.label_grid(float(np.abs(y).max()) if n else 0.0, n_global)
    Fm = np.zeros(n)
    r = y.copy()
    trees, weights, Es = [], [1.0] + [float(step_size)] * (max_iter - 1), []
    for t in range(max_iter):
        if t > 0:
            E = residual_exponent(float(np.abs(r).max()) if n else 0.0)
        Es.append(E)
        q, q2 = ro.to_grid(r, E, S, S2)
        Sk, S2k = S - E, S2 - 2 * E
        nodes = go.grow_tree(t, bins, W[t if W.shape[0] > 1 else 0], q, q2, feat_bins, feat_kind, m, max_depth, min_inst, min_gain,
                             seed, Sk, S2k)
        for nd in nodes.values():
            nd["payload"] = go.leaf_value(nd, weights[t], Sk)
            nd["value"] = go.leaf_value(nd, 1.0, Sk)
        trees.append(nodes)
        Fm = Fm + np.array([nodes[int(i)]["payload"] for i in go.walk(nodes, bins)])
        r = residual(y, Fm, loss)
    return trees, weights, Es, S, S2, Fm


def fit(x, y, arity, max_iter=20, step_size=0.1, max_depth=5, max_bins=32, min_inst=1, min_gain=0.0, subsampling_rate=1.0,
        strategy="all", seed=0, loss="squared"):
    """end to end on a dense matrix: -> dict(trees, weights, E, S, S2, margin, thresholds, n_thr, bins, ...)"""
    x = np.ascontiguousarray(x, np.float64)
    y = np.asarray(y, np.float64)
    n, F = x.shape
    arity = np.asarray(arity, np.int32)
    if not np.isfinite(y).all():
        raise ValueError("a label is NaN or infinite")
    mpb, kind, m = oracle.build_metadata(n, F, 2, arity, max_bins, 1, "all" if strategy == "auto" else strategy)
    frac = min(1.0, max(mpb * mpb, 10000) / n) if (arity == 0).any() else 1.0
    thr, n_thr, _ = oracle.find_splits(x, seed, int(frac * 4294967296.0), arity, mpb)
    tp, bad = oracle.bin_rows(x, thr, n_thr, arity, mpb)
    assert bad == 0
    bins = tp[:, :F]
    feat_bins = np.where(arity > 0, arity, n_thr + 1).astype(np.int32)
    if subsampling_rate < 1.0:
        W = oracle.bag_weights(seed, max_iter, n, go.subsample_cdf(subsampling_rate)).astype(np.int64)
    else:
        W = np.ones((1, n), np.int64)
    trees, weights, Es, S, S2, Fm = boost(bins, y, W, feat_bins, kind, m, max_iter, step_size, max_depth, min_inst, min_gain,
                                          seed, loss, n)
    return dict(trees=trees, weights=weights, E=Es, S=S, S2=S2, margin=Fm, thresholds=thr, n_thr=n_thr, bins=bins,
                feat_bins=feat_bins, feat_kind=kind, m=m, max_bins=mpb, arity=arity)


def prefix_predictions(model, bins):
    """-> [prediction of the first k trees for k = 1..T]: Σ in tree order from +0.0"""
    Fm, out = np.zeros(bins.shape[0]), []
    for nodes in model["trees"]:
        Fm = Fm + np.array([nodes[int(i)]["payload"] for i in go.walk(nodes, bins)])
        out.append(Fm)
    return out


def prefix_predictions_x(model, x):
    tp, _ = oracle.bin_rows(np.ascontiguousarray(x, np.float64), model["thresholds"], model["n_thr"], model["arity"],
                            model["max_bins"])
    return prefix_predictions(model, tp[:, :x.shape[1]])


def predict_x(model, x):
    return prefix_predictions_x(model, x)[-1]


def export(model):
    """canonical arrays ordered by (tree, node id), as GBTRegressionModel.export gives them"""
    return go.export(model)


def feature_importances(model, F):
    v = np.zeros(F)
    for nodes in model["trees"]:
        for nd in nodes.values():
            if not nd["leaf"]:
                v[nd["feat"]] += nd["gain"] * float(nd["stats"][0])
    return v / v.sum() if v.sum() > 0 else v
