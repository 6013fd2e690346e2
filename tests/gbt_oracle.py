"""Sequential numpy restatement of GBTClassifier as b200flow trains it (DESIGN.md §5e): Spark 3's GradientBoostedTrees.boost
with LogLoss over regression trees (RandomForest.run, numTrees = 1, Variance), residuals on the fixed-point grid, and the
shared exp of csrc/portable_exp.h.  findSplits, binning, the Bernoulli subsample draws and the feature subsets come from the
C oracle (oracle/), which the forest tests already pin; everything else is restated here operation for operation, so the
device model must equal it bit for bit.  Rows are not de-duplicated and histograms are summed exactly (integers)."""
import math

import numpy as np

import oracle

DBL_MAX = np.finfo(np.float64).max
EPSILON = 2.220446049250313e-16

_O_THRESHOLD = 7.09782712893383973096e+02
_U_THRESHOLD = -7.45133219101941108420e+02
_INV_LN2 = 1.44269504088896338700e+00
_LN2_HI = 6.93147180369123816490e-01
_LN2_LO = 1.90821492927058770002e-10
_P = (1.66666666666666019037e-01, -2.77777777770155933842e-03, 6.61375632143793436117e-05, -1.65339022054652515390e-06,
      4.13813679705723846039e-08)


def pexp(x):
    """csrc/portable_exp.h on an array (elementwise IEEE operations, no FMA)."""
    x = np.asarray(x, np.float64)
    with np.errstate(all="ignore"):
        xs = np.where(np.isfinite(x), x, 0.0)
        kd = np.rint(xs * _INV_LN2)
        hi = xs - kd * _LN2_HI
        lo = kd * _LN2_LO
        r = hi - lo
        t = r * r
        c = r - t * (_P[0] + t * (_P[1] + t * (_P[2] + t * (_P[3] + t * _P[4]))))
        y = 1.0 - ((lo - (r * c) / (2.0 - c)) - hi)
        out = np.ldexp(y, kd.astype(np.int64).clip(-2000, 2000).astype(np.int32))   # one rounding, as the two-step scaling
    out = np.where(x > _O_THRESHOLD, np.inf, out)
    out = np.where(x < _U_THRESHOLD, 0.0, out)
    return np.where(np.isnan(x), x, out)


def grid_shift(n_global):
    lg = int(math.ceil(math.log2(max(int(n_global), 2))))
    return 60 - lg, 58 - lg


def to_grid(r, S, S2):
    """r -> (q, q2) int64"""
    r = np.where(np.isnan(r), 0.0, r)
    q = np.rint(r * 2.0 ** S).astype(np.int64)
    rh = q.astype(np.float64) * 2.0 ** -S
    return q, np.rint(rh * rh * 2.0 ** S2).astype(np.int64)


def residual(y, F):
    with np.errstate(all="ignore"):
        return 4.0 * y / (1.0 + pexp(2.0 * y * F))


def _limbs(v, count):
    """v (int64) cut into (shift, float64 limb) pairs narrow enough that a float64 sum of `count` limbs is exact
    (limb · count < 2^53); the top limb keeps the sign, and all-zero limbs are left out"""
    bits = max(1, 53 - int(np.ceil(np.log2(max(count, 2)))))
    out, sh = [], 0
    while sh < 64:
        limb = (v >> sh) if sh + bits >= 64 else ((v >> sh) & ((1 << bits) - 1))
        if limb.any():
            out.append((sh, limb.astype(np.float64)))
        sh += bits
    return out


def node_hist(bins, w, q, q2, n_bins):
    """int64 [m, n_bins, 3] of {Σw, Σw·q, Σw·q2} per (feature of bins [rows, m], bin), exact: the limbs' float64 bincounts
    are put back together with wrapping int64 arithmetic (every total fits in int64)"""
    n, m = bins.shape
    w = w.astype(np.int64)
    with np.errstate(over="ignore"):
        parts = [_limbs(v, n) for v in (w, w * q, w * q2)]
    cols = np.asfortranarray(bins).astype(np.intp)
    out = np.zeros((m, n_bins, 3), np.int64)
    for j in range(m):
        for k, limbs in enumerate(parts):
            for sh, limb in limbs:
                out[j, :, k] += np.bincount(cols[:, j], weights=limb, minlength=n_bins).astype(np.int64) << np.int64(sh)
    return out


def variance(cnt, s1, s2, S, S2):
    """Variance.calculate on int64 stats (arrays), 0 where count == 0"""
    c = np.asarray(cnt).astype(np.float64)
    s = np.asarray(s1).astype(np.float64) * 2.0 ** -S
    sq = np.asarray(s2).astype(np.float64) * 2.0 ** -S2
    with np.errstate(all="ignore"):
        v = (sq - s * s / c) / c
    return np.where(c == 0.0, 0.0, v)


def best_split(hist, subset, feat_bins, feat_kind, tot, S, S2, min_inst, min_gain):
    """-> (gain, position j, split index, L stats, categorical mask or None) or None; first max over (feature, split)"""
    parent = float(variance(tot[0], tot[1], tot[2], S, S2))
    best = None
    for j, f in enumerate(subset):
        nb = int(feat_bins[f])
        if nb < 2:
            continue
        raw = hist[j][:nb]
        cat = feat_kind[f] != 0
        if cat:
            with np.errstate(all="ignore"):
                cen = np.where(raw[:, 0] == 0, DBL_MAX, (raw[:, 1].astype(np.float64) * 2.0 ** -S) / raw[:, 0].astype(np.float64))
            order = np.argsort(cen, kind="stable")
        else:
            order = np.arange(nb)
        cum = np.cumsum(raw[order], axis=0)[:nb - 1]
        L, R = cum, tot[None, :] - cum
        lc, rc = L[:, 0].astype(np.float64), R[:, 0].astype(np.float64)
        il = variance(L[:, 0], L[:, 1], L[:, 2], S, S2)
        ir = variance(R[:, 0], R[:, 1], R[:, 2], S, S2)
        t = lc + rc
        with np.errstate(all="ignore"):
            g = parent - (lc / t) * il - (rc / t) * ir
        ok = (lc >= min_inst) & (rc >= min_inst) & ~(g < min_gain)
        if not ok.any():
            continue
        gv = np.where(ok, g, -np.inf)
        sp = int(np.argmax(gv))
        if best is None or gv[sp] > best[0]:
            mask = None
            if cat:
                mask = np.zeros(4, np.uint64)
                for c in order[:sp + 1]:
                    mask[c >> 6] |= np.uint64(1) << np.uint64(c & 63)
            best = (float(gv[sp]), j, sp, L[sp].copy(), mask)
    return parent, best


def grow_tree(t, bins, w, q, q2, feat_bins, feat_kind, m, max_depth, min_inst, min_gain, seed, S, S2):
    """one regression tree on binned rows (only rows with w > 0 count): {nid: node dict}"""
    F = bins.shape[1]
    nodes = {}
    frontier = [(1, np.nonzero(w > 0)[0], None)]
    level = 0
    n_bins = int(feat_bins.max())
    while frontier:
        nxt = []
        for nid, rows, _ in frontier:
            subset = oracle.feature_subset(seed, t, nid, F, m) if m < F else np.arange(F)
            hist = node_hist(bins[rows][:, subset], w[rows], q[rows], q2[rows], n_bins)
            tot = hist[0].sum(0)
            parent, best = best_split(hist, subset, feat_bins, feat_kind, tot, S, S2, min_inst, min_gain)
            gain = best[0] if best is not None else -DBL_MAX
            nd = dict(stats=tot, gain=gain, leaf=True, feat=-1, kind=0, bin_thr=0, mask=np.zeros(4, np.uint64))
            nodes[nid] = nd
            if best is None or not gain > 0.0 or level >= max_depth:
                continue
            _, j, sp, L, mask = best
            f = int(subset[j])
            nd.update(leaf=False, feat=f, kind=1 if mask is not None else 0, bin_thr=sp, mask=mask if mask is not None else nd["mask"])
            R = tot - L
            il, ir = float(variance(L[0], L[1], L[2], S, S2)), float(variance(R[0], R[1], R[2], S, S2))
            b = bins[rows, f]
            go_left = (b <= sp) if mask is None else _left_table(mask)[b]
            for child, st, imp, sel in ((2 * nid, L, il, go_left), (2 * nid + 1, R, ir, ~go_left)):
                if level + 1 == max_depth or abs(imp) < EPSILON:
                    nodes[child] = dict(stats=st, gain=0.0, leaf=True, feat=-1, kind=0, bin_thr=0, mask=np.zeros(4, np.uint64))
                else:
                    nxt.append((child, rows[sel], None))
        frontier = nxt
        level += 1
    return nodes


def _left_table(mask):
    """bin -> goes left, for a categorical split's mask"""
    return np.array([(int(mask[v >> 6]) >> (v & 63)) & 1 for v in range(256)], bool)


def walk(nodes, bins):
    """leaf node id of every binned row"""
    nid = np.ones(bins.shape[0], np.int64)
    for k in sorted(nodes):                          # parents before children
        nd = nodes[k]
        if nd["leaf"]:
            continue
        at = nid == k
        b = bins[at, nd["feat"]]
        left = (b <= nd["bin_thr"]) if nd["kind"] == 0 else _left_table(nd["mask"])[b]
        nid[at] = 2 * k + np.where(left, 0, 1)
    return nid


def leaf_value(nd, weight, S):
    st = nd["stats"]
    with np.errstate(all="ignore"):
        return weight * ((np.float64(st[1]) * 2.0 ** -S) / np.float64(st[0]))      # 0/0 = NaN for an empty node


def boost(bins, labels, W, feat_bins, feat_kind, m, max_iter, step_size, max_depth, min_inst, min_gain, seed, n_global=None):
    """GradientBoostedTrees.boost on binned rows.  W: int weights [max_iter or 1, n].  -> (trees, tree weights, F, S)"""
    n = bins.shape[0]
    S, S2 = grid_shift(n if n_global is None else n_global)
    y = np.where(np.asarray(labels) > 0, 1.0, -1.0)
    Fm = np.zeros(n)
    q, q2 = to_grid(y, S, S2)
    trees, weights = [], [1.0] + [float(step_size)] * (max_iter - 1)
    for t in range(max_iter):
        w = W[t if W.shape[0] > 1 else 0]
        nodes = grow_tree(t, bins, w, q, q2, feat_bins, feat_kind, m, max_depth, min_inst, min_gain, seed, S, S2)
        for nd in nodes.values():
            nd["payload"] = leaf_value(nd, weights[t], S)
        trees.append(nodes)
        leaf = walk(nodes, bins)
        Fm = Fm + np.array([nodes[int(i)]["payload"] for i in leaf])
        q, q2 = to_grid(residual(y, Fm), S, S2)
    return trees, weights, Fm, S


def subsample_cdf(rate):
    cdf = np.full(32, 0xFFFFFFFF, np.uint32)
    cdf[0] = int(math.floor((1.0 - rate) * 4294967296.0))
    return cdf


def fit(x, labels, arity, max_iter=20, step_size=0.1, max_depth=5, max_bins=32, min_inst=1, min_gain=0.0, subsampling_rate=1.0,
        strategy="all", seed=0):
    """end to end on a dense matrix: -> dict(trees, weights, margin, S, thresholds, n_thr, bins, feat_bins, feat_kind, m)"""
    x = np.ascontiguousarray(x, np.float64)
    n, F = x.shape
    arity = np.asarray(arity, np.int32)
    mpb, kind, m = oracle.build_metadata(n, F, 2, arity, max_bins, 1, "all" if strategy == "auto" else strategy)
    frac = min(1.0, max(mpb * mpb, 10000) / n) if (arity == 0).any() else 1.0
    thr, n_thr, _ = oracle.find_splits(x, seed, int(frac * 4294967296.0), arity, mpb)
    tp, bad = oracle.bin_rows(x, thr, n_thr, arity, mpb, labels)
    assert bad == 0
    feat_bins = np.where(arity > 0, arity, n_thr + 1).astype(np.int32)
    if subsampling_rate < 1.0:
        W = oracle.bag_weights(seed, max_iter, n, subsample_cdf(subsampling_rate)).astype(np.int64)
    else:
        W = np.ones((1, n), np.int64)
    # rows with equal (bins, label) are one record with their summed weights: the histograms are integer sums, so the trees
    # do not change, and it keeps the restatement tractable at KDD99-full size
    uniq, inv = np.unique(np.ascontiguousarray(tp[:, :F + 1]).view(np.dtype((np.void, F + 1))).ravel(), return_inverse=True)
    ub = uniq.view(np.uint8).reshape(-1, F + 1)
    Wu = np.stack([np.bincount(inv.ravel(), weights=wt, minlength=len(uniq)) for wt in W]).astype(np.int64)
    trees, weights, Fu, S = boost(ub[:, :F], ub[:, F], Wu, feat_bins, kind, m, max_iter, step_size, max_depth, min_inst, min_gain, seed,
                                  n_global=n)
    bins, Fm = tp[:, :F], Fu[inv.ravel()]
    return dict(trees=trees, weights=weights, margin=Fm, S=S, thresholds=thr, n_thr=n_thr, bins=bins, feat_bins=feat_bins,
                feat_kind=kind, m=m, max_bins=mpb)


def predict(model, bins):
    """-> (margin, raw [n, 2], probability [n, 2], prediction) as GBTClassificationModel computes them"""
    Fm = np.zeros(bins.shape[0])
    for nodes in model["trees"]:
        Fm = Fm + np.array([nodes[int(i)]["payload"] for i in walk(nodes, bins)])
    p0 = 1.0 / (1.0 + pexp(-2.0 * -Fm))
    return Fm, np.stack([-Fm, Fm], 1), np.stack([p0, 1.0 - p0], 1), (Fm > 0.0).astype(np.float64)


def export(model):
    """canonical arrays ordered by (tree, node id), as GBTModel.export gives them"""
    rows = []
    for t, nodes in enumerate(model["trees"]):
        for nid in sorted(nodes):
            rows.append((t, nid, nodes[nid]))
    return dict(tree=np.array([r[0] for r in rows], np.int32), nid=np.array([r[1] for r in rows], np.uint32),
                feat=np.array([r[2]["feat"] for r in rows], np.int32), kind=np.array([r[2]["kind"] for r in rows], np.int32),
                bin_thr=np.array([r[2]["bin_thr"] for r in rows], np.int32),
                is_leaf=np.array([1 if r[2]["leaf"] else 0 for r in rows], np.int32),
                mask=np.array([r[2]["mask"] for r in rows], np.uint64).reshape(-1, 4),
                gain=np.array([r[2]["gain"] for r in rows], np.float64), payload=np.array([r[2]["payload"] for r in rows], np.float64),
                stats=np.array([r[2]["stats"] for r in rows], np.int64).reshape(-1, 3))
