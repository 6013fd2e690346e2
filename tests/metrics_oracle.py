"""numpy restatement of Spark's BinaryClassificationMetrics and MulticlassMetrics as the evaluators use them (DESIGN.md §5b,
§6): the reference the device results are compared with.  Test infrastructure only; the product never imports it."""
import numpy as np


def binary_oracle(scores, labels=None, pos=None, neg=None, num_bins=1000):
    """-> dict(areaUnderROC, areaUnderPR, score, tp, fp, P, N): the areas and the (down-sampled) curve points of one
    segment.  Distinct scores in descending order (-0.0 == +0.0) with integer counts; numBins > 0 keeps ranks g-1, 2g-1,
    ... and the last, g = n_distinct // numBins, when g >= 2; trapezoids (x2 - x1) * (y2 + y1) / 2.0 summed in curve
    order from 0.0."""
    s = np.asarray(scores, np.float64).ravel()
    if labels is not None:
        y = np.asarray(labels, np.float64).ravel() > 0.5
        pos, neg = y.astype(np.int64), (~y).astype(np.int64)
    pos, neg = np.asarray(pos, np.int64).ravel(), np.asarray(neg, np.int64).ravel()
    keep = (pos + neg) != 0
    s, pos, neg = s[keep], pos[keep], neg[keep]
    if np.isnan(s).any():
        raise ValueError("NaN score")
    if s.size == 0:
        raise ValueError("empty dataset")
    s = np.where(s == 0.0, 0.0, s)
    uniq, inv = np.unique(s, return_inverse=True)
    dpos = np.zeros(uniq.size, np.int64); np.add.at(dpos, inv, pos)
    dneg = np.zeros(uniq.size, np.int64); np.add.at(dneg, inv, neg)
    uniq, dpos, dneg = uniq[::-1], dpos[::-1], dneg[::-1]
    nd = uniq.size
    g = nd // num_bins if num_bins > 0 else 0
    if g >= 2:
        ranks = np.arange(g - 1, nd, g)
        if ranks.size == 0 or ranks[-1] != nd - 1:
            ranks = np.append(ranks, nd - 1)
    else:
        ranks = np.arange(nd)
    ctp, cfp = np.cumsum(dpos)[ranks], np.cumsum(dneg)[ranks]
    P, N = int(dpos.sum()), int(dneg.sum())
    tpr = ctp / np.float64(P) if P else np.zeros(ranks.size)
    fpr = cfp / np.float64(N) if N else np.zeros(ranks.size)
    tot = (ctp + cfp).astype(np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        prec = np.where(tot == 0, 1.0, ctp / tot)

    def area(x, y):
        terms = (x[1:] - x[:-1]) * (y[1:] + y[:-1]) / 2.0
        return float(np.add.accumulate(np.concatenate([[0.0], terms]))[-1])

    roc = area(np.concatenate([[0.0], fpr, [1.0]]), np.concatenate([[0.0], tpr, [1.0]]))
    pr = area(np.concatenate([[0.0], tpr]), np.concatenate([[prec[0]], prec]))
    return dict(areaUnderROC=roc, areaUnderPR=pr, score=uniq[ranks], tp=ctp, fp=cfp, P=P, N=N)


def multiclass_oracle(pred, label, metric_label=0.0, beta=1.0):
    """MulticlassMetrics, label by label in plain Python floats (Spark's formulas)."""
    pred, label = np.asarray(pred, np.float64), np.asarray(label, np.float64)
    N = float(label.size)
    labels = sorted(set(label.tolist()))
    sup = {l: float((label == l).sum()) for l in labels}
    tp = {l: float(((label == l) & (pred == l)).sum()) for l in labels}
    fp = {l: float(((label != l) & (pred == l)).sum()) for l in labels}

    def precision(l):
        return 0.0 if tp[l] + fp[l] == 0 else tp[l] / (tp[l] + fp[l])

    def recall(l):
        return tp[l] / sup[l]

    def fpr(l):
        return float(np.float64(fp[l]) / np.float64(N - sup[l])) if N - sup[l] else float("nan")

    def fmeasure(l, b):
        p, r = precision(l), recall(l)
        return 0.0 if p + r == 0 else (1 + b * b) * p * r / (b * b * p + r)

    # The weighted sums use numpy's .sum() over the labels in ascending order, as metrics_from_confusion does (and as its
    # weightedPrecision / weightedRecall always have): pairwise above 8 labels, so at many labels this checks the product's
    # reduction order rather than Spark's sequential sum over its label map (whose order is a hash order anyway).
    def weighted(f):
        return float(np.array([f(l) * (sup[l] / N) for l in labels]).sum())

    out = dict(weightedFalsePositiveRate=weighted(fpr), weightedFMeasure=weighted(lambda l: fmeasure(l, beta)),
               weightedTruePositiveRate=weighted(recall),
               hammingLoss=float((pred != label).sum()) / N)
    if metric_label in sup:
        m = metric_label
        out.update(truePositiveRateByLabel=recall(m), falsePositiveRateByLabel=fpr(m), precisionByLabel=precision(m),
                   recallByLabel=recall(m), fMeasureByLabel=fmeasure(m, beta))
    return out


def log_loss_oracle(label, prob, eps=1e-15):
    label, prob = np.asarray(label), np.asarray(prob, np.float64)
    p = prob[np.arange(label.size), label.astype(np.int64)]
    loss = np.where(p < eps, -np.log(eps), np.where(p > 1 - eps, -np.log1p(-eps), -np.log(np.where(p > 0, p, 1.0))))
    return float(loss.mean())
