"""CPU checks of the evaluation semantics (DESIGN.md §5b, §6): the numpy restatement reproduces pyspark's doctest answers and
sklearn, the down-sampling edges, and the confusion-derived multiclass metrics of b200flow.forest.metrics_from_confusion."""
import numpy as np
import pytest

from metrics_oracle import binary_oracle, log_loss_oracle, multiclass_oracle

sk = pytest.importorskip("sklearn.metrics")

DOCTEST_BINARY = [(0.1, 0.0), (0.1, 1.0), (0.4, 0.0), (0.6, 0.0), (0.6, 1.0), (0.6, 1.0), (0.8, 1.0)]
DOCTEST_MULTI = [(0.0, 0.0), (0.0, 1.0), (0.0, 0.0), (1.0, 0.0), (1.0, 1.0), (1.0, 1.0), (1.0, 1.0), (2.0, 2.0), (2.0, 0.0)]
DOCTEST_LOGLOSS = [(1.0, [0.1, 0.8, 0.1]), (2.0, [0.9, 0.05, 0.05]), (0.0, [0.8, 0.2, 0.0]), (1.0, [0.3, 0.65, 0.05])]


def _cm(pred, label):
    C = int(max(np.max(pred), np.max(label))) + 1
    cm = np.zeros((C, C), np.int64)
    np.add.at(cm, (np.asarray(label, np.int64), np.asarray(pred, np.int64)), 1)
    return cm


def test_binary_doctest_answers():
    s, y = np.array(DOCTEST_BINARY).T
    o = binary_oracle(s, y)
    assert o["areaUnderROC"] == 0.7083333333333333
    assert o["areaUnderPR"] == 0.8339285714285714


@pytest.mark.parametrize("kind", ["random", "tied", "inf_negzero"])
def test_binary_roc_matches_sklearn(kind):
    rng = np.random.default_rng(7)
    n = 20000
    if kind == "random":
        s = rng.random(n)
    elif kind == "tied":
        s = rng.integers(0, 13, n) / 4.0
    else:
        s = rng.choice([-np.inf, np.inf, -0.0, 0.0, 0.5, -1.5, 2.0], n)
    y = (rng.random(n) < 0.3).astype(np.float64)
    o = binary_oracle(s, y, num_bins=0)
    want = sk.roc_auc_score(y, np.unique(s, return_inverse=True)[1])     # ranks: sklearn refuses inf, the area is the same
    assert abs(o["areaUnderROC"] - want) <= 1e-12


def test_negative_zero_is_positive_zero():
    y = np.array([1, 0, 1, 0], np.float64)
    a = binary_oracle(np.array([0.0, -0.0, 1.0, 0.0]), y, num_bins=0)
    assert a["score"].tolist() == [1.0, 0.0] and a["tp"].tolist() == [1, 2] and a["fp"].tolist() == [0, 2]


@pytest.mark.parametrize("nd_mult,extra,g", [(2, -1, 1), (2, 0, 2), (3, 1, 3)])
def test_down_sampling_edges(nd_mult, extra, g):
    bins = 5
    nd = nd_mult * bins + extra
    s = np.arange(nd, dtype=np.float64)
    y = (np.arange(nd) % 3 == 0).astype(np.float64)
    o = binary_oracle(s, y, num_bins=bins)
    assert nd // bins == g or (g == 1 and nd // bins < 2)
    full = binary_oracle(s, y, num_bins=0)
    if g == 1:
        assert len(o["score"]) == nd and o["areaUnderROC"] == full["areaUnderROC"]
    else:
        want = list(range(g - 1, nd, g))
        if want[-1] != nd - 1:
            want.append(nd - 1)                               # the final partial chunk
        assert len(o["score"]) == len(want)
        desc = s[::-1]
        assert o["score"].tolist() == desc[want].tolist()
        assert o["tp"].tolist() == np.cumsum(y[::-1] > 0.5)[want].tolist()


def test_one_class_only():
    s = np.array([0.2, 0.4, 0.4, 0.9])
    allneg = binary_oracle(s, np.zeros(4))                     # P = 0: TPR = 0 everywhere
    assert allneg["P"] == 0 and allneg["areaUnderROC"] == 0.0 and allneg["areaUnderPR"] == 0.0
    allpos = binary_oracle(s, np.ones(4))                      # N = 0: FPR = 0 until the closing (1, 1)
    assert allpos["N"] == 0 and allpos["areaUnderROC"] == 1.0 and allpos["areaUnderPR"] == 1.0


def test_oracle_rejects_nan_and_empty():
    with pytest.raises(ValueError):
        binary_oracle(np.array([0.1, np.nan]), np.array([0.0, 1.0]))
    with pytest.raises(ValueError):
        binary_oracle(np.zeros(0), np.zeros(0))


def test_multiclass_doctest_answers():
    from b200flow.forest import metrics_from_confusion
    pred, lab = np.array(DOCTEST_MULTI).T
    cm = _cm(pred, lab)
    m = metrics_from_confusion(cm)
    assert abs(m["f1"] - 0.6613756613756614) < 1e-15 and abs(m["accuracy"] - 0.6666666666666666) < 1e-15
    assert metrics_from_confusion(cm, metric_label=1.0)["truePositiveRateByLabel"] == 0.75
    assert abs(m["hammingLoss"] - 0.3333333333333333) < 1e-15
    lab_ll = np.array([r[0] for r in DOCTEST_LOGLOSS])
    prob = np.array([r[1] for r in DOCTEST_LOGLOSS])
    assert abs(log_loss_oracle(lab_ll, prob) - 0.9682005730687164) < 1e-12


@pytest.mark.parametrize("C,beta", [(2, 1.0), (5, 0.5), (23, 2.0)])
def test_multiclass_metrics_match_oracle_and_sklearn(C, beta):
    from b200flow.forest import metrics_from_confusion
    rng = np.random.default_rng(C)
    lab = rng.integers(0, C, 3000)
    lab[lab == C - 1] = 0                                        # a class never seen as a label ...
    pred = np.where(rng.random(3000) < 0.6, lab, rng.integers(0, C, 3000))   # ... but predicted
    cm = _cm(pred, lab)
    labels = sorted(set(lab.tolist()))
    p, r, f, _ = sk.precision_recall_fscore_support(lab, pred, labels=labels, beta=beta, average=None, zero_division=0)
    before = metrics_from_confusion(cm)
    for li, l in enumerate(labels):
        m = metrics_from_confusion(cm, metric_label=float(l), beta=beta)
        o = multiclass_oracle(pred, lab, metric_label=float(l), beta=beta)
        for k in ("truePositiveRateByLabel", "falsePositiveRateByLabel", "precisionByLabel", "recallByLabel", "fMeasureByLabel",
                  "weightedFalsePositiveRate", "weightedFMeasure", "weightedTruePositiveRate", "hammingLoss"):
            assert m[k] == o[k] or (np.isnan(m[k]) and np.isnan(o[k])), (k, l)
        assert abs(m["precisionByLabel"] - p[li]) < 1e-12 and abs(m["recallByLabel"] - r[li]) < 1e-12
        assert abs(m["fMeasureByLabel"] - f[li]) < 1e-12
        for k in ("f1", "accuracy", "weightedPrecision", "weightedRecall", "macroF1"):
            assert m[k] == before[k]                               # the existing metrics do not move
    assert abs(before["hammingLoss"] - sk.hamming_loss(lab, pred)) < 1e-15
    assert "recallByLabel" not in metrics_from_confusion(cm, metric_label=float(C - 1))   # not a true label


def test_evaluator_params_and_direction():
    from pyspark.ml.evaluation import BinaryClassificationEvaluator, MulticlassClassificationEvaluator
    b = BinaryClassificationEvaluator()
    assert b.getMetricName() == "areaUnderROC" and b.getNumBins() == 1000 and b.getRawPredictionCol() == "rawPrediction"
    assert b.isLargerBetter() and b.setMetricName("areaUnderPR").isLargerBetter()
    m = MulticlassClassificationEvaluator()
    assert m.getMetricLabel() == 0.0 and m.getBeta() == 1.0 and m.getEps() == 1e-15 and m.getProbabilityCol() == "probability"
    for name, larger in (("f1", True), ("recallByLabel", True), ("hammingLoss", False), ("logLoss", False)):
        assert m.copy({"metricName": name}).isLargerBetter() is larger
