"""Evaluation on the GPU: b200flow.metrics.binary_metrics (the radix sort-and-scan of csrc/metrics.cu) against the numpy
restatement with ==, the shim's BinaryClassificationEvaluator and the new MulticlassClassificationEvaluator metrics on model
predictions, the pyspark doctests through createDataFrame, and the validators with the new metrics."""
import numpy as np
import pytest
import torch

from metrics_oracle import binary_oracle, log_loss_oracle, multiclass_oracle
from test_tuning_gpu import _count_fits, _frame, _generic_cv

pytestmark = pytest.mark.gpu


def _scores(kind, S, n, rng):
    if kind == "distinct":
        return rng.permutation(S * n).reshape(S, n) / float(S * n) - 0.25
    if kind == "values1000":
        return rng.integers(0, 1000, (S, n)) / 999.0
    return rng.choice([-np.inf, np.inf, -0.0, 0.0, 1e-300, -2.5, 0.75, 3.0], (S, n))


def _check(got, want, s=None):
    roc, pr = (got["areaUnderROC"], got["areaUnderPR"]) if s is None else (got["areaUnderROC"][s], got["areaUnderPR"][s])
    cur = got["curves"] if s is None else got["curves"][s]
    assert roc == want["areaUnderROC"] and pr == want["areaUnderPR"]
    assert np.array_equal(cur["score"], want["score"]) and np.array_equal(cur["tp"], want["tp"])
    assert np.array_equal(cur["fp"], want["fp"])
    assert not np.signbit(cur["score"][cur["score"] == 0]).any()                 # -0.0 comes out as +0.0


@pytest.mark.parametrize("n", [1, 7, 100000, 1200000])
@pytest.mark.parametrize("kind", ["distinct", "values1000", "inf_negzero"])
@pytest.mark.parametrize("S", [1, 9])
def test_binary_metrics_equal_the_oracle(n, kind, S):
    from b200flow.metrics import binary_metrics
    rng = np.random.default_rng(n + S)
    sc = _scores(kind, S, n, rng)
    y = (rng.random(n) < 0.35).astype(np.float64)
    if n == 7:
        y[:2] = [0.0, 1.0]
    ts, ty = torch.from_numpy(sc).cuda(), torch.from_numpy(y).cuda()
    for bins in (0, 1, 7, 1000):
        if S == 1:
            got = binary_metrics(ts[0], ty, num_bins=bins, curves=True)
            _check(got, binary_oracle(sc[0], y, num_bins=bins))
        else:
            got = binary_metrics(ts, ty, num_bins=bins, curves=True)
            for s in range(S):
                _check(got, binary_oracle(sc[s], y, num_bins=bins), s)


def test_binary_metrics_counts_and_single_class():
    from b200flow.metrics import binary_metrics
    rng = np.random.default_rng(3)
    sc = rng.integers(0, 50, 5000) / 7.0
    pos, neg = rng.integers(0, 4, 5000), rng.integers(0, 3, 5000)           # some rows with zero counts are ignored
    got = binary_metrics(torch.from_numpy(sc).cuda(), pos=torch.from_numpy(pos).cuda(), neg=torch.from_numpy(neg).cuda(),
                         num_bins=0, curves=True)
    _check(got, binary_oracle(sc, pos=pos, neg=neg, num_bins=0))
    for y in (np.zeros(5000), np.ones(5000)):                                # P = 0, N = 0
        got = binary_metrics(torch.from_numpy(sc).cuda(), torch.from_numpy(y).cuda(), num_bins=7, curves=True)
        _check(got, binary_oracle(sc, y, num_bins=7))


def test_binary_metrics_many_segments():
    """S > 256: the segment id takes two radix passes."""
    from b200flow.metrics import binary_metrics
    rng = np.random.default_rng(300)
    S, n = 300, 257
    sc = rng.integers(0, 40, (S, n)) / 13.0
    y = (rng.random((S, n)) < 0.5).astype(np.float64)
    for bins in (0, 7):
        got = binary_metrics(torch.from_numpy(sc).cuda(), torch.from_numpy(y).cuda(), num_bins=bins, curves=True)
        for s in range(S):
            _check(got, binary_oracle(sc[s], y[s], num_bins=bins), s)


def test_binary_metrics_nan_and_empty_raise():
    from b200flow.metrics import InvalidScoresError, binary_metrics
    with pytest.raises(InvalidScoresError):
        binary_metrics(torch.tensor([0.1, float("nan"), 0.3], dtype=torch.float64, device="cuda"),
                       torch.tensor([0.0, 1.0, 1.0], dtype=torch.float64, device="cuda"))
    with pytest.raises(InvalidScoresError):
        binary_metrics(torch.zeros(0, dtype=torch.float64, device="cuda"), torch.zeros(0, dtype=torch.float64, device="cuda"))
    zero = torch.zeros(5, dtype=torch.int32, device="cuda")                  # rows, but none with a count
    with pytest.raises(InvalidScoresError):
        binary_metrics(torch.rand(5, dtype=torch.float64, device="cuda"), pos=zero, neg=zero)


def _spark():
    from pyspark.sql import SparkSession
    return SparkSession.builder.getOrCreate()


def test_doctests_through_create_data_frame():
    from pyspark.ml.evaluation import BinaryClassificationEvaluator, MulticlassClassificationEvaluator
    from pyspark.ml.linalg import Vectors
    from pyspark.sql.utils import IllegalArgumentException
    spark = _spark()
    rows = [(0.1, 0.0), (0.1, 1.0), (0.4, 0.0), (0.6, 0.0), (0.6, 1.0), (0.6, 1.0), (0.8, 1.0)]
    df = spark.createDataFrame([(Vectors.dense([1.0 - s, s]), l) for s, l in rows], ["raw", "label"])
    ev = BinaryClassificationEvaluator(rawPredictionCol="raw")
    assert ev.evaluate(df) == 0.7083333333333333
    assert ev.evaluate(df, {ev.metricName: "areaUnderPR"}) == 0.8339285714285714
    lists = spark.createDataFrame([([1.0 - s, s], l) for s, l in rows], ["raw", "label"])    # number lists work the same
    assert ev.evaluate(lists) == 0.7083333333333333
    numeric = spark.createDataFrame(rows, ["raw", "label"])                                  # a numeric score column
    assert ev.evaluate(numeric) == 0.7083333333333333
    with pytest.raises(IllegalArgumentException):
        ev.evaluate(spark.createDataFrame([(Vectors.dense([0.5]), 1.0)], ["raw", "label"]))
    with pytest.raises(IllegalArgumentException):
        ev.evaluate(spark.createDataFrame([(float("nan"), 1.0), (0.2, 0.0)], ["raw", "label"]))
    with pytest.raises(IllegalArgumentException):
        BinaryClassificationEvaluator(rawPredictionCol="raw", weightCol="w").evaluate(df)
    mc = spark.createDataFrame([(0.0, 0.0), (0.0, 1.0), (0.0, 0.0), (1.0, 0.0), (1.0, 1.0), (1.0, 1.0), (1.0, 1.0), (2.0, 2.0),
                                (2.0, 0.0)], ["prediction", "label"])
    m = MulticlassClassificationEvaluator()
    assert abs(m.evaluate(mc) - 0.6613756613756614) < 1e-15
    assert m.evaluate(mc, {m.metricName: "truePositiveRateByLabel", m.metricLabel: 1.0}) == 0.75
    assert abs(m.evaluate(mc, {m.metricName: "hammingLoss"}) - 0.3333333333333333) < 1e-15
    with pytest.raises(IllegalArgumentException):
        m.evaluate(mc, {m.metricName: "recallByLabel", m.metricLabel: 7.0})
    for bad in (float("nan"), float("inf"), -1.0):
        with pytest.raises(IllegalArgumentException):
            m.evaluate(mc, {m.metricName: "recallByLabel", m.metricLabel: bad})
    ll = spark.createDataFrame([(1.0, Vectors.dense([0.1, 0.8, 0.1])), (2.0, Vectors.dense([0.9, 0.05, 0.05])),
                                (0.0, Vectors.dense([0.8, 0.2, 0.0])), (1.0, Vectors.dense([0.3, 0.65, 0.05]))],
                               ["label", "probability"])
    assert abs(m.evaluate(ll, {m.metricName: "logLoss"}) - 0.9682005730687164) < 1e-12


def _two_class_frame(lazy):
    from pyspark.ml.feature import VectorAssembler
    df, feats = _frame(20000, 2, seed=23)
    df = VectorAssembler(inputCols=feats, outputCol="features").transform(df).select(["features", "label_num"])
    if not lazy:
        df._cols["features"].data
    return df


@pytest.mark.parametrize("lazy", [True, False])
@pytest.mark.parametrize("kind", ["rf", "dt", "lr", "nb"])
def test_binary_evaluator_on_model_predictions(kind, lazy):
    from pyspark.ml.classification import DecisionTreeClassifier, LogisticRegression, NaiveBayes, RandomForestClassifier
    from pyspark.ml.evaluation import BinaryClassificationEvaluator
    if kind in ("lr", "nb") and lazy:
        pytest.skip("LR / NB read the dense vector")
    df = _two_class_frame(lazy)
    est = {"rf": lambda: RandomForestClassifier(labelCol="label_num", maxBins=70, numTrees=8, maxDepth=6, seed=2),
           "dt": lambda: DecisionTreeClassifier(labelCol="label_num", maxBins=70, maxDepth=6),
           "lr": lambda: LogisticRegression(labelCol="label_num", maxIter=5),
           "nb": lambda: NaiveBayes(labelCol="label_num")}[kind]()
    out = est.fit(df).transform(df)
    raw = out._column_tensor("rawPrediction")[:, 1].cpu().numpy()
    lab = out._column_tensor("label_num").cpu().numpy()
    for name in ("areaUnderROC", "areaUnderPR"):
        for bins in (0, 1000):
            ev = BinaryClassificationEvaluator(labelCol="label_num", metricName=name, numBins=bins)
            assert ev.evaluate(out) == binary_oracle(raw, lab, num_bins=bins)[name], (name, bins)


@pytest.mark.parametrize("C", [5, 23])
def test_new_multiclass_metrics_on_rf_predictions(C):
    from pyspark.ml.classification import RandomForestClassifier
    from pyspark.ml.evaluation import MulticlassClassificationEvaluator
    from pyspark.ml.feature import VectorAssembler
    df, feats = _frame(20000, C, seed=C)
    df = VectorAssembler(inputCols=feats, outputCol="features").transform(df).select(["features", "label_num"])
    out = RandomForestClassifier(labelCol="label_num", maxBins=70, numTrees=6, maxDepth=5, seed=1).fit(df).transform(df)
    pred = out._column_tensor("prediction").cpu().numpy()
    lab = out._column_tensor("label_num").cpu().numpy()
    prob = out._column_tensor("probability").cpu().numpy()
    ev = MulticlassClassificationEvaluator(labelCol="label_num")
    for ml in (0.0, 1.0, float(C - 2)):
        for beta in (1.0, 0.5):
            want = multiclass_oracle(pred, lab, metric_label=ml, beta=beta)
            for name, v in want.items():
                got = ev.evaluate(out, {ev.metricName: name, ev.metricLabel: ml, ev.beta: beta})
                assert got == v or (np.isnan(got) and np.isnan(v)), (name, ml, beta)
    ll = ev.evaluate(out, {ev.metricName: "logLoss"})
    want = log_loss_oracle(lab, prob)
    assert abs(ll - want) <= 1e-12 * abs(want)


@pytest.mark.parametrize("metric", ["recallByLabel", "hammingLoss", "areaUnderROC", "areaUnderPR", "logLoss"])
def test_validators_with_new_metrics(metric, monkeypatch):
    from pyspark.ml.classification import RandomForestClassifier
    from pyspark.ml.evaluation import BinaryClassificationEvaluator, MulticlassClassificationEvaluator
    from pyspark.ml.tuning import CrossValidator, ParamGridBuilder, TrainValidationSplit
    df = _two_class_frame(True) if metric.startswith("area") else None
    if df is None:
        from pyspark.ml.feature import VectorAssembler
        d5, feats = _frame(20000, 5, seed=8)
        df = VectorAssembler(inputCols=feats, outputCol="features").transform(d5).select(["features", "label_num"])
    est = RandomForestClassifier(labelCol="label_num", maxBins=70, seed=4)
    grid = ParamGridBuilder().addGrid(est.numTrees, [2, 6]).addGrid(est.maxDepth, [1, 4, 7]).build()
    if metric.startswith("area"):
        ev = BinaryClassificationEvaluator(labelCol="label_num", metricName=metric)
    else:
        ev = MulticlassClassificationEvaluator(labelCol="label_num", metricName=metric, metricLabel=1.0)
    fits = _count_fits(monkeypatch)
    model = CrossValidator(estimator=est, estimatorParamMaps=grid, evaluator=ev, numFolds=3, seed=2019).fit(df)
    fast = metric != "logLoss"
    assert fits[0] == (3 + 1 if fast else 3 * len(grid) + 1)                 # one fit per fold on the fast path
    want = _generic_cv(est, grid, ev, df, 3, 2019)
    assert model.avgMetrics == want and len(set(want)) > 1
    best = int(np.argmax(want)) if ev.isLargerBetter() else int(np.argmin(want))
    direct = est.fit(df, grid[best])._forest.export()
    got = model.bestModel._forest.export()
    assert all(np.array_equal(got[k], direct[k]) for k in direct)
    tvs = TrainValidationSplit(estimator=est, estimatorParamMaps=grid, evaluator=ev, trainRatio=0.7, seed=5).fit(df)
    train, val = df.randomSplit([0.7, 0.3], seed=5)
    assert tvs.validationMetrics == [ev.evaluate(est.fit(train, m).transform(val)) for m in grid]


@pytest.mark.parametrize("dt", [False, True])
@pytest.mark.parametrize("lazy", [True, False])
def test_grid_binary_metrics_equal_standalone_fits(dt, lazy):
    """every (numTrees, maxDepth) point of grid_binary_metrics == fitting that point alone + transform + evaluator."""
    from pyspark.ml.classification import DecisionTreeClassifier, RandomForestClassifier
    from pyspark.ml.evaluation import BinaryClassificationEvaluator
    from pyspark.ml.tuning import _grid_on_val
    df = _two_class_frame(lazy)
    train, val = df.randomSplit([0.7, 0.3], seed=11)
    if dt:
        est = DecisionTreeClassifier(labelCol="label_num", maxBins=70)
        tree_cuts, depth_cuts = [1], [0, 2, 5, 9]
        big = est.copy({"maxDepth": 9})
    else:
        est = RandomForestClassifier(labelCol="label_num", maxBins=70, seed=4)
        tree_cuts, depth_cuts = [3, 7, 20], [0, 2, 5, 9]
        big = est.copy({"numTrees": 20, "maxDepth": 9})
    forest = big.fit(train)._forest
    for bins in (0, 1000):
        auc = _grid_on_val(forest, big, val, tree_cuts, depth_cuts, bins)
        for i, T in enumerate(tree_cuts):
            for j, d in enumerate(depth_cuts):
                m = est.fit(train, {"maxDepth": d} if dt else {"numTrees": T, "maxDepth": d}).transform(val)
                for k, name in enumerate(("areaUnderROC", "areaUnderPR")):
                    want = BinaryClassificationEvaluator(labelCol="label_num", metricName=name, numBins=bins).evaluate(m)
                    assert auc[i, j, k] == want, (T, d, name, bins)


def test_grid_binary_metrics_blocks_of_tree_cuts(monkeypatch):
    """a score budget below one tree cut's scores processes the grid one tree cut at a time: the same areas."""
    from b200flow.forest import ForestModel
    from pyspark.ml.classification import RandomForestClassifier
    from pyspark.ml.tuning import _grid_on_val
    df = _two_class_frame(True)
    est = RandomForestClassifier(labelCol="label_num", maxBins=70, seed=4, numTrees=9, maxDepth=6)
    forest = est.fit(df)._forest
    whole = _grid_on_val(forest, est, df, [2, 5, 9], [1, 3, 6], 1000)
    monkeypatch.setattr(ForestModel, "GRID_SCORE_BUDGET", 8)
    assert np.array_equal(_grid_on_val(forest, est, df, [2, 5, 9], [1, 3, 6], 1000), whole)
