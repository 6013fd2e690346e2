"""GBTRegressor on the device against the numpy restatement (tests/gbt_regression_oracle.py), bit for bit: structure,
thresholds, category masks, the fp64 bits of payloads and gains, the int64 node stats, every tree's grid exponent, the
training margins and the held-out predictions; de-duplication on and off, slot groups, records without spare bytes and the
record-path transform; evaluateEachIteration against the evaluator on every prefix model; and the pyspark shim with
Pipeline, CrossValidator and TrainValidationSplit."""
import numpy as np
import pytest
import torch

import gbt_regression_oracle as gro
import regression_oracle as ro
from b200flow import encode as enc, forest as fr, gbt_regression as bgr, metrics as bm, synth
from util import kdd_luts_gpu, kdd_plan

DEV = "cuda"
KEYS = ("tree", "nid", "feat", "kind", "bin_thr", "is_leaf", "mask", "stats")


def _kdd(n, seed):
    rec, dicts = synth.make_kdd(n, 2, seed=seed, device=DEV)
    schema = synth.kdd_schema()
    luts, ordered = kdd_luts_gpu(rec, schema, dicts)
    plan = kdd_plan(schema, luts, ordered)
    arity = [0] * 38 + [len(ordered[c]) for c in synth.KDD_CATEGORICAL]
    x, _, _ = plan.run(rec, torch.float64)
    return rec, plan, arity, x, torch.log1p(x[:, 2])              # label: log1p(dst_bytes)


def _cicids(n, seed):
    rec, dicts = synth.make_cicids(n, 2, seed=seed, device=DEV, dtype="f64")
    schema = synth.cicids_schema(78, "f64")
    counts = enc.category_counts(rec, schema, "Label", 2).cpu().numpy()
    ordered, lut = enc.string_index_order(counts, dicts["Label"])
    plan = enc.EncodePlan(schema)
    for f in schema.names[:-1]:
        plan.add_numeric(f)
    plan.set_label("Label", lut)
    x, _, _ = plan.run(rec, torch.float64)
    return x[:, 1:].contiguous(), x[:, 0].contiguous(), [0] * 77        # label: the first column (Flow Duration)


def _oracle(x, y, arity, p):
    return gro.fit(x.cpu().numpy(), y.cpu().numpy(), arity, max_iter=p.max_iter, step_size=p.step_size, max_depth=p.max_depth,
                   max_bins=p.max_bins, min_inst=p.min_instances_per_node, min_gain=p.min_info_gain,
                   subsampling_rate=p.subsampling_rate, strategy=p.feature_subset_strategy, seed=p.seed, loss=p.loss)


def _row_margin(model):
    m = model.train_margin
    return (m if model.train_uid is None else m[model.train_uid.long()]).cpu().numpy()


def _assert_same_model(model, want):
    got, exp = model.export(), gro.export(want)
    for k in KEYS:
        assert np.array_equal(got[k], exp[k]), k
    assert np.array_equal(got["payload"].view(np.int64), exp["payload"].view(np.int64))
    assert np.array_equal(got["gain"].view(np.int64), exp["gain"].view(np.int64))
    assert np.array_equal(model.forest.thresholds.cpu().numpy(), want["thresholds"])
    assert (model.E, model.S, model.S2) == (want["E"], want["S"], want["S2"])
    assert model.train_stats["E"] == want["E"] and model.tree_weights == want["weights"]
    assert np.array_equal(_row_margin(model).view(np.int64), want["margin"].view(np.int64))
    assert np.allclose(model.feature_importances(), gro.feature_importances(want, model.F), rtol=1e-12, atol=1e-15)


CASES = {
    "squared": dict(),
    "absolute": dict(loss="absolute"),
    "depth0": dict(max_depth=0),
    "depth1_absolute": dict(max_depth=1, loss="absolute"),
    "one_iteration": dict(max_iter=1),
    "subsample_sqrt": dict(subsampling_rate=0.7, feature_subset_strategy="sqrt"),
    "min_inst": dict(min_instances_per_node=20),
    "min_gain": dict(min_info_gain=0.01),
    "negative_labels": dict(label=lambda y: -3.0 * y - 0.5),
    "labels_near_1e9": dict(label=lambda y: 1e9 + 1000.0 * y),
    "constant_labels": dict(label=lambda y: torch.full_like(y, 2.75)),
    "constant_labels_absolute": dict(label=lambda y: torch.full_like(y, -6.5), loss="absolute"),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASES))
def test_device_model_equals_the_restatement(case):
    kw = dict(CASES[case])
    label = kw.pop("label", None)
    rec, plan, arity, x, y = _kdd(12000, 7)
    if label is not None:
        y = label(y)
    p = bgr.GBTRegressorParams(**{**dict(max_iter=5, step_size=0.3, max_depth=4, max_bins=70, seed=11), **kw})
    model = bgr.fit_gbt_regressor(x[:10000], y[:10000], arity, p)
    want = _oracle(x[:10000], y[:10000], arity, p)
    _assert_same_model(model, want)
    pred = model.predict(x[10000:])
    assert np.array_equal(pred.cpu().numpy().view(np.int64), gro.predict_x(want, x[10000:].cpu().numpy()).view(np.int64))
    if case.startswith("constant_labels"):
        assert model.export()["is_leaf"].all() and model.E[1:] == [0] * 4
    if case == "absolute":                              # r = ±1 from iteration 1 on: the grid changes scale after tree 0
        assert model.E[0] >= 3 and model.E[1:] == [0] * 4


@pytest.mark.gpu
@pytest.mark.parametrize("max_bins", [78, 33])
def test_cicids_f64_equals_the_restatement(max_bins):
    x, y, arity = _cicids(8000, 5)
    for loss in ("squared", "absolute"):
        p = bgr.GBTRegressorParams(max_iter=3, max_depth=4, max_bins=max_bins, seed=9, loss=loss)
        model = bgr.fit_gbt_regressor(x, y, arity, p)
        want = _oracle(x, y, arity, p)
        _assert_same_model(model, want)
        assert np.array_equal(model.predict(x[:500]).cpu().numpy().view(np.int64),
                              gro.predict_x(want, x[:500].cpu().numpy()).view(np.int64))


@pytest.mark.gpu
def test_deduplication_slot_groups_and_record_path_give_the_same_model(monkeypatch):
    rec, plan, arity, x, y = _kdd(15000, 3)
    y = torch.round(y * 4.0) / 4.0                                   # repeated labels: records do merge
    p = bgr.GBTRegressorParams(max_iter=4, max_depth=5, max_bins=70, seed=2, subsampling_rate=0.8)
    dense = bgr.fit_gbt_regressor(x, y, arity, p)
    assert dense.train_stats["unique_rows"] < 15000
    want = dense.export()
    monkeypatch.setattr(fr, "DEDUP", False)
    rows = bgr.fit_gbt_regressor(x, y, arity, p)
    assert rows.train_stats["unique_rows"] == 15000
    monkeypatch.setattr(fr, "DEDUP", True)
    monkeypatch.setattr(fr, "HIST_BUDGET_BYTES", 2 * 41 * 70 * 24)      # two slots per group
    grouped = bgr.fit_gbt_regressor(x, y, arity, p)
    for other in (rows, grouped):
        got = other.export()
        for k in want:
            assert np.array_equal(np.asarray(got[k]).view(np.uint8), np.asarray(want[k]).view(np.uint8)), k
        assert other.E == dense.E
        assert np.array_equal(_row_margin(other).view(np.int64), _row_margin(dense).view(np.int64))
    assert torch.equal(dense.predict_records(rec, plan), dense.predict(x))
    _assert_same_model(dense, _oracle(x, y, arity, p))


@pytest.mark.gpu
def test_wide_records_without_spare_bytes_fit_without_deduplication():
    # F = 60: F + 1 = 61 leaves 3 spare bytes in the 64-byte record, too few for the label: every row stays its own record
    g = torch.Generator(device=DEV).manual_seed(4)
    x = torch.randint(0, 4, (6000, 60), device=DEV, generator=g).to(torch.float64)
    y = x[:, 0] * 1.5 - x[:, 1] + torch.randn(6000, device=DEV, generator=g, dtype=torch.float64)
    for loss in ("squared", "absolute"):
        p = bgr.GBTRegressorParams(max_iter=3, max_depth=4, seed=3, loss=loss)
        model = bgr.fit_gbt_regressor(x, y, [0] * 60, p)
        assert model.train_stats["unique_rows"] == 6000
        _assert_same_model(model, _oracle(x, y, [0] * 60, p))


@pytest.mark.gpu
def test_non_finite_labels_and_huge_residuals_are_refused():
    _, _, arity, x, y = _kdd(3000, 13)
    for bad in (float("nan"), float("inf"), float("-inf")):
        yb = y.clone(); yb[17] = bad
        with pytest.raises(ValueError, match="finite"):
            bgr.fit_gbt_regressor(x, yb, arity, bgr.GBTRegressorParams(max_iter=2, max_bins=70))
    yh = torch.where(torch.arange(3000, device=DEV) % 2 == 0, 0.9, -0.9).to(torch.float64) * 2.0 ** 300
    with pytest.raises(ValueError, match="residual"):                 # depth 0: tree 0 is ~0, so r = 2y is beyond 2^300
        bgr.fit_gbt_regressor(x, yh, arity, bgr.GBTRegressorParams(max_iter=2, max_depth=0, max_bins=70))


@pytest.mark.gpu
@pytest.mark.parametrize("loss", ["squared", "absolute"])
def test_evaluate_each_iteration_equals_the_evaluator_on_every_prefix(loss):
    rec, plan, arity, x, y = _kdd(12000, 21)
    p = bgr.GBTRegressorParams(max_iter=5, max_depth=4, max_bins=70, seed=6, loss=loss, subsampling_rate=0.9)
    model = bgr.fit_gbt_regressor(x[:9000], y[:9000], arity, p)
    xt, yt = x[9000:], y[9000:]
    key = "mse" if loss == "squared" else "mae"
    prefixes = gro.prefix_predictions_x(_oracle(x[:9000], y[:9000], arity, p), xt.cpu().numpy())
    for metric_loss, k in (("squared", "mse"), ("absolute", "mae")):
        got = model.evaluate_each_iteration(xt, yt, metric_loss)
        assert got == [ro.metrics(yt.cpu().numpy(), pr)[k] for pr in prefixes], metric_loss
    # a model fitted with fewer iterations is the prefix: its evaluator value is the same entry, bit for bit
    every = model.evaluate_each_iteration(xt, yt, loss)
    for T in (1, 3):
        short = bgr.fit_gbt_regressor(x[:9000], y[:9000], arity, bgr.GBTRegressorParams(**{**p.__dict__, "max_iter": T}))
        assert bm.regression_metrics(yt, short.predict(xt))[key] == every[T - 1]
    assert bm.regression_metrics(yt, model.predict(xt))[key] == every[-1]


def _frame(n, seed):
    from pyspark.sql import DataFrame
    rec, dicts = synth.make_kdd(n, 2, seed=seed, device="cuda:0")
    return DataFrame.fromRecords(rec, synth.kdd_schema(), dicts)


def _stages():
    from pyspark.ml.feature import StringIndexer, VectorAssembler
    cats = synth.KDD_CATEGORICAL
    st = [StringIndexer(inputCol=c, outputCol=c + "_num") for c in cats]
    nums = [c for c in synth.KDD_COLUMNS if c not in cats + ["label", "dst_bytes"]]
    st.append(VectorAssembler(inputCols=nums + [c + "_num" for c in cats], outputCol="features"))
    return st


@pytest.mark.gpu
def test_shim_pipeline_evaluator_and_model_selection():
    from pyspark.ml import Pipeline
    from pyspark.ml.evaluation import RegressionEvaluator
    from pyspark.ml.feature import IllegalArgumentException
    from pyspark.ml.regression import GBTRegressionModel, GBTRegressor
    from pyspark.ml.tuning import CrossValidator, ParamGridBuilder, TrainValidationSplit, fold_frames
    df = _frame(20000, 5)
    gb = GBTRegressor(labelCol="dst_bytes", maxIter=4, maxBins=70, seed=3)
    model = Pipeline(stages=_stages() + [gb]).fit(df)
    out = model.transform(df)
    m = model.stages[-1]
    assert isinstance(m, GBTRegressionModel)
    assert m.getNumTrees == 4 and m.treeWeights == [1.0, 0.1, 0.1, 0.1] and m.numFeatures == 40
    assert m.totalNumNodes == m._reg.n_nodes
    assert abs(float(np.sum(m.featureImportances.toArray())) - 1.0) < 1e-12
    dbg = m.toDebugString
    assert dbg.startswith("GBTRegressionModel with 4 trees") and "Tree 3 (weight 0.1)" in dbg
    ex = m._reg.export()
    leaf0 = np.nonzero((ex["tree"] == 0) & (ex["is_leaf"] == 1))[0][0]
    assert ("Predict: %r" % float(m._reg.leaf_values(ex)[leaf0])) in dbg
    assert repr(m) == "GBTRegressionModel with 4 trees"
    feats = Pipeline(stages=_stages()).fit(df).transform(df)
    sel = feats.select("features", "dst_bytes")
    dense = m.transform(sel)
    assert torch.equal(out._column_tensor("prediction"), dense._column_tensor("prediction"))
    ev = RegressionEvaluator(labelCol="dst_bytes", metricName="mse")
    each = m.evaluateEachIteration(sel, "squared")
    assert len(each) == 4 and each[-1] == ev.evaluate(out)
    assert m.evaluateEachIteration(sel, "absolute")[-1] == RegressionEvaluator(labelCol="dst_bytes", metricName="mae").evaluate(out)
    with pytest.raises(IllegalArgumentException):
        m.evaluateEachIteration(sel, "huber")
    with pytest.raises(IllegalArgumentException):
        GBTRegressor(labelCol="dst_bytes", lossType="huber").fit(sel)
    # CrossValidator over maxIter x maxDepth: the generic path, and the argmin wins
    g2 = GBTRegressor(labelCol="dst_bytes", maxBins=70, seed=4)
    grid = ParamGridBuilder().addGrid(g2.maxIter, [2, 5]).addGrid(g2.maxDepth, [2, 4]).build()
    cvm = CrossValidator(estimator=g2, estimatorParamMaps=grid, evaluator=ev, numFolds=2, seed=9).fit(sel)
    want = [0.0] * 4
    for train, val in fold_frames(sel, 2, 9):
        for i, pm in enumerate(grid):
            want[i] += ev.evaluate(g2.fit(train, pm).transform(val))
    assert cvm.avgMetrics == [v / 2 for v in want]
    best = int(np.argmin(cvm.avgMetrics))
    assert cvm.bestModel.getNumTrees == grid[best][g2.maxIter]
    tvm = TrainValidationSplit(estimator=g2, estimatorParamMaps=grid, evaluator=ev, trainRatio=0.75, seed=2).fit(sel)
    assert len(tvm.validationMetrics) == 4 and isinstance(tvm.bestModel, GBTRegressionModel)
