"""DecisionTreeRegressor / RandomForestRegressor on the device against the numpy restatement (tests/regression_oracle.py),
bit for bit: structure, thresholds, category masks, the fp64 bits of payloads and gains, the int64 node stats, and the
predictions and leaf variances on held-out rows; de-duplication on and off, slot groups, the record-path transform;
RegressionEvaluator against the restated exact sums; and the pyspark shim with Pipeline and CrossValidator."""
import math

import numpy as np
import pytest
import torch

import oracle
import regression_oracle as ro
from b200flow import encode as enc, forest as fr, metrics as bm, regression as br, synth
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


def _fit(x, y, arity, p, dt=False):
    return (br.fit_dt_regressor if dt else br.fit_rf_regressor)(x, y, arity, p)


def _oracle(x, y, arity, p, dt=False):
    return ro.fit(x.cpu().numpy(), y.cpu().numpy(), arity, num_trees=1 if dt else p.num_trees, max_depth=p.max_depth,
                  max_bins=p.max_bins, min_inst=p.min_instances_per_node, min_gain=p.min_info_gain,
                  subsampling_rate=p.subsampling_rate, strategy="all" if dt else p.feature_subset_strategy, seed=p.seed,
                  bootstrap=not dt)


def _assert_same_model(model, want):
    got, exp = model.export(), ro.export(want)
    for k in KEYS:
        assert np.array_equal(got[k], exp[k]), k
    assert np.array_equal(got["payload"].view(np.int64), exp["payload"].view(np.int64))
    assert np.array_equal(got["gain"].view(np.int64), exp["gain"].view(np.int64))
    assert np.array_equal(model.forest.thresholds.cpu().numpy(), want["thresholds"])
    assert (model.E, model.S, model.S2) == (want["E"], want["S"], want["S2"])
    assert np.allclose(model.feature_importances(), ro.feature_importances(want, model.F), rtol=1e-12, atol=1e-15)


def _assert_same_output(model, want, x_test):
    pred, var = ro.predict_x(want, x_test.cpu().numpy())
    assert np.array_equal(model.predict(x_test).cpu().numpy().view(np.int64), pred.view(np.int64))
    if model.var_forest is not None:
        p2, v2 = model.predict_with_variance(x=x_test)
        assert np.array_equal(p2.cpu().numpy().view(np.int64), pred.view(np.int64))
        assert np.array_equal(v2.cpu().numpy().view(np.int64), var.view(np.int64))


CASES = {
    "forest": dict(),
    "decision_tree": dict(dt=True, max_depth=6),
    "depth0": dict(max_depth=0),
    "depth1": dict(max_depth=1, dt=True),
    "one_tree_forest": dict(num_trees=1),
    "subsample_all": dict(subsampling_rate=0.7, feature_subset_strategy="all"),
    "sqrt_min_inst": dict(feature_subset_strategy="sqrt", min_instances_per_node=20),
    "onethird_min_gain": dict(feature_subset_strategy="onethird", min_info_gain=0.01),
    "negative_labels": dict(label=lambda y: -3.0 * y - 0.5),
    "labels_near_1e9": dict(label=lambda y: 1e9 + 1000.0 * y, dt=True),
    "constant_labels": dict(label=lambda y: torch.full_like(y, 2.75)),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASES))
def test_device_model_equals_the_restatement(case):
    kw = dict(CASES[case])
    dt, label = kw.pop("dt", False), kw.pop("label", None)
    rec, plan, arity, x, y = _kdd(12000, 7)
    if label is not None:
        y = label(y)
    p = br.RegressorParams(**{**dict(num_trees=5, max_depth=4, max_bins=70, seed=11, feature_subset_strategy="auto"), **kw})
    model = _fit(x[:10000], y[:10000], arity, p, dt)
    want = _oracle(x[:10000], y[:10000], arity, p, dt)
    _assert_same_model(model, want)
    _assert_same_output(model, want, x[10000:])
    if case == "constant_labels":
        assert model.export()["is_leaf"].all()


@pytest.mark.gpu
@pytest.mark.parametrize("max_bins", [78, 33])
def test_cicids_f64_equals_the_restatement(max_bins):
    x, y, arity = _cicids(8000, 5)
    p = br.RegressorParams(num_trees=3, max_depth=4, max_bins=max_bins, seed=9)
    model = _fit(x, y, arity, p)
    _assert_same_model(model, _oracle(x, y, arity, p))
    dt = _fit(x, y, arity, p, dt=True)
    want = _oracle(x, y, arity, p, dt=True)
    _assert_same_model(dt, want)
    _assert_same_output(dt, want, x[:500])


@pytest.mark.gpu
def test_deduplication_slot_groups_and_record_path_give_the_same_model(monkeypatch):
    rec, plan, arity, x, y = _kdd(15000, 3)
    y = torch.round(y * 4.0) / 4.0                                   # repeated labels: records do merge
    p = br.RegressorParams(num_trees=4, max_depth=5, max_bins=70, seed=2)
    dense = _fit(x, y, arity, p)
    assert dense.train_stats["unique_rows"] < 15000
    want = dense.export()
    monkeypatch.setattr(fr, "DEDUP", False)
    rows = _fit(x, y, arity, p)
    assert rows.train_stats["unique_rows"] == 15000
    monkeypatch.setattr(fr, "DEDUP", True)
    monkeypatch.setattr(fr, "HIST_BUDGET_BYTES", 2 * 41 * 70 * 24)      # two slots per group
    grouped = _fit(x, y, arity, p)
    for other in (rows, grouped):
        got = other.export()
        for k in want:
            assert np.array_equal(np.asarray(got[k]).view(np.uint8), np.asarray(want[k]).view(np.uint8)), k
    assert torch.equal(dense.predict_records(rec, plan), dense.predict(x))
    dt = _fit(x, y, arity, p, dt=True)
    pr, vr = dt.predict_with_variance(rec=rec, plan=plan)
    pd, vd = dt.predict_with_variance(x=x)
    assert torch.equal(pr, pd) and torch.equal(vr, vd) and torch.equal(pd, dt.predict(x))
    _assert_same_model(dense, _oracle(x, y, arity, p))


@pytest.mark.gpu
def test_wide_records_without_spare_bytes_fit_without_deduplication():
    # F = 60: F + 1 = 61 leaves 3 spare bytes in the 64-byte record, too few for the label: every row stays its own record
    g = torch.Generator(device=DEV).manual_seed(4)
    x = torch.randint(0, 4, (6000, 60), device=DEV, generator=g).to(torch.float64)
    y = x[:, 0] * 1.5 - x[:, 1] + torch.randn(6000, device=DEV, generator=g, dtype=torch.float64)
    p = br.RegressorParams(num_trees=3, max_depth=4, seed=3)
    model = _fit(x, y, [0] * 60, p)
    assert model.train_stats["unique_rows"] == 6000
    _assert_same_model(model, _oracle(x, y, [0] * 60, p))


@pytest.mark.gpu
def test_non_finite_labels_are_refused():
    _, _, arity, x, y = _kdd(3000, 13)
    for bad in (float("nan"), float("inf")):
        yb = y.clone(); yb[17] = bad
        with pytest.raises(ValueError, match="finite"):
            _fit(x, yb, arity, br.RegressorParams(num_trees=2, max_bins=70))


@pytest.mark.gpu
def test_evaluator_equals_the_restatement_on_a_million_rows():
    g = torch.Generator(device=DEV).manual_seed(8)
    n = 1_200_000
    y = torch.randn(n, device=DEV, generator=g, dtype=torch.float64) * 1e3 + 50.0
    torch.manual_seed(8)
    err = torch.distributions.StudentT(torch.tensor(1.5, dtype=torch.float64)).sample((n,)).to(DEV)
    p = y + err
    yh, ph = y.cpu().numpy(), p.cpu().numpy()
    for origin in (False, True):
        got = bm.regression_metrics(y, p, through_origin=origin)
        want = ro.metrics(yh, ph, through_origin=origin)
        for k in want:
            assert got[k] == want[k], (k, got[k], want[k])
    # shard layout does not matter: the sums are exact
    perm = torch.randperm(n, device=DEV, generator=g)
    assert bm.regression_metrics(y[perm], p[perm]) == bm.regression_metrics(y, p)
    p2 = p.clone(); p2[5] = float("nan")
    assert all(math.isnan(v) for v in bm.regression_metrics(y, p2).values())
    assert all(math.isnan(v) for v in bm.regression_metrics(y[:0], p[:0]).values())


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
def test_shim_pipeline_evaluator_and_cross_validator():
    from pyspark.ml import Pipeline
    from pyspark.ml.evaluation import RegressionEvaluator
    from pyspark.ml.feature import IllegalArgumentException, _materialize
    from pyspark.ml.regression import DecisionTreeRegressor, RandomForestRegressor
    from pyspark.ml.tuning import CrossValidator, ParamGridBuilder, fold_frames
    df = _frame(20000, 5)
    rf = RandomForestRegressor(labelCol="dst_bytes", numTrees=4, maxBins=70, seed=3)
    model = Pipeline(stages=_stages() + [rf]).fit(df)
    out = model.transform(df)
    m = model.stages[-1]
    assert m.getNumTrees == 4 and m.treeWeights == [1.0] * 4 and m.numFeatures == 40
    assert abs(float(np.sum(m.featureImportances.toArray())) - 1.0) < 1e-12 and "Tree 3 (weight 1.0)" in m.toDebugString
    assert repr(m) == "RandomForestRegressionModel with 4 trees"
    feats = Pipeline(stages=_stages()).fit(df).transform(df)
    dense = m.transform(feats.select("features", "dst_bytes"))
    assert torch.equal(out._column_tensor("prediction"), dense._column_tensor("prediction"))
    ev = RegressionEvaluator(labelCol="dst_bytes")
    rmse = ev.evaluate(out)
    y = out._column_tensor("dst_bytes").to(torch.float64)
    assert rmse == ro.metrics(y.cpu().numpy(), out._column_tensor("prediction").cpu().numpy())["rmse"]
    dt = DecisionTreeRegressor(labelCol="dst_bytes", maxBins=70, varianceCol="v", seed=1).fit(feats)
    o2 = dt.transform(feats)
    v = o2._column_tensor("v")
    assert torch.equal(v, dt._reg.predict_with_variance(x=_materialize(feats, "features"))[1])
    assert v.shape[0] == 20000 and bool((v >= -1e-9 * v.abs().max()).all())      # Variance.calculate: rounding may dip below 0
    assert dt.depth <= 5 and dt.numNodes == dt.totalNumNodes and "DecisionTreeRegressionModel of depth" in dt.toDebugString
    with pytest.raises(IllegalArgumentException):
        DecisionTreeRegressor(labelCol="dst_bytes", impurity="gini").fit(feats)
    # CrossValidator over numTrees x maxDepth with rmse: the generic path, and the argmin wins
    r2 = RandomForestRegressor(labelCol="dst_bytes", maxBins=70, seed=4)
    grid = ParamGridBuilder().addGrid(r2.numTrees, [2, 5]).addGrid(r2.maxDepth, [2, 4]).build()
    sel = feats.select("features", "dst_bytes")
    cvm = CrossValidator(estimator=r2, estimatorParamMaps=grid, evaluator=ev, numFolds=2, seed=9).fit(sel)
    want = [0.0] * 4
    for train, val in fold_frames(sel, 2, 9):
        for i, pm in enumerate(grid):
            want[i] += ev.evaluate(r2.fit(train, pm).transform(val))
    assert cvm.avgMetrics == [v / 2 for v in want]
    best = int(np.argmin(cvm.avgMetrics))
    assert cvm.bestModel.getNumTrees == grid[best][r2.numTrees]
