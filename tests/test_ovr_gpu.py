"""OneVsRest on the device.  The class-batched GBT trainer (b200flow.gbt.fit_gbt_ovr) against K separate binary fits on the
relabelled rows, bit for bit: structure, thresholds, the fp64 bits of payloads and gains, the int64 node stats and the tree
weights; one case also against the numpy restatement (tests/gbt_oracle.py).  The joint transform against the sub-models'
transforms.  The pyspark shim: OneVsRest(GBTClassifier) against hand-made per-class fits, the generic path (LogisticRegression,
NaiveBayes, more than 256 classes), the evaluator and CrossValidator."""
import numpy as np
import pytest
import torch

import gbt_oracle as go
from b200flow import encode as enc, forest as fr, gbt as bg, synth
from util import kdd_luts_gpu, kdd_plan

DEV = "cuda"


def _kdd(n, seed, n_classes=5):
    rec, dicts = synth.make_kdd(n, n_classes, seed=seed, device=DEV)
    schema = synth.kdd_schema()
    luts, ordered = kdd_luts_gpu(rec, schema, dicts)
    plan = kdd_plan(schema, luts, ordered)
    arity = [0] * 38 + [len(ordered[c]) for c in synth.KDD_CATEGORICAL]
    return rec, plan, arity, len(ordered["label"])


def _cicids(n, seed, n_classes=15):
    rec, dicts = synth.make_cicids(n, n_classes, seed=seed, device=DEV, dtype="f64")
    schema = synth.cicids_schema(78, "f64")
    counts = enc.category_counts(rec, schema, "Label", n_classes).cpu().numpy()
    ordered, lut = enc.string_index_order(counts, dicts["Label"])
    plan = enc.EncodePlan(schema)
    for f in schema.names[:-1]:
        plan.add_numeric(f)
    plan.set_label("Label", lut)
    return rec, plan, [0] * 78, len(ordered)


def _assert_same_export(a, b):
    ea, eb = a.export(), b.export()
    assert sorted(ea) == sorted(eb)
    for k in ea:
        assert np.array_equal(np.asarray(ea[k]).view(np.uint8), np.asarray(eb[k]).view(np.uint8)), k
    assert a.tree_weights == b.tree_weights
    assert torch.equal(a.forest.thresholds, b.forest.thresholds)


def _assert_equals_separate_fits(ovr, x, y, K, arity, p):
    assert len(ovr.models) == K
    for k in range(K):
        _assert_same_export(ovr.models[k], bg.fit_gbt(x, (y == k).to(torch.int32), arity, p))


def _spark_argmax(r):
    """Vector.argmax row by row, in plain Python: index 0 first, then only a strictly greater value moves it"""
    out = np.zeros(r.shape[0])
    for i, row in enumerate(r.tolist()):
        best, arg = row[0], 0
        for k, v in enumerate(row[1:], 1):
            if v > best:
                best, arg = v, k
        out[i] = arg
    return out


CASES = {
    "default": dict(),
    "subsample_sqrt": dict(subsampling_rate=0.7, feature_subset_strategy="sqrt"),
    "depth0": dict(max_depth=0, max_iter=3),
    "depth1": dict(max_depth=1),
    "one_iteration": dict(max_iter=1, max_depth=6),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASES))
def test_batched_fit_equals_the_separate_fits(case):
    rec, plan, arity, K = _kdd(10000, 7)
    x, y, _ = plan.run(rec, torch.float64)
    kw = dict(max_iter=5, max_depth=4, max_bins=70, seed=11)
    kw.update(CASES[case])
    p = bg.GBTParams(**kw)
    ovr = bg.fit_gbt_ovr(x, y, K, arity, p)
    _assert_equals_separate_fits(ovr, x, y, K, arity, p)
    # the training margins of class k are its separate fit's, row by row
    for k in range(K):
        m = ovr.models[k]
        assert torch.equal(m.train_margin[m.train_uid.long()].view(torch.int64), m.margin(x).view(torch.int64))


@pytest.mark.gpu
def test_every_sub_model_equals_the_restatement():
    rec, plan, arity, K = _kdd(6000, 29)
    x, y, _ = plan.run(rec, torch.float64)
    p = bg.GBTParams(max_iter=4, max_depth=4, max_bins=70, subsampling_rate=0.8, feature_subset_strategy="sqrt", seed=5)
    ovr = bg.fit_gbt_ovr(x, y, K, arity, p)
    xn, yn = x.cpu().numpy(), y.cpu().numpy()
    for k in range(K):
        want = go.fit(xn, (yn == k).astype(np.int32), arity, max_iter=p.max_iter, step_size=p.step_size, max_depth=p.max_depth,
                      max_bins=p.max_bins, subsampling_rate=p.subsampling_rate, strategy=p.feature_subset_strategy, seed=p.seed)
        got, exp = ovr.models[k].export(), go.export(want)
        for key in ("tree", "nid", "feat", "kind", "bin_thr", "is_leaf", "mask", "stats"):
            assert np.array_equal(got[key], exp[key]), (k, key)
        assert np.array_equal(got["payload"].view(np.int64), exp["payload"].view(np.int64)), k
        assert np.array_equal(got["gain"].view(np.int64), exp["gain"].view(np.int64)), k
        assert ovr.models[k].tree_weights == want["weights"]


@pytest.mark.gpu
def test_class_absent_from_the_training_rows():
    rec, plan, arity, K = _kdd(8000, 3)
    x, y, _ = plan.run(rec, torch.float64)
    p = bg.GBTParams(max_iter=4, max_depth=3, max_bins=70, seed=8)
    ovr = bg.fit_gbt_ovr(x, y, K + 1, arity, p)                # class K: in the metadata, on no row
    _assert_equals_separate_fits(ovr, x, y, K + 1, arity, p)
    raw, _ = ovr.predict(x)
    assert bool((raw[:, K] < 0).all())


@pytest.mark.gpu
def test_record_path_equals_dense_path_and_transforms_match_the_sub_models():
    rec, plan, arity, K = _kdd(14000, 17)
    x, y, _ = plan.run(rec, torch.float64)
    p = bg.GBTParams(max_iter=5, max_depth=5, max_bins=70, seed=2)
    dense = bg.fit_gbt_ovr(x[:12000], y[:12000], K, arity, p)
    fused = bg.fit_gbt_ovr_records(rec[:12000].contiguous(), plan, K, arity, p)
    assert fused.train_stats["unique_rows"] < 12000
    for a, b in zip(dense.models, fused.models):
        _assert_same_export(a, b)
    held_x, held_rec = x[12000:], rec[12000:].contiguous()
    for model, (raw, pred) in ((dense, dense.predict(held_x)), (fused, fused.predict_records(held_rec, plan))):
        assert raw.shape == (2000, K)
        for k in range(K):
            want = model.models[k].predict(held_x)[0][:, 1]
            assert torch.equal(raw[:, k].view(torch.int64), want.view(torch.int64)), k
        assert np.array_equal(pred.cpu().numpy(), _spark_argmax(raw.cpu().numpy()))


@pytest.mark.gpu
def test_cicids_f64_records_fifteen_classes():
    rec, plan, arity, K = _cicids(8000, 5)
    assert K == 15
    x, y, _ = plan.run(rec, torch.float64)
    p = bg.GBTParams(max_iter=3, max_depth=4, max_bins=78, seed=9)
    ovr = bg.fit_gbt_ovr_records(rec, plan, K, arity, p)
    _assert_equals_separate_fits(ovr, x, y, K, arity, p)


@pytest.mark.gpu
def test_histogram_budget_slot_groups_give_the_same_models(monkeypatch):
    rec, plan, arity, K = _kdd(10000, 19)
    x, y, _ = plan.run(rec, torch.float64)
    p = bg.GBTParams(max_iter=3, max_depth=5, max_bins=70, seed=6)
    want = bg.fit_gbt_ovr(x, y, K, arity, p)
    monkeypatch.setattr(fr, "HIST_BUDGET_BYTES", 3 * 41 * 70 * 24)      # three slots per group: groups cut across classes
    got = bg.fit_gbt_ovr(x, y, K, arity, p)
    for a, b in zip(want.models, got.models):
        _assert_same_export(a, b)


@pytest.mark.gpu
def test_a_label_beyond_the_class_count_is_refused():
    rec, plan, arity, K = _kdd(3000, 13)
    x, y, _ = plan.run(rec, torch.float64)
    with pytest.raises(ValueError, match="not in"):
        bg.fit_gbt_ovr(x, y, K - 1, arity, bg.GBTParams(max_iter=2, max_depth=2, max_bins=70))


# ------------------------------------------------------------------ the shim
def _frame(n, seed, n_classes=5):
    from pyspark.sql import DataFrame
    rec, dicts = synth.make_kdd(n, n_classes, seed=seed, device="cuda:0")
    return DataFrame.fromRecords(rec, synth.kdd_schema(), dicts)


def _stages():
    from pyspark.ml.feature import StringIndexer, VectorAssembler
    cats = synth.KDD_CATEGORICAL
    st = [StringIndexer(inputCol=c, outputCol=c + "_num") for c in cats + ["label"]]
    nums = [c for c in synth.KDD_COLUMNS if c not in cats + ["label"]]
    st.append(VectorAssembler(inputCols=nums + [c + "_num" for c in cats], outputCol="features"))
    return st


def _relabelled(df, lcol, k, name="bin_label"):
    from pyspark.sql import ColumnData
    cols = dict(df._cols)
    y = df._column_tensor(lcol)
    cols[name] = ColumnData("numeric", (y == k).to(torch.float64), "f64", {"ml_attr": {"type": "nominal", "vals": ["0.0", "1.0"]}})
    return df._with(cols=cols)


@pytest.mark.gpu
def test_shim_gbt_equals_hand_made_fits_and_evaluates():
    from pyspark.ml import Pipeline
    from pyspark.ml.classification import GBTClassifier, OneVsRest
    from pyspark.ml.evaluation import MulticlassClassificationEvaluator
    df = _frame(15000, 5)
    gbt = GBTClassifier(maxIter=4, maxDepth=4, maxBins=70)
    model = Pipeline(stages=_stages() + [OneVsRest(classifier=gbt, labelCol="label_num")]).fit(df)
    ovr = model.stages[-1]
    assert ovr._joint is not None and ovr.numClasses == 5
    out = model.transform(df)
    feats = Pipeline(stages=_stages()).fit(df).transform(df)
    raw = out._column_tensor("rawPrediction")
    assert "probability" not in out.columns
    for k in range(5):
        hand = GBTClassifier(maxIter=4, maxDepth=4, maxBins=70, labelCol="bin_label").fit(_relabelled(feats, "label_num", k))
        sub = ovr.models[k]
        a, b = sub._gbt.export(), hand._gbt.export()
        for key in a:
            assert np.array_equal(np.asarray(a[key]).view(np.uint8), np.asarray(b[key]).view(np.uint8)), (k, key)
        assert sub.toDebugString == hand.toDebugString
        assert np.array_equal(sub.featureImportances.toArray(), hand.featureImportances.toArray())
        hraw = hand.transform(feats)._column_tensor("rawPrediction")[:, 1]
        assert torch.equal(raw[:, k].view(torch.int64), hraw.view(torch.int64))
        sraw = sub.transform(feats)._column_tensor("rawPrediction")[:, 1]
        assert torch.equal(sraw.view(torch.int64), hraw.view(torch.int64))
    acc = MulticlassClassificationEvaluator(labelCol="label_num", metricName="accuracy").evaluate(out)
    f1 = MulticlassClassificationEvaluator(labelCol="label_num").evaluate(out)
    assert acc > 0.8 and 0.0 < f1 <= 1.0


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["lr", "nb"])
def test_shim_generic_path_equals_the_hand_loop(which):
    from pyspark.ml import Pipeline
    from pyspark.ml.classification import LogisticRegression, NaiveBayes, OneVsRest
    from pyspark.ml.evaluation import MulticlassClassificationEvaluator
    df = _frame(6000, 9)
    feats = Pipeline(stages=_stages()).fit(df).transform(df).select("features", "label_num")
    make = (lambda **kw: LogisticRegression(maxIter=15, **kw)) if which == "lr" else (lambda **kw: NaiveBayes(**kw))
    ovr = OneVsRest(classifier=make(), labelCol="label_num").fit(feats)
    assert ovr._joint is None and len(ovr.models) == 5
    out = ovr.transform(feats)
    raw = out._column_tensor("rawPrediction")
    for k in range(5):
        hand = make(labelCol="bin_label").fit(_relabelled(feats, "label_num", k))
        want = hand.transform(feats)._column_tensor("rawPrediction")[:, 1]
        assert torch.equal(raw[:, k].view(torch.int64), want.view(torch.int64)), k
    assert np.array_equal(out._column_tensor("prediction").cpu().numpy(), _spark_argmax(raw.cpu().numpy()))
    MulticlassClassificationEvaluator(labelCol="label_num").evaluate(out)


@pytest.mark.gpu
def test_shim_cross_validator_over_the_inner_classifier():
    from pyspark.ml import Pipeline
    from pyspark.ml.classification import GBTClassifier, OneVsRest
    from pyspark.ml.evaluation import MulticlassClassificationEvaluator
    from pyspark.ml.tuning import CrossValidator, ParamGridBuilder, fold_frames
    df = _frame(8000, 21)
    sel = Pipeline(stages=_stages()).fit(df).transform(df).select("features", "label_num")
    gbt = GBTClassifier(maxIter=3, maxBins=70, seed=4)
    ovr = OneVsRest(classifier=gbt, labelCol="label_num")
    grid = ParamGridBuilder().addGrid(gbt.maxDepth, [2, 3]).build()
    ev = MulticlassClassificationEvaluator(labelCol="label_num")
    cvm = CrossValidator(estimator=ovr, estimatorParamMaps=grid, evaluator=ev, numFolds=2, seed=9).fit(sel)
    want = [0.0, 0.0]
    for train, val in fold_frames(sel, 2, 9):
        for i, depth in enumerate([2, 3]):
            m = OneVsRest(classifier=GBTClassifier(maxIter=3, maxBins=70, seed=4, maxDepth=depth), labelCol="label_num").fit(train)
            want[i] += ev.evaluate(m.transform(val))
    assert cvm.avgMetrics == [v / 2 for v in want]
    assert cvm.bestModel.models[0]._gbt.export()["nid"].max() < 16       # the best model's trees have at most depth 3


@pytest.mark.gpu
def test_more_than_256_classes_take_the_generic_path():
    from pyspark.ml import Pipeline
    from pyspark.ml.classification import GBTClassifier, OneVsRest
    from pyspark.sql import ColumnData
    df = _frame(1200, 2)
    feats = Pipeline(stages=_stages()).fit(df).transform(df).select("features")
    cols = dict(feats._cols)
    y = torch.arange(1200, device="cuda:0", dtype=torch.float64).remainder(257)
    cols["label"] = ColumnData("numeric", y, "f64")
    frame = feats._with(cols=cols)
    model = OneVsRest(classifier=GBTClassifier(maxIter=1, maxDepth=1, maxBins=70)).fit(frame)
    assert model._joint is None and model.numClasses == 257
    out = model.transform(frame)
    raw = out._column_tensor("rawPrediction")
    assert raw.shape == (1200, 257)
    hand = GBTClassifier(maxIter=1, maxDepth=1, maxBins=70, labelCol="bin_label").fit(_relabelled(frame, "label", 256))
    want = hand.transform(frame)._column_tensor("rawPrediction")[:, 1]
    assert torch.equal(raw[:, 256].view(torch.int64), want.view(torch.int64))
