"""GBTClassifier on the device against the numpy restatement (tests/gbt_oracle.py), bit for bit: structure, thresholds,
the fp64 bits of payloads and gains, the int64 node stats, tree weights, and raw / probability / prediction on held-out
rows; the training margin against the transform margin; the de-duplicated fit against the row-level one; the variance
histogram kernel against torch.index_add_; and the pyspark shim with both evaluators and CrossValidator."""
import numpy as np
import pytest
import torch

import gbt_oracle as go
from b200flow import encode as enc, forest as fr, gbt as bg, synth
from util import kdd_luts_gpu, kdd_plan

DEV = "cuda"
KEYS = ("tree", "nid", "feat", "kind", "bin_thr", "is_leaf", "mask", "stats")


def _kdd(n, seed):
    rec, dicts = synth.make_kdd(n, 2, seed=seed, device=DEV)
    schema = synth.kdd_schema()
    luts, ordered = kdd_luts_gpu(rec, schema, dicts)
    plan = kdd_plan(schema, luts, ordered)
    arity = [0] * 38 + [len(ordered[c]) for c in synth.KDD_CATEGORICAL]
    return rec, plan, arity


def _cicids(n, seed):
    rec, dicts = synth.make_cicids(n, 2, seed=seed, device=DEV, dtype="f64")
    schema = synth.cicids_schema(78, "f64")
    counts = enc.category_counts(rec, schema, "Label", 2).cpu().numpy()
    ordered, lut = enc.string_index_order(counts, dicts["Label"])
    plan = enc.EncodePlan(schema)
    for f in schema.names[:-1]:
        plan.add_numeric(f)
    plan.set_label("Label", lut)
    return rec, plan, [0] * 78


def _oracle(x, y, arity, p):
    return go.fit(x.cpu().numpy(), y.cpu().numpy(), arity, max_iter=p.max_iter, step_size=p.step_size, max_depth=p.max_depth,
                  max_bins=p.max_bins, min_inst=p.min_instances_per_node, min_gain=p.min_info_gain,
                  subsampling_rate=p.subsampling_rate, strategy=p.feature_subset_strategy, seed=p.seed)


def _assert_same_model(model, want):
    got, exp = model.export(), go.export(want)
    for k in KEYS:
        assert np.array_equal(got[k], exp[k]), k
    assert np.array_equal(got["payload"].view(np.int64), exp["payload"].view(np.int64))
    assert np.array_equal(got["gain"].view(np.int64), exp["gain"].view(np.int64))
    assert model.tree_weights == want["weights"]
    assert np.array_equal(model.forest.thresholds.cpu().numpy(), want["thresholds"])


def _assert_same_output(model, want, x_test):
    import oracle
    tp, _ = oracle.bin_rows(x_test.cpu().numpy(), want["thresholds"], want["n_thr"], model.forest.arity, want["max_bins"])
    mg, raw, prob, pred = go.predict(want, tp[:, :model.F])
    r, pr, pd = model.predict(x_test)
    assert np.array_equal(r.cpu().numpy().view(np.int64), raw.view(np.int64))
    assert np.array_equal(pr.cpu().numpy().view(np.int64), prob.view(np.int64))
    assert np.array_equal(pd.cpu().numpy(), pred)


CASES = {
    "kdd": dict(),
    "subsample_sqrt": dict(subsampling_rate=0.7, feature_subset_strategy="sqrt"),
    "depth0": dict(max_depth=0, max_iter=3),
    "depth1": dict(max_depth=1),
    "one_iteration": dict(max_iter=1, max_depth=6),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASES))
def test_device_model_equals_the_restatement(case):
    rec, plan, arity = _kdd(12000, 7)
    x, y, _ = plan.run(rec, torch.float64)
    kw = dict(max_iter=6, max_depth=4, max_bins=70, seed=11)
    kw.update(CASES[case])
    p = bg.GBTParams(**kw)
    model = bg.fit_gbt(x[:10000], y[:10000], arity, p)
    want = _oracle(x[:10000], y[:10000], arity, p)
    _assert_same_model(model, want)
    _assert_same_output(model, want, x[10000:])
    # the training margin of every row is the transform margin, bit for bit
    train_margin = model.train_margin[model.train_uid.long()]
    assert torch.equal(train_margin.view(torch.int64), model.margin(x[:10000]).view(torch.int64))
    assert np.array_equal(train_margin.cpu().numpy().view(np.int64), want["margin"].view(np.int64))


@pytest.mark.gpu
def test_record_path_and_deduplication_give_the_same_model(monkeypatch):
    rec, plan, arity = _kdd(15000, 3)
    x, y, _ = plan.run(rec, torch.float64)
    p = bg.GBTParams(max_iter=5, max_depth=5, max_bins=70, seed=2)
    dense = bg.fit_gbt(x, y, arity, p)
    fused = bg.fit_gbt_records(rec, plan, arity, p)
    assert fused.train_stats["unique_rows"] < 15000
    monkeypatch.setattr(fr, "DEDUP", False)
    rows = bg.fit_gbt(x, y, arity, p)
    for other in (fused, rows):
        a, b = dense.export(), other.export()
        for k in a:
            assert np.array_equal(np.asarray(a[k]).view(np.uint8), np.asarray(b[k]).view(np.uint8)), k
    raw_f, prob_f, pred_f = fused.predict_records(rec, plan)
    raw_d, prob_d, pred_d = dense.predict(x)
    assert torch.equal(raw_f, raw_d) and torch.equal(prob_f, prob_d) and torch.equal(pred_f, pred_d)
    _assert_same_model(dense, _oracle(x, y, arity, p))


@pytest.mark.gpu
def test_cicids_f64_records_equal_the_restatement():
    rec, plan, arity = _cicids(8000, 5)
    x, y, _ = plan.run(rec, torch.float64)
    p = bg.GBTParams(max_iter=4, max_depth=4, max_bins=78, seed=9)
    model = bg.fit_gbt_records(rec, plan, arity, p)
    _assert_same_model(model, _oracle(x, y, arity, p))


@pytest.mark.gpu
def test_odd_bin_count_equals_the_restatement():
    # maxBins 33 on continuous data: n_bins is odd, so the scoring warps' scratch blocks need their 16-byte rounding
    rec, plan, arity = _cicids(8000, 21)
    x, y, _ = plan.run(rec, torch.float64)
    p = bg.GBTParams(max_iter=3, max_depth=4, max_bins=33, seed=4)
    model = bg.fit_gbt(x, y, arity, p)
    assert model.n_bins % 2 == 1
    _assert_same_model(model, _oracle(x, y, arity, p))


@pytest.mark.gpu
def test_histogram_budget_slot_groups_give_the_same_model(monkeypatch):
    rec, plan, arity = _kdd(12000, 19)
    x, y, _ = plan.run(rec, torch.float64)
    p = bg.GBTParams(max_iter=3, max_depth=5, max_bins=70, seed=6)
    want = bg.fit_gbt(x, y, arity, p).export()
    monkeypatch.setattr(fr, "HIST_BUDGET_BYTES", 2 * 41 * 70 * 24)      # two slots per group
    got = bg.fit_gbt(x, y, arity, p).export()
    for k in want:
        assert np.array_equal(np.asarray(got[k]).view(np.uint8), np.asarray(want[k]).view(np.uint8)), k


@pytest.mark.gpu
def test_single_label_training_set():
    rec, plan, arity = _kdd(3000, 13)
    x, y, _ = plan.run(rec, torch.float64)
    y = torch.ones_like(y)
    p = bg.GBTParams(max_iter=3, max_depth=3, max_bins=70, seed=1)
    model = bg.fit_gbt(x, y, arity, p)
    want = _oracle(x, y, arity, p)
    _assert_same_model(model, want)
    ex = model.export()
    assert ex["is_leaf"][ex["tree"] == 0].all() and bool((model.predict(x)[2] == 1.0).all())   # later trees may split on rounding


@pytest.mark.gpu
@pytest.mark.parametrize("m,n_bins", [(41, 70), (100, 256)])       # (100, 256): 600 KB per slot, in feature passes
def test_hist_level_equals_index_add(m, n_bins):
    g = torch.Generator(device=DEV).manual_seed(m)
    U, F, n_slots = 50000, max(m, 41), 3
    stride = fr.tp_stride(F)
    tp = torch.randint(0, n_bins, (U, stride), dtype=torch.uint8, device=DEV, generator=g)
    rq = torch.randint(-(1 << 44), 1 << 44, (U, 2), dtype=torch.int64, device=DEV, generator=g)
    rec = torch.randint(0, U, (120000,), dtype=torch.int32, device=DEV, generator=g)
    w = torch.randint(0, 5, (120000,), dtype=torch.int32, device=DEV, generator=g)
    ent = torch.stack([rec, w], 1).contiguous()
    bounds = torch.tensor([0, 30000, 30001, 120000], dtype=torch.int64, device=DEV)
    seg_begin, seg_end = bounds[:-1].contiguous(), bounds[1:].contiguous()
    subset = torch.stack([torch.randperm(F, device=DEV, generator=g)[:m].sort().values for _ in range(n_slots)]).to(torch.int16)
    nch = ((seg_end - seg_begin + fr.CHUNK_ROWS - 1) // fr.CHUNK_ROWS).to(torch.int32)
    chunk_off = torch.zeros(n_slots + 1, dtype=torch.int64, device=DEV)
    chunk_off[1:] = torch.cumsum(nch, 0)
    hist = torch.zeros(n_slots * m * n_bins * 3, dtype=torch.int64, device=DEV)
    from b200flow._lib import call, ptr
    call("b200flow_gbt_hist_level", ptr(tp), stride, ptr(ent), ptr(rq), n_slots, ptr(seg_begin), ptr(seg_end), ptr(chunk_off),
         int(chunk_off[-1]), fr.CHUNK_ROWS, ptr(subset), m, n_bins, ptr(hist))
    want = torch.zeros(n_slots * m * n_bins, 3, dtype=torch.int64, device=DEV)
    slot = torch.repeat_interleave(torch.arange(n_slots, device=DEV), (seg_end - seg_begin))
    ww = w.to(torch.int64)
    vals = torch.stack([ww, ww * rq[rec.long(), 0], ww * rq[rec.long(), 1]], 1)
    for j in range(m):
        f = subset[slot, j].long()
        b = tp[rec.long(), f].long()
        want.index_add_(0, (slot * m + j) * n_bins + b, vals)
    assert torch.equal(hist.view(-1, 3), want)


def _frame(n, seed):
    from pyspark.sql import DataFrame
    rec, dicts = synth.make_kdd(n, 2, seed=seed, device="cuda:0")
    return DataFrame.fromRecords(rec, synth.kdd_schema(), dicts)


def _stages():
    from pyspark.ml.feature import StringIndexer, VectorAssembler
    cats = synth.KDD_CATEGORICAL
    st = [StringIndexer(inputCol=c, outputCol=c + "_num") for c in cats + ["label"]]
    nums = [c for c in synth.KDD_COLUMNS if c not in cats + ["label"]]
    st.append(VectorAssembler(inputCols=nums + [c + "_num" for c in cats], outputCol="features"))
    return st


@pytest.mark.gpu
def test_shim_pipeline_evaluators_and_cross_validator():
    from pyspark.ml import Pipeline
    from pyspark.ml.classification import GBTClassifier
    from pyspark.ml.evaluation import BinaryClassificationEvaluator, MulticlassClassificationEvaluator
    from pyspark.ml.feature import IllegalArgumentException
    from pyspark.ml.tuning import CrossValidator, ParamGridBuilder, fold_frames
    df = _frame(20000, 5)
    gbt = GBTClassifier(labelCol="label_num", maxIter=5, maxBins=70, seed=3)
    model = Pipeline(stages=_stages() + [gbt]).fit(df)
    out = model.transform(df)
    m = model.stages[-1]
    assert m.getNumTrees == 5 and m.treeWeights == [1.0, 0.1, 0.1, 0.1, 0.1] and m.numClasses == 2 and m.numFeatures == 41
    assert abs(float(np.sum(m.featureImportances.toArray())) - 1.0) < 1e-12 and "Tree 4 (weight 0.1)" in m.toDebugString
    raw = out._column_tensor("rawPrediction").cpu().numpy()
    prob = out._column_tensor("probability").cpu().numpy()
    pred = out._column_tensor("prediction").cpu().numpy()
    assert np.array_equal(raw[:, 0], -raw[:, 1]) and np.array_equal(pred, (raw[:, 1] > 0).astype(np.float64))
    assert np.array_equal(prob[:, 1], 1.0 - prob[:, 0])
    acc = MulticlassClassificationEvaluator(labelCol="label_num", metricName="accuracy").evaluate(out)
    auc = BinaryClassificationEvaluator(labelCol="label_num").evaluate(out)
    assert acc > 0.9 and 0.9 < auc <= 1.0
    feats = Pipeline(stages=_stages()).fit(df).transform(df)
    with pytest.raises(IllegalArgumentException):             # three classes
        three = _frame(3000, 2)
        from pyspark.ml.feature import StringIndexer
        GBTClassifier(labelCol="service_num").fit(Pipeline(stages=_stages()).fit(three).transform(three))
    g2 = GBTClassifier(labelCol="label_num", maxBins=70, seed=4)
    grid = ParamGridBuilder().addGrid(g2.maxDepth, [2, 4]).addGrid(g2.stepSize, [0.1, 0.3]).build()
    ev = MulticlassClassificationEvaluator(labelCol="label_num")
    sel = feats.select("features", "label_num")
    cvm = CrossValidator(estimator=g2.setMaxIter(3), estimatorParamMaps=grid, evaluator=ev, numFolds=2, seed=9).fit(sel)
    want = [0.0] * 4
    for train, val in fold_frames(sel, 2, 9):
        for i, pm in enumerate(grid):
            want[i] += ev.evaluate(g2.fit(train, pm).transform(val))
    assert cvm.avgMetrics == [v / 2 for v in want]
