"""Model selection on the GPU: the sub-forest premise on CUDA-fitted forests, ForestModel.grid_confusion against standalone
fits of every (numTrees, maxDepth) point, and the shim's CrossValidator / TrainValidationSplit against the generic
fit -> transform -> evaluate loop over the same folds (DESIGN.md §5a)."""
import hashlib

import numpy as np
import pytest
import torch

from test_tuning import cut_export, sorted_export
from util import forests_equal, kdd_luts_gpu, kdd_plan

pytestmark = pytest.mark.gpu

TREE_CUTS = [3, 7, 20]
DEPTH_CUTS = [0, 2, 5, 9]


def forest_hash(ex):
    """sha256 of a canonical export (the fields bench.py hashes)."""
    h = hashlib.sha256()
    for k in ("tree", "nid", "feat", "kind", "bin_thr", "is_leaf", "counts"):
        h.update(np.ascontiguousarray(np.asarray(ex[k]).astype(np.int64)).tobytes())
    h.update(np.ascontiguousarray(np.asarray(ex["mask"]).astype(np.uint64)).tobytes())
    h.update(np.ascontiguousarray(np.asarray(ex["gain"], np.float64)[np.asarray(ex["is_leaf"]) == 0]).tobytes())
    return h.hexdigest()[:16]


def _kdd(n, C, seed):
    from b200flow import synth
    rec, dicts = synth.make_kdd(n, C, seed=seed, device="cuda")
    schema = synth.kdd_schema()
    luts, ordered = kdd_luts_gpu(rec, schema, dicts)
    plan = kdd_plan(schema, luts, ordered)
    arity = [0] * 38 + [len(ordered[c]) for c in synth.KDD_CATEGORICAL]
    return rec, plan, arity, len(ordered["label"])


def _params(T, d, dt=False):
    from b200flow import forest as fr
    if dt:
        return fr.ForestParams(num_trees=1, max_depth=d, max_bins=70, feature_subset_strategy="all", bootstrap=False, seed=9)
    return fr.ForestParams(num_trees=T, max_depth=d, max_bins=70, seed=2019)


# ------------------------------------------------------------------ 4. the premise on CUDA-fitted forests
@pytest.mark.parametrize("C,dt", [(5, False), (23, False), (5, True)])
def test_sub_forest_premise_on_cuda_forests(C, dt):
    from b200flow import forest as fr
    rec, plan, arity, C = _kdd(60000, C, seed=3)
    big = fr.fit_forest_records(rec, plan, C, arity, _params(12, 9, dt)).export()
    assert np.floor(np.log2(big["nid"].max())) == 9
    for T, d in ((1, 3), (1, 6), (1, 0), (1, 9)) if dt else ((5, 3), (12, 6), (2, 0), (2, 9)):   # RF: T >= 2 (§5a)
        small = sorted_export(fr.fit_forest_records(rec, plan, C, arity, _params(T, d, dt)).export())
        got = cut_export(big, T, d)
        assert forests_equal(got, small) == [], (T, d)
        assert forest_hash(got) == forest_hash(small)


# ------------------------------------------------------------------ 5. grid_confusion against standalone fits
def _standalone_cms(fit, predict, label, C, tree_cuts, depth_cuts, dt=False):
    from b200flow import forest as fr
    out = np.zeros((len(tree_cuts), len(depth_cuts), C, C), np.int64)
    for i, T in enumerate(tree_cuts):
        for j, d in enumerate(depth_cuts):
            model = fit(_params(T, d, dt))
            out[i, j] = fr.confusion_matrix(predict(model), label.to(torch.float64), C).cpu().numpy()
    return out


@pytest.mark.parametrize("C", [5, 23])
def test_grid_confusion_record_path(C):
    from b200flow import forest as fr
    rec, plan, arity, C = _kdd(200000, C, seed=5)
    train, val = rec[:150000].contiguous(), rec[100000:].contiguous()
    _, _, _, lab = fr.fit_forest_records(train, plan, C, arity, _params(1, 1)).predict_records(val, plan, want_label=True)
    assert torch.unique(val, dim=0).shape[0] < val.shape[0]                      # the validation rows repeat
    fit = lambda p: fr.fit_forest_records(train, plan, C, arity, p)
    big = fit(_params(max(TREE_CUTS), max(DEPTH_CUTS)))
    got = big.grid_confusion(val, TREE_CUTS, DEPTH_CUTS, plan=plan).numpy()
    want = _standalone_cms(fit, lambda m: m.predict_records(val, plan)[2], lab, C, TREE_CUTS, DEPTH_CUTS)
    assert got.shape == want.shape and np.array_equal(got, want)
    assert got[0, 0].sum() == val.shape[0] and len({got[i, j].tobytes() for i in range(3) for j in range(4)}) > 6
    # the result does not depend on how the depth cuts are split over launches
    assert np.array_equal(big.grid_confusion(val, TREE_CUTS, DEPTH_CUTS, plan=plan, max_depth_cuts_per_launch=1).numpy(), got)


@pytest.mark.parametrize("C", [5, 23])
def test_grid_confusion_dense_path(C):
    from b200flow import forest as fr
    rec, plan, arity, C = _kdd(200000, C, seed=6)
    x, y, _ = plan.run(rec, torch.float64)
    xt, yt, xv, yv = x[:150000], y[:150000], x[100000:].contiguous(), y[100000:].contiguous()
    fit = lambda p: fr.fit_forest(xt, yt, C, arity, p)
    got = fit(_params(max(TREE_CUTS), max(DEPTH_CUTS))).grid_confusion(xv, TREE_CUTS, DEPTH_CUTS, labels=yv).numpy()
    want = _standalone_cms(fit, lambda m: m.predict(xv)[2], yv, C, TREE_CUTS, DEPTH_CUTS)
    assert np.array_equal(got, want)


def test_grid_confusion_decision_tree():
    from b200flow import forest as fr
    rec, plan, arity, C = _kdd(200000, 23, seed=7)
    train, val = rec[:150000].contiguous(), rec[100000:].contiguous()
    _, _, _, lab = fr.fit_forest_records(train, plan, C, arity, _params(1, 1)).predict_records(val, plan, want_label=True)
    fit = lambda p: fr.fit_forest_records(train, plan, C, arity, p)
    big = fit(_params(1, max(DEPTH_CUTS), dt=True))
    assert big.dt_mode
    got = big.grid_confusion(val, [1], DEPTH_CUTS, plan=plan).numpy()
    want = _standalone_cms(fit, lambda m: m.predict_records(val, plan)[2], lab, C, [1], DEPTH_CUTS, dt=True)
    assert np.array_equal(got, want)


def test_grid_confusion_many_classes_global_atomics_and_split_launches():
    """100 classes: the I x J x C x C matrices (3 x 8 x 100 x 100 x 8 B) exceed shared memory, so counts go to global memory
    atomics; 8 depth cuts of 100 fp64 votes per row do not fit one launch even at 32 threads (8 x 100 x 8 x 32 B > 200 KB),
    so the depth cuts are split over two launches."""
    from b200flow import forest as fr
    rec, plan, arity, _ = _kdd(60000, 23, seed=8)
    x, _, _ = plan.run(rec, torch.float64)
    g = torch.Generator(device="cuda"); g.manual_seed(1)
    C = 100
    y = torch.randint(0, C, (x.shape[0],), device="cuda", generator=g, dtype=torch.int32)
    y = torch.where(x[:, 38] < 1, y % 3, y)                                   # some structure: one protocol has 3 labels
    xt, yt, xv, yv = x[:40000], y[:40000], x[30000:].contiguous(), y[30000:].contiguous()
    depth_cuts = [0, 1, 2, 3, 4, 5, 7, 9]
    fit = lambda p: fr.fit_forest(xt, yt, C, arity, p)
    big = fit(_params(max(TREE_CUTS), max(depth_cuts)))
    got = big.grid_confusion(xv, TREE_CUTS, depth_cuts, labels=yv).numpy()
    want = _standalone_cms(fit, lambda m: m.predict(xv)[2], yv, C, TREE_CUTS, depth_cuts)
    assert np.array_equal(got, want)
    # a matrix side larger than C (validation labels the fit never saw) keeps the counts in the top-left corner
    wide = big.grid_confusion(xv, TREE_CUTS, depth_cuts[:2], labels=yv, cm_side=C + 3).numpy()
    assert wide.shape[2:] == (C + 3, C + 3) and np.array_equal(wide[:, :, :C, :C], got[:, :2]) and wide[:, :, C:].sum() == 0


# ------------------------------------------------------------------ 6. the shim's validators against the generic loop
def _frame(n, C, seed):
    from b200flow import synth
    from pyspark.ml import Pipeline
    from pyspark.ml.feature import StringIndexer, VectorAssembler
    from pyspark.sql import DataFrame
    rec, dicts = synth.make_kdd(n, C, seed=seed, device="cuda")
    df = DataFrame.fromRecords(rec, synth.kdd_schema(), dicts)
    cats = synth.KDD_CATEGORICAL
    df = Pipeline(stages=[StringIndexer(inputCol=c, outputCol=c + "_num") for c in cats + ["label"]]).fit(df).transform(df)
    feats = [c for c in df.columns if c not in cats + ["label", "label_num"]]
    return df, feats


def _generic_cv(est, maps, ev, df, k, seed):
    """CrossValidator restated: fold ids from the seeded split of the global row index, per map fit -> transform -> evaluate."""
    from b200flow.rows import random_split_ids
    fid = random_split_ids(df.count(), [1.0] * k, seed, 0, df._device())
    sums = [0.0] * len(maps)
    for i in range(k):
        train, val = df._compact(fid != i), df._compact(fid == i)
        for j, m in enumerate(maps):
            sums[j] += ev.evaluate(est.fit(train, m).transform(val))
    return [s / k for s in sums]


def _count_fits(monkeypatch):
    from b200flow import forest as fr
    n = [0]
    for name in ("fit_forest", "fit_forest_records"):
        orig = getattr(fr, name)

        def wrapped(*a, _orig=orig, **kw):
            n[0] += 1
            return _orig(*a, **kw)
        monkeypatch.setattr(fr, name, wrapped)
    return n


@pytest.mark.parametrize("kind", ["rf", "dt"])
@pytest.mark.parametrize("lazy", [True, False])
def test_cross_validator_and_tvs_equal_the_generic_loop(kind, lazy, monkeypatch):
    from pyspark.ml.classification import DecisionTreeClassifier, RandomForestClassifier
    from pyspark.ml.evaluation import MulticlassClassificationEvaluator
    from pyspark.ml.feature import VectorAssembler
    from pyspark.ml.tuning import CrossValidator, ParamGridBuilder, TrainValidationSplit
    df, feats = _frame(30000, 23, seed=31)
    df = VectorAssembler(inputCols=feats, outputCol="features").transform(df).select(["features", "label_num"])
    if not lazy:
        df._cols["features"].data                                      # materialise: the dense path
    assert df._cols["features"].lazy == lazy
    if kind == "rf":
        est = RandomForestClassifier(labelCol="label_num", maxBins=70, seed=4)
        grid = ParamGridBuilder().addGrid(est.numTrees, [2, 6]).addGrid(est.maxDepth, [1, 4, 7]).build()
        grid.append({est.numTrees: 1, est.maxDepth: 3})                   # numTrees == 1: a fit group of its own
    else:
        est = DecisionTreeClassifier(labelCol="label_num", maxBins=70)
        grid = ParamGridBuilder().addGrid(est.maxDepth, [0, 3, 8]).build()
    ev = MulticlassClassificationEvaluator(labelCol="label_num", metricName="f1")
    fits = _count_fits(monkeypatch)
    cv = CrossValidator(estimator=est, estimatorParamMaps=grid, evaluator=ev, numFolds=3, seed=2019)
    model = cv.fit(df)
    groups = 2 if kind == "rf" else 1
    assert fits[0] == 3 * groups + 1                                         # one fit per fold and group, plus the refit
    want = _generic_cv(est, grid, ev, df, 3, 2019)
    assert model.avgMetrics == want and len(set(want)) > 2
    best = int(np.argmax(want))
    direct = est.fit(df, grid[best])._forest.export()
    got = model.bestModel._forest.export()
    assert all(np.array_equal(got[k], direct[k]) for k in direct)
    assert model.subModels is None and model.transform(df).count() == df.count()
    # TrainValidationSplit: one randomSplit([r, 1 - r], seed)
    tvs = TrainValidationSplit(estimator=est, estimatorParamMaps=grid, evaluator=ev, trainRatio=0.7, seed=5).fit(df)
    train, val = df.randomSplit([0.7, 1.0 - 0.7], seed=5)
    assert tvs.validationMetrics == [ev.evaluate(est.fit(train, m).transform(val)) for m in grid]
    # collectSubModels takes the generic loop and gives the same metrics
    cv_sub = CrossValidator(estimator=est, estimatorParamMaps=grid, evaluator=ev, numFolds=3, seed=2019, collectSubModels=True).fit(df)
    assert cv_sub.avgMetrics == want and len(cv_sub.subModels) == 3 and len(cv_sub.subModels[0]) == len(grid)


def test_cross_validator_generic_loop_for_lr_and_pipeline():
    from pyspark.ml import Pipeline
    from pyspark.ml.classification import LogisticRegression, RandomForestClassifier
    from pyspark.ml.evaluation import MulticlassClassificationEvaluator
    from pyspark.ml.feature import VectorAssembler
    from pyspark.ml.tuning import CrossValidator, ParamGridBuilder
    df, feats = _frame(12000, 5, seed=41)
    ev = MulticlassClassificationEvaluator(labelCol="label_num", metricName="accuracy")
    va = VectorAssembler(inputCols=feats, outputCol="features")
    vdf = va.transform(df).select(["features", "label_num"])
    lr = LogisticRegression(labelCol="label_num", maxIter=5)
    grid = ParamGridBuilder().addGrid(lr.regParam, [0.0, 0.3]).build()
    m = CrossValidator(estimator=lr, estimatorParamMaps=grid, evaluator=ev, numFolds=2, seed=3).fit(vdf)
    assert m.avgMetrics == _generic_cv(lr, grid, ev, vdf, 2, 3)
    rf = RandomForestClassifier(labelCol="label_num", maxBins=70, seed=1)
    pipe = Pipeline(stages=[va, rf])
    grid = ParamGridBuilder().addGrid(rf.numTrees, [2, 5]).addGrid(rf.maxDepth, [2, 5]).build()
    m = CrossValidator(estimator=pipe, estimatorParamMaps=grid, evaluator=ev, numFolds=2, seed=3).fit(df)
    want = _generic_cv(pipe, grid, ev, df, 2, 3)
    assert m.avgMetrics == want and len(set(want)) > 1
    assert m.bestModel.stages[-1]._forest.T == grid[int(np.argmax(want))][rf.numTrees]
