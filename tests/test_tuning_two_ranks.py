"""CrossValidator with TWO RANKS ON ONE GPU (gloo group, as in tests/test_two_ranks_one_gpu.py): each rank holds a block of
the rows; fold ids are keyed by the global row index, the fits all-reduce their histograms and grid_confusion all-reduces
its counts, so avgMetrics and the best model equal the single-process result exactly."""
import numpy as np
import pytest

from ranks import block, run

pytestmark = pytest.mark.gpu

N = 30000


def _cv(rec, dicts):
    from b200flow import synth
    from pyspark.ml import Pipeline
    from pyspark.ml.classification import RandomForestClassifier
    from pyspark.ml.evaluation import MulticlassClassificationEvaluator
    from pyspark.ml.feature import StringIndexer, VectorAssembler
    from pyspark.ml.tuning import CrossValidator, ParamGridBuilder
    from pyspark.sql import DataFrame
    df = DataFrame.fromRecords(rec, synth.kdd_schema(), dicts)
    cats = synth.KDD_CATEGORICAL
    df = Pipeline(stages=[StringIndexer(inputCol=c, outputCol=c + "_num") for c in cats + ["label"]]).fit(df).transform(df)
    feats = [c for c in df.columns if c not in cats + ["label", "label_num"]]
    df = VectorAssembler(inputCols=feats, outputCol="features").transform(df).select(["features", "label_num"])
    rf = RandomForestClassifier(labelCol="label_num", maxBins=70, seed=4)
    grid = ParamGridBuilder().addGrid(rf.numTrees, [2, 5]).addGrid(rf.maxDepth, [2, 6]).build()
    ev = MulticlassClassificationEvaluator(labelCol="label_num", metricName="f1")
    m = CrossValidator(estimator=rf, estimatorParamMaps=grid, evaluator=ev, numFolds=3, seed=2019).fit(df)
    return m.avgMetrics, m.bestModel._forest.export()


def _ranks(rank, grp, dev):
    from b200flow import synth
    rec, dicts = synth.make_kdd(N, 5, seed=17, device="cuda:0")
    lo, hi = block(rank, 11000, N)                                          # uneven blocks
    avg, ex = _cv(rec[lo:hi].contiguous(), dicts)
    return [float.hex(v) for v in avg], ex


def test_cross_validator_two_ranks_equals_single_process(tmp_path):
    got_avg, got = run(tmp_path, _ranks, timeout=300)[0]
    from b200flow import synth
    rec, dicts = synth.make_kdd(N, 5, seed=17, device="cuda:0")
    avg, ex = _cv(rec, dicts)
    assert got_avg == [float.hex(v) for v in avg]
    assert all(np.array_equal(got[k], ex[k]) for k in ex)
