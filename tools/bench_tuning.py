"""Time a 3-fold CrossValidator over numTrees {20, 50, 100} x maxDepth {5, 10, 16} on a seeded KDD99-full-shaped synthetic
set (5 classes by default), twice: through the pyspark.ml shim (one forest fit per fold + grid_confusion, then the refit) and as the
hand-written generic loop (fit -> transform -> evaluate for every fold and map, then the refit).  After one untimed run of
each arm, the arms alternate --repeats times; the median of each is reported with every run's time.  Also prints the fit
counts, whether avgMetrics are equal, and the card name and power limit read in the same run.  One JSON line.

    python tools/bench_tuning.py [--rows 4898431] [--folds 3] [--repeats 3] [--metric f1] [--classes 5]

--metric areaUnderROC / areaUnderPR scores with a BinaryClassificationEvaluator (its fast path: grid_binary_metrics); any
other name is a MulticlassClassificationEvaluator metric.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "spark-network-traffic-classifier_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402


def card():
    out = {"name": torch.cuda.get_device_name(0)}
    try:
        import pynvml as nv
        nv.nvmlInit()
        h = nv.nvmlDeviceGetHandleByIndex(torch.cuda.current_device())
        out["power_limit_w"] = nv.nvmlDeviceGetEnforcedPowerLimit(h) / 1000.0
        out["max_sm_mhz"] = nv.nvmlDeviceGetMaxClockInfo(h, nv.NVML_CLOCK_SM)
    except Exception as e:                                    # the times stay valid; the power limit is then unknown
        out["power_limit_w"] = "unavailable: %s" % type(e).__name__
    return out


def frame(n, seed, classes=5):
    from b200flow import synth
    from pyspark.ml import Pipeline
    from pyspark.ml.feature import StringIndexer, VectorAssembler
    from pyspark.sql import DataFrame
    rec, dicts = synth.make_kdd(n, classes, seed=seed, device="cuda")
    df = DataFrame.fromRecords(rec, synth.kdd_schema(), dicts)
    cats = synth.KDD_CATEGORICAL
    df = Pipeline(stages=[StringIndexer(inputCol=c, outputCol=c + "_num") for c in cats + ["label"]]).fit(df).transform(df)
    feats = [c for c in df.columns if c not in cats + ["label", "label_num"]]
    return VectorAssembler(inputCols=feats, outputCol="features").transform(df).select(["features", "label_num"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=4898431)
    ap.add_argument("--folds", type=int, default=3)
    ap.add_argument("--seed", type=int, default=2019)
    ap.add_argument("--repeats", type=int, default=3, help="timed runs of each arm, alternated; the median is reported")
    ap.add_argument("--metric", default="f1", help="evaluator metric (areaUnderROC / areaUnderPR: the binary evaluator)")
    ap.add_argument("--classes", type=int, default=5, help="label classes of the synthetic set")
    a = ap.parse_args()
    from b200flow import forest as fr
    from b200flow.rows import random_split_ids
    from pyspark.ml.classification import RandomForestClassifier
    from pyspark.ml.evaluation import BinaryClassificationEvaluator, MulticlassClassificationEvaluator
    from pyspark.ml.tuning import CrossValidator, ParamGridBuilder

    fits = [0]
    for name in ("fit_forest", "fit_forest_records"):
        orig = getattr(fr, name)

        def wrapped(*args, _orig=orig, **kw):
            fits[0] += 1
            return _orig(*args, **kw)
        setattr(fr, name, wrapped)

    df = frame(a.rows, a.seed, a.classes)
    rf = RandomForestClassifier(labelCol="label_num", featuresCol="features", maxBins=70, seed=a.seed)
    grid = ParamGridBuilder().addGrid(rf.numTrees, [20, 50, 100]).addGrid(rf.maxDepth, [5, 10, 16]).build()
    if a.metric in ("areaUnderROC", "areaUnderPR"):
        ev = BinaryClassificationEvaluator(labelCol="label_num", metricName=a.metric)
    else:
        ev = MulticlassClassificationEvaluator(labelCol="label_num", metricName=a.metric)
    better = 1 if ev.isLargerBetter() else -1

    def fast():
        fits[0] = 0
        cv = CrossValidator(estimator=rf, estimatorParamMaps=grid, evaluator=ev, numFolds=a.folds, seed=a.seed).fit(df)
        return cv.avgMetrics, cv.bestModel, fits[0]

    def generic():
        fits[0] = 0
        fid = random_split_ids(df.count(), [1.0] * a.folds, a.seed, 0, df._device())
        sums = [0.0] * len(grid)
        for i in range(a.folds):
            train, val = df._compact(fid != i), df._compact(fid == i)
            for j, m in enumerate(grid):
                sums[j] += ev.evaluate(rf.fit(train, m).transform(val))
        avg = [s / a.folds for s in sums]
        return avg, rf.fit(df, grid[max(range(len(avg)), key=lambda j: (better * avg[j], -j))]), fits[0]

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        return time.perf_counter() - t0, out

    timed(fast); timed(generic)                                # warm-up: every shape both arms use
    times = {"fast": [], "generic": []}
    for _ in range(a.repeats):                                 # alternate the arms
        t, (avg_f, best_f, fast_fits) = timed(fast); times["fast"].append(t)
        t, (avg, best, gen_fits) = timed(generic); times["generic"].append(t)
    fast_s, gen_s = sorted(times["fast"])[a.repeats // 2], sorted(times["generic"])[a.repeats // 2]
    same_best = bool(best._forest.T == best_f._forest.T and
                     all((best._forest.export()[k] == best_f._forest.export()[k]).all() for k in ("nid", "feat", "counts")))
    print(json.dumps({"metric": "3-fold CrossValidator, numTrees {20,50,100} x maxDepth {5,10,16}", "rows": a.rows,
                      "evaluator_metric": a.metric, "classes": a.classes,
                      "fast_s": round(fast_s, 3), "generic_s": round(gen_s, 3),
                      "fast_runs_s": [round(t, 3) for t in times["fast"]],
                      "generic_runs_s": [round(t, 3) for t in times["generic"]], "speedup": round(gen_s / fast_s, 2),
                      "fits_fast": fast_fits, "fits_generic": gen_fits, "avgMetrics_equal": avg_f == avg,
                      "bestModel_equal": same_best, "avgMetrics": avg_f, "card": card()}))


if __name__ == "__main__":
    main()
