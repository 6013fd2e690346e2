"""Time BinaryClassificationEvaluator.evaluate (b200flow.metrics.binary_metrics: the sm_90a radix sort-and-scan) with
numBins=1000 and numBins=0, on (1) the RandomForest scores of a KDD99-full-shaped test split (2 classes, 4,898,431 rows split
75 / 25, about 1.22 M test rows) and (2) 2^26 uniform random scores with random labels.  Beside each, torch.sort of the same
scores (descending) is timed: the library sort alone, without the grouping, counting and curve the evaluator does.  Every
time is the median of --repeats runs after one untimed run, host clock around work that ends in a device synchronise.
Prints the card name and power limit read in the same run.  One JSON line.

    python tools/bench_eval.py [--rows 4898431] [--big-log2 26] [--repeats 5]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "spark-network-traffic-classifier_b200"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

from bench_tuning import card  # noqa: E402


def median_time(fn, repeats):
    fn()
    ts = []
    for _ in range(repeats):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return round(sorted(ts)[len(ts) // 2] * 1e3, 3), [round(t * 1e3, 3) for t in ts]


def rf_predictions(n, seed):
    from b200flow import synth
    from pyspark.ml import Pipeline
    from pyspark.ml.classification import RandomForestClassifier
    from pyspark.ml.feature import StringIndexer, VectorAssembler
    from pyspark.sql import DataFrame
    rec, dicts = synth.make_kdd(n, 2, seed=seed, device="cuda")
    df = DataFrame.fromRecords(rec, synth.kdd_schema(), dicts)
    cats = synth.KDD_CATEGORICAL
    df = Pipeline(stages=[StringIndexer(inputCol=c, outputCol=c + "_num") for c in cats + ["label"]]).fit(df).transform(df)
    feats = [c for c in df.columns if c not in cats + ["label", "label_num"]]
    df = VectorAssembler(inputCols=feats, outputCol="features").transform(df).select(["features", "label_num"])
    train, test = df.randomSplit([0.75, 0.25], seed=seed)
    model = RandomForestClassifier(labelCol="label_num", maxBins=70, numTrees=20, maxDepth=10, seed=seed).fit(train)
    return model.transform(test)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=4898431)
    ap.add_argument("--big-log2", type=int, default=26)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--seed", type=int, default=2019)
    a = ap.parse_args()
    from b200flow.metrics import binary_metrics
    from pyspark.ml.evaluation import BinaryClassificationEvaluator
    out = {"card": card(), "unit": "ms, median of %d runs" % a.repeats}

    pred = rf_predictions(a.rows, a.seed)
    scores = pred._column_tensor("rawPrediction")[:, 1].contiguous()
    res = {"rows": int(scores.numel()), "distinct_scores": int(torch.unique(scores).numel())}
    for bins in (1000, 0):
        ev = BinaryClassificationEvaluator(labelCol="label_num", numBins=bins)
        res["evaluate_bins%d" % bins], res["evaluate_bins%d_runs" % bins] = median_time(lambda: ev.evaluate(pred), a.repeats)
        res["areaUnderROC_bins%d" % bins] = ev.evaluate(pred)
    res["torch_sort"], _ = median_time(lambda: torch.sort(scores, descending=True, stable=True), a.repeats)
    out["kdd_rf_test_split"] = res

    n = 1 << a.big_log2
    g = torch.Generator(device="cuda").manual_seed(a.seed)
    big = torch.rand(n, dtype=torch.float64, device="cuda", generator=g)
    lab = (torch.rand(n, dtype=torch.float64, device="cuda", generator=g) < 0.3).to(torch.float64)
    res = {"rows": n}
    for bins in (1000, 0):
        res["binary_metrics_bins%d" % bins], res["binary_metrics_bins%d_runs" % bins] = \
            median_time(lambda: binary_metrics(big, lab, num_bins=bins), a.repeats)
    res["torch_sort"], _ = median_time(lambda: torch.sort(big, descending=True, stable=True), a.repeats)
    out["random_2^%d" % a.big_log2] = res
    print(json.dumps(out))


if __name__ == "__main__":
    main()
