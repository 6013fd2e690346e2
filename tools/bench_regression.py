"""Time RandomForestRegressor on a KDD99-full-shaped set: --rows flows (default 4,898,431, synth.make_kdd(n, 2)) assembled by
the shim pipeline StringIndexer -> VectorAssembler (40 features without dst_bytes, 3 of them categorical), maxBins 70, the
label log1p(dst_bytes); 20 trees at depth 5 (Spark's defaults) and at depth 10.

It reports
  * fit (host clock around a synchronised fit, after one untimed fit), transform of every row and RegressionEvaluator
    (rmse) on the predictions (CUDA events, median of --repeats);
  * CUDA-event time per phase of the fit (variance histograms, split scoring, node-pool growth, partition);
  * RandomForestClassifier's fit on the same features (20 trees, depth 5, label = attack or not), for scale;
  * GBTClassifier's fit (tools/bench_gbt.py's setting: 20 iterations, depth 5) with the shared level loop, and, with
    --gbt-before FILE (a gbt.py from before the level loop was shared), with that module in the same process;
  * the CPU restatement (tests/regression_oracle.py) on the first --oracle-rows rows: its time and whether the device model
    and the evaluator equal it bit for bit.
One JSON line, with the card's name and power limit read in the same run.

    python tools/bench_regression.py [--rows 4898431] [--oracle-rows 20000] [--repeats 5] [--gbt-before FILE]
"""
import argparse
import importlib.util
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "spark-network-traffic-classifier_b200"), os.path.join(ROOT, "tools"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench_tuning import card  # noqa: E402


def features(n, seed):
    from b200flow import synth
    from pyspark.ml import Pipeline
    from pyspark.ml.classification import _arity_from_attrs
    from pyspark.ml.feature import StringIndexer, VectorAssembler
    from pyspark.sql import DataFrame
    rec, dicts = synth.make_kdd(n, 2, seed=seed, device="cuda:0")
    df = DataFrame.fromRecords(rec, synth.kdd_schema(), dicts)
    cats = synth.KDD_CATEGORICAL
    stages = [StringIndexer(inputCol=c, outputCol=c + "_num") for c in cats + ["label"]]
    nums = [c for c in synth.KDD_COLUMNS if c not in cats + ["label", "dst_bytes"]]
    stages.append(VectorAssembler(inputCols=nums + [c + "_num" for c in cats], outputCol="features"))
    out = Pipeline(stages=stages).fit(df).transform(df)
    x = out._cols["features"].data.to(torch.float64).contiguous()
    y = torch.log1p(out._column_tensor("dst_bytes").to(torch.float64)).contiguous()
    cls = out._column_tensor("label_num").to(torch.int32).contiguous()
    return x, y, cls, _arity_from_attrs(out._cols["features"].meta.get("attrs"), x.shape[1])


def timed_fit(fn):
    fn()                                                 # untimed: first-call costs
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return r, (time.perf_counter() - t0) * 1e3


def events(fn, repeats):
    ts = []
    for _ in range(repeats):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts))


def phases(fn):
    from b200flow import forest as fr
    fr.PROFILE = {}
    fn()
    torch.cuda.synchronize()
    out = {k: round(sum(a.elapsed_time(b) for a, b in v), 2) for k, v in fr.PROFILE.items()}
    fr.PROFILE = None
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=4_898_431)
    ap.add_argument("--oracle-rows", type=int, default=20000)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--gbt-before", default=None, help="a gbt.py from before the level loop was shared, timed alongside")
    a = ap.parse_args()
    from b200flow import forest as fr, gbt as bg, metrics as bm, regression as br
    torch.cuda.set_device(0)
    x, y, cls, arity = features(a.rows, 1)
    out = dict(tool="bench_regression", rows=a.rows, features=x.shape[1], card=card())
    for depth in (5, 10):
        p = br.RegressorParams(num_trees=20, max_depth=depth, max_bins=70, seed=7)
        model, ms = timed_fit(lambda: br.fit_rf_regressor(x, y, arity, p))
        r = dict(fit_ms=round(ms, 1), nodes=model.n_nodes, unique_rows=model.train_stats["unique_rows"],
                 levels=model.train_stats["levels"], E=model.E, S=model.S)
        r["phases_ms"] = phases(lambda: br.fit_rf_regressor(x, y, arity, p))
        r["transform_ms"] = round(events(lambda: model.predict(x), a.repeats), 2)
        pred = model.predict(x)
        r["evaluator_ms"] = round(events(lambda: bm.regression_metrics(y, pred), a.repeats), 2)
        r["rmse"] = bm.regression_metrics(y, pred)["rmse"]
        out["rf_depth%d" % depth] = r
    fp = fr.ForestParams(num_trees=20, max_depth=5, max_bins=70, seed=7)
    _, ms = timed_fit(lambda: fr.fit_forest(x, cls, int(cls.max().item()) + 1, arity, fp))
    out["rf_classifier_fit_ms"] = round(ms, 1)
    gp = bg.GBTParams(max_iter=20, max_depth=5, max_bins=70, seed=7)
    binary = (cls > 0).to(torch.int32)
    _, ms = timed_fit(lambda: bg.fit_gbt(x, binary, arity, gp))
    out["gbt_fit_ms"] = round(ms, 1)
    if a.gbt_before:
        spec = importlib.util.spec_from_file_location("b200flow.gbt_before", a.gbt_before)
        before = importlib.util.module_from_spec(spec)
        sys.modules["b200flow.gbt_before"] = before
        spec.loader.exec_module(before)
        m_before, ms_b = timed_fit(lambda: before.fit_gbt(x, binary, arity, gp))
        _, ms_a = timed_fit(lambda: bg.fit_gbt(x, binary, arity, gp))      # again, after: the two interleave
        out["gbt_fit_before_ms"], out["gbt_fit_after_ms"] = round(ms_b, 1), round(ms_a, 1)
        ea, eb = bg.fit_gbt(x, binary, arity, gp).export(), m_before.export()
        out["gbt_same_bits"] = all(np.array_equal(np.asarray(ea[k]).view(np.uint8), np.asarray(eb[k]).view(np.uint8)) for k in ea)
    if a.oracle_rows:
        import regression_oracle as ro
        k = min(a.oracle_rows, a.rows)
        p = br.RegressorParams(num_trees=20, max_depth=5, max_bins=70, seed=7)
        model = br.fit_rf_regressor(x[:k].contiguous(), y[:k].contiguous(), arity, p)
        t0 = time.perf_counter()
        want = ro.fit(x[:k].cpu().numpy(), y[:k].cpu().numpy(), arity, num_trees=20, max_depth=5, max_bins=70, seed=7)
        out["oracle_rows"], out["oracle_s"] = k, round(time.perf_counter() - t0, 1)
        got, exp = model.export(), ro.export(want)
        out["oracle_same_bits"] = all(np.array_equal(np.asarray(got[c]).view(np.uint8), np.asarray(exp[c]).view(np.uint8))
                                      for c in ("tree", "nid", "feat", "kind", "bin_thr", "is_leaf", "mask", "stats", "payload", "gain"))
        pred = model.predict(x[:k].contiguous())
        mg, mw = bm.regression_metrics(y[:k], pred), ro.metrics(y[:k].cpu().numpy(), pred.cpu().numpy())
        out["oracle_metrics_same"] = all(mg[c] == mw[c] for c in mw)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
