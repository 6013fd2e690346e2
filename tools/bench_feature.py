"""Time the preprocessing stages (DESIGN.md §5s) on a KDD-shaped batch from b200flow/synth.py: --rows rows (default
4,898,431, the KDD99-full row count) with their 38 numeric fields read in place from the raw records, plus one f32 column
that is 90 % zeros (the heavily tied case of the rank select's histograms).
  * "steps": the library primitives of b200flow/quantile.py;
  * "stages": the fit and the transform of every pyspark.ml.feature stage over the same DataFrame, host syncs included:
    Imputer (mean, median, mode) and QuantileDiscretizer / Bucketizer over the 38 fields, RobustScaler, MaxAbsScaler and
    MinMaxScaler over a lazy VectorAssembler of them (a fit reads the vector through one encode pass that is not kept).
For each it reports the host-timed median of --repeats after a warm-up (ending in a device synchronise) and the HBM bytes
the algorithm needs, from the shapes: one read of the columns per statistics pass, nine per rank select (the count pass and
eight digit passes), the read and the 8 sort passes of 8-byte keys (read and written) for mode, the columns read and the
output written by each transform, and for the vector stages the encode pass (records in, f32 vector out, widened to f64).
The card's name and power limit are read in the same run.  One JSON line.

    python tools/bench_feature.py [--rows 4898431] [--repeats 5]
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

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench_tuning import card  # noqa: E402


def median_time(fn, repeats):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return sorted(ts)[len(ts) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=4898431)
    ap.add_argument("--repeats", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_feature needs a CUDA device")
    from b200flow import quantile as q
    from b200flow import synth
    n = a.rows
    rec, dicts = synth.make_kdd(n, 23, seed=1, device="cuda")
    schema = synth.kdd_schema()
    fields = [c for c in synth.KDD_COLUMNS if c not in synth.KDD_CATEGORICAL and c != "label"]
    cs = q.record_columns(rec, schema, fields)
    D = cs.D
    rng = np.random.default_rng(2)
    zeros = torch.from_numpy(np.where(rng.random(n) < 0.9, 0.0, rng.exponential(100.0, n)).astype(np.float32)).cuda()
    col_bytes = n * D * 4                                            # every numeric KDD field is 4 bytes
    st = q.column_stats(cs)
    scale = [1.0 / r if r else 0.0 for r in st.max - st.min]
    splits = [list(s) for s in (np.unique(np.concatenate([[-np.inf], v, [np.inf]])) for v in
                                q.quantiles(cs, [i / 10 for i in range(1, 10)]))]
    steps = {
        "column_stats_mean": (lambda: q.column_stats(cs, with_mean=True), 2 * col_bytes),
        "median": (lambda: q.quantiles(cs, [0.5]), 9 * col_bytes),
        "deciles": (lambda: q.quantiles(cs, [i / 10 for i in range(1, 10)]), 9 * col_bytes),
        "buckets_200": (lambda: q.quantiles(cs, [i / 200 for i in range(1, 200)]), 9 * col_bytes),
        "zeros_column_median": (lambda: q.quantiles(zeros, [0.5]), 9 * n * 4),
        "zeros_column_buckets_200": (lambda: q.quantiles(zeros, [i / 200 for i in range(1, 200)]), 9 * n * 4),
        "zeros_column_mode": (lambda: q.mode(zeros), n * 4 + 8 * 2 * 8 * n),     # read, then 8 sort passes over 8-byte keys
        "bucketize": (lambda: q.bucketize(cs, splits), col_bytes + n * D * 8 + n),
        "impute_fill": (lambda: q.fill(cs, [0.0] * D), 2 * col_bytes),
        "min_max": (lambda: q.min_max(cs, st.min, scale, 0.0, 0.5), col_bytes + n * D * 8),
    }
    stages = stage_steps(rec, schema, dicts, fields, n, D)
    res = {"card": card(), "rows": n, "columns": D, "record_bytes": schema.row_bytes, "steps": {}, "stages": {}}
    for part, table in (("steps", steps), ("stages", stages)):
        for name, (fn, nbytes) in table.items():
            t = median_time(fn, a.repeats)
            res[part][name] = {"ms": round(1e3 * t, 3), "algorithmic_bytes": int(nbytes),
                               "GB_per_s": round(nbytes / t / 1e9, 1)}
            print(part, name, json.dumps(res[part][name]), file=sys.stderr, flush=True)
    print(json.dumps(res))


def stage_steps(rec, schema, dicts, fields, n, D):
    """{name: (callable, algorithmic bytes)} of every stage's fit and transform"""
    from pyspark.ml.feature import (Imputer, MaxAbsScaler, MinMaxScaler, QuantileDiscretizer, RobustScaler,
                                    VectorAssembler)
    from pyspark.sql import DataFrame
    df = DataFrame.fromRecords(rec, schema, dicts)
    col_bytes = n * D * 4
    vdf = VectorAssembler(inputCols=fields, outputCol="features", handleInvalid="keep").transform(df)
    vec_bytes = n * schema.row_bytes + n * D * 4 + n * D * 4 + n * D * 8       # encode to f32, widen to f64
    plan_bytes = n * schema.row_bytes + n * D * 8                              # the scaled plan over the records
    outs = [c + "_o" for c in fields]
    out = {}
    for strategy, fit_bytes in (("mean", 2 * col_bytes), ("median", 9 * col_bytes),
                                ("mode", D * (n * 4 + 8 * 2 * 8 * n))):
        est = Imputer(inputCols=fields, outputCols=outs, strategy=strategy)
        out["imputer_%s_fit" % strategy] = (lambda est=est: est.fit(df), fit_bytes)
    im = Imputer(inputCols=fields, outputCols=outs, strategy="median").fit(df)
    out["imputer_transform"] = (lambda: im.transform(df), 2 * col_bytes)
    qd = QuantileDiscretizer(inputCols=fields, outputCols=outs, numBuckets=10, handleInvalid="keep")
    out["quantile_discretizer_fit"] = (lambda: qd.fit(df), 9 * col_bytes)
    bz = qd.fit(df)
    out["bucketizer_transform"] = (lambda: bz.transform(df), col_bytes + n * D * 8 + n + 2 * n * D * 8)   # + column copies
    for name, est, fit_bytes in (("robust_scaler", RobustScaler(inputCol="features", outputCol="s"), vec_bytes + 9 * n * D * 8),
                                 ("max_abs_scaler", MaxAbsScaler(inputCol="features", outputCol="s"), vec_bytes + n * D * 8),
                                 ("min_max_scaler", MinMaxScaler(inputCol="features", outputCol="s"), vec_bytes + n * D * 8)):
        out[name + "_fit"] = (lambda est=est: est.fit(vdf), fit_bytes)
        m = est.fit(vdf)
        tr_bytes = vec_bytes + 2 * n * D * 8 if name == "min_max_scaler" else plan_bytes
        out[name + "_transform"] = (lambda m=m: m.transform(vdf), tr_bytes)
    return out


if __name__ == "__main__":
    main()
