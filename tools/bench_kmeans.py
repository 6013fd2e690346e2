"""Time KMeans on a KDD99-full-shaped training split: --rows flows (default 3,673,823 = 75 % of 4,898,431) encoded by the shim
pipeline StringIndexer -> OneHotEncoder -> VectorAssembler -> StandardScaler (D = 119 one-hot-encoded features), then
b200flow.kmeans.kmeans_fit with tol = 0 so that Lloyd runs all --max-iter iterations, for each k of --ks.

Per k it reports
  * the fit time (host clock around a fit that ends in a device synchronise, after one untimed fit),
  * per-iteration kernel times with CUDA events: the assign kernel, the grouped sum of the centers (G = k, W = D) and the
    grouped sum of the cost (G = 1), each the median of --repeats launches on the fitted centers,
  * the achieved fp64 instruction rate of assign: 3 · n · k · D instructions (sub, mul, add per term) over its time,
  * the numpy restatement (tests/kmeans_oracle.py) on the first --oracle-rows rows with the same centers: whether clusters
    and distances are equal bit for bit.
The card name and power limit are read in the same run.  One JSON line per k.

    python tools/bench_kmeans.py [--rows 3673823] [--ks 23,100] [--max-iter 20] [--repeats 10] [--oracle-rows 20000]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "spark-network-traffic-classifier_b200"), os.path.join(ROOT, "tools"),
          os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench_tuning import card  # noqa: E402


def features(n, seed):
    from b200flow import synth
    from pyspark.ml import Pipeline
    from pyspark.ml.feature import OneHotEncoder, StandardScaler, StringIndexer, VectorAssembler
    from pyspark.sql import DataFrame
    rec, dicts = synth.make_kdd(n, 23, seed=seed, device="cuda:0")
    df = DataFrame.fromRecords(rec, synth.kdd_schema(), dicts)
    cats = synth.KDD_CATEGORICAL
    stages = [StringIndexer(inputCol=c, outputCol=c + "_num") for c in cats]
    stages.append(OneHotEncoder(inputCols=[c + "_num" for c in cats], outputCols=[c + "_oh" for c in cats]))
    nums = [c for c in synth.KDD_COLUMNS if c not in cats + ["label"]]
    stages.append(VectorAssembler(inputCols=nums + [c + "_oh" for c in cats], outputCol="raw"))
    stages.append(StandardScaler(inputCol="raw", outputCol="features", withMean=True, withStd=True))
    out = Pipeline(stages=stages).fit(df).transform(df)
    return out._cols["features"].data.to(torch.float64).contiguous()


def event_ms(fn, repeats):
    fn()
    ts = []
    for _ in range(repeats):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return round(sorted(ts)[len(ts) // 2], 4)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=3673823)
    ap.add_argument("--ks", default="23,100")
    ap.add_argument("--max-iter", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=10)
    ap.add_argument("--oracle-rows", type=int, default=20000)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_kmeans.py needs a CUDA device")
    import kmeans_oracle as ko
    from b200flow import kmeans as bk
    dev_card = card()
    x = features(a.rows, 2019)
    n, D = x.shape
    sh = bk._Shards(n, 0, None, x.device)
    for k in [int(v) for v in a.ks.split(",")]:
        bk.kmeans_fit(x, k, max_iter=a.max_iter, tol=0.0, seed=1)                  # warm-up
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = bk.kmeans_fit(x, k, max_iter=a.max_iter, tol=0.0, seed=1)
        torch.cuda.synchronize()
        fit_s = time.perf_counter() - t0
        c = res.centers
        kk = c.shape[0]
        assign_ms = event_ms(lambda: bk.assign(x, c), a.repeats)
        cl, d = bk.assign(x, c)
        sums_ms = event_ms(lambda: bk.grouped_sum(x, cl, kk, sh), a.repeats)
        cost_ms = event_ms(lambda: bk.grouped_sum(d.reshape(-1, 1), None, 1, sh), a.repeats)
        m = min(a.oracle_rows, n)
        xs = x[:m].cpu().numpy()
        ocl, od = ko.assign(xs, c.cpu().numpy())
        instr = 3.0 * n * kk * D
        print(json.dumps({
            "rows": n, "D": D, "k": k, "k_fitted": kk, "num_iter": res.num_iter, "training_cost": res.training_cost,
            "fit_s": round(fit_s, 4), "assign_ms": assign_ms, "center_sums_ms": sums_ms, "cost_sum_ms": cost_ms,
            "assign_fp64_ginstr_per_s": round(instr / (assign_ms * 1e-3) / 1e9, 1),
            "oracle_rows": m, "oracle_equal": bool(np.array_equal(cl[:m].cpu().numpy(), ocl) and
                                                   np.array_equal(d[:m].cpu().numpy().view(np.int64), od.view(np.int64))),
            "card": dev_card}), flush=True)


if __name__ == "__main__":
    main()
