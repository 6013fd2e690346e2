"""Time PCA on the shapes of the two datasets: KDD99-full's training split (3,673,823 flows = 75 % of 4,898,431) encoded to
D = 119 (one-hot, bench_kmeans.features) and to D = 41 (indexed categoricals), and CICIDS2017-full (2,830,743 flows,
D = 78), all standardised f64, for each k of --ks.

Per shape it reports CUDA-event medians, each over enough repetitions to fill --window seconds after a warm-up:
  * mean_ms: the column sums (b200flow_group_sums, G = 1, W = D) and their chain,
  * gram_ms: b200flow_centered_gram over all chunks in batches of the partial budget, and the chain,
  * fit_ms: the whole pca_fit, host eigendecomposition included (host clock around a fit that ends in a synchronise),
  * project_ms per k: b200flow_pca_project.
For the Gram and the projection it reports the algorithmic bytes (8 n D in and the partial rows out; 8 n (D + k)) and FLOPs
(n D (D + 1) for the upper triangle; 2 n D k) computed from the shapes, the achieved rates, which of the two bounds the
kernel (the larger of bytes over 3.35 TB/s and FLOPs over 67 TFLOP/s), and the share of that bound reached.  Both peaks are
NVIDIA's data-sheet figures for the H100 SXM at 700 W, not measurements; the card's name and power limit are read in the
same run.  It also reports whether a fit on the first --oracle-rows rows matches tests/pca_oracle.py (relative 1e-10).
One JSON line per shape.

    python tools/bench_pca.py [--shapes kdd119,kdd41,cicids78] [--ks 8,32] [--window 2.0] [--oracle-rows 20000]
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

PEAK_HBM = 3.35e12          # data sheet, H100 SXM
PEAK_FP64_TC = 67e12        # data sheet, H100 SXM at 700 W
KDD_TRAIN_ROWS, CICIDS_ROWS = 3673823, 2830743


def features(shape, rows):
    from b200flow import synth
    from pyspark.ml import Pipeline
    from pyspark.ml.feature import StandardScaler, StringIndexer, VectorAssembler
    from pyspark.sql import DataFrame
    if shape == "kdd119":
        from bench_kmeans import features as onehot
        return onehot(rows or KDD_TRAIN_ROWS, 2019)
    if shape == "kdd41":
        rec, dicts = synth.make_kdd(rows or KDD_TRAIN_ROWS, 23, seed=2019, device="cuda:0")
        df = DataFrame.fromRecords(rec, synth.kdd_schema(), dicts)
        cats = synth.KDD_CATEGORICAL
        stages = [StringIndexer(inputCol=c, outputCol=c + "_num") for c in cats]
        cols = [c for c in synth.KDD_COLUMNS if c not in cats + ["label"]] + [c + "_num" for c in cats]
    elif shape == "cicids78":
        rec, dicts = synth.make_cicids(rows or CICIDS_ROWS, 15, seed=2019, device="cuda:0", dtype="f64")
        df = DataFrame.fromRecords(rec, synth.cicids_schema(78, "f64"), dicts)
        stages, cols = [], ["f%02d" % i for i in range(78)]
    else:
        raise SystemExit("unknown shape %r" % shape)
    stages.append(VectorAssembler(inputCols=cols, outputCol="raw"))
    stages.append(StandardScaler(inputCol="raw", outputCol="features", withMean=True, withStd=True))
    out = Pipeline(stages=stages).fit(df).transform(df)
    return out._cols["features"].data.to(torch.float64).contiguous()


def window_ms(fn, window):
    """(median ms, repetitions) of fn by CUDA events: one untimed call, then at least 5 and until `window` seconds."""
    fn()
    torch.cuda.synchronize()
    ts, t0 = [], time.perf_counter()
    while len(ts) < 5 or time.perf_counter() - t0 < window:
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return sorted(ts)[len(ts) // 2], len(ts)


def bound(nbytes, flops, ms):
    """achieved rates, the binding data-sheet limit and the share of it reached."""
    t_mem, t_cmp = nbytes / PEAK_HBM, flops / PEAK_FP64_TC
    return {"bytes": int(nbytes), "flops": int(flops), "tb_per_s": round(nbytes / (ms * 1e-3) / 1e12, 3),
            "tflops": round(flops / (ms * 1e-3) / 1e12, 2),
            "bound_by": "HBM bandwidth (data sheet 3.35 TB/s)" if t_mem >= t_cmp else "fp64 tensor cores (data sheet 67 TFLOP/s)",
            "share_of_datasheet_bound": round(max(t_mem, t_cmp) / (ms * 1e-3), 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="kdd119,kdd41,cicids78")
    ap.add_argument("--rows", type=int, default=0, help="rows of every shape (default: the datasets' sizes)")
    ap.add_argument("--ks", default="8,32")
    ap.add_argument("--window", type=float, default=2.0)
    ap.add_argument("--oracle-rows", type=int, default=20000)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_pca.py needs a CUDA device")
    import pca_oracle as po
    from b200flow import dist as bdist, pca as bp
    dev_card = card()
    for shape in a.shapes.split(","):
        x = features(shape, a.rows)
        n, D = x.shape
        sh = bdist.Shards(n, 0, None, x.device)
        ks = [k for k in (int(v) for v in a.ks.split(",")) if k <= D]
        mean_ms, mean_reps = window_ms(lambda: bp.column_sums(x, sh), a.window)
        mean = bp.column_sums(x, sh) * (1.0 / n)
        gram_ms, gram_reps = window_ms(lambda: bp.centered_gram_total(x, mean, sh), a.window)
        k0 = ks[0]
        bp.pca_fit(x, k0)                                                     # untimed
        torch.cuda.synchronize()
        fits = []
        t_end = time.perf_counter() + a.window
        while len(fits) < 3 or time.perf_counter() < t_end:
            t0 = time.perf_counter()
            fit = bp.pca_fit(x, k0)
            torch.cuda.synchronize()
            fits.append((time.perf_counter() - t0) * 1e3)
        nc = (n + bdist.CHUNK - 1) // bdist.CHUNK
        res = {"shape": shape, "rows": n, "D": D, "chunks": nc,
               "mean_ms": round(mean_ms, 3), "mean_reps": mean_reps,
               "mean_tb_per_s": round(8.0 * n * D / (mean_ms * 1e-3) / 1e12, 3),
               "gram_ms": round(gram_ms, 3), "gram_reps": gram_reps,
               "gram": bound(8.0 * n * D + 8.0 * nc * (D * (D + 1) // 2), 1.0 * n * D * (D + 1), gram_ms),
               "fit_ms": round(sorted(fits)[len(fits) // 2], 3), "fit_reps": len(fits), "fit_k": k0, "project": {}}
        for k in ks:
            pc = torch.from_numpy(np.ascontiguousarray(bp.components(fit.cov, k)[0])).to(x.device)
            ms, reps = window_ms(lambda: bp.project(x, pc), a.window)
            res["project"][str(k)] = dict(ms=round(ms, 3), reps=reps, **bound(8.0 * n * (D + k), 2.0 * n * D * k, ms))
        m = min(a.oracle_rows, n)
        xo = x[:m].cpu().numpy()
        got, want = bp.pca_fit(x[:m].contiguous(), k0), po.fit(xo, k0)
        res["oracle_rows"] = m
        res["oracle_cov_match"] = bool(np.max(np.abs(got.cov - want[3])) <= 1e-10 * np.max(np.abs(want[3])) and
                                       np.max(np.abs(got.explained_variance - want[1])) <= 1e-10)
        res["explained_variance"] = [float(v) for v in fit.explained_variance]
        res["card"] = dev_card
        print(json.dumps(res), flush=True)
        del x
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
