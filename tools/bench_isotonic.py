"""Time IsotonicRegression (b200flow.isotonic, DESIGN.md §5p) at three shapes of --rows rows (default 4,898,431, the
KDD99-full row count), from seeded data:
  * distinct: uniform features, almost all distinct, a noisy increasing label;
  * calibration: forest-like probabilities, 21 distinct scores with 60 % of the rows at 0.0 (one tie run of ~2.9 M rows
    summed on one thread), a Bernoulli label;
  * junction: an increasing series with one heavy, very low point just right of the middle, so the top merge level pools
    the whole left half on one thread.
For each shape it reports the card's name and power limit (read in the same run), the host-timed fit (ending in the
device synchronise of reading the model back) and transform (ending in torch.cuda.synchronize) at the library's chunk
size, the median of --repeats after a warm-up; the tie-pool and PAV kernel times of one fit from torch.profiler in a run
of their own; and, for scale, the host time of numpy's stable argsort plus scipy.optimize.isotonic_regression on the same
rows.  For the distinct and junction shapes it also times the fit at each chunk size of --chunks.  One JSON line.

    python tools/bench_isotonic.py [--rows 4898431] [--repeats 5] [--chunks 16,32,64,128,256]
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


def shape(kind, n, seed=1):
    rng = np.random.default_rng(seed)
    if kind == "distinct":
        x = rng.uniform(0.0, 1.0, n)
        y = x + rng.normal(0.0, 0.3, n)
    elif kind == "calibration":
        x = np.where(rng.random(n) < 0.6, 0.0, np.round(rng.beta(0.7, 0.7, n) * 20) / 20)
        y = (rng.random(n) < np.clip(x * 0.9 + 0.05, 0, 1)).astype(np.float64)
    else:
        x = np.arange(n, dtype=np.float64)
        y = x.copy()
        y[n // 2 + 1] = -1e3 * n
    w = np.ones(n)
    if kind == "junction":
        w[n // 2 + 1] = 1e3
    return x, y, w


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


def kernel_ms(fn):
    """{kernel group: summed device ms} of one call, from torch.profiler"""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    groups = {"tie_pool": ("iso_tie_kernel",), "pav": ("iso_pav_chunk_kernel", "iso_pav_merge_kernel"),
              "sort": ("radix_hist_kernel", "radix_scatter_kernel"), "all": ("",)}
    out = {k: 0.0 for k in groups}
    for e in prof.events():
        if e.device_type.name != "CUDA":
            continue
        for k, names in groups.items():
            if any(s in e.name for s in names):
                out[k] += e.device_time_total / 1000.0 if hasattr(e, "device_time_total") else e.cuda_time_total / 1000.0
    return {k: round(v, 3) for k, v in out.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=4898431)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--chunks", default="16,32,64,128,256")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_isotonic needs a CUDA device")
    from scipy.optimize import isotonic_regression
    from b200flow import isotonic as biso
    res = {"card": card(), "rows": a.rows, "shapes": {}}
    for kind in ("distinct", "calibration", "junction"):
        x, y, w = shape(kind, a.rows)
        xt, yt, wt = (torch.from_numpy(v).cuda() for v in (x, y, w))
        fit = biso.isotonic_fit(xt, yt, wt)
        r = {"model_points": int(fit.boundaries.shape[0]),
             "fit_ms": round(1e3 * median_time(lambda: biso.isotonic_fit(xt, yt, wt), a.repeats), 3),
             "transform_ms": round(1e3 * median_time(lambda: biso.isotonic_predict(xt, fit), a.repeats), 3),
             "kernel_ms": kernel_ms(lambda: biso.isotonic_fit(xt, yt, wt))}
        if kind != "calibration":
            r["fit_ms_by_chunk"] = {c: round(1e3 * median_time(lambda: biso.isotonic_fit(xt, yt, wt, chunk=int(c)),
                                                               a.repeats), 3) for c in a.chunks.split(",")}
        t0 = time.perf_counter()
        o = np.argsort(x, kind="stable")
        isotonic_regression(y[o], weights=w[o], increasing=True)
        r["host_scipy_ms"] = round(1e3 * (time.perf_counter() - t0), 1)
        res["shapes"][kind] = r
        print(kind, json.dumps(r), file=sys.stderr, flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
