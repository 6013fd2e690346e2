"""Time the feature-selection passes on KDD-shaped data (b200flow.synth.make_kdd, 4,898,431 flows = KDD99-full, 23 classes):
D = 41 (indexed categoricals) and D = 119 (one-hot), f64, label = the class index.

Per shape it reports CUDA-event medians, each over enough repetitions to fill --window seconds after a warm-up:
  * distinct_ms: b200flow_distinct_values over every column, the table fill included;
  * contingency_ms: b200flow_contingency_counts over the columns with at most 10000 distinct values (the chi-square input);
  * class_sums_ms: b200flow_group_sums (G = classes) and the chain, in batches of the partial budget;
  * centered_ms: b200flow_group_centered_moments with the class means and the chain;
  * centered_g256_ms: the same pass with 256 groups (row i in group i % 256, zero centres), the kernel's widest shape;
  * fit_ms: a whole UnivariateFeatureSelector(continuous, categorical).fit (ANOVA), the label dictionary included (host
    clock around a fit that ends in a synchronise).
For every pass it reports the bytes one read of its input needs (8 n W for the W columns it reads, plus 8 n for the label)
and the achieved bytes/s against NVIDIA's data-sheet 3.35 TB/s for the H100 SXM (not a measurement).  The card's name and
power limit are read in the same run.  One JSON line per shape.

    python tools/bench_select.py [--shapes kdd41,kdd119] [--rows 4898431] [--window 2.0]
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

PEAK_HBM = 3.35e12          # data sheet, H100 SXM
KDD_ROWS = 4898431


def features(shape, rows):
    """(x f64 [n, D], label f64 [n]) on cuda:0."""
    from b200flow import encode as enc, synth
    rec, dicts = synth.make_kdd(rows, 23, seed=2019, device="cuda:0")
    plan = enc.EncodePlan(synth.kdd_schema())
    for c in synth.KDD_COLUMNS:
        if c not in synth.KDD_CATEGORICAL and c != "label":
            plan.add_numeric(c)
    for c in synth.KDD_CATEGORICAL:
        lut = np.arange(len(dicts[c]), dtype=np.int32)
        if shape == "kdd119":
            plan.add_onehot(c, lut, len(dicts[c]), drop_last=True)
        else:
            plan.add_index(c, lut)
    plan.set_label("label", np.arange(len(dicts["label"]), dtype=np.int32))
    x, y, _ = plan.run(rec, torch.float64)
    return x, y.to(torch.float64)


def event_ms(fn, window):
    fn()
    torch.cuda.synchronize()
    t0 = time.time()
    fn()
    torch.cuda.synchronize()
    reps = max(3, int(window / max(time.time() - t0, 1e-4)))
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def run(shape, rows, window):
    from b200flow import dist as bdist, selection as bs
    from b200flow._lib import call, ptr
    from pyspark.ml.feature import UnivariateFeatureSelector
    from pyspark.sql import ColumnData, DataFrame
    x, y = features(shape, rows)
    n, D = x.shape
    dev = x.device
    sh = bdist.Shards(n, 0, None, dev)
    labels, ids = bs.label_dictionary(y, sh, "bench")
    L = len(labels)
    _, counts, _ = bs.distinct_tables(x)
    low = [j for j in range(D) if int(counts[j]) <= bs.MAX_CATEGORIES]
    xl = x[:, low].contiguous()
    dicts = bs.dictionaries(xl, sh, "bench")
    off = np.concatenate([[0], np.cumsum([len(d) for d in dicts])]).astype(np.int32)
    d_all, off_t = torch.from_numpy(np.concatenate(dicts)).to(dev), torch.from_numpy(off).to(dev)
    cnt = torch.zeros(int(off[-1]) * L, dtype=torch.int64, device=dev)

    def contingency():
        cnt.zero_()
        call("b200flow_contingency_counts", ptr(xl), n, len(low), len(low), ptr(ids), L, ptr(d_all), ptr(off_t), int(off[-1]),
             ptr(cnt))

    sums, nk = bs.group_sums_total(x, ids, L, sh)
    means = (sums / torch.from_numpy(nk.astype(np.float64)).to(dev)[:, None]).contiguous()
    ms = {"distinct_ms": event_ms(lambda: bs.distinct_tables(x), window),
          "contingency_ms": event_ms(contingency, window),
          "class_sums_ms": event_ms(lambda: bs.group_sums_total(x, ids, L, sh), window),
          "centered_ms": event_ms(lambda: bs.centered_moments_total(x, ids, L, means, None, 0.0, sh), window)}
    # the widest class count the kernels take: 256 groups (row i in group i % 256) leave 24 columns per CTA
    ids256 = (torch.arange(n, device=dev) % 256).to(torch.int32)
    means256 = torch.zeros((256, D), dtype=torch.float64, device=dev)
    ms["centered_g256_ms"] = event_ms(lambda: bs.centered_moments_total(x, ids256, 256, means256, None, 0.0, sh), window)
    df = DataFrame(n, None, None, {}, {"features": ColumnData("vector", x, "f64"), "label": ColumnData("numeric", y, "f64")})
    sel = UnivariateFeatureSelector(selectionMode="numTopFeatures").setFeatureType("continuous").setLabelType("categorical") \
        .setSelectionThreshold(20)
    sel.fit(df)
    fits = []
    for _ in range(3):
        torch.cuda.synchronize()
        t0 = time.time()
        sel.fit(df)
        torch.cuda.synchronize()
        fits.append((time.time() - t0) * 1e3)
    widths = {"distinct_ms": D, "contingency_ms": len(low), "class_sums_ms": D, "centered_ms": D, "centered_g256_ms": D}
    out = {"shape": shape, "rows": n, "D": D, "classes": L, "chi_square_columns": len(low), "fit_ms": float(np.median(fits))}
    for k, v in ms.items():
        b = 8 * n * widths[k] + (8 * n if k != "distinct_ms" else 0)
        out[k] = round(v, 3)
        out[k.replace("_ms", "_bytes")] = b
        out[k.replace("_ms", "_TBps")] = round(b / (v * 1e-3) / 1e12, 3)
        out[k.replace("_ms", "_of_datasheet")] = round(b / (v * 1e-3) / PEAK_HBM, 3)
    out["card"] = card()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="kdd41,kdd119")
    ap.add_argument("--rows", type=int, default=KDD_ROWS)
    ap.add_argument("--window", type=float, default=2.0)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_select needs a CUDA device")
    for s in a.shapes.split(","):
        print(json.dumps(run(s, a.rows, a.window)), flush=True)


if __name__ == "__main__":
    main()
