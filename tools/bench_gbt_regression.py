"""Time GBTRegressor on a KDD99-full-shaped set: tools/bench_regression.py's data (--rows flows, default 4,898,431, assembled
by StringIndexer -> VectorAssembler into 40 features without dst_bytes, 3 of them categorical; label log1p(dst_bytes)),
maxBins 70, 20 iterations at depth 5 (Spark's defaults), for both losses.

It reports
  * fit (host clock around a synchronised fit, after one untimed fit);
  * CUDA-event time per phase of the fit: variance histograms, split scoring, node-pool growth, partition, the margin /
    residual update with its max |r| (gbr_update), the residual grid (gbr_grid), and the per-iteration host read of the
    reduced max (gbr_sync: device time from the read's start until the stream resumes);
  * transform of every row and evaluateEachIteration over every row (CUDA events, median of --repeats);
  * GBTClassifier's fit on the same features (20 iterations, depth 5, label = attack or not), for scale;
  * the CPU restatement (tests/gbt_regression_oracle.py) on the first --oracle-rows rows: whether the device model, its
    training margins and its predictions equal it bit for bit.
One JSON line, with the card's name and power limit read in the same run.

    python tools/bench_gbt_regression.py [--rows 4898431] [--oracle-rows 20000] [--repeats 5]
"""
import argparse
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

from bench_regression import events, features, phases, timed_fit  # noqa: E402
from bench_tuning import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=4_898_431)
    ap.add_argument("--oracle-rows", type=int, default=20000)
    ap.add_argument("--repeats", type=int, default=5)
    a = ap.parse_args()
    from b200flow import gbt as bg, gbt_regression as bgr
    torch.cuda.set_device(0)
    x, y, cls, arity = features(a.rows, 1)
    out = dict(tool="bench_gbt_regression", rows=a.rows, features=x.shape[1], card=card())
    for loss in ("squared", "absolute"):
        p = bgr.GBTRegressorParams(max_iter=20, max_depth=5, max_bins=70, seed=7, loss=loss)
        model, ms = timed_fit(lambda: bgr.fit_gbt_regressor(x, y, arity, p))
        r = dict(fit_ms=round(ms, 1), nodes=model.n_nodes, unique_rows=model.train_stats["unique_rows"],
                 levels=model.train_stats["levels"], E=model.E, S=model.S)
        r["phases_ms"] = phases(bg, lambda: bgr.fit_gbt_regressor(x, y, arity, p))
        r["transform_ms"] = round(events(lambda: model.predict(x), a.repeats), 2)
        r["evaluate_each_iteration_ms"] = round(events(lambda: model.evaluate_each_iteration(x, y, loss), a.repeats), 2)
        r["final_loss"] = model.evaluate_each_iteration(x, y, loss)[-1]
        out[loss] = r
    gp = bg.GBTParams(max_iter=20, max_depth=5, max_bins=70, seed=7)
    binary = (cls > 0).to(torch.int32)
    _, ms = timed_fit(lambda: bg.fit_gbt(x, binary, arity, gp))
    out["gbt_classifier_fit_ms"] = round(ms, 1)
    if a.oracle_rows:
        import gbt_regression_oracle as gro
        k = min(a.oracle_rows, a.rows)
        xk, yk = x[:k].contiguous(), y[:k].contiguous()
        same = {}
        for loss in ("squared", "absolute"):
            p = bgr.GBTRegressorParams(max_iter=20, max_depth=5, max_bins=70, seed=7, loss=loss)
            model = bgr.fit_gbt_regressor(xk, yk, arity, p)
            t0 = time.perf_counter()
            want = gro.fit(xk.cpu().numpy(), yk.cpu().numpy(), arity, max_iter=20, max_depth=5, max_bins=70, seed=7, loss=loss)
            out["oracle_s_" + loss] = round(time.perf_counter() - t0, 1)
            got, exp = model.export(), gro.export(want)
            margin = model.train_margin if model.train_uid is None else model.train_margin[model.train_uid.long()]
            same[loss] = (all(np.array_equal(np.asarray(got[c]).view(np.uint8), np.asarray(exp[c]).view(np.uint8))
                              for c in ("tree", "nid", "feat", "kind", "bin_thr", "is_leaf", "mask", "stats", "payload", "gain"))
                          and model.E == want["E"]
                          and np.array_equal(margin.cpu().numpy().view(np.int64), want["margin"].view(np.int64))
                          and np.array_equal(model.predict(xk).cpu().numpy().view(np.int64),
                                             gro.predict_x(want, xk.cpu().numpy()).view(np.int64)))
        out["oracle_rows"], out["oracle_same_bits"] = k, same
        out["equal"] = all(same.values())
    print(json.dumps(out))


if __name__ == "__main__":
    main()
