"""Time BisectingKMeans on a KDD99-full-shaped training split: --rows flows (default 3,673,823 = 75 % of 4,898,431) encoded by
the shim pipeline StringIndexer -> OneHotEncoder -> VectorAssembler -> StandardScaler (D = 119), the same features as
tools/bench_kmeans.py, then b200flow.bisecting_kmeans.bkm_fit for each k of --ks.

Per k it reports
  * the fit time (host clock around a fit that ends in a device synchronise, after one untimed fit),
  * the levels that divided clusters and the leaves produced,
  * the median CUDA-event time of one bkm_assign pass (every row picking between the root's two fitted children, the
    first level's pass) and of one bkm_predict walk of the fitted tree, each with its
    achieved bytes/s: both are bandwidth-bound passes whose floor is the n·D·8 bytes of x they must read, against the
    H100 SXM's 3.35 TB/s,
  * oracle_equal: the numpy restatement (tests/bisecting_kmeans_oracle.py) fitted on the first --oracle-rows rows equals
    the device fit of those rows bit for bit (tree, centers, costs, walk),
  * the card name and power limit, read in the same run.
One JSON line per k.

    python tools/bench_bisecting_kmeans.py [--rows 3673823] [--ks 8,23] [--max-iter 20] [--repeats 10] [--oracle-rows 20000]
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

from bench_kmeans import event_ms, features  # noqa: E402
from bench_tuning import card  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def _equal(res, want, xs):
    import bisecting_kmeans_oracle as bo
    t, w = res.tree, want["tree"]
    same = all(np.array_equal(getattr(t, key), w[key]) for key in ("heap", "left", "right", "leaf", "size"))
    same = same and np.array_equal(t.center.view(np.int64), w["center"].view(np.int64))
    same = same and np.array_equal(t.cost.view(np.int64), w["cost"].view(np.int64))
    wl, wd = bo.predict_tree(xs, w)
    return bool(same and float(res.training_cost).hex() == float(want["training_cost"]).hex() and
                np.array_equal(res.leaf.cpu().numpy(), wl) and np.array_equal(res.dist.cpu().numpy().view(np.int64), wd.view(np.int64)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=3673823)
    ap.add_argument("--ks", default="8,23")
    ap.add_argument("--max-iter", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=10)
    ap.add_argument("--oracle-rows", type=int, default=20000)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_bisecting_kmeans.py needs a CUDA device")
    import bisecting_kmeans_oracle as bo
    from b200flow import bisecting_kmeans as bb
    dev_card = card()
    x = features(a.rows, 2019)
    n, D = x.shape
    for k in [int(v) for v in a.ks.split(",")]:
        bb.bkm_fit(x, k, max_iter=a.max_iter, seed=1)                             # warm-up
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = bb.bkm_fit(x, k, max_iter=a.max_iter, seed=1)
        torch.cuda.synchronize()
        fit_s = time.perf_counter() - t0
        tree = res.tree
        # one assign pass in which every row divides: the first level, the root against its two fitted children
        slot = np.full(tree.heap.shape[0], -1, np.int32)
        slot[0] = 0
        kids = [c for c in (tree.left[0], tree.right[0])]
        centers = np.stack([tree.center[max(c, 0)] for c in kids])
        present = np.array([c >= 0 for c in kids], np.uint8)
        args = (x, torch.zeros(n, dtype=torch.int32, device=x.device), torch.from_numpy(slot).to(x.device),
                torch.from_numpy(centers).to(x.device), torch.from_numpy(present).to(x.device))
        assign_ms = event_ms(lambda: bb.bkm_assign(*args), a.repeats)
        predict_ms = event_ms(lambda: bb.bkm_predict(x, tree), a.repeats)
        x_bytes = float(n) * D * 8
        m = min(a.oracle_rows, n)
        xs = x[:m].contiguous()
        xh = xs.cpu().numpy()
        small = bb.bkm_fit(xs, k, max_iter=a.max_iter, seed=1)
        want = bo.fit(xh, k, max_iter=a.max_iter, seed=1)
        print(json.dumps({
            "rows": n, "D": D, "k": k, "max_iter": a.max_iter, "levels": res.levels, "leaves": tree.num_leaves,
            "training_cost": res.training_cost, "fit_s": round(fit_s, 4),
            "assign_ms": assign_ms,
            "assign_gb_per_s": round(x_bytes / (assign_ms * 1e-3) / 1e9, 1),
            "predict_ms": predict_ms, "predict_gb_per_s": round(x_bytes / (predict_ms * 1e-3) / 1e9, 1),
            "bound": "bandwidth: n*D*8 bytes of x per pass against %.2f TB/s HBM3" % (HBM_BYTES_PER_S / 1e12),
            "bound_ms": round(x_bytes / HBM_BYTES_PER_S * 1e3, 3),
            "oracle_rows": m, "oracle_equal": _equal(small, want, xh), "card": dev_card}), flush=True)


if __name__ == "__main__":
    main()
