"""Time LinearRegression on a KDD99-full-shaped set: --rows flows (default 4,898,431) encoded by the shim pipeline
StringIndexer -> OneHotEncoder -> VectorAssembler -> StandardScaler (D = 119, f64), with a seeded linear label and
heavy-tailed (Student t, 3 dof) noise.

It reports
  * one loss + gradient evaluation (b200flow.linreg.loss_grad_totals: the fused kernel and the chunk chain) in squared and
    Huber mode, with CUDA events, the median of --repeats, alternated in the same run with a plain torch fp64 arm computing
    the same totals, and the largest difference between the two relative to the largest total;
  * the achieved bytes/s of each evaluation from n D 8 bytes per pass, against the data sheet's 3.35 TB/s (a 700 W figure;
    the card's power limit is read in the same run);
  * host-timed fits after one untimed fit each: normal equations, L-BFGS, L-BFGS + L1 and Huber, with iteration counts;
  * the transform (one margin per row), CUDA events, median of --repeats, and the peak bytes of the normal path's staged
    [x, y] batch.
One JSON line.

    python tools/bench_linreg.py [--rows 4898431] [--repeats 20]
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

from bench_svc import features  # noqa: E402
from bench_tuning import card  # noqa: E402

PEAK_HBM = 3.35e12


def torch_totals(x, y, shift, inv, ys, yt, w, b, sigma, eps, huber):
    """the same [D + 3] totals as loss_grad_totals, with torch fp64 ops"""
    xs = ((x - shift) if shift is not None else x) * inv
    m = xs @ w
    if not huber:
        d = m - (y - ys) * yt
        return torch.cat([(d * d).sum().reshape(1), d @ xs, d.sum().reshape(1), torch.zeros(1, dtype=x.dtype, device=x.device)])
    z = (y - m - b) / sigma
    inner = z.abs() <= eps
    loss = torch.where(inner, sigma + z * z * sigma, sigma + (2 * eps * z.abs() - eps * eps) * sigma)
    a = torch.where(inner, -2.0 * z, -2.0 * eps * torch.sign(z))
    s = torch.where(inner, 1.0 - z * z, torch.full_like(z, 1.0 - eps * eps))
    return torch.cat([loss.sum().reshape(1), a @ xs, a.sum().reshape(1), s.sum().reshape(1)])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=4898431)
    ap.add_argument("--repeats", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_linreg.py needs a CUDA device")
    from b200flow import dist as bdist, linreg as blr, pca
    dev_card = card()
    x, _ = features(a.rows, 23, 2019)
    n, D = x.shape
    rng = np.random.default_rng(5)
    beta = torch.from_numpy(rng.normal(0.0, 1.0, D)).cuda()
    noise = torch.from_numpy(rng.standard_t(3, n)).cuda()
    y = (x @ beta + 3.0 + noise).contiguous()
    sh = bdist.Shards(n, 0, None, x.device)
    mx = x.mean(0)
    sd = x.std(0)
    inv = torch.where(sd > 0, 1.0 / torch.where(sd > 0, sd, torch.ones_like(sd)), torch.zeros_like(sd)).contiguous()
    w = torch.from_numpy(rng.normal(0.0, 0.05, D)).cuda()
    bs = torch.tensor([0.3, 2.0], dtype=torch.float64, device="cuda")
    ys, yt = float(y.mean()), 1.0 / float(y.std())
    med = lambda ts: sorted(ts)[len(ts) // 2]                             # noqa: E731
    evals = {}
    for mode, huber in (("squared", False), ("huber", True)):
        args = (None, inv, 0.0, 1.0, w, bs, 1.35, blr.HUBER) if huber else (mx, inv, ys, yt, w, None, 0.0, blr.SQUARED)
        ours = lambda: blr.loss_grad_totals(x, y, *args[:6], args[6], args[7], sh)         # noqa: E731
        ref = (lambda: torch_totals(x, y, None, inv, 0.0, 1.0, w, 0.3, 2.0, 1.35, True)) if huber else \
            (lambda: torch_totals(x, y, mx, inv, ys, yt, w, 0.0, 1.0, 0.0, False))
        for f in (ours, ref, ours, ref):
            f()
        torch.cuda.synchronize()
        t_ours, t_ref = [], []
        for _ in range(a.repeats):
            for f, ts in ((ours, t_ours), (ref, t_ref)):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                f()
                e1.record()
                e1.synchronize()
                ts.append(e0.elapsed_time(e1))
        got, want = ours(), ref()
        ms = med(t_ours)
        nbytes = n * D * 8.0
        evals[mode] = {"ms": round(ms, 3), "torch_fp64_ms": round(med(t_ref), 3),
                       "max_rel_diff": float(((got - want).abs().max() / want.abs().max()).item()),
                       "gb_per_s": round(nbytes / (ms * 1e-3) / 1e9, 1),
                       "share_of_hbm_datasheet": round(nbytes / PEAK_HBM / (ms * 1e-3), 3)}
    fits = {}
    for name, p in (("normal", blr.LinRegParams()), ("lbfgs", blr.LinRegParams(solver="l-bfgs")),
                    ("lbfgs_l1", blr.LinRegParams(solver="l-bfgs", reg_param=0.01, elastic_net_param=1.0)),
                    ("huber", blr.LinRegParams(loss="huber", reg_param=0.01))):
        blr.linreg_fit(x, y, p)                                            # untimed fit
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        f = blr.linreg_fit(x, y, p)
        torch.cuda.synchronize()
        fits[name] = {"s": round(time.perf_counter() - t0, 3), "iterations": f.iterations, "solver": f.solver,
                      "objective": f.objective_history[-1], "scale": f.scale}
    fit = blr.linreg_fit(x, y, blr.LinRegParams())
    tr = []
    blr.linreg_predict(x, fit)
    for _ in range(a.repeats):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        blr.linreg_predict(x, fit)
        e1.record()
        e1.synchronize()
        tr.append(e0.elapsed_time(e1))
    staged = min(pca.stage_rows(D), n) * (D + 1) * 8
    print(json.dumps({"rows": n, "D": D, "eval": evals, "fits": fits, "transform_ms": round(med(tr), 3),
                      "normal_staging_bytes": staged, "card": dev_card}), flush=True)


if __name__ == "__main__":
    main()
