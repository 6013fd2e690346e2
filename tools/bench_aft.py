"""Time AFTSurvivalRegression on a KDD99-full-shaped set: --rows flows (default 4,898,431) encoded by the shim pipeline
StringIndexer -> OneHotEncoder -> VectorAssembler -> StandardScaler (D = 119), with seeded Weibull lifetimes
(log t = x . beta + b + sigma log E, E ~ Exp(1)) right-censored at an independent exponential time.

It reports, for f64 features and their f32 copy,
  * one loss + gradient evaluation (b200flow.aft.loss_grad_totals: the fused kernel and the chunk chain), with CUDA events,
    the median of --repeats, alternated in the same run with a plain torch fp64 arm computing the same totals, and the
    largest difference between the two relative to the largest total;
  * the achieved bytes/s of the evaluation from n (D 8 or 4 + 12) bytes per pass (features, log t and the censor),
    against the data sheet's 3.35 TB/s (a 700 W figure; the card's power limit is read in the same run);
  * a host-timed fit after one untimed fit, with its iterations and the fitted scale;
  * the transform with quantiles (the prediction and nine quantiles per row), CUDA events, median of --repeats.
One JSON line.

    python tools/bench_aft.py [--rows 4898431] [--repeats 20]
"""
import argparse
import json
import math
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


def torch_totals(x, log_t, censor, shift, inv, w, b, sigma):
    """the same [D + 3] totals as aft.loss_grad_totals, with torch fp64 ops"""
    xs = ((x - shift) if shift is not None else x) * inv
    z = (log_t - xs @ w - b) / sigma
    ez = torch.exp(z)
    d = censor.to(torch.float64)
    loss = d * math.log(sigma) - d * z + ez
    a = (d - ez) / sigma
    s = d + (d - ez) * z
    return torch.cat([loss.sum().reshape(1), a @ xs, a.sum().reshape(1), s.sum().reshape(1)])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=4898431)
    ap.add_argument("--repeats", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_aft.py needs a CUDA device")
    from b200flow import aft as baft, dist as bdist
    dev_card = card()
    x, _ = features(a.rows, 23, 2019)
    n, D = x.shape
    rng = np.random.default_rng(5)
    beta = torch.from_numpy(rng.normal(0.0, 0.05, D)).cuda()
    gen = torch.Generator(device="cuda").manual_seed(7)
    e = torch.empty(n, dtype=torch.float64, device="cuda").exponential_(1.0, generator=gen)
    t = torch.exp(x @ beta + 1.5 + 0.7 * torch.log(e))
    cen = torch.empty(n, dtype=torch.float64, device="cuda").exponential_(1.0, generator=gen) * float(t.median()) * 3.0
    censor = (t <= cen).to(torch.float64)
    t = torch.minimum(t, cen).contiguous()
    sh = bdist.Shards(n, 0, None, x.device)
    mx = x.mean(0)
    sd = x.std(0)
    inv = torch.where(sd > 0, 1.0 / torch.where(sd > 0, sd, torch.ones_like(sd)), torch.zeros_like(sd)).contiguous()
    log_t, ci = torch.log(t).contiguous(), censor.to(torch.int32).contiguous()
    w = torch.from_numpy(rng.normal(0.0, 0.05, D)).cuda()
    b, sigma = 0.3, 1.2
    bs = torch.tensor([b, sigma, math.log(sigma)], dtype=torch.float64, device="cuda")
    med = lambda ts: sorted(ts)[len(ts) // 2]                             # noqa: E731

    def cuda_ms(f):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        f()
        e1.record()
        e1.synchronize()
        return e0.elapsed_time(e1)

    out = {"rows": n, "D": D, "censored_share": round(1.0 - float(censor.mean()), 4)}
    for name, xd in (("f64", x), ("f32", x.float().contiguous())):
        ours = lambda: baft.loss_grad_totals(xd, log_t, ci, mx, inv, w, bs, sh)            # noqa: E731
        ref = lambda: torch_totals(x, log_t, censor, mx, inv, w, b, sigma)                 # noqa: E731
        for f in (ours, ref, ours, ref):
            f()
        torch.cuda.synchronize()
        t_ours, t_ref = [], []
        for _ in range(a.repeats):
            t_ours.append(cuda_ms(ours))
            t_ref.append(cuda_ms(ref))
        got, want = ours(), ref()
        ms = med(t_ours)
        nbytes = n * (D * xd.element_size() + 12.0)
        arm = {"eval_ms": round(ms, 3), "torch_fp64_ms": round(med(t_ref), 3),
               "max_rel_diff": float(((got - want).abs().max() / want.abs().max()).item()),
               "gb_per_s": round(nbytes / (ms * 1e-3) / 1e9, 1), "share_of_hbm_datasheet": round(nbytes / PEAK_HBM / (ms * 1e-3), 3)}
        p = baft.AFTParams()
        baft.aft_fit(xd, t, censor, p)                                     # untimed fit
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fit = baft.aft_fit(xd, t, censor, p)
        torch.cuda.synchronize()
        arm.update(fit_s=round(time.perf_counter() - t0, 3), iterations=fit.iterations, scale=fit.scale,
                   objective=fit.objective_history[-1])

        def transform():
            lam = baft.aft_predict(xd, fit)
            return lam, baft.aft_predict_quantiles(xd, fit, baft.QUANTILES, lam=lam)

        transform()
        arm["transform_quantiles_ms"] = round(med([cuda_ms(transform) for _ in range(a.repeats)]), 3)
        out[name] = arm
    out["card"] = dev_card
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
