"""Time GeneralizedLinearRegression on a KDD99-full-shaped set: --rows flows (default 4,898,431) encoded by the shim
pipeline StringIndexer -> OneHotEncoder -> VectorAssembler -> StandardScaler (D = 119, f64), with Poisson, gamma and
Bernoulli labels drawn from a seeded coefficient vector.

It reports
  * one IRLS rows pass (b200flow.glm.rows_total in REWEIGHT mode, poisson/log) and one weighted Gram pass
    (pca.centered_gram_total with w) with CUDA events, the median of --repeats, each alternated in the same run with a
    plain torch fp64 arm computing the same totals, and the largest difference relative to the largest total;
  * bytes/s of the rows pass (x, y and the two [n] outputs: n (8 D + 8 + 16) bytes) against the data sheet's 3.35 TB/s
    HBM, and FLOP/s of the Gram pass (2 n (D + 1)(D + 2) / 2 multiply-adds as FLOPs) against the 67 TFLOP/s fp64
    tensor-core data-sheet figure, with the bound that applies (both 700 W figures; the card's power limit is read in the
    same run);
  * host-timed fits after one untimed fit each, poisson/log, gamma/log and binomial/logit, with iteration counts.
One JSON line.

    python tools/bench_glm.py [--rows 4898431] [--repeats 10]
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
PEAK_FP64_TC = 67e12


def torch_reweight(x, y, coef, b):
    """the same [D + 2] totals as REWEIGHT mode for poisson/log, with torch fp64 ops"""
    eta = x @ coef + b
    mu = torch.exp(eta).clamp_min(1e-16)
    z = eta + (y - mu) / mu
    w = mu
    return torch.cat([w.sum().reshape(1), w @ x, (w * z).sum().reshape(1)])


def torch_gram(x, z, w, mx, mz):
    a = torch.cat([x - mx, (z - mz)[:, None]], 1)
    return (a * w[:, None]).t() @ a


def timed(fns, repeats):
    med = lambda ts: sorted(ts)[len(ts) // 2]                             # noqa: E731
    for f in fns + fns:
        f()
    torch.cuda.synchronize()
    ts = [[] for _ in fns]
    for _ in range(repeats):
        for f, t in zip(fns, ts):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            f()
            e1.record()
            e1.synchronize()
            t.append(e0.elapsed_time(e1))
    return [med(t) for t in ts]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=4898431)
    ap.add_argument("--repeats", type=int, default=10)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_glm.py needs a CUDA device")
    from b200flow import dist as bdist, glm as bg, pca
    dev_card = card()
    x, _ = features(a.rows, 23, 2019)
    n, D = x.shape
    rng = np.random.default_rng(5)
    beta = torch.from_numpy(rng.normal(0.0, 0.3, D) / np.sqrt(D)).cuda()
    eta = x @ beta + 0.2
    g = torch.Generator(device="cuda").manual_seed(5)
    labels = {"poisson": torch.poisson(torch.exp(eta), generator=g),
              "gamma": torch.distributions.Gamma(torch.full_like(eta, 2.0), 2.0 / torch.exp(eta)).sample(),
              "binomial": (torch.rand(n, device="cuda", dtype=torch.float64, generator=g) < torch.sigmoid(eta)).double()}
    sh = bdist.Shards(n, 0, None, x.device)
    spec = bg.resolve(bg.GLMParams(family="poisson"))
    y = labels["poisson"].contiguous()
    coef = (beta * 0.9).contiguous()
    ours = lambda: bg.rows_total(x, y, None, None, coef, 0.2, spec, bg.REWEIGHT, sh)        # noqa: E731
    ref = lambda: torch_reweight(x, y, coef, 0.2)                                         # noqa: E731
    t_rows, t_rows_ref = timed([ours, ref], a.repeats)
    got, want = ours()[0], ref()
    rows_bytes = n * (8.0 * D + 8 + 16)
    zw = ours()[1]
    z, w = zw[:, 0].contiguous(), zw[:, 1].contiguous()
    mx = (w @ x) / w.sum()
    mz = float((w @ z) / w.sum())
    gram = lambda: pca.centered_gram_total(x, mx, sh, y=z, y_mean=mz, w=w)                # noqa: E731
    gref = lambda: torch_gram(x, z, w, mx, mz)                                            # noqa: E731
    t_gram, t_gram_ref = timed([gram, gref], a.repeats)
    q, G = gram().cpu().numpy(), gref().cpu().numpy()
    iu = np.triu_indices(D + 1)
    gdiff = float(np.max(np.abs(q[iu[0] + iu[1] * (iu[1] + 1) // 2] - G[iu])) / np.max(np.abs(G)))
    flops = 2.0 * n * (D + 1) * (D + 2) / 2
    gram_bytes = n * 8.0 * (D + 2)
    gram_bound = max(flops / PEAK_FP64_TC, gram_bytes / PEAK_HBM)
    passes = {"rows_pass": {"ms": round(t_rows, 3), "torch_fp64_ms": round(t_rows_ref, 3),
                            "max_rel_diff": float(((got - want).abs().max() / want.abs().max()).item()),
                            "gb_per_s": round(rows_bytes / (t_rows * 1e-3) / 1e9, 1),
                            "share_of_hbm_datasheet": round(rows_bytes / PEAK_HBM / (t_rows * 1e-3), 3), "bound": "HBM"},
              "weighted_gram": {"ms": round(t_gram, 3), "torch_fp64_ms": round(t_gram_ref, 3), "max_rel_diff": gdiff,
                                "tflop_per_s": round(flops / (t_gram * 1e-3) / 1e12, 2),
                                "gb_per_s": round(gram_bytes / (t_gram * 1e-3) / 1e9, 1),
                                "share_of_datasheet_bound": round(gram_bound / (t_gram * 1e-3), 3),
                                "bound": "fp64 tensor core" if flops / PEAK_FP64_TC > gram_bytes / PEAK_HBM else "HBM"}}
    fits = {}
    for name, p in (("poisson_log", bg.GLMParams(family="poisson")), ("gamma_log", bg.GLMParams(family="gamma", link="log")),
                    ("binomial_logit", bg.GLMParams(family="binomial"))):
        yy = labels[name.split("_")[0]].contiguous()
        bg.glm_fit(x, yy, p)                                                 # untimed fit
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        f = bg.glm_fit(x, yy, p)
        torch.cuda.synchronize()
        fits[name] = {"s": round(time.perf_counter() - t0, 3), "iterations": f.iterations,
                      "cholesky": f.diag_inv_atwa is not None}
    print(json.dumps({"rows": n, "D": D, "passes": passes, "fits": fits, "card": dev_card}), flush=True)


if __name__ == "__main__":
    main()
