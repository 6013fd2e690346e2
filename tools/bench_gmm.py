"""Time GaussianMixture on a KDD99-full-shaped training split: --rows flows (default 3,673,823 = 75 % of 4,898,431) encoded by
the shim pipeline StringIndexer -> OneHotEncoder -> VectorAssembler -> StandardScaler (D = 119, bench_kmeans.features), then
b200flow.gmm.gmm_fit with tol = 0 so that EM runs all --max-iter iterations, for each k of --ks.

Per k it reports
  * the fit time (host clock around a fit that ends in a device synchronise, after one untimed fit),
  * per-iteration CUDA-event medians of --repeats: the E-step kernel, the moments kernel, the chunk chain and the host
    eigendecompositions + broadcast, on the fitted parameters,
  * achieved fp64 rates from shape-computed FLOPs, 2 n k Dp^2 for the E-step (Dp = ceil8(D)) and n k Da (Da + 8) for the
    upper-triangle moments (Da = ceil8(D + 1)), and their share of the data sheet's 67 TFLOP/s fp64 tensor-core peak (a
    700 W figure, not a measured one; the card's power limit is read in the same run),
  * a plain torch fp64 arm (batched matmuls for the same whitening and Gram) alternated with the kernels, and the largest
    difference of its sums from the kernels' relative to the largest sum,
  * whether one EM step on the first --oracle-rows rows matches tests/gmm_oracle.py (relative 1e-10).
One JSON line per k.

    python tools/bench_gmm.py [--rows 3673823] [--ks 5,23] [--max-iter 10] [--repeats 10] [--oracle-rows 20000]
"""
import argparse
import json
import math
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

PEAK_FP64_TC = 67e12


def torch_sums(x, means, roots, c):
    """LL, W, S and the full Q of every component with torch fp64 matmuls (the same E-step, in log space), one component
    at a time so that one [n, D] whitened block is live."""
    k = means.shape[0]
    s = torch.empty((x.shape[0], k), dtype=torch.float64, device=x.device)
    for i in range(k):
        y = (x - means[i]) @ roots[i].t()
        s[:, i] = c[i] - 0.5 * (y * y).sum(1)
    t = torch.logaddexp(torch.tensor(math.log(2.220446049250313e-16), dtype=torch.float64, device=x.device), s)
    lse = torch.logsumexp(t, 1)
    r = torch.exp(t - lse[:, None])
    Q = torch.stack([(x * r[:, i:i + 1]).t() @ x for i in range(k)])
    return lse.sum(), r.sum(0), r.t() @ x, Q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=3673823)
    ap.add_argument("--ks", default="5,23")
    ap.add_argument("--max-iter", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=10)
    ap.add_argument("--oracle-rows", type=int, default=20000)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_gmm.py needs a CUDA device")
    import gmm_oracle as go
    from b200flow import dist as bdist, gmm as bg
    dev_card = card()
    x = features(a.rows, 2019)
    n, D = x.shape
    Dp, Da = (D + 7) // 8 * 8, (D + 8) // 8 * 8
    sh = bdist.Shards(n, 0, None, x.device)
    xo = x[:a.oracle_rows].cpu().numpy()
    for k in [int(v) for v in a.ks.split(",")]:
        bg.gmm_fit(x, k, max_iter=a.max_iter, tol=0.0, seed=1)               # untimed
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fit = bg.gmm_fit(x, k, max_iter=a.max_iter, tol=0.0, seed=1)
        torch.cuda.synchronize()
        fit_s = time.perf_counter() - t0
        mu = torch.from_numpy(fit.means).cuda()
        roots, c = fit.roots, fit.log_consts
        P = bg.width(k, D)
        nc = (n + 4095) // 4096
        nb = max(1, bg.PARTIALS_BUDGET // (8 * (P + 4096 * k)))
        rows = min(n, nb * 4096)
        parts = torch.empty((min(nc, nb), P), dtype=torch.float64, device="cuda")
        resp = torch.empty((rows, k), dtype=torch.float64, device="cuda")
        xb = x[:rows]
        scale = n / rows                                                      # one batch, scaled to all the rows
        e_ms = event_ms(lambda: bg.estep(xb, mu, roots, c, 0, resp=resp, partials=parts), a.repeats) * scale
        m_ms = event_ms(lambda: bg.moments(xb, resp, 0, parts), a.repeats) * scale
        ch_ms = event_ms(lambda: bdist.chunk_chain(parts, parts.shape[0], 1, P, sh), a.repeats) * scale
        h_ms = event_ms(lambda: bg._constants(fit.covariances, fit.weights, sh, x.device), a.repeats)
        ours = lambda: bg.em_sums(x, mu, roots, c, sh)                        # noqa: E731
        ref = lambda: torch_sums(x, mu, roots, c)                             # noqa: E731
        t_ours, t_ref = [], []
        for f, ts in ((ours, t_ours), (ref, t_ref)) * (a.repeats // 2 + 1):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            f()
            e1.record()
            e1.synchronize()
            ts.append(e0.elapsed_time(e1))
        med = lambda ts: sorted(ts[1:])[len(ts[1:]) // 2]                    # noqa: E731
        tot = ours().cpu().numpy()
        ll, W, S, Q = ref()
        per = 1 + D + D * (D + 1) // 2
        iu = np.triu_indices(D)
        pos = iu[0] + iu[1] * (iu[1] + 1) // 2
        Qn = Q.cpu().numpy()
        diffs = []
        for i in range(k):
            b = 1 + i * per
            diffs.append(abs(tot[b] - float(W[i])) / max(1.0, abs(float(W[i]))))
            diffs.append(np.max(np.abs(tot[b + 1:b + 1 + D] - S[i].cpu().numpy())) / max(1.0, float(S[i].abs().max())))
            q = Qn[i][iu]
            diffs.append(np.max(np.abs(tot[b + 1 + D:b + per][pos] - q)) / max(1.0, np.abs(q).max()))
        diffs.append(abs(tot[0] - float(ll)) / abs(float(ll)))
        got = (lambda t: (float(t[0]),) + bg.m_step(t, k, D))(
            bg.em_sums(torch.from_numpy(xo).cuda(), mu, roots, c, bdist.Shards(xo.shape[0], 0, None, x.device)).cpu().numpy())
        want = go.em_step(xo, fit.weights, fit.means, fit.covariances)
        oracle_ok = abs(got[0] - want[0]) <= 1e-10 * abs(want[0]) and all(
            np.max(np.abs(g - e)) <= 1e-10 * np.max(np.abs(e)) for g, e in zip(got[1:], want[1:]))
        fe, fm = 2.0 * n * k * Dp * Dp, 1.0 * n * k * Da * (Da + 8)
        print(json.dumps({
            "rows": n, "D": D, "k": k, "max_iter": a.max_iter, "num_iter": fit.num_iter, "fit_s": round(fit_s, 3),
            "estep_ms": round(e_ms, 3), "moments_ms": round(m_ms, 3), "chain_ms": round(ch_ms, 3),
            "host_eigh_bcast_ms": round(h_ms, 3), "batch_chunks": min(nc, nb),
            "estep_tflops": round(fe / (e_ms * 1e-3) / 1e12, 2), "moments_tflops": round(fm / (m_ms * 1e-3) / 1e12, 2),
            "estep_share_of_datasheet_67_tflops": round(fe / (e_ms * 1e-3) / PEAK_FP64_TC, 4),
            "moments_share_of_datasheet_67_tflops": round(fm / (m_ms * 1e-3) / PEAK_FP64_TC, 4),
            "em_sums_ms": round(med(t_ours), 3), "torch_fp64_ms": round(med(t_ref), 3),
            "max_rel_diff_vs_torch": float(max(diffs)), "oracle_step_match": bool(oracle_ok),
            "log_likelihood": fit.log_likelihood, "card": dev_card}), flush=True)


if __name__ == "__main__":
    main()
