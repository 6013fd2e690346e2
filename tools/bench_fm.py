"""Time FMClassifier and OneVsRest(FMClassifier) on a KDD99-full-shaped set: --rows flows (default 4,898,431) with
--classes labels (default 23, as KDD99) encoded by the shim pipeline StringIndexer -> OneHotEncoder -> VectorAssembler ->
StandardScaler (D = 119, f64), with --factor-size factors (default 8, Spark's default).

It reports
  * one loss + gradient evaluation (b200flow.fm.fm_loss_grad_totals: the fused kernel and the chunk chain) at K = 1 and
    K = --classes columns, with CUDA events, the median of --repeats, alternated in the same run with a plain torch fp64
    arm (cuBLAS matmuls and elementwise ops over row blocks) computing the same totals, and the largest difference between
    the two relative to the largest total;
  * the achieved bytes/s and FLOP/s of each evaluation, from the padded shapes the kernel runs (below), and the least time
    the data sheet allows (the larger of bytes / 3.35 TB/s and FLOPs / 67 TFLOP/s, 700 W figures; the card's power limit
    is read in the same run) and which of the two bounds it;
  * a binary fit (normal vs attack) at the defaults, host-timed after one untimed fit;
  * OneVsRest(FMClassifier) at maxIter = --ovr-max-iter: the class-batched fit against K standalone fits run one after
    the other, both host-timed, and a hash of every model of each (they must be equal);
  * the OneVsRest transform (K raw values in one launch and the first argmax), CUDA events, median of --repeats;
  * FMRegressor: one squared-error evaluation (b200flow.fm.fm_regression_loss_grad_totals) against the torch fp64 arm,
    as above, and a fit at the defaults but stepSize 0.01, host-timed after one untimed fit, of a seeded label with a
    pairwise and a linear part.  --regressor-only skips the classifier arms.
One JSON line.

    python tools/bench_fm.py [--rows 4898431] [--classes 23] [--factor-size 8] [--repeats 10] [--ovr-max-iter 30]
                             [--regressor-only]
"""
import argparse
import hashlib
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

from bench_svc import PEAK_FP64_TC, PEAK_HBM, features, pad8  # noqa: E402
from bench_tuning import card  # noqa: E402

TORCH_ROWS = 1 << 19


def work(n, D, kf, K):
    """(bytes, FLOPs) of one loss + gradient pass from the kernel's padded shapes: each class block reads x once (8 B per
    feature) and its labels; per row, S = X U and Q = X^2 U^2 over pad8(kb (k + 1)) columns per block, the gradient
    [X, 1]^T [g S | g] over the same columns and X^2^T g over pad8(kb), each over pad8(D + 1) features, 2 FLOPs per
    multiply-add"""
    from b200flow import _lib
    kb, blocks, _ = _lib.fm_config(D, kf, K)
    dp, nc, kc = pad8(D + 1), blocks * pad8(kb * (kf + 1)), blocks * pad8(kb)
    return blocks * n * (D * 8.0 + 4.0), 2.0 * n * dp * (3 * nc + kc)


def torch_totals(x, y, pos, w, kf):
    """the same totals as fm_loss_grad_totals ([K, D (k + 1) + D + 3]) with cuBLAS and torch ops, over row blocks; pos None:
    fm_regression_loss_grad_totals' squared error against the f64 labels y"""
    n, D = x.shape
    K, nv = w.shape[0], D * kf
    U = torch.cat([w[:, :nv].reshape(K, D, kf), w[:, nv:nv + D].reshape(K, D, 1)], 2).permute(1, 0, 2).reshape(D, -1)
    U2, b = U * U, w[:, -1]
    out = torch.zeros((K, D * (kf + 1) + D + 3), dtype=torch.float64, device=x.device)
    for s in range(0, n, TORCH_ROWS):
        xc, yc = x[s:s + TORCH_ROWS], y[s:s + TORCH_ROWS]
        m = xc.shape[0]
        x2 = xc * xc
        S = (xc @ U).view(m, K, kf + 1)
        Q = (x2 @ U2).view(m, K, kf + 1)
        r = b + S[:, :, kf] + 0.5 * (S[:, :, :kf] * S[:, :, :kf] - Q[:, :, :kf]).sum(2)
        if pos is None:
            d = r - yc[:, None]
            g = 2.0 * d
            loss = (d * d).sum(0)
        else:
            yk = (yc.long()[:, None] == pos.long()[None, :]).to(torch.float64)
            g = torch.sigmoid(r) - yk
            loss = torch.where(yk > 0, torch.nn.functional.softplus(-r), torch.nn.functional.softplus(r)).sum(0)
        M = S * g[:, :, None]
        M[:, :, kf] = g
        G = (xc.t() @ M.view(m, -1)).view(D, K, kf + 1)
        out[:, 0] += loss
        out[:, 1] += m
        out[:, 2:2 + nv] += G[:, :, :kf].permute(1, 0, 2).reshape(K, nv)
        out[:, 2 + nv:2 + nv + D] += G[:, :, kf].t()
        out[:, 2 + nv + D] += g.sum(0)
        out[:, 3 + nv + D:] += (x2.t() @ g).t()
    return out


def model_hash(fits):
    h = hashlib.sha256()
    for f in fits:
        for a in (f.factors, f.linear, [f.intercept]):
            h.update(np.ascontiguousarray(a, np.float64).tobytes())
    return h.hexdigest()[:16]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=4898431)
    ap.add_argument("--classes", type=int, default=23)
    ap.add_argument("--factor-size", type=int, default=8)
    ap.add_argument("--repeats", type=int, default=10)
    ap.add_argument("--ovr-max-iter", type=int, default=30)
    ap.add_argument("--regressor-only", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fm.py needs a CUDA device")
    from b200flow import dist as bdist, fm as bfm
    from pyspark.ml.classification import _first_argmax
    dev_card = card()
    x, y = features(a.rows, a.classes, 2019)
    n, D = x.shape
    K, kf = int(y.max().item()) + 1, a.factor_size
    sh = bdist.Shards(n, 0, None, x.device)
    rng = np.random.default_rng(1)
    med = lambda ts: sorted(ts)[len(ts) // 2]                             # noqa: E731

    def timed_eval(ours, ref, nbytes, flops):
        for f in (ours, ref, ours, ref):                                   # warm-up: modules, cuBLAS algorithms
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
        diff = float(((got - want).abs().max() / want.abs().max()).item())
        ms = med(t_ours)
        tb, tf = nbytes / PEAK_HBM, flops / PEAK_FP64_TC
        return {"ms": round(ms, 3), "torch_fp64_ms": round(med(t_ref), 3), "max_rel_diff": diff,
                "gb_per_s": round(nbytes / (ms * 1e-3) / 1e9, 1), "fp64_tflops": round(flops / (ms * 1e-3) / 1e12, 2),
                "datasheet_bound_ms": round(max(tb, tf) * 1e3, 3), "bound": "fp64" if tf >= tb else "hbm",
                "share_of_bound": round(max(tb, tf) / (ms * 1e-3), 4)}

    # FMRegressor: a label with a pairwise and a linear part, and noise
    beta = torch.from_numpy(rng.normal(0.0, 0.3, D)).cuda()
    yr = (x[:, 0] * x[:, 1] + x @ beta + 0.5 * torch.from_numpy(rng.normal(0.0, 1.0, n)).cuda()).contiguous()
    wr = torch.from_numpy(rng.normal(0.0, 0.05, (1, D * (kf + 1) + 1))).cuda()
    nbytes, flops = work(n, D, kf, 1)
    regressor = {"eval": timed_eval(lambda: bfm.fm_regression_loss_grad_totals(x, yr, wr, kf, 1.0, 43, sh),
                                    lambda: torch_totals(x, yr, None, wr, kf), nbytes + 4.0 * n, flops)}
    pr = bfm.FMParams(factor_size=kf, step_size=0.01, seed=11)            # stepSize 1.0 diverges on these heavy tails
    bfm.fm_regression_fit(x, yr, pr)                                       # untimed fit
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    rfit = bfm.fm_regression_fit(x, yr, pr)
    torch.cuda.synchronize()
    regressor.update(fit_s=round(time.perf_counter() - t0, 3), step_size=pr.step_size, iterations=rfit.iterations,
                     first_objective=rfit.objective_history[0], objective=rfit.objective_history[-1],
                     label_variance=float(yr.var().item()))
    if a.regressor_only:
        print(json.dumps({"rows": n, "D": D, "factor_size": kf, "regressor": regressor, "card": dev_card}), flush=True)
        return
    evals = {}
    for k in (1, K):
        pos = torch.arange(k, dtype=torch.int32, device="cuda")
        w = torch.from_numpy(rng.normal(0.0, 0.05, (k, D * (kf + 1) + 1))).cuda()
        nbytes, flops = work(n, D, kf, k)
        evals["K%d" % k] = timed_eval(lambda: bfm.fm_loss_grad_totals(x, y, pos, w, kf, 1.0, 43, sh),
                                      lambda: torch_totals(x, y, pos, w, kf), nbytes, flops)
    # binary fit at the defaults: normal (label 0 after StringIndexer's frequency order) vs attack
    yb = (y != 0).to(torch.int32)
    p = bfm.FMParams(factor_size=kf, seed=11)
    bfm.fm_fit_classes(x, yb, [1], p)                                      # untimed fit
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fit = bfm.fm_fit_classes(x, yb, [1], p)[0]
    torch.cuda.synchronize()
    binary_s = time.perf_counter() - t0
    # OneVsRest: class-batched vs K standalone fits
    po = bfm.FMParams(factor_size=kf, max_iter=a.ovr_max_iter, seed=11)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    batched = bfm.fm_fit_classes(x, y, range(K), po)
    torch.cuda.synchronize()
    batched_s = time.perf_counter() - t0
    t0 = time.perf_counter()
    seq = [bfm.fm_fit_classes(x, (y == k).to(torch.int32), [1], po)[0] for k in range(K)]
    torch.cuda.synchronize()
    seq_s = time.perf_counter() - t0
    weights = torch.from_numpy(np.stack([np.concatenate([f.factors.reshape(-1), f.linear, [f.intercept]]) for f in batched]))
    tr = []
    bfm.fm_raw(x, weights, kf)
    for _ in range(a.repeats):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        raw = bfm.fm_raw(x, weights, kf)
        pred = _first_argmax(raw)
        e1.record()
        e1.synchronize()
        tr.append(e0.elapsed_time(e1))
    acc = float((pred.to(torch.int32) == y).double().mean().item())
    print(json.dumps({
        "rows": n, "D": D, "classes": K, "factor_size": kf, "eval": evals,
        "binary_fit_s": round(binary_s, 3), "binary_iterations": fit.iterations, "binary_objective": fit.objective_history[-1],
        "ovr_max_iter": a.ovr_max_iter, "ovr_batched_s": round(batched_s, 3), "ovr_sequential_s": round(seq_s, 3),
        "ovr_batched_hash": model_hash(batched), "ovr_sequential_hash": model_hash(seq),
        "ovr_iterations": sorted({f.iterations for f in batched}),
        "transform_ms": round(med(tr), 3), "train_accuracy": round(acc, 4), "regressor": regressor, "card": dev_card}),
        flush=True)


if __name__ == "__main__":
    main()
