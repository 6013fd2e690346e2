"""Time LinearSVC and OneVsRest(LinearSVC) on a KDD99-full-shaped set: --rows flows (default 4,898,431) with --classes
labels (default 23, as KDD99) encoded by the shim pipeline StringIndexer -> OneHotEncoder -> VectorAssembler ->
StandardScaler (D = 119, f64).

It reports
  * one hinge loss + subgradient evaluation (b200flow.svc.loss_grad_totals: the fused kernel and the chunk chain) at K = 1
    and K = --classes columns, with CUDA events, the median of --repeats, alternated in the same run with a plain torch
    fp64 arm (cuBLAS matmuls and elementwise ops) computing the same totals, and the largest difference between the two
    relative to the largest total;
  * the achieved bytes/s and FLOP/s of each evaluation, from bytes = n D 8 and FLOPs = 4 n pad8(D + 1) pad8(K) per pass,
    and the least time the data sheet allows (the larger of bytes / 3.35 TB/s and FLOPs / 67 TFLOP/s, 700 W figures; the
    card's power limit is read in the same run);
  * a binary fit (normal vs attack) at the defaults, host-timed after one untimed fit;
  * OneVsRest(LinearSVC) at maxIter = --ovr-max-iter: the class-batched fit against K standalone fits run one after the
    other, both host-timed, and a hash of every coefficient and intercept of each (they must be equal);
  * the OneVsRest transform (K margins in one launch and the first argmax), CUDA events, median of --repeats.
One JSON line.

    python tools/bench_svc.py [--rows 4898431] [--classes 23] [--repeats 20] [--ovr-max-iter 30]
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

from bench_tuning import card  # noqa: E402

PEAK_FP64_TC = 67e12
PEAK_HBM = 3.35e12


def features(n, classes, seed):
    from b200flow import synth
    from pyspark.ml import Pipeline
    from pyspark.ml.feature import OneHotEncoder, StandardScaler, StringIndexer, VectorAssembler
    from pyspark.sql import DataFrame
    rec, dicts = synth.make_kdd(n, classes, seed=seed, device="cuda:0")
    df = DataFrame.fromRecords(rec, synth.kdd_schema(), dicts)
    cats = synth.KDD_CATEGORICAL
    stages = [StringIndexer(inputCol=c, outputCol=c + "_num") for c in cats + ["label"]]
    stages.append(OneHotEncoder(inputCols=[c + "_num" for c in cats], outputCols=[c + "_oh" for c in cats]))
    nums = [c for c in synth.KDD_COLUMNS if c not in cats + ["label"]]
    stages.append(VectorAssembler(inputCols=nums + [c + "_oh" for c in cats], outputCol="raw"))
    stages.append(StandardScaler(inputCol="raw", outputCol="features", withMean=True, withStd=True))
    out = Pipeline(stages=stages).fit(df).transform(df)
    return out._cols["features"].data.to(torch.float64).contiguous(), out._column_tensor("label_num").to(torch.int32)


def torch_totals(x, y, pos, inv, w):
    """the same totals as loss_grad_totals ([K, D + 2]: hinge loss, subgradient) with cuBLAS and torch ops."""
    D = x.shape[1]
    xs = x * inv
    m = torch.addmm(w[:, D], xs, w[:, :D].t())
    yp = torch.where(y.long()[:, None] == pos.long()[None, :], 1.0, -1.0).to(torch.float64)
    h = 1.0 - yp * m
    act = (h > 0).to(torch.float64)
    a = -yp * act
    return torch.cat([(h * act).sum(0)[:, None], (a.t() @ xs), a.sum(0)[:, None]], 1)


def pad8(v):
    return (v + 7) // 8 * 8


def model_hash(fits):
    h = hashlib.sha256()
    for f in fits:
        h.update(np.ascontiguousarray(f.coef, np.float64).tobytes())
        h.update(np.float64(f.intercept).tobytes())
    return h.hexdigest()[:16]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=4898431)
    ap.add_argument("--classes", type=int, default=23)
    ap.add_argument("--repeats", type=int, default=20)
    ap.add_argument("--ovr-max-iter", type=int, default=30)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_svc.py needs a CUDA device")
    from b200flow import dist as bdist, selection, svc as bsvc
    from pyspark.ml.classification import _first_argmax
    dev_card = card()
    x, y = features(a.rows, a.classes, 2019)
    n, D = x.shape
    K = int(y.max().item()) + 1
    sh = bdist.Shards(n, 0, None, x.device)
    std = np.sqrt(selection.variances(x))
    inv = torch.from_numpy(np.where(std > 0, 1.0 / np.where(std > 0, std, 1.0), 0.0)).cuda()
    rng = np.random.default_rng(1)
    med = lambda ts: sorted(ts)[len(ts) // 2]                             # noqa: E731
    evals = {}
    for k in (1, K):
        pos = torch.arange(k, dtype=torch.int32, device="cuda")
        w = torch.from_numpy(rng.normal(0.0, 0.05, (k, D + 1))).cuda()
        ours, ref = lambda: bsvc.loss_grad_totals(x, y, pos, inv, w, sh), lambda: torch_totals(x, y, pos, inv, w)
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
        nbytes, flops = n * D * 8.0, 4.0 * n * pad8(D + 1) * pad8(k)
        bound = max(nbytes / PEAK_HBM, flops / PEAK_FP64_TC)
        evals["K%d" % k] = {"ms": round(ms, 3), "torch_fp64_ms": round(med(t_ref), 3), "max_rel_diff": diff,
                            "gb_per_s": round(nbytes / (ms * 1e-3) / 1e9, 1), "fp64_tflops": round(flops / (ms * 1e-3) / 1e12, 2),
                            "datasheet_bound_ms": round(bound * 1e3, 3), "share_of_bound": round(bound / (ms * 1e-3), 4)}
    # binary fit: normal (label 0 after StringIndexer's frequency order) vs attack
    yb = (y != 0).to(torch.int32)
    p = bsvc.SVCParams()
    bsvc.svc_fit_classes(x, yb, [1], p)                                    # untimed fit
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fit = bsvc.svc_fit_classes(x, yb, [1], p)[0]
    torch.cuda.synchronize()
    binary_s = time.perf_counter() - t0
    # OneVsRest: class-batched vs K standalone fits
    po = bsvc.SVCParams(max_iter=a.ovr_max_iter)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    batched = bsvc.svc_fit_classes(x, y, range(K), po)
    torch.cuda.synchronize()
    batched_s = time.perf_counter() - t0
    t0 = time.perf_counter()
    seq = [bsvc.svc_fit_classes(x, (y == k).to(torch.int32), [1], po)[0] for k in range(K)]
    torch.cuda.synchronize()
    seq_s = time.perf_counter() - t0
    weights = torch.from_numpy(np.stack([np.concatenate([f.coef, [f.intercept]]) for f in batched]))
    tr = []
    bsvc.svc_margins(x, weights)
    for _ in range(a.repeats):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        raw = bsvc.svc_margins(x, weights)
        pred = _first_argmax(raw)
        e1.record()
        e1.synchronize()
        tr.append(e0.elapsed_time(e1))
    acc = float((pred.to(torch.int32) == y).double().mean().item())
    print(json.dumps({
        "rows": n, "D": D, "classes": K, "eval": evals,
        "binary_fit_s": round(binary_s, 3), "binary_iterations": fit.iterations, "binary_objective": fit.objective_history[-1],
        "ovr_max_iter": a.ovr_max_iter, "ovr_batched_s": round(batched_s, 3), "ovr_sequential_s": round(seq_s, 3),
        "ovr_batched_hash": model_hash(batched), "ovr_sequential_hash": model_hash(seq),
        "ovr_iterations": [f.iterations for f in batched],
        "transform_ms": round(med(tr), 3), "train_accuracy": round(acc, 4), "card": dev_card}), flush=True)


if __name__ == "__main__":
    main()
