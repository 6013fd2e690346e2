"""Time the MultilayerPerceptronClassifier on a KDD99-full-shaped set: --rows flows (default 4,898,431) encoded by the shim
pipeline StringIndexer -> OneHotEncoder -> VectorAssembler -> StandardScaler (D = 119), the first 75 % as the training
rows and the rest as the test rows, layers = --layers (default 119,64,32,5).

It reports
  * one loss + gradient evaluation (b200flow.mlp.loss_grad_sums: the fused kernel and the chunk chain) with CUDA events,
    the median of --repeats, alternated in the same run with a plain torch fp64 arm (cuBLAS matmuls and elementwise ops)
    computing the same loss and gradient, and the largest difference between the two relative to the largest gradient;
  * the achieved fp64 rate from FLOPs = 2 n (3 sum in_l out_l - in_1 out_1) and its share of the data sheet's 67 TFLOP/s
    fp64 tensor-core peak (a 700 W figure; the card's power limit is read in the same run);
  * a full fit at the defaults (maxIter = 100, l-bfgs), host-timed after one untimed fit, and its iteration count;
  * transform (b200flow.mlp.mlp_raw) of the test rows, CUDA events, median of --repeats.
One JSON line.

    python tools/bench_mlp.py [--rows 4898431] [--layers 119,64,32,5] [--repeats 20]
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

import torch  # noqa: E402

from bench_tuning import card  # noqa: E402

PEAK_FP64_TC = 67e12


def features(n, seed):
    from b200flow import synth
    from pyspark.ml import Pipeline
    from pyspark.ml.feature import OneHotEncoder, StandardScaler, StringIndexer, VectorAssembler
    from pyspark.sql import DataFrame
    rec, dicts = synth.make_kdd(n, 5, seed=seed, device="cuda:0")
    df = DataFrame.fromRecords(rec, synth.kdd_schema(), dicts)
    cats = synth.KDD_CATEGORICAL
    stages = [StringIndexer(inputCol=c, outputCol=c + "_num") for c in cats + ["label"]]
    stages.append(OneHotEncoder(inputCols=[c + "_num" for c in cats], outputCols=[c + "_oh" for c in cats]))
    nums = [c for c in synth.KDD_COLUMNS if c not in cats + ["label"]]
    stages.append(VectorAssembler(inputCols=nums + [c + "_oh" for c in cats], outputCol="raw"))
    stages.append(StandardScaler(inputCol="raw", outputCol="features", withMean=True, withStd=True))
    out = Pipeline(stages=stages).fit(df).transform(df)
    return out._cols["features"].data.to(torch.float64).contiguous(), out._column_tensor("label_num").to(torch.int32)


def torch_loss_grad(x, y, layers, w):
    """the same sums as loss_grad_sums ([P + 1]: loss, then the gradient in Spark's layout) with cuBLAS and torch ops."""
    params, off = [], 0
    for a, b in zip(layers[:-1], layers[1:]):
        params.append((w[off:off + a * b].view(a, b).t(), w[off + a * b:off + a * b + b]))
        off += (a + 1) * b
    acts = [x]
    for l, (W, b) in enumerate(params):
        z = torch.addmm(b, acts[-1], W.t())
        if l < len(params) - 1:
            acts.append(torch.sigmoid(z))
    loss = (torch.logsumexp(z, 1) - z.gather(1, y.long()[:, None])[:, 0]).sum()
    delta = torch.softmax(z, 1)
    delta[torch.arange(x.shape[0], device=x.device), y.long()] -= 1.0
    grads = [None] * len(params)
    for l in range(len(params) - 1, -1, -1):
        a = acts[l]
        grads[l] = torch.cat([(delta.t() @ a).t().reshape(-1), delta.sum(0)])
        if l:
            delta = (delta @ params[l][0]) * a * (1.0 - a)
    return torch.cat([loss.reshape(1)] + grads)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=4898431)
    ap.add_argument("--layers", default="119,64,32,5")
    ap.add_argument("--repeats", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_mlp.py needs a CUDA device")
    from b200flow import dist as bdist, mlp as bm
    dev_card = card()
    layers = [int(v) for v in a.layers.split(",")]
    x_all, y_all = features(a.rows, 2019)
    n_train = a.rows * 3 // 4
    x, y = x_all[:n_train].contiguous(), y_all[:n_train].contiguous()
    xt = x_all[n_train:].contiguous()
    del x_all
    n = x.shape[0]
    assert x.shape[1] == layers[0], "features have D = %d, layers[0] = %d" % (x.shape[1], layers[0])
    sh = bdist.Shards(n, 0, None, x.device)
    w = torch.from_numpy(bm.init_weights(layers, 1)).cuda()
    ours, ref = lambda: bm.loss_grad_sums(x, y, layers, w, sh), lambda: torch_loss_grad(x, y, layers, w)
    for f in (ours, ref, ours, ref):                                       # warm-up: modules, cuBLAS algorithms
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
    med = lambda ts: sorted(ts)[len(ts) // 2]                             # noqa: E731
    k, r = ours(), ref()
    grad_diff = float(((k[1:] - r[1:]).abs().max() / r[1:].abs().max()).item())
    loss_diff = float(((k[0] - r[0]).abs() / r[0].abs()).item())
    flops = 2.0 * n * (3 * sum(i * o for i, o in zip(layers[:-1], layers[1:])) - layers[0] * layers[1])
    ms = med(t_ours)
    bm.mlp_fit(x, y, layers, seed=1)                                       # untimed fit
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fit = bm.mlp_fit(x, y, layers, seed=1)
    torch.cuda.synchronize()
    fit_s = time.perf_counter() - t0
    tr = []
    bm.mlp_raw(fit.weights, layers, xt)
    for _ in range(a.repeats):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        bm.mlp_raw(fit.weights, layers, xt)
        e1.record()
        e1.synchronize()
        tr.append(e0.elapsed_time(e1))
    acc = float((bm.mlp_raw(fit.weights, layers, xt).argmax(1).to(torch.int32) == y_all[n_train:].cuda()).double().mean().item())
    print(json.dumps({
        "train_rows": n, "test_rows": xt.shape[0], "layers": layers, "P": bm.n_params(layers),
        "loss_grad_ms": round(ms, 3), "gflop": round(flops / 1e9, 2), "fp64_tflops": round(flops / (ms * 1e-3) / 1e12, 2),
        "share_of_67_tflops": round(flops / (ms * 1e-3) / PEAK_FP64_TC, 4),
        "torch_fp64_ms": round(med(t_ref), 3), "max_rel_grad_diff": grad_diff, "rel_loss_diff": loss_diff,
        "fit_s": round(fit_s, 3), "fit_iterations": fit.iterations, "final_loss": fit.objective_history[-1],
        "transform_ms": round(med(tr), 3), "test_accuracy": round(acc, 4), "card": dev_card}), flush=True)


if __name__ == "__main__":
    main()
