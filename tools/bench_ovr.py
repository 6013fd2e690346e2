"""Time OneVsRest(GBTClassifier) on a KDD99-full-shaped set: --rows flows (default 4,898,431, synth.make_kdd(n, K)) assembled by
the shim pipeline StringIndexer -> VectorAssembler (41 features, 3 of them categorical), GBT maxIter 20, maxDepth 5,
maxBins 70, for K = 5 and K = 23 classes.

Per K it reports
  * fit: the class-batched trainer (b200flow.gbt.fit_gbt_ovr, one level loop for the K problems) against the generic loop
    (K fit_gbt calls on the relabelled labels, label == k, which is what OneVsRest does for any other classifier): one
    untimed run of each arm, then --repeats alternated timed runs (host clock around a synchronised fit), median and range;
  * whether the two arms' K models are equal (every export array, byte for byte);
  * CUDA-event time per phase of one fit of each arm;
  * transform of every row: the joint predict (one tree walk over the K·T trees with C = K) against K sub-model predicts
    plus the argmax (CUDA events, alternated, median).
One JSON line, with the card's name and power limit read in the same run.

    python tools/bench_ovr.py [--rows 4898431] [--classes 5,23] [--repeats 3]
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

from bench_tuning import card  # noqa: E402


def features(n, K, seed):
    from b200flow import synth
    from pyspark.ml import Pipeline
    from pyspark.ml.classification import _arity_from_attrs
    from pyspark.ml.feature import StringIndexer, VectorAssembler
    from pyspark.sql import DataFrame
    rec, dicts = synth.make_kdd(n, K, seed=seed, device="cuda:0")
    df = DataFrame.fromRecords(rec, synth.kdd_schema(), dicts)
    cats = synth.KDD_CATEGORICAL
    stages = [StringIndexer(inputCol=c, outputCol=c + "_num") for c in cats + ["label"]]
    nums = [c for c in synth.KDD_COLUMNS if c not in cats + ["label"]]
    stages.append(VectorAssembler(inputCols=nums + [c + "_num" for c in cats], outputCol="features"))
    out = Pipeline(stages=stages).fit(df).transform(df)
    x = out._cols["features"].data.to(torch.float64).contiguous()
    n_classes = len(out._cols["label_num"].meta["ml_attr"]["vals"])
    return x, out._column_tensor("label_num").to(torch.int32), n_classes, _arity_from_attrs(out._cols["features"].meta.get("attrs"), x.shape[1])


def host_timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, r


def event_ms(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(); fn(); e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def phases(fn):
    from b200flow import forest as fr
    fr.PROFILE = {}
    fn()
    torch.cuda.synchronize()
    out = {k: round(sum(e0.elapsed_time(e1) for e0, e1 in v), 3) for k, v in fr.PROFILE.items()}
    fr.PROFILE = None
    return out


def summary(ts):
    return dict(median=float(np.median(ts)), min=float(np.min(ts)), max=float(np.max(ts)), runs=len(ts))


def one(K_req, rows, repeats, bg):
    from pyspark.ml.classification import _first_argmax
    x, y, K, arity = features(rows, K_req, 2019)
    p = bg.GBTParams(max_iter=20, max_depth=5, max_bins=70, seed=2019)
    batched = lambda: bg.fit_gbt_ovr(x, y, K, arity, p)                          # noqa: E731
    generic = lambda: [bg.fit_gbt(x, (y == k).to(torch.int32), arity, p) for k in range(K)]   # noqa: E731
    _, ovr = host_timed(batched)                                                 # untimed: warm-up of each arm
    _, sep = host_timed(generic)
    t_b, t_g = [], []
    for _ in range(repeats):                                                     # alternated in the same run
        t_b.append(host_timed(batched)[0])
        t_g.append(host_timed(generic)[0])
    equal = True
    for a, b in zip(ovr.models, sep):
        ea, eb = a.export(), b.export()
        equal = equal and sorted(ea) == sorted(eb) and all(
            np.array_equal(np.asarray(ea[c]).view(np.uint8), np.asarray(eb[c]).view(np.uint8)) for c in ea)
        equal = equal and a.tree_weights == b.tree_weights and torch.equal(a.forest.thresholds, b.forest.thresholds)
    out = dict(classes=K, fit_batched_s=summary(t_b), fit_generic_s=summary(t_g),
               speedup=float(np.median(t_g) / np.median(t_b)), models_equal=bool(equal),
               train_stats=ovr.train_stats, phases_batched_ms=phases(batched), phases_generic_ms=phases(generic))

    def joint():
        return ovr.predict(x)

    def loop():
        raw = torch.stack([m.predict(x)[0][:, 1] for m in sep], 1)
        return raw, _first_argmax(raw)
    jr, jp = joint(); lr, lp = loop()
    out["transform_equal"] = bool(torch.equal(jr.view(torch.int64), lr.view(torch.int64)) and torch.equal(jp, lp))
    tj, tl = [], []
    for _ in range(max(repeats, 5)):
        tj.append(event_ms(joint)); tl.append(event_ms(loop))
    out["transform_joint_ms"], out["transform_loop_ms"] = summary(tj), summary(tl)
    out["train_accuracy"] = float((jp == y.to(torch.float64)).to(torch.float64).mean().item())
    del x, y
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=4_898_431)
    ap.add_argument("--classes", default="5,23")
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    from b200flow import gbt as bg
    torch.cuda.set_device(0)
    out = dict(card=card(), rows=a.rows, max_iter=20, max_depth=5, max_bins=70)
    out["runs"] = [one(int(k), a.rows, a.repeats, bg) for k in a.classes.split(",")]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
