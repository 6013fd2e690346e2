"""Time GBTClassifier on a KDD99-full-shaped binary set: --rows flows (default 4,898,431, synth.make_kdd(n, 2)) assembled by
the shim pipeline StringIndexer -> VectorAssembler (41 features, 3 of them categorical), maxBins 70, maxIter 20, maxDepth 5.

It reports
  * fit (host clock around a synchronised fit, after one untimed fit) and transform of every row (CUDA events, median);
  * CUDA-event time per phase of the fit: variance histograms, split scoring, node-pool growth, partition, update;
  * the histogram kernel on the root level of the data's unique records (every record with its multiplicity, all 41
    features): its algorithmic bytes/s — per entry the 8-byte entry, the 16-byte {q, q2} and the 64-byte record — next to a
    torch.index_add_ int64 arm building the same histogram, which must be bit-equal (the sums are integers);
  * the CPU restatement (tests/gbt_oracle.py: the C oracle's findSplits and binning, the boosting in numpy) on the same
    rows (or the first --oracle-rows), its time and whether the device model equals it bit for bit.
One JSON line, with the card's name and power limit read in the same run.

    python tools/bench_gbt.py [--rows 4898431] [--oracle-rows 0] [--repeats 10]
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


def features(n, seed):
    from b200flow import synth
    from pyspark.ml import Pipeline
    from pyspark.ml.feature import StringIndexer, VectorAssembler
    from pyspark.sql import DataFrame
    rec, dicts = synth.make_kdd(n, 2, seed=seed, device="cuda:0")
    df = DataFrame.fromRecords(rec, synth.kdd_schema(), dicts)
    cats = synth.KDD_CATEGORICAL
    stages = [StringIndexer(inputCol=c, outputCol=c + "_num") for c in cats + ["label"]]
    nums = [c for c in synth.KDD_COLUMNS if c not in cats + ["label"]]
    stages.append(VectorAssembler(inputCols=nums + [c + "_num" for c in cats], outputCol="features"))
    out = Pipeline(stages=stages).fit(df).transform(df)
    attrs = out._cols["features"].meta.get("attrs")
    from pyspark.ml.classification import _arity_from_attrs
    x = out._cols["features"].data.to(torch.float64).contiguous()
    return x, out._column_tensor("label_num").to(torch.int32), _arity_from_attrs(attrs, x.shape[1])


def events(fn, repeats):
    ts = []
    for _ in range(repeats):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts))


def hist_arms(x, y, arity, p, repeats):
    """the root-level histogram of the unique records, by the kernel and by index_add_"""
    from b200flow import forest as fr
    from b200flow._lib import call, ptr
    rows = fr._TrainingRows(fr._DenseSource(x, y), 2, arity, p.max_bins, 1, "all", p.seed, 0, None).read()
    tp, U, F, n_bins = rows.tp, rows.U, rows.F, rows.n_bins
    mult = torch.bincount(rows.uid.long(), minlength=U).to(torch.int32)
    ent = torch.stack([torch.arange(U, dtype=torch.int32, device=x.device), mult], 1).contiguous()
    S, S2 = (60 - int(np.ceil(np.log2(x.shape[0])))), (58 - int(np.ceil(np.log2(x.shape[0]))))
    rq = torch.zeros((U, 2), dtype=torch.int64, device=x.device)
    margin = torch.zeros(U, dtype=torch.float64, device=x.device)
    call("b200flow_gbt_update", ptr(tp), tp.shape[1], F, U, None, None, None, -1, S, S2, ptr(margin), ptr(rq))
    seg_b = torch.zeros(1, dtype=torch.int64, device=x.device)
    seg_e = torch.full((1,), U, dtype=torch.int64, device=x.device)
    n_ch = (U + fr.CHUNK_ROWS - 1) // fr.CHUNK_ROWS
    chunk_off = torch.tensor([0, n_ch], dtype=torch.int64, device=x.device)
    subset = torch.arange(F, dtype=torch.int16, device=x.device).reshape(1, F)
    hist = torch.zeros(F * n_bins * 3, dtype=torch.int64, device=x.device)

    def kernel():
        hist.zero_()
        call("b200flow_gbt_hist_level", ptr(tp), tp.shape[1], ptr(ent), ptr(rq), 1, ptr(seg_b), ptr(seg_e), ptr(chunk_off), n_ch,
             fr.CHUNK_ROWS, ptr(subset), F, n_bins, ptr(hist))
    ref = torch.zeros(F * n_bins, 3, dtype=torch.int64, device=x.device)
    w = mult.to(torch.int64)
    vals = torch.stack([w, w * rq[:, 0], w * rq[:, 1]], 1)
    idx = (torch.arange(F, device=x.device)[None, :] * n_bins + tp[:U, :F].long()).reshape(-1)
    vals_f = vals.repeat_interleave(F, 0)

    def torch_arm():
        ref.zero_()
        ref.index_add_(0, idx, vals_f)
    kernel(); torch_arm(); torch.cuda.synchronize()
    equal = bool(torch.equal(hist.view(-1, 3), ref))
    t_k, t_t = [], []
    for _ in range(repeats):                                   # alternated in the same run
        t_k.append(events(kernel, 1)); t_t.append(events(torch_arm, 1))
    byt = U * (8 + 16 + tp.shape[1])
    return dict(unique_records=U, features=F, n_bins=n_bins, kernel_ms=float(np.median(t_k)), index_add_ms=float(np.median(t_t)),
                algorithmic_bytes=byt, kernel_GBps=byt / (float(np.median(t_k)) * 1e6), bit_equal=equal)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=4_898_431)
    ap.add_argument("--oracle-rows", type=int, default=0, help="rows for the numpy restatement (0: all of them)")
    ap.add_argument("--repeats", type=int, default=10)
    a = ap.parse_args()
    from b200flow import forest as fr, gbt as bg
    torch.cuda.set_device(0)
    out = dict(card=card(), rows=a.rows)
    x, y, arity = features(a.rows, 2019)
    p = bg.GBTParams(max_iter=20, max_depth=5, max_bins=70, seed=2019)
    bg.fit_gbt(x, y, arity, p)                                   # untimed: module load, allocator warm-up
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    model = bg.fit_gbt(x, y, arity, p)
    torch.cuda.synchronize()
    out["fit_s"] = time.perf_counter() - t0
    out["train_stats"] = model.train_stats
    fr.PROFILE = {}
    bg.fit_gbt(x, y, arity, p)
    torch.cuda.synchronize()
    out["phases_ms"] = {k: round(sum(e0.elapsed_time(e1) for e0, e1 in v), 3) for k, v in fr.PROFILE.items()}
    fr.PROFILE = None
    out["transform_ms"] = events(lambda: model.predict(x), a.repeats)
    pred = model.predict(x)[2]
    out["train_accuracy"] = float((pred == y.to(torch.float64)).to(torch.float64).mean().item())
    out["histogram"] = hist_arms(x, y, arity, p, a.repeats)
    # the CPU restatement on the same rows
    import gbt_oracle as go
    k = min(a.oracle_rows or a.rows, a.rows)
    t0 = time.perf_counter()
    want = go.fit(x[:k].cpu().numpy(), y[:k].cpu().numpy(), arity, max_iter=20, max_depth=5, max_bins=70, seed=2019)
    out["oracle_rows"], out["oracle_fit_s"] = k, time.perf_counter() - t0
    got = bg.fit_gbt(x[:k], y[:k], arity, p).export()
    exp = go.export(want)
    out["oracle_equal"] = all(np.array_equal(np.asarray(got[c]).view(np.uint8), np.asarray(exp[c]).view(np.uint8)) for c in exp)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
