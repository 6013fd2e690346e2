#!/usr/bin/env python
"""Micro-benchmark of the fused encode kernel against the HBM roofline (north-star target: >= 70 % of the data-sheet HBM
peak at 1 GPU).  Plans: KDD script-faithful (index + assemble, 41 slots), KDD full (index + one-hot + scale + assemble,
119 slots), KDD -> fp64 out, CICIDS (78 f32 fields).  Each plan runs `--iters` back-to-back launches over a record batch
larger than L2, timed with CUDA events.  Prints one JSON line per plan."""
import argparse, json, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "spark-network-traffic-classifier_b200")); sys.path.insert(0, ROOT)
import numpy as np, torch
from b200flow import encode as enc, synth


def timed(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser(); ap.add_argument("--rows", type=int, default=4898431); ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    peak = 3350.0                                               # GB/s: H100 SXM data sheet (HBM3), not measured
    rec, dicts = synth.make_kdd(a.rows, 5, seed=2019, device="cuda")
    schema = synth.kdd_schema()
    luts, ordered = {}, {}
    for c in synth.KDD_CATEGORICAL + ["label"]:
        cnt = enc.category_counts(rec, schema, c, len(dicts[c])).cpu().numpy()
        ordered[c], luts[c] = enc.string_index_order(cnt, dicts[c])

    def plan(onehot):
        p = enc.EncodePlan(schema)
        for c in synth.KDD_COLUMNS:
            if c not in synth.KDD_CATEGORICAL and c != "label":
                p.add_numeric(c)
        for c in synth.KDD_CATEGORICAL:
            p.add_onehot(c, luts[c], len(ordered[c])) if onehot else p.add_index(c, luts[c])
        p.set_label("label", luts["label"])
        return p
    cases = []
    pf = plan(False); cases.append(("kdd_faithful_f32", pf, rec, torch.float32))
    po = plan(True)
    x, _, _ = po.run(rec, torch.float64)
    mean, std = enc.column_moments(x); del x
    std = std.cpu().numpy(); po.set_scaling(mean.cpu().numpy(), np.where(std != 0, 1.0 / np.where(std != 0, std, 1), 0.0))
    cases.append(("kdd_full_onehot_scaled_f32", po, rec, torch.float32))
    cases.append(("kdd_faithful_f64", pf, rec, torch.float64))
    rc, dc = synth.make_cicids(min(a.rows, 2830743), 15, seed=2019, device="cuda")
    sc = synth.cicids_schema()
    cnt = enc.category_counts(rc, sc, "Label", 15).cpu().numpy()
    _, lutc = enc.string_index_order(cnt, dc["Label"])
    pc = enc.EncodePlan(sc)
    for f in sc.names[:-1]:
        pc.add_numeric(f)
    pc.set_label("Label", lutc)
    cases.append(("cicids_f32", pc, rc, torch.float32))
    for name, p, r, dt in cases:
        n = r.shape[0]
        out = torch.empty((n, p.n_out), dtype=dt, device="cuda")
        ms = timed(lambda: p.run(r, dt, out=out, want_valid=False), a.iters)
        byts = n * p.algorithmic_bytes_per_row(dt)
        print(json.dumps({"plan": name, "rows": n, "n_out": p.n_out, "bytes_per_row": p.algorithmic_bytes_per_row(dt), "ms": ms,
                          "rows_per_s": n / ms * 1e3, "achieved_gbs": byts / ms / 1e6, "peak_gbs": peak, "frac": byts / ms / 1e6 / peak}))
        del out


if __name__ == "__main__":
    main()
