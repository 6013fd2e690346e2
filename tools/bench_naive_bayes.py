"""Time NaiveBayes on the workloads of the reference scripts: a CICIDS-shaped training split (b200flow.synth.make_cicids,
2,120,000 flows = 75 % of CICIDS2017, D = 78, f32) for gaussian, and a KDD-shaped split (make_kdd, 3,673,823 flows = 75 % of
KDD99-full, 23 classes) for weighted multinomial and complement on the 38 numeric features and bernoulli on the five binary
flags plus the one-hot categoricals.

Per case it reports:
  * fit_ms / transform_ms: a host clock around a whole nb_fit / nb_raw that ends in a synchronise, median of 3 after one
    untimed run;
  * moments_ms / raw_ms: CUDA-event medians of one b200flow_nb_moments launch over all rows (the pass without centres) and
    one b200flow_nb_raw launch, with the bytes one read of the inputs and the write of the outputs need, and the achieved
    bytes/s against NVIDIA's data-sheet 3.35 TB/s for the H100 SXM (not a measurement);
  * torch_multinomial_fit_ms: the existing torch fit (b200flow.linear.nb_fit, unweighted) on the same features, for context;
  * oracle_equal: the fit on the first 20,000 rows equals tests/naive_bayes_oracle.py bit for bit (pi, theta, sigma).
The card's name and power limit are read in the same run.  One JSON line per case.

    python tools/bench_naive_bayes.py [--cases gaussian,multinomial_w,complement,bernoulli] [--scale 1.0] [--window 2.0]
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

from bench_select import event_ms  # noqa: E402
from bench_tuning import card  # noqa: E402

PEAK_HBM = 3.35e12          # data sheet, H100 SXM
CICIDS_ROWS, KDD_ROWS = 2120000, 3673823


def cicids(rows):
    from b200flow import encode as enc, synth
    rec, dicts = synth.make_cicids(rows, 15, seed=2019, device="cuda:0")
    plan = enc.EncodePlan(synth.cicids_schema())
    for i in range(78):
        plan.add_numeric("f%02d" % i)
    plan.set_label("Label", np.arange(len(dicts["Label"]), dtype=np.int32))
    x, y, _ = plan.run(rec, torch.float32)
    return x, y.to(torch.float64), len(dicts["Label"])


def kdd(rows):
    """(numeric features f64, binary flags + one-hot f64, label, classes)"""
    from b200flow import encode as enc, synth
    rec, dicts = synth.make_kdd(rows, 23, seed=2019, device="cuda:0")
    plan = enc.EncodePlan(synth.kdd_schema())
    numeric = [c for c in synth.KDD_COLUMNS if c not in synth.KDD_CATEGORICAL and c != "label"]
    for c in numeric:
        plan.add_numeric(c)
    for c in synth.KDD_CATEGORICAL:
        plan.add_onehot(c, np.arange(len(dicts[c]), dtype=np.int32), len(dicts[c]), drop_last=True)
    plan.set_label("label", np.arange(len(dicts["label"]), dtype=np.int32))
    x, y, _ = plan.run(rec, torch.float64)
    flags = [numeric.index(c) for c in sorted(synth.KDD_BINARY)]
    xb = torch.cat([x[:, flags], x[:, len(numeric):]], 1).contiguous()
    return x[:, :len(numeric)].contiguous(), xb, y.to(torch.float64), len(dicts["label"])


def host_ms(fn):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(3):
        torch.cuda.synchronize()
        t0 = time.time()
        fn()
        torch.cuda.synchronize()
        ts.append((time.time() - t0) * 1e3)
    return float(np.median(ts))


def run(case, x, y, C, w, window):
    from b200flow import linear, naive_bayes as nb
    from b200flow._lib import call, ptr
    import naive_bayes_oracle as nbo
    mt = {"multinomial_w": "multinomial"}.get(case, case)
    n, D = x.shape
    dev = x.device
    fit = nb.nb_fit(x, y, C, mt, 1.0, weights=w)
    score = (lambda: linear.nb_raw(fit, x)) if mt == "multinomial" else (lambda: nb.nb_raw(fit, x))
    out = {"case": case, "model_type": mt, "weighted": w is not None, "rows": n, "D": D, "classes": C,
           "dtype": str(x.dtype).replace("torch.", ""),
           "fit_ms": round(host_ms(lambda: nb.nb_fit(x, y, C, mt, 1.0, weights=w)), 3),
           "transform_ms": round(host_ms(score), 3),
           "torch_multinomial_fit_ms": round(host_ms(lambda: linear.nb_fit(x, y, C, 1.0)), 3) if mt != "gaussian" else None}
    ids = y.to(torch.int32).contiguous()
    p, code, ld = nb._rows(x)
    nc = (n + 4095) // 4096
    parts = torch.empty((nc, C, D + 1), dtype=torch.float64, device=dev)
    moments = lambda: call("b200flow_nb_moments", p, code, n, D, ld, ptr(ids), ptr(w), C, None, 0, ptr(parts), None)  # noqa: E731
    ms = event_ms(moments, window)
    b = n * D * x.element_size() + 4 * n + (8 * n if w is not None else 0) + nc * C * (D + 1) * 8
    out.update(moments_ms=round(ms, 3), moments_bytes=b, moments_TBps=round(b / (ms * 1e-3) / 1e12, 3),
               moments_of_datasheet=round(b / (ms * 1e-3) / PEAK_HBM, 3))
    if mt != "multinomial":
        raw = torch.empty((n, C), dtype=torch.float64, device=dev)
        model = {"gaussian": 0, "bernoulli": 1, "complement": 2}[mt]
        ms = event_ms(lambda: call("b200flow_nb_raw", p, code, n, D, ld, model, ptr(fit._a), ptr(fit._b), ptr(fit._c0),
                                   ptr(fit._c1), ptr(fit._present_u8), C, ptr(raw), None), window)
        b = n * D * x.element_size() + n * C * 8
        out.update(raw_ms=round(ms, 3), raw_bytes=b, raw_TBps=round(b / (ms * 1e-3) / 1e12, 3),
                   raw_of_datasheet=round(b / (ms * 1e-3) / PEAK_HBM, 3))
    m = 20000
    small = nb.nb_fit(x[:m], y[:m], C, mt, 1.0, weights=None if w is None else w[:m])
    want = nbo.fit(x[:m].double().cpu().numpy(), y[:m].cpu().numpy(), C, mt, 1.0, None if w is None else w[:m].cpu().numpy())
    out["oracle_equal"] = all(getattr(small, k).cpu().numpy().tobytes() == getattr(want, k).tobytes() for k in ("pi", "theta", "sigma"))
    out["card"] = card()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", default="gaussian,multinomial_w,complement,bernoulli")
    ap.add_argument("--scale", type=float, default=1.0, help="fraction of the full row counts")
    ap.add_argument("--window", type=float, default=2.0)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_naive_bayes needs a CUDA device")
    cases = a.cases.split(",")
    if "gaussian" in cases:
        x, y, C = cicids(int(CICIDS_ROWS * a.scale))
        print(json.dumps(run("gaussian", x, y, C, None, a.window)), flush=True)
        del x, y
    rest = [c for c in cases if c != "gaussian"]
    if rest:
        xn, xb, y, C = kdd(int(KDD_ROWS * a.scale))
        g = torch.Generator(device="cuda:0"); g.manual_seed(7)
        w = torch.rand(xn.shape[0], device="cuda:0", generator=g, dtype=torch.float64) * 2.0
        for c in rest:
            x = xb if c == "bernoulli" else xn
            print(json.dumps(run(c, x, y, C, w if c == "multinomial_w" else None, a.window)), flush=True)


if __name__ == "__main__":
    main()
