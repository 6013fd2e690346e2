"""The fused level kernel on the reference scripts' own forest shapes (KDD 23-class, CICIDS 14/15-class,
DecisionTree feature passes — kdd99.py:61,64, cicids17.py:65,68) and the fused encode -> bins path (raw records -> TreePoint
bins without the dense matrix; SURVEY.md 8d).  Every GPU result is compared with the CPU oracle through the C ABI."""
import numpy as np
import pytest
import torch

import oracle
from b200flow import _lib, encode as enc, forest as fr, synth
from util import forests_equal, kdd_luts_gpu, kdd_plan, oracle_encode

DEV = "cuda"


# ------------------------------------------------------------------------------- launch shapes (host-only: no GPU needed)
def test_route_hist_config_covers_the_reference_scripts_shapes():
    # (F, m, n_bins, C): KDD 5-class bench config, kdd99.py:64 (23 classes), cicids17.py:68 (14 classes after the filters),
    # BASELINE config 4 (15 classes) — all must run the fused kernel in ONE feature pass
    for shape in [(41, 7, 70, 5), (41, 7, 70, 23), (78, 9, 78, 14), (78, 9, 78, 15), (41, 7, 70, 2), (78, 9, 78, 6)]:
        cfg = _lib.route_hist_config(*shape)
        assert cfg is not None, shape
        chunk, m_pass = cfg
        assert m_pass == shape[1] and chunk in (256, 512, 1024)
    # the launch shapes measured fastest on the H100 (DESIGN.md 3): 8x2 for the narrow nodes, 16x1 / 32x1 for the wide ones
    assert [_lib.route_hist_config(*s)[0] for s in [(41, 7, 70, 5), (78, 9, 78, 6), (41, 7, 70, 23), (78, 9, 78, 15)]] == [512, 512, 512, 1024]
    # DecisionTree: every feature in every node -> feature passes, the first of which routes
    chunk, m_pass = _lib.route_hist_config(41, 41, 70, 23)
    assert 1 <= m_pass < 41 and 2 * m_pass * 70 * 23 * 4 <= 227 * 1024
    chunk, m_pass = _lib.route_hist_config(78, 78, 78, 15)
    assert 1 <= m_pass < 78
    # one feature's pair of child histograms beyond shared memory: no fused path
    assert _lib.route_hist_config(41, 7, 256, 200) is None
    assert _lib.route_hist_config(300, 18, 32, 2) is None              # records wider than the staged tile supports


# ------------------------------------------------------------------------------- helpers
def _kdd_records(n, n_classes, seed):
    rec, dicts = synth.make_kdd(n, n_classes, seed=seed, device=DEV)
    schema = synth.kdd_schema()
    luts, ordered = kdd_luts_gpu(rec, schema, dicts)
    plan = kdd_plan(schema, luts, ordered)
    arity = [0] * 38 + [len(ordered[c]) for c in synth.KDD_CATEGORICAL]
    return rec, plan, arity, len(ordered["label"])


def _cicids_records(n, n_classes, seed, dtype="f32", nan_fraction=0.0):
    rec, dicts = synth.make_cicids(n, n_classes, seed=seed, device=DEV, dtype=dtype, nan_fraction=nan_fraction)
    schema = synth.cicids_schema(78, dtype)
    counts = enc.category_counts(rec, schema, "Label", n_classes).cpu().numpy()
    ordered, lut = enc.string_index_order(counts, dicts["Label"])
    plan = enc.EncodePlan(schema)
    for f in schema.names[:-1]:
        plan.add_numeric(f)
    plan.set_label("Label", lut)
    return rec, plan, [0] * 78, len(ordered)


def _oracle_fit(x_np, y_np, C, arity, p):
    return oracle.fit_forest(x_np, y_np, C, arity, num_trees=p.num_trees, max_bins=p.max_bins, max_depth=p.max_depth,
                             min_instances=p.min_instances_per_node, min_info_gain=p.min_info_gain, seed=p.seed,
                             strategy=p.feature_subset_strategy, subsampling_rate=p.subsampling_rate)


# ------------------------------------------------------------------------------- fused level kernel, script shapes
@pytest.mark.gpu
@pytest.mark.parametrize("kind,n_classes,depth", [("kdd", 23, 9), ("cicids", 14, 8), ("cicids", 15, 8)])
def test_script_forest_shapes_run_fused_and_match_oracle(kind, n_classes, depth):
    # 20 trees x the script's class count on >= 200 k rows, node for node against the oracle (VERDICT r1, next-round item 1)
    n = 200000
    rec, plan, arity, C = _kdd_records(n, n_classes, 41) if kind == "kdd" else _cicids_records(n, n_classes, 43)
    x, y, _ = plan.run(rec, torch.float64)
    p = fr.ForestParams(num_trees=20, max_bins=70 if kind == "kdd" else 78, max_depth=depth, seed=2019)
    model = fr.fit_forest(x, y, C, arity, p)
    assert model.train_stats["route_passes"] == 1 and model.train_stats["route_chunk"] > 0      # the fused kernel, one pass
    fo, meta = _oracle_fit(x.cpu().numpy(), y.cpu().numpy(), C, arity, p)
    assert forests_equal(model.export(), fo.export()) == []
    xt = x[:50000]
    tp_o, _ = oracle.bin_rows(xt.cpu().numpy(), meta["thresholds"], meta["n_thr"], meta["arity"], meta["max_bins"])
    raw_o, prob_o, pred_o = fo.predict(tp_o)
    raw, prob, pred = model.predict(xt)
    assert np.array_equal(pred.cpu().numpy(), pred_o) and np.array_equal(raw.cpu().numpy(), raw_o)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["8x2", "8x1", "16x2", "16x1", "32x1"])
def test_every_launch_shape_builds_the_same_forest(shape, monkeypatch):
    # warps per CTA x entries per lane: all five shapes of route_cfg must give the forest of the unfused kernels
    rec, plan, arity, C = _kdd_records(60000, 5, 17)
    x, y, _ = plan.run(rec, torch.float64)
    p = fr.ForestParams(num_trees=7, max_bins=70, max_depth=9, seed=5)
    monkeypatch.setattr(fr, "FUSED", False)
    want = fr.fit_forest(x, y, C, arity, p).export()
    monkeypatch.setattr(fr, "FUSED", True)
    monkeypatch.setenv("B200FLOW_ROUTE_SHAPE", shape)
    m = fr.fit_forest(x, y, C, arity, p)
    nw, ks = (int(v) for v in shape.split("x"))
    assert m.train_stats["route_chunk"] == nw * ks * 32
    got = m.export()
    assert forests_equal(got, want) == [] and np.array_equal(got["gain"], want["gain"])


@pytest.mark.gpu
@pytest.mark.parametrize("kind,classes", [("kdd", 5), ("kdd", 23), ("bytes78", 6), ("bytes78", 15)])
def test_histogram_update_variants_build_the_same_forest(kind, classes, monkeypatch):
    # featureSubsetStrategy="all": feature passes wider than 12, so the fused kernel runs its generic runtime loop instead of
    # the rotated-feature update, on KDD's 32-byte packed records and on 78 features of 78 bins (7 bits: byte records)
    if kind == "kdd":
        rec, plan, arity, C = _kdd_records(60000, classes, 29)
        x, y, _ = plan.run(rec, torch.float64)
        p = fr.ForestParams(num_trees=6, max_bins=70, max_depth=9, seed=3, feature_subset_strategy="all")
        fmt = ("packed", 32)
    else:
        g = torch.Generator(device=DEV); g.manual_seed(classes)
        x = torch.rand((60000, 78), dtype=torch.float64, device=DEV, generator=g)
        y = ((x[:, :6] > 0.5).sum(1) + (x[:, 6] + x[:, 7] > 1.0)) % classes
        C, arity = classes, [0] * 78
        y = y.to(torch.int32)
        p = fr.ForestParams(num_trees=4, max_bins=78, max_depth=8, seed=3, feature_subset_strategy="all")
        fmt = ("bytes", fr.tp_stride(78))
    monkeypatch.setattr(fr, "FUSED", False)
    want = fr.fit_forest(x, y, C, arity, p).export()
    monkeypatch.setattr(fr, "FUSED", True)
    m = fr.fit_forest(x, y, C, arity, p)
    F = len(arity)
    assert (m.train_stats["record_format"], m.train_stats["record_bytes"]) == fmt
    assert -(-F // m.train_stats["route_passes"]) > 12                     # balanced passes: each wider than 12 features
    got = m.export()
    assert forests_equal(got, want) == [] and np.array_equal(got["gain"], want["gain"])


@pytest.mark.gpu
def test_decision_tree_feature_passes_match_oracle():
    # kdd99.py:61 DecisionTreeClassifier on 23 classes: 41 features x 70 bins x 23 classes = 264 KB per node -> feature passes
    rec, plan, arity, C = _kdd_records(60000, 23, 91)
    x, y, _ = plan.run(rec, torch.float64)
    p = fr.ForestParams(num_trees=1, max_bins=70, max_depth=7, bootstrap=False, seed=1)
    model = fr.fit_forest(x, y, C, arity, p)
    assert model.train_stats["route_passes"] > 1
    fo, meta = _oracle_fit(x.cpu().numpy(), y.cpu().numpy(), C, arity, p)
    assert forests_equal(model.export(), fo.export()) == []


# ------------------------------------------------------------------------------- fused encode -> bins
@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 31, 97, 4096, 50021])
def test_encode_bins_equals_oracle_encode_then_bin(n):
    rec, plan, arity, C = _kdd_records(max(n, 3000), 5, 23)
    x, y, _ = plan.run(rec, torch.float64)
    model = fr.fit_forest(x, y, C, arity, fr.ForestParams(num_trees=1, max_bins=70, max_depth=0, bootstrap=False, seed=3))
    rec = rec[:n].contiguous()
    want_x, want_y, _ = oracle_encode(plan, rec.cpu().numpy())
    tp_o, bad_o = oracle.bin_rows(want_x, model.thresholds.cpu().numpy(), model.n_thr.cpu().numpy(), arity, 70, want_y)
    src = fr._RecordSource(rec, plan)
    bad = torch.zeros(2, dtype=torch.int32, device=DEV)
    tp, lab = src.bin(model.thresholds, model.n_thr, model._arity_dev, 70, bad, want_label_out=True)
    assert tp.shape == (n, 64) and bad_o == 0 and bad.cpu().tolist() == [0, 0]
    assert np.array_equal(tp.cpu().numpy()[:, :42], tp_o[:, :42]) and not tp[:, 42:].any()
    assert np.array_equal(lab.cpu().numpy(), want_y)


@pytest.mark.gpu
@pytest.mark.parametrize("kind,dtype", [("kdd", "f32"), ("cicids", "f32"), ("cicids", "f64")])
def test_fit_and_predict_from_records_equal_the_dense_path(kind, dtype):
    n = 80000
    rec, plan, arity, C = _kdd_records(n, 5, 29) if kind == "kdd" else _cicids_records(n, 15, 31, dtype)
    p = fr.ForestParams(num_trees=6, max_bins=70 if kind == "kdd" else 78, max_depth=8, seed=2019)
    x, y, _ = plan.run(rec, torch.float64)
    dense = fr.fit_forest(x, y, C, arity, p)
    fused = fr.fit_forest_records(rec, plan, C, arity, p)
    assert torch.equal(dense.thresholds, fused.thresholds) and torch.equal(dense.n_thr, fused.n_thr)     # R4 from raw records
    ed, ef = dense.export(), fused.export()
    assert forests_equal(ef, ed) == [] and np.array_equal(ef["gain"], ed["gain"])
    fo, meta = _oracle_fit(x.cpu().numpy(), y.cpu().numpy(), C, arity, p)                                 # and both equal the oracle
    assert forests_equal(ef, fo.export()) == []
    raw_d, prob_d, pred_d = dense.predict(x[:30000])
    raw_f, prob_f, pred_f, lab = fused.predict_records(rec[:30000].contiguous(), plan, want_label=True)
    assert torch.equal(raw_d, raw_f) and torch.equal(prob_d, prob_f) and torch.equal(pred_d, pred_f)
    assert torch.equal(lab, y[:30000])


@pytest.mark.gpu
def test_f64_records_bin_differently_from_their_f32_copies():
    # SURVEY 7 hard part: Spark's inferSchema makes the CICIDS columns doubles.  A value with more than 7 significant digits
    # can sit on the other side of a midpoint threshold once rounded to f32, so the f64 record path must bin the doubles
    # themselves: equal to the oracle on the f64 values, and NOT equal to binning the f32-rounded values everywhere.
    n = 120000
    rec, plan, arity, C = _cicids_records(n, 15, 37, "f64")
    x64, y, _ = plan.run(rec, torch.float64)
    m = fr.fit_forest_records(rec, plan, C, arity, fr.ForestParams(num_trees=1, max_bins=78, max_depth=0, bootstrap=False, seed=9))
    thr, n_thr = m.thresholds.cpu().numpy(), m.n_thr.cpu().numpy()
    bad = torch.zeros(2, dtype=torch.int32, device=DEV)
    tp, _ = fr._RecordSource(rec, plan).bin(m.thresholds, m.n_thr, m._arity_dev, 78, bad)
    tp_o, _ = oracle.bin_rows(x64.cpu().numpy(), thr, n_thr, arity, 78, y.cpu().numpy())
    assert np.array_equal(tp.cpu().numpy()[:, :79], tp_o[:, :79])
    x32 = x64.to(torch.float32).to(torch.float64)
    tp_32, _ = oracle.bin_rows(x32.cpu().numpy(), thr, n_thr, arity, 78, y.cpu().numpy())
    assert (tp_32[:, :78] != tp_o[:, :78]).sum() > 0


@pytest.mark.gpu
def test_encode_bins_counts_nan_and_routes_unseen_categories_right():
    rec, plan, arity, C = _kdd_records(20000, 5, 53)
    x, y, _ = plan.run(rec, torch.float64)
    p = fr.ForestParams(num_trees=4, max_bins=70, max_depth=6, seed=1)
    model = fr.fit_forest_records(rec, plan, C, arity, p)
    bad_rec = rec[:2000].clone()
    bad_rec.view(torch.float32)[5, 0] = float("nan"); bad_rec.view(torch.float32)[9, 4] = float("nan")
    bad_rec.view(torch.int32)[11, 2] = 9999                                            # service code outside the dictionary
    plan.check_nan = 1
    with pytest.raises(fr.InvalidRowsError):
        model.predict_records(bad_rec, plan, on_invalid="error")
    raw, prob, pred, _ = model.predict_records(bad_rec, plan)                         # default: unseen category goes right
    assert pred.shape[0] == 2000 and bool(torch.isfinite(raw).all())
    ok = torch.ones(2000, dtype=torch.bool, device=DEV); ok[[5, 9, 11]] = False
    _, _, pred_ref = model.predict(x[:2000])
    assert torch.equal(pred[ok], pred_ref[ok])
    with pytest.raises(fr.InvalidRowsError):
        fr.fit_forest_records(bad_rec, plan, C, arity, p)
    plan.check_nan = 0
    # a categorical value outside [0, arity) at transform time: binned outside every left set, counted, not fatal
    xb = x[:100].clone(); xb[3, 39] = 200.0; xb[4, 38] = 1.5
    tp, nbad = model.bin(xb)
    assert int(nbad.item()) == 2 and int(tp[3, 39]) == arity[39] and int(tp[4, 38]) == arity[38]
    model.predict(xb)
    with pytest.raises(ValueError):
        fr.fit_forest(xb, y[:100], C, arity, p)
