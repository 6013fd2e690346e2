"""Parity of the CUDA hot path (through the C ABI) against the CPU oracle on the same seeded inputs.
Bar: bit-exact for bins / histograms / splits / labels and fp64 outputs; <= 1e-6 relative for fp32 features."""
import numpy as np
import pytest
import torch

import oracle
from b200flow import _lib, encode as enc, forest as fr, synth
from util import forests_equal, kdd_luts_gpu, kdd_luts_oracle, kdd_plan, oracle_encode

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _kdd(n, n_classes=5, seed=3):
    rec, dicts = synth.make_kdd(n, n_classes, seed=seed, device=DEV)
    return rec, dicts, synth.kdd_schema()


# ------------------------------------------------------------------------------- encode
@pytest.mark.parametrize("n", [1, 3, 63, 64, 65, 1000, 40007])
def test_encode_script_faithful_matches_oracle(n):
    rec, dicts, schema = _kdd(n)
    rec_np = rec.cpu().numpy()
    luts_g, ord_g = kdd_luts_gpu(rec, schema, dicts)
    luts_o, ord_o = kdd_luts_oracle(rec_np, schema, dicts)
    assert ord_g == ord_o and all((luts_g[k] == luts_o[k]).all() for k in luts_o)      # R1 exact
    plan = kdd_plan(schema, luts_g, ord_g)
    want, want_lab, want_valid = oracle_encode(plan, rec_np)
    got64, lab, valid = plan.run(rec, torch.float64)
    assert np.array_equal(got64.cpu().numpy(), want)                                   # fp64 out: bit-exact
    assert np.array_equal(lab.cpu().numpy(), want_lab) and np.array_equal(valid.cpu().numpy(), want_valid)
    got32, _, _ = plan.run(rec, torch.float32)
    assert np.allclose(got32.cpu().numpy(), want, rtol=1e-6, atol=0)


@pytest.mark.parametrize("n", [5, 2048, 100003])
def test_encode_full_onehot_scaled_matches_oracle(n):
    rec, dicts, schema = _kdd(n, seed=11)
    rec_np = rec.cpu().numpy()
    luts, ordered = kdd_luts_gpu(rec, schema, dicts)
    plan = kdd_plan(schema, luts, ordered, onehot=True)
    assert plan.n_out == 38 + sum(len(ordered[c]) - 1 for c in synth.KDD_CATEGORICAL)
    x, _, _ = plan.run(rec, torch.float64)
    mean, std = enc.column_moments(x)                                                  # R3c fit
    o_mean, o_std = oracle.moments(x.cpu().numpy())
    assert np.allclose(mean.cpu().numpy(), o_mean, rtol=1e-9, atol=1e-12)
    assert np.allclose(std.cpu().numpy(), o_std, rtol=1e-9, atol=1e-12)
    scale = np.where(o_std != 0, 1.0 / np.where(o_std != 0, o_std, 1.0), 0.0)
    plan.set_scaling(o_mean, scale)                                                    # withMean + withStd, fused
    want, _, _ = oracle_encode(plan, rec_np)
    got64, _, _ = plan.run(rec, torch.float64)
    assert np.array_equal(got64.cpu().numpy(), want)
    got32, _, _ = plan.run(rec, torch.float32)
    err = np.abs(got32.cpu().numpy() - want)
    assert (err <= 1e-6 * np.abs(want) + 1e-30).all()                                  # 1e-6 relative (north_star)


def test_encode_full_size_properties():
    # KDD99-full row count: the fused encode is checked through properties that need no CPU pass over 4.9 M rows —
    # numeric slots are the raw fields bit for bit, an index slot is lut[code], a dropLast one-hot block has one 1 exactly when
    # the rank is not the last one (and it sits at the rank), the label is lut[label code], and the scaled vector has
    # mean 0 / unit sample variance per column.
    n = 4898431
    rec, dicts, schema = _kdd(n, seed=2019)
    luts, ordered = kdd_luts_gpu(rec, schema, dicts)
    faithful = kdd_plan(schema, luts, ordered)
    x, y, _ = faithful.run(rec, torch.float32, want_valid=False)
    raw = rec.view(torch.int32)
    numeric = [c for c in synth.KDD_COLUMNS if c not in synth.KDD_CATEGORICAL and c != "label"]
    for j, c in enumerate(numeric):
        assert torch.equal(x[:, j].view(torch.int32), raw[:, schema.offsets[c] // 4])
    for j, c in enumerate(synth.KDD_CATEGORICAL):
        lut = torch.from_numpy(np.asarray(luts[c], np.int32)).to(DEV)
        assert torch.equal(x[:, 38 + j], lut[raw[:, schema.offsets[c] // 4].long()].to(torch.float32))
    lab_lut = torch.from_numpy(np.asarray(luts["label"], np.int32)).to(DEV)
    assert torch.equal(y, lab_lut[raw[:, schema.offsets["label"] // 4].long()])
    del x
    full = kdd_plan(schema, luts, ordered, onehot=True, label=False)
    xo, _, _ = full.run(rec, torch.float32, want_valid=False)
    col = 38
    for c in synth.KDD_CATEGORICAL:
        K = len(ordered[c]); blk = xo[:, col:col + K - 1]
        rank = torch.from_numpy(np.asarray(luts[c], np.int32)).to(DEV)[raw[:, schema.offsets[c] // 4].long()]
        assert torch.equal(blk.sum(1), (rank < K - 1).to(torch.float32))
        hot = torch.where(rank < K - 1, rank, torch.zeros_like(rank)).long()
        assert torch.equal(blk.gather(1, hot[:, None])[:, 0], (rank < K - 1).to(torch.float32))
        col += K - 1
    mean, std = enc.column_moments(xo)
    m, sd = mean.cpu().numpy(), std.cpu().numpy()
    full.set_scaling(m, np.where(sd != 0, 1.0 / np.where(sd != 0, sd, 1.0), 0.0))
    del xo
    xs, _, _ = full.run(rec, torch.float64, want_valid=False)
    live = torch.from_numpy(sd != 0).to(DEV)
    assert xs.mean(0).abs().max().item() < 1e-9
    assert ((xs.var(0, unbiased=True) - 1.0).abs()[live]).max().item() < 1e-9 and (xs[:, ~live] == 0).all()


def test_category_counts_multi_equals_single_columns():
    rec, dicts, schema = _kdd(50021)
    cols = synth.KDD_CATEGORICAL + ["label"]
    multi = enc.category_counts_multi(rec, schema, cols, [len(dicts[c]) for c in cols])
    rec_np = rec.cpu().numpy()
    for c, m in zip(cols, multi):
        single = enc.category_counts(rec, schema, c, len(dicts[c]))
        assert torch.equal(m, single)
        assert np.array_equal(m.cpu().numpy(), oracle.category_counts(rec_np, schema.row_bytes, schema.offsets[c], len(dicts[c])))


def test_encode_invalid_codes_and_nan_rows():
    rec, dicts, schema = _kdd(5000, seed=5)
    luts, ordered = kdd_luts_gpu(rec, schema, dicts)
    lut = luts["service"].copy(); lut[lut == lut.max()] = -1                           # pretend the rarest was unseen at fit
    luts["service"] = lut
    r32 = rec.view(torch.int32)
    r32[7, 2] = 999; r32[9, 2] = -4                                                    # codes outside the dictionary
    rec.view(torch.float32)[11, 0] = float("nan"); rec.view(torch.float32)[12, 4] = float("inf")
    plan = kdd_plan(schema, luts, ordered); plan.check_nan = 1
    want, want_lab, want_valid = oracle_encode(plan, rec.cpu().numpy())
    got, lab, valid = plan.run(rec, torch.float64)
    assert np.array_equal(valid.cpu().numpy(), want_valid)
    assert want_valid[7] == 0 and want_valid[9] == 0 and want_valid[11] == 0 and want_valid[12] == 1
    ok = want_valid == 1
    assert np.array_equal(got.cpu().numpy()[ok], want[ok])


def test_cicids_encode_f32_records():
    rec, dicts = synth.make_cicids(30001, 15, seed=4, device=DEV, nan_fraction=0.01)
    schema = synth.cicids_schema()
    counts = enc.category_counts(rec, schema, "Label", 15).cpu().numpy()
    assert np.array_equal(counts, oracle.category_counts(rec.cpu().numpy(), schema.row_bytes, schema.offsets["Label"], 15))
    ordered, lut = enc.string_index_order(counts, dicts["Label"])
    plan = enc.EncodePlan(schema)
    for f in schema.names[:-1]:
        plan.add_numeric(f)
    plan.set_label("Label", lut); plan.check_nan = 1
    want, wl, wv = oracle_encode(plan, rec.cpu().numpy())
    got, lab, valid = plan.run(rec, torch.float64)
    assert np.array_equal(valid.cpu().numpy(), wv) and 0 < (wv == 0).sum() < 2000
    assert np.array_equal(np.nan_to_num(got.cpu().numpy(), nan=-1.0), np.nan_to_num(want, nan=-1.0))
    assert np.array_equal(lab.cpu().numpy(), wl)


# ------------------------------------------------------------------------------- tree prep
def _features(n, n_classes, seed, kind="kdd"):
    if kind == "kdd":
        rec, dicts, schema = _kdd(n, n_classes, seed)
        luts, ordered = kdd_luts_gpu(rec, schema, dicts)
        plan = kdd_plan(schema, luts, ordered)
        x, y, _ = plan.run(rec, torch.float64)
        arity = [0] * 38 + [len(ordered[c]) for c in synth.KDD_CATEGORICAL]
        return x, y, arity, len(ordered["label"])
    rec, dicts = synth.make_cicids(n, n_classes, seed=seed, device=DEV)
    schema = synth.cicids_schema()
    counts = enc.category_counts(rec, schema, "Label", n_classes).cpu().numpy()
    ordered, lut = enc.string_index_order(counts, dicts["Label"])
    plan = enc.EncodePlan(schema)
    for f in schema.names[:-1]:
        plan.add_numeric(f)
    plan.set_label("Label", lut)
    x, y, _ = plan.run(rec, torch.float64)
    return x, y, [0] * 78, len(ordered)


def test_find_splits_and_binning_exact():
    x, y, arity, C = _features(60000, 5, 21)
    p = fr.ForestParams(num_trees=1, max_bins=70, max_depth=0, seed=99, bootstrap=False)
    m = fr.fit_forest(x, y, C, arity, p)
    xs = x.cpu().numpy()
    keep = int(min(1.0, max(70 * 70, 10000) / x.shape[0]) * 4294967296.0)
    thr, n_thr, ns = oracle.find_splits(xs, 99, keep, arity, 70)
    assert np.array_equal(m.n_thr.cpu().numpy(), n_thr)
    assert np.array_equal(m.thresholds.cpu().numpy(), thr)                            # fp64 midpoints, bit-exact
    tp_o, bad = oracle.bin_rows(xs, thr, n_thr, arity, 70, y.cpu().numpy())
    tp_g, bad_g = m.bin(x, y)
    assert bad == 0 and int(bad_g.item()) == 0
    F = x.shape[1]
    assert np.array_equal(tp_g.cpu().numpy()[:, :F + 1], tp_o[:, :F + 1]) and not tp_g[:, F + 1:].any()
    # float32 features bin identically to their widened fp64 values
    x32 = x.to(torch.float32)
    tp32, _ = m.bin(x32, y)
    tp_o32, _ = oracle.bin_rows(x32.cpu().numpy().astype(np.float64), thr, n_thr, arity, 70, y.cpu().numpy())
    assert np.array_equal(tp32.cpu().numpy()[:, :F + 1], tp_o32[:, :F + 1])


@pytest.mark.parametrize("n,max_bins", [(300, 32), (9000, 70), (60000, 100), (120000, 150), (120000, 256)])
def test_find_splits_small_and_large_samples(n, max_bins):
    # <= 16384 sampled rows: shared-memory sort + bisection walk; more: the global-memory kernel.  Columns: all-distinct
    # reals (every run has length 1), heavy ties, a constant, and few distinct values (fewer than maxBins).
    g = torch.Generator(device="cpu").manual_seed(n + max_bins)
    cols = [torch.randn(n, generator=g, dtype=torch.float64), torch.randint(0, 500, (n,), generator=g).to(torch.float64) ** 2,
            torch.zeros(n, dtype=torch.float64), torch.randint(0, 20, (n,), generator=g).to(torch.float64) * 0.25,
            torch.floor(torch.rand(n, generator=g, dtype=torch.float64) ** 6 * 1e6)]
    x = torch.stack(cols, 1).contiguous()
    y = (x[:, 0] > 0).to(torch.int32)
    p = fr.ForestParams(num_trees=1, max_bins=max_bins, max_depth=0, seed=7, bootstrap=False)
    m = fr.fit_forest(x.to(DEV), y.to(DEV), 2, [0] * 5, p)
    mpb = min(max_bins, n)
    keep = int(min(1.0, max(mpb * mpb, 10000) / n) * 4294967296.0)
    thr, n_thr, ns = oracle.find_splits(x.numpy(), 7, keep, [0] * 5, mpb)
    assert np.array_equal(m.n_thr.cpu().numpy(), n_thr)
    assert np.array_equal(m.thresholds.cpu().numpy(), thr)


def test_bagging_weights_and_entries_match_oracle():
    n, T, seed = 5000, 7, 1234
    cdf = fr.poisson_cdf_table(1.0)
    assert np.array_equal(cdf, oracle.poisson_cdf_table(1.0))
    w = oracle.bag_weights(seed, T, n, cdf, row_offset=17)
    cdf_t = torch.from_numpy(cdf.view(np.int32).copy()).to(DEV)
    W = torch.zeros(T * n, dtype=torch.int32, device=DEV)
    _lib.call("b200flow_bag_weights", seed, T, 17, n, _lib.ptr(cdf_t), cdf.ctypes.data, None, None, n, _lib.ptr(W))       # identity uid
    assert np.array_equal(W.cpu().numpy().reshape(T, n), w.astype(np.int32))
    # duplicate groups: weights of the rows of a group are summed into its unique record
    uid = torch.randint(0, 37, (n,), dtype=torch.int32, device=DEV)
    W2 = torch.zeros(T * 37, dtype=torch.int32, device=DEV)
    _lib.call("b200flow_bag_weights", seed, T, 17, n, _lib.ptr(cdf_t), cdf.ctypes.data, _lib.ptr(uid), None, 37, _lib.ptr(W2))
    want = np.zeros((T, 37), np.int64)
    for t in range(T):
        np.add.at(want[t], uid.cpu().numpy(), w[t])
    assert np.array_equal(W2.cpu().numpy().reshape(T, 37), want)
    # the same through the grouped order (rows of a group adjacent): identical sums
    gsize = torch.empty(37, dtype=torch.int32, device=DEV); cursor = torch.empty(37, dtype=torch.int32, device=DEV)
    goff = torch.empty(38, dtype=torch.int64, device=DEV)
    perm = torch.empty(n, dtype=torch.int32, device=DEV); uperm = torch.empty(n, dtype=torch.int32, device=DEV)
    _lib.call("b200flow_group_rows", _lib.ptr(uid), n, 37, _lib.ptr(gsize), _lib.ptr(goff), _lib.ptr(cursor), _lib.ptr(perm), _lib.ptr(uperm))
    assert torch.equal(torch.sort(perm)[0], torch.arange(n, dtype=torch.int32, device=DEV)) and torch.equal(uperm, uid[perm.long()])
    assert bool((uperm[1:] >= uperm[:-1]).all())
    W3 = torch.zeros(T * 37, dtype=torch.int32, device=DEV)
    _lib.call("b200flow_bag_weights", seed, T, 17, n, _lib.ptr(cdf_t), cdf.ctypes.data, _lib.ptr(uperm), _lib.ptr(perm), 37, _lib.ptr(W3))
    assert torch.equal(W3, W2)
    # entries = non-zero (unique, weight) pairs per tree, in unique-id order
    nb = (n + 1023) // 1024
    blk = torch.zeros(T * nb, dtype=torch.int32, device=DEV)
    _lib.call("b200flow_bag_count", _lib.ptr(W), T, n, _lib.ptr(blk))
    off = torch.zeros(T * nb + 1, dtype=torch.int64, device=DEV); tot = torch.zeros(1, dtype=torch.int64, device=DEV)
    _lib.call("b200flow_exclusive_scan_i32_to_i64", _lib.ptr(blk), T * nb, _lib.ptr(off), _lib.ptr(tot))
    E = int(tot.item())
    assert E == int((w > 0).sum())
    ent = torch.empty((E, 2), dtype=torch.int32, device=DEV)
    _lib.call("b200flow_bag_fill", _lib.ptr(W), T, n, _lib.ptr(off), _lib.ptr(ent))
    ent, off = ent.cpu().numpy(), off.cpu().numpy()
    for t in range(T):
        b, e = off[t * nb], off[(t + 1) * nb]
        idx = np.nonzero(w[t])[0]
        assert np.array_equal(ent[b:e, 0], idx) and np.array_equal(ent[b:e, 1], w[t][idx])


def test_dedup_rows_groups_identical_records():
    n, F = 50000, 41
    stride = fr.tp_stride(F)
    g = torch.Generator(device=DEV); g.manual_seed(3)
    base = torch.randint(0, 70, (900, stride), dtype=torch.uint8, device=DEV, generator=g)
    base[:, F + 1:] = 0
    pick = torch.randint(0, 900, (n,), device=DEV, generator=g)
    pick[:20000] = 5                                                                   # one huge duplicate group
    tp = base[pick].contiguous()
    cap = 1 << 17
    table = torch.empty(cap, dtype=torch.int32, device=DEV); minrow = torch.empty(cap, dtype=torch.int32, device=DEV)
    slot_of = torch.empty(n, dtype=torch.int32, device=DEV); rep = torch.empty(n, dtype=torch.int32, device=DEV)
    flag = torch.empty(n, dtype=torch.int32, device=DEV); pos = torch.empty(n + 1, dtype=torch.int64, device=DEV)
    uid = torch.empty(n, dtype=torch.int32, device=DEV); tpu = torch.empty_like(tp); tot = torch.zeros(1, dtype=torch.int64, device=DEV)
    _lib.call("b200flow_dedup_rows", _lib.ptr(tp), n, stride, F + 1, _lib.ptr(table), _lib.ptr(minrow), cap, _lib.ptr(slot_of),
              _lib.ptr(rep), _lib.ptr(flag), _lib.ptr(pos), _lib.ptr(tot), _lib.ptr(uid), _lib.ptr(tpu))
    U = int(tot.item())
    tp_n, uid_n, tpu_n = tp.cpu().numpy(), uid.cpu().numpy(), tpu.cpu().numpy()[:U]
    uniq, first, inv = np.unique(tp_n, axis=0, return_index=True, return_inverse=True)
    assert U == len(uniq)
    assert np.array_equal(tpu_n[uid_n], tp_n)                                          # every row maps to its own record
    order = np.argsort(first)                                                          # ids follow each group's first row
    rank = np.empty(len(uniq), np.int64); rank[order] = np.arange(len(uniq))
    assert np.array_equal(uid_n, rank[inv.reshape(-1)])


def test_scan_large():
    n = 1_000_003
    a = torch.randint(0, 5, (n,), dtype=torch.int32, device=DEV)
    out = torch.empty(n + 1, dtype=torch.int64, device=DEV); tot = torch.zeros(1, dtype=torch.int64, device=DEV)
    _lib.call("b200flow_exclusive_scan_i32_to_i64", _lib.ptr(a), n, _lib.ptr(out), _lib.ptr(tot))
    ref = torch.cumsum(a.to(torch.int64), 0)
    assert torch.equal(out[1:], ref) and int(out[0]) == 0 and int(tot) == int(ref[-1])


@pytest.mark.parametrize("F,m", [(41, 7), (78, 9), (78, 26), (5, 2), (300, 100)])
def test_feature_subsets_match_oracle(F, m):
    S = 500
    tree = torch.randint(0, 100, (S,), dtype=torch.int32, device=DEV)
    nid = torch.randint(1, 1 << 20, (S,), dtype=torch.int32, device=DEV)
    sub = torch.empty((S, m), dtype=torch.int16, device=DEV)
    _lib.call("b200flow_feature_subsets", 4242, S, _lib.ptr(tree), _lib.ptr(nid), F, m, _lib.ptr(sub))
    sub = sub.cpu().numpy(); tree = tree.cpu().numpy(); nid = nid.cpu().numpy()
    for s in range(0, S, 7):
        assert np.array_equal(sub[s], oracle.feature_subset(4242, int(tree[s]), int(nid[s]), F, m))


def test_hist_level_direct():
    n, F, C, NB, m = 30000, 41, 5, 70, 7
    g = torch.Generator(device=DEV); g.manual_seed(5)
    stride = fr.tp_stride(F)
    tp = torch.randint(0, NB, (n, stride), dtype=torch.uint8, device=DEV, generator=g)
    tp[:, F] = torch.randint(0, C, (n,), dtype=torch.uint8, device=DEV, generator=g)
    tp[:20000, :F] = tp[0, :F]                                                         # duplicate-heavy (smurf-like) rows
    ent = torch.randperm(n, device=DEV, generator=g)[:25000].to(torch.int32)
    w = torch.randint(1, 5, (25000,), dtype=torch.uint8, device=DEV, generator=g)
    bounds = [0, 3, 3, 9000, 25000]                                                    # 4 slots incl. an empty one
    S = 4
    seg_b = torch.tensor(bounds[:-1], dtype=torch.int64, device=DEV); seg_e = torch.tensor(bounds[1:], dtype=torch.int64, device=DEV)
    nch = ((seg_e - seg_b + 2047) // 2048).to(torch.int32)
    coff = torch.zeros(S + 1, dtype=torch.int64, device=DEV); tot = torch.zeros(1, dtype=torch.int64, device=DEV)
    _lib.call("b200flow_exclusive_scan_i32_to_i64", _lib.ptr(nch), S, _lib.ptr(coff), _lib.ptr(tot))
    sub = torch.stack([torch.sort(torch.randperm(F, device=DEV, generator=g)[:m])[0] for _ in range(S)]).to(torch.int16)
    hist = torch.zeros(S * m * NB * C, dtype=torch.int32, device=DEV)
    packed = torch.stack([ent, w.to(torch.int32)], 1).contiguous()                     # {record index, weight} pairs
    _lib.call("b200flow_hist_level", _lib.ptr(tp), stride, F, _lib.ptr(packed), S, _lib.ptr(seg_b), _lib.ptr(seg_e),
              _lib.ptr(coff), int(tot.item()), 2048, _lib.ptr(sub), m, NB, C, _lib.ptr(hist))
    hist = hist.cpu().numpy().reshape(S, m, NB, C)
    tp_n, ent_n, w_n, sub_n = tp.cpu().numpy(), ent.cpu().numpy(), w.cpu().numpy(), sub.cpu().numpy()
    for s in range(S):
        want = oracle.hist_node(tp_n, F, ent_n[bounds[s]:bounds[s + 1]], w_n[bounds[s]:bounds[s + 1]], sub_n[s], NB, C)
        assert np.array_equal(hist[s], want)


# ------------------------------------------------------------------------------- forests
def _fit_both(x, y, C, arity, **kw):
    p = fr.ForestParams(**kw)
    model = fr.fit_forest(x, y, C, arity, p)
    T = p.num_trees
    fo, meta = oracle.fit_forest(x.cpu().numpy(), y.cpu().numpy(), C, arity, num_trees=T, max_bins=p.max_bins,
                                 max_depth=p.max_depth, min_instances=p.min_instances_per_node, min_info_gain=p.min_info_gain,
                                 seed=p.seed, strategy=p.feature_subset_strategy, subsampling_rate=p.subsampling_rate)
    return model, fo, meta


def _check_predictions(model, fo, meta, xt, dt_mode=False):
    tp_o, _ = oracle.bin_rows(xt.cpu().numpy(), meta["thresholds"], meta["n_thr"], meta["arity"], meta["max_bins"])
    raw_o, prob_o, pred_o = fo.predict(tp_o, dt_mode=dt_mode)
    raw, prob, pred = model.predict(xt)
    assert np.array_equal(pred.cpu().numpy(), pred_o)                                  # labels bit-exact
    assert np.array_equal(raw.cpu().numpy(), raw_o) and np.array_equal(prob.cpu().numpy(), prob_o)
    return pred_o


def test_decision_tree_deterministic_anchor_kdd_binary():
    # <= 10 000 rows, maxBins^2 <= 10 000: no RNG at all in MLlib (SURVEY §4) — DT = T=1, all features
    x, y, arity, C = _features(9000, 2, 31)
    model, fo, meta = _fit_both(x, y, C, arity, num_trees=1, max_bins=70, max_depth=5, bootstrap=False, seed=1)
    assert forests_equal(model.export(), fo.export()) == []
    _check_predictions(model, fo, meta, x[:3000], dt_mode=True)


@pytest.mark.parametrize("depth", [2, 4])
def test_decision_tree_cuda_matches_exact_cart(depth):
    # independent anchor (tests/test_oracle_vs_sklearn.py): with fewer distinct values than maxBins every midpoint is a
    # candidate threshold, so the CUDA DecisionTree must equal scikit-learn's exact CART node for node
    sktree = pytest.importorskip("sklearn.tree")
    rng = np.random.default_rng(depth)
    xn = rng.integers(0, 20, size=(3000, 6)).astype(np.float64)
    score = (xn[:, 0] > 9.5) * 1.0 + (xn[:, 2] > 4.5) * 1.0 + (xn[:, 4] > 14.5) * 0.7 + rng.normal(0, 0.6, 3000)
    yn = np.digitize(score, [0.8, 1.7]).astype(np.int32)
    model = fr.fit_forest(torch.from_numpy(xn).to(DEV), torch.from_numpy(yn).to(DEV), 3, [0] * 6,
                          fr.ForestParams(num_trees=1, max_bins=32, max_depth=depth, bootstrap=False, seed=depth))
    sk = sktree.DecisionTreeClassifier(criterion="gini", max_depth=depth, random_state=0).fit(xn, yn)
    assert model.n_nodes == sk.tree_.node_count
    raw, prob, pred = model.predict(torch.from_numpy(xn).to(DEV))
    assert np.array_equal(pred.cpu().numpy(), sk.predict(xn).astype(np.float64))
    assert np.abs(prob.cpu().numpy() - sk.predict_proba(xn)).max() < 1e-15


@pytest.mark.parametrize("n_classes,depth,trees", [(2, 5, 20), (5, 8, 10), (23, 6, 6)])
def test_random_forest_kdd_matches_oracle(n_classes, depth, trees):
    x, y, arity, C = _features(40000, n_classes, 77 + n_classes)
    model, fo, meta = _fit_both(x, y, C, arity, num_trees=trees, max_bins=70, max_depth=depth, seed=2019)
    # protocol_type (arity 3): unordered when multiclass, ordered when binary (F7 / A.1)
    assert meta["feat_kind"][38] == (2 if C > 2 else 1) and meta["feat_kind"][39] == 1
    assert forests_equal(model.export(), fo.export()) == []
    xt, yt, _, _ = _features(15000, n_classes, 500 + n_classes)
    pred = _check_predictions(model, fo, meta, xt)
    cm = fr.confusion_matrix(torch.from_numpy(pred).to(DEV), yt.to(torch.float64), C)
    cm_o = oracle.confusion(pred, yt.cpu().numpy().astype(np.float64), C)
    assert np.array_equal(cm.cpu().numpy(), cm_o)
    mg, mo = fr.metrics_from_confusion(cm.cpu().numpy()), oracle.metrics(cm_o)
    for k in mo:
        assert abs(mg[k] - mo[k]) < 1e-12
    assert mo["accuracy"] > 0.9


def test_random_forest_deep_kdd():
    x, y, arity, C = _features(60000, 5, 123)
    model, fo, meta = _fit_both(x, y, C, arity, num_trees=5, max_bins=70, max_depth=16, seed=7)
    assert forests_equal(model.export(), fo.export()) == []
    assert model.n_nodes > 2000
    _check_predictions(model, fo, meta, x[:20000])


def test_random_forest_cicids_matches_oracle():
    x, y, arity, C = _features(50000, 15, 9, kind="cicids")
    model, fo, meta = _fit_both(x, y, C, arity, num_trees=20, max_bins=78, max_depth=5, seed=2019)
    assert model.m == 9 and forests_equal(model.export(), fo.export()) == []
    _check_predictions(model, fo, meta, x[:10000])


def test_decision_tree_cicids_all_features_and_min_instances():
    x, y, arity, C = _features(30000, 6, 10, kind="cicids")
    model, fo, meta = _fit_both(x, y, C, arity, num_trees=1, max_bins=32, max_depth=7, bootstrap=False,
                                min_instances_per_node=25, min_info_gain=0.001, seed=3)
    assert model.m == 78 and forests_equal(model.export(), fo.export()) == []
    _check_predictions(model, fo, meta, x[:5000], dt_mode=True)


def test_decision_tree_wide_histogram_multipass():
    # 23 classes x 41 features x 70 bins = 264 KB per node: the histogram kernel must tile features over passes
    x, y, arity, C = _features(25000, 23, 91)
    model, fo, meta = _fit_both(x, y, C, arity, num_trees=1, max_bins=70, max_depth=5, bootstrap=False, seed=1)
    assert forests_equal(model.export(), fo.export()) == []
    _check_predictions(model, fo, meta, x[:4000], dt_mode=True)


def test_unfused_level_loop_equals_fused(monkeypatch):
    # route_hist_level (fused) and partition_level + hist_level (fallback for wide nodes) must build the same forest
    x, y, arity, C = _features(40000, 5, 64)
    p = fr.ForestParams(num_trees=6, max_bins=70, max_depth=9, seed=13)
    a = fr.fit_forest(x, y, C, arity, p).export()
    monkeypatch.setattr(fr, "FUSED", False)
    b = fr.fit_forest(x, y, C, arity, p).export()
    assert forests_equal(a, b) == []
    assert np.array_equal(a["gain"], b["gain"])


def test_dedup_does_not_change_the_forest(monkeypatch):
    # the level loop on unique records + summed weights must give the forest of the row-by-row loop
    x, y, arity, C = _features(50000, 5, 71)
    p = fr.ForestParams(num_trees=6, max_bins=70, max_depth=10, seed=29)
    m1 = fr.fit_forest(x, y, C, arity, p)
    assert m1.train_stats["unique_rows"] < 0.8 * m1.train_stats["rows"]                # the synthetic flows do repeat
    monkeypatch.setattr(fr, "DEDUP", False)
    m2 = fr.fit_forest(x, y, C, arity, p)
    assert m2.train_stats["unique_rows"] == m2.train_stats["rows"]
    assert forests_equal(m1.export(), m2.export()) == [] and np.array_equal(m1.export()["gain"], m2.export()["gain"])


def test_large_batch_size_independent_properties(monkeypatch):
    # Sizes the oracle cannot finish in seconds (1.2 M rows, 24 trees, depth 12) are checked through properties that do not
    # depend on the size: (1) the product path (fused level kernel, unique records, sharded-style padding)
    # builds byte for byte the forest of the plainest path (row-by-row, unfused hist + partition kernels); (2) the root
    # histogram of every tree sums to its bag weight total: sum of the roots' class counts == sum of the entries' weights;
    # (3) predictions do not depend on de-duplicating the test records, and raw votes sum to the number of trees.
    x, y, arity, C = _features(1200000, 5, 909)
    p = fr.ForestParams(num_trees=24, max_bins=70, max_depth=12, seed=77)
    fast = fr.fit_forest(x, y, C, arity, p)
    ex_fast = fast.export()
    roots = ex_fast["nid"] == 1
    assert int(roots.sum()) == 24
    w = oracle.bag_weights(77, 24, x.shape[0], oracle.poisson_cdf_table(1.0))          # [T, n] Poisson weights (host, cheap)
    assert np.array_equal(ex_fast["counts"][roots].sum(1), w.astype(np.int64).sum(1))
    xt = x[:300000]
    raw_a, prob_a, pred_a = fast.predict(xt)
    assert np.allclose(raw_a.sum(1).cpu().numpy(), 24.0, rtol=0, atol=1e-9)
    monkeypatch.setattr(fr, "DEDUP", False)
    monkeypatch.setattr(fr, "FUSED", False)
    plain = fr.fit_forest(x, y, C, arity, p)
    ex_plain = plain.export()
    assert forests_equal(ex_fast, ex_plain) == [] and np.array_equal(ex_fast["gain"], ex_plain["gain"])
    raw_b, prob_b, pred_b = plain.predict(xt)
    assert torch.equal(raw_a, raw_b) and torch.equal(prob_a, prob_b) and torch.equal(pred_a, pred_b)


def test_forest_fp32_features_equal_fp64_features():
    x, y, arity, C = _features(30000, 5, 55)
    p = fr.ForestParams(num_trees=4, max_bins=70, max_depth=6, seed=5)
    a = fr.fit_forest(x, y, C, arity, p).export()
    b = fr.fit_forest(x.to(torch.float32), y, C, arity, p).export()                    # KDD values are fp32-exact
    assert forests_equal(a, b) == []


def test_sharded_histograms_sum_to_unsharded():
    # multi-GPU property on one device: training on row shards with global row offsets, histograms added,
    # equals the unsharded histogram (integer sums) — checked through level-0 node counts and bagging.
    x, y, arity, C = _features(20000, 5, 8)
    p = fr.ForestParams(num_trees=3, max_bins=70, max_depth=0, seed=11)
    full = fr.fit_forest(x, y, C, arity, p).export()["counts"]
    # NOTE thresholds depend on the global sample; depth 0 only needs bagging + label counts
    a = fr.fit_forest(x[:7000], y[:7000], C, arity, p, row_offset=0).export()["counts"]
    b = fr.fit_forest(x[7000:], y[7000:], C, arity, p, row_offset=7000).export()["counts"]
    assert np.array_equal(a + b, full)


def test_max_bins_too_small_raises():
    x, y, arity, C = _features(2000, 2, 2)
    with pytest.raises(ValueError, match="maxBins"):
        fr.fit_forest(x, y, C, arity, fr.ForestParams(num_trees=1, max_bins=32, bootstrap=False))


# ------------------------------------------------------------------------------- split / compaction
def test_random_split_and_compaction():
    n = 100003
    cum = np.array([0.75, 1.0])
    sid = torch.empty(n, dtype=torch.uint8, device=DEV)
    _lib.call("b200flow_random_split", 2019, 5, n, cum.ctypes.data, 2, _lib.ptr(sid))
    want = oracle.random_split(2019, n, cum, row_offset=5)
    assert np.array_equal(sid.cpu().numpy(), want) and abs((want == 0).mean() - 0.75) < 0.01
    rows = torch.arange(n * 6, dtype=torch.int32, device=DEV).reshape(n, 6).contiguous()
    nb = (n + 1023) // 1024
    scratch = torch.zeros(nb + 1 + (nb + 1) // 2 + 1, dtype=torch.int64, device=DEV)
    for part in (0, 1):
        out = torch.empty_like(rows); kept = torch.zeros(1, dtype=torch.int64, device=DEV)
        flag = (sid == part).to(torch.uint8)
        _lib.call("b200flow_compact_rows", _lib.ptr(rows), n, 24, _lib.ptr(flag), 1, _lib.ptr(out), _lib.ptr(scratch), _lib.ptr(kept))
        k = int(kept.item())
        assert k == int((want == part).sum())
        assert torch.equal(out[:k], rows[torch.from_numpy(want == part).to(DEV)])
