"""Feature selection on the device: each csrc/selection.cu kernel against the numpy restatement (tests/selection_oracle.py)
with canaries around the buffers (dictionaries and counts exact, centred partials bit for bit), the distinct-value limit,
full fits of the three tests and three selectors on KDD-shaped data, and a lazy VectorAssembler -> UnivariateFeatureSelector
-> RandomForestClassifier pipeline that still trains and predicts from the raw records."""
import numpy as np
import pytest
import torch

import selection_oracle as so

pytestmark = pytest.mark.gpu

CANARY = 7.0


def _dev(a):
    return torch.as_tensor(np.ascontiguousarray(a)).cuda()


def _mixed(n, D, seed):
    """columns of cardinality 1, 2, 5, 40, 3000 and 9000 (at most), with -0.0 mixed into the zeros."""
    rng = np.random.default_rng(seed)
    cards = [1, 2, 5, 40, 3000, 9000]
    x = np.empty((n, D))
    for j in range(D):
        c = cards[j % len(cards)]
        x[:, j] = rng.integers(0, c, n) * (0.5 if c < 9000 else 0.37) - (c // 2)
    x[rng.random((n, D)) < 0.1] = -0.0
    return x


def _tables(x):
    from b200flow import selection as bs
    tab, cnt, ovf = bs.distinct_tables(_dev(x))
    return tab.cpu().numpy(), cnt.cpu().numpy(), ovf.cpu().numpy()


@pytest.mark.parametrize("D", [1, 41, 119, 256])
@pytest.mark.parametrize("n", [1, 4095, 4097, 100000])
def test_distinct_values_and_contingency_counts_are_exact(n, D):
    from b200flow import selection as bs
    x = _mixed(n, D, n + D)
    y = np.random.default_rng(D).integers(0, 7, n).astype(np.float64)
    tab, cnt, ovf = _tables(x)
    for j in range(D):
        keys = tab[j][tab[j] != -1].view(np.float64)
        want = so.dictionary(x[:, j])
        assert np.array_equal(np.sort(keys), want) and cnt[j] == len(want) and ovf[j] == 0, j
        assert not np.any(np.signbit(keys) & (keys == 0.0))
    sh = _one(n)
    dicts = bs.dictionaries(_dev(x), sh, "test")
    labels, ids = bs.label_dictionary(_dev(y), sh, "test")
    assert np.array_equal(labels, so.dictionary(y))
    assert np.array_equal(ids.cpu().numpy(), np.searchsorted(labels, y).astype(np.int32))
    want_l, want_t = so.contingency(x, y)
    got = bs.contingency_tables(_dev(x), ids, len(labels), dicts, sh)
    for j in range(D):
        assert np.array_equal(dicts[j], so.dictionary(x[:, j]))
        assert got[j].dtype == np.int64 and np.array_equal(got[j], want_t[j]), j


def _one(n):
    from b200flow import dist as bdist
    return bdist.Shards(n, 0, None, torch.device("cuda"))


@pytest.mark.parametrize("W", [4, 6])
def test_contingency_counts_write_only_their_cells(W):
    """W = 4: the counters fit in shared memory; W = 6 (a column of up to 9000 values): they are counted in global memory."""
    from b200flow._lib import call, ptr
    x = _mixed(5000, W, 3)
    y = np.random.default_rng(2).integers(0, 3, 5000).astype(np.float64)
    dicts = [so.dictionary(x[:, j]) for j in range(W)]
    o = np.concatenate([[0], np.cumsum([len(d) for d in dicts])]).astype(np.int32)
    nv, L = int(o[-1]), 3
    ids = np.searchsorted(so.dictionary(y), y).astype(np.int32)
    buf = torch.full((nv * L + 2,), 7, dtype=torch.int64, device="cuda")
    buf[1:-1] = 0
    xt, it, dt, ot = _dev(x), _dev(ids), _dev(np.concatenate(dicts)), _dev(o)
    call("b200flow_contingency_counts", ptr(xt), 5000, W, W, ptr(it), L, ptr(dt), ptr(ot), nv, ptr(buf[1:-1]))
    got = buf.cpu().numpy()
    assert got[0] == 7 and got[-1] == 7
    _, want = so.contingency(x, y)
    for j in range(W):
        assert np.array_equal(got[1:-1].reshape(nv, L)[o[j]:o[j + 1]], want[j]), j


@pytest.mark.parametrize("n,W", [(1, 1), (4097, 41), (100000, 119)])
def test_distinct_values_write_only_their_own_tables_and_counters(n, W):
    """canary rows around the tables and canary entries around the counters and overflow flags stay untouched."""
    from b200flow import selection as bs
    from b200flow._lib import call, ptr
    x = _mixed(n, W, 5)
    tab = torch.full((W + 2, bs.TABLE_SLOTS), -1, dtype=torch.int64, device="cuda")
    tab[0] = 12345
    tab[-1] = 12345
    cnt = torch.full((W + 2,), 77, dtype=torch.int32, device="cuda")
    ovf = torch.full((W + 2,), 77, dtype=torch.int32, device="cuda")
    cnt[1:-1] = 0
    ovf[1:-1] = 0
    xt = _dev(x)
    call("b200flow_distinct_values", ptr(xt), n, W, W, ptr(tab[1:-1]), ptr(cnt[1:-1]), ptr(ovf[1:-1]))
    t, c, o = tab.cpu().numpy(), cnt.cpu().numpy(), ovf.cpu().numpy()
    assert np.all(t[0] == 12345) and np.all(t[-1] == 12345)
    assert c[0] == 77 and c[-1] == 77 and o[0] == 77 and o[-1] == 77
    for j in range(W):
        keys = t[1 + j][t[1 + j] != -1].view(np.float64)
        assert np.array_equal(np.sort(keys), so.dictionary(x[:, j])) and c[1 + j] == len(keys) and o[1 + j] == 0, j


def test_distinct_value_limit():
    from b200flow import selection as bs
    x = np.zeros((30000, 3))
    x[:, 0] = np.arange(30000) % 10000                # exactly 10000 values
    x[:, 1] = np.arange(30000) % 10001                # one too many
    x[:, 2] = np.arange(30000)                        # far too many
    _, cnt, ovf = _tables(x)
    assert cnt[0] == 10000 and ovf.tolist() == [0, 1, 1]
    sh = _one(30000)
    assert len(bs.dictionaries(_dev(x[:, :1]), sh, "test")[0]) == 10000
    with pytest.raises(bs.TooManyValuesError, match="column 1"):
        bs.dictionaries(_dev(x), sh, "test")


@pytest.mark.parametrize("row_offset", [0, 4096 * 3 + 1000])
@pytest.mark.parametrize("n,D,G", [(1, 1, 1), (4095, 41, 5), (4097, 119, 23), (100000, 41, 3), (9000, 256, 256)])
def test_centered_moment_partials_equal_the_restatement(n, D, G, row_offset):
    from b200flow import selection as bs
    rng = np.random.default_rng(n + D)
    x = rng.normal(size=(n, D)) * rng.uniform(0.1, 5.0, D) + rng.normal(0, 10, D)
    ids = rng.integers(0, G, n).astype(np.int32)
    centers = rng.normal(size=(G, D))
    nc = len(so.chunks(n, row_offset))
    buf = torch.full((nc + 2, G, D), CANARY, dtype=torch.float64, device="cuda")
    bs.centered_moments(_dev(x), _dev(ids), G, _dev(centers), None, 0.0, row_offset, buf[1:nc + 1])
    got = buf.cpu().numpy()
    assert np.all(got[0] == CANARY) and np.all(got[-1] == CANARY)
    want = so.centered_partials(x, ids, G, centers, None, 0.0, row_offset)
    assert got[1:-1].tobytes() == want.tobytes()
    y = rng.normal(size=n) * 3 + x[:, 0]
    buf = torch.full((nc + 2, 1, 2 * D + 1), CANARY, dtype=torch.float64, device="cuda")
    bs.centered_moments(_dev(x), None, 1, _dev(centers[:1]), _dev(y), 0.25, row_offset, buf[1:nc + 1])
    got = buf.cpu().numpy()
    assert np.all(got[0] == CANARY) and np.all(got[-1] == CANARY)
    assert got[1:-1].tobytes() == so.centered_partials(x, None, 1, centers[:1], y, 0.25, row_offset).tobytes()


def _kdd(n, seed=7):
    """KDD-shaped features: the 38 numeric columns and the three indexed categorical ones, and the class label."""
    from b200flow import encode as enc, synth
    rec, dicts = synth.make_kdd(n, 5, seed=seed, device="cuda:0")
    schema = synth.kdd_schema()
    plan = enc.EncodePlan(schema)
    for c in synth.KDD_COLUMNS:
        if c not in synth.KDD_CATEGORICAL and c != "label":
            plan.add_numeric(c)
    for c in synth.KDD_CATEGORICAL:
        plan.add_index(c, np.arange(len(dicts[c]), dtype=np.int32))
    plan.set_label("label", np.arange(len(dicts["label"]), dtype=np.int32))
    x, y, _ = plan.run(rec, torch.float64)
    return x, y.to(torch.float64)


def test_full_fits_equal_the_restatement_bit_for_bit():
    from b200flow import selection as bs
    x, y = _kdd(30000)
    xh, yh = x.cpu().numpy(), y.cpu().numpy()
    cat = [j for j in range(x.shape[1]) if len(so.dictionary(xh[:, j])) <= 60]
    xc = x[:, cat].contiguous()
    res = bs.chi_square_test(xc, y)
    for a, b in zip((res.p_values, res.dof, res.statistics), so.chi_square(xh[:, cat], yh)):
        assert a.tobytes() == np.asarray(b).astype(a.dtype).tobytes()
    res = bs.anova_test(x, y)
    for a, b in zip((res.p_values, res.dof, res.statistics), so.anova(xh, yh)):
        assert np.asarray(a).tobytes() == np.asarray(b).astype(a.dtype).tobytes()
    yc = xh[:, 0] * 1e-3 + xh[:, 4] * 1e-6 + np.random.default_rng(1).normal(size=len(yh))
    res = bs.f_value_test(x, _dev(yc))
    for a, b in zip((res.p_values, res.dof, res.statistics), so.f_value(xh, yc)):
        assert np.asarray(a).tobytes() == np.asarray(b).astype(a.dtype).tobytes()
    assert bs.variances(x).tobytes() == so.variances(xh).tobytes()


def test_batched_partials_give_the_same_bits(monkeypatch):
    from b200flow import selection as bs
    x, y = _kdd(3 * 4096 + 77)
    one = bs.anova_test(x, y)
    monkeypatch.setattr(bs, "PARTIALS_BUDGET", 1)                   # one chunk per batch
    many = bs.anova_test(x, y)
    assert one.statistics.tobytes() == many.statistics.tobytes() and one.p_values.tobytes() == many.p_values.tobytes()


def test_limits_are_refused():
    from b200flow import _lib, selection as bs
    with pytest.raises(_lib.UnsupportedParamError):
        bs.anova_test(torch.zeros((10, 257), dtype=torch.float64, device="cuda"), torch.zeros(10, dtype=torch.float64,
                                                                                               device="cuda"))
    with pytest.raises(ValueError, match="finite"):
        bs.chi_square_test(_dev(np.full((10, 3), np.nan)), _dev(np.zeros(10)))
    with pytest.raises(ValueError, match="finite"):
        bs.f_value_test(_dev(np.zeros((10, 3))), _dev(np.full(10, np.inf)))
    with pytest.raises(_lib.UnsupportedParamError, match="256 distinct labels"):
        bs.chi_square_test(_dev(np.zeros((300, 2))), _dev(np.arange(300.0)))
    with pytest.raises(ValueError, match="two classes"):
        bs.anova_test(_dev(np.ones((10, 2))), _dev(np.zeros(10)))


def test_shim_tests_and_selectors_then_forest():
    from b200flow import selection as bs, synth
    from pyspark.ml import Pipeline
    from pyspark.ml.classification import RandomForestClassifier
    from pyspark.ml.feature import (ChiSqSelector, IllegalArgumentException, SparkException, StringIndexer,
                                    UnivariateFeatureSelector, VarianceThresholdSelector, VectorAssembler, _peek)
    from pyspark.ml.linalg import DenseVector
    from pyspark.ml.stat import ANOVATest, ChiSquareTest, FValueTest
    from test_kmeans_gpu import _kdd_frame
    df = _kdd_frame(20000, 11)
    cats = synth.KDD_CATEGORICAL
    nums = [c for c in synth.KDD_COLUMNS if c not in cats + ["label"]]
    idx = [StringIndexer(inputCol=c, outputCol=c + "_i") for c in cats + ["label"]]
    for s in idx:
        df = s.fit(df).transform(df)
    cols = nums + [c + "_i" for c in cats]
    out = VectorAssembler(inputCols=cols, outputCol="features").transform(df)
    x, y = _peek(out, "features"), _peek(out, "label_i")[:, 0].contiguous()
    assert out._cols["features"].lazy and out._cols["label_i"].lazy

    row = ANOVATest.test(out, "features", "label_i").head()
    want = bs.anova_test(x, y)
    assert isinstance(row.pValues, DenseVector) and np.array_equal(row.pValues.toArray(), want.p_values, equal_nan=True)
    assert row.degreesOfFreedom == [20000 - 1] * len(cols) and np.array_equal(row.fValues.toArray(), want.statistics,
                                                                              equal_nan=True)
    flat = FValueTest.test(out, "features", "label_i", flatten=True)
    assert flat.columns == ["featureIndex", "pValue", "degreesOfFreedom", "fValue"] and flat.count() == len(cols)
    assert out._cols["features"].lazy and out._cols["label_i"].lazy            # the tests leave the columns lazy
    cat_df = VectorAssembler(inputCols=[c + "_i" for c in cats], outputCol="cf").transform(df)
    chi = ChiSquareTest.test(cat_df, "cf", "label_i").head()
    assert chi.statistics.toArray().shape == (3,) and all(d > 0 for d in chi.degreesOfFreedom)
    with pytest.raises(IllegalArgumentException, match="does not exist"):
        ChiSquareTest.test(out, "nope", "label_i")
    with pytest.raises(SparkException, match="more than 10000"):
        ChiSquareTest.test(VectorAssembler(inputCols=["src_bytes"], outputCol="sb").transform(
            _wide_frame()), "sb", "label")

    sel = UnivariateFeatureSelector(featuresCol="features", outputCol="selected", labelCol="label_i",
                                    selectionMode="numTopFeatures").setFeatureType("continuous") \
        .setLabelType("categorical").setSelectionThreshold(8)
    pipe = Pipeline(stages=[sel, RandomForestClassifier(featuresCol="selected", labelCol="label_i", numTrees=5, maxDepth=6,
                                                        seed=3)]).fit(out)
    sm, forest = pipe.stages
    chosen = sm.selectedFeatures
    assert chosen == bs.select(want.p_values, "numTopFeatures", 8) and len(chosen) == 8
    res = sm.transform(out)
    sc = res._cols["selected"]
    assert sc.lazy and sc.prov[0] == "plan" and sc.prov[1].n_out == 8
    assert [a.get("name") for a in sc.meta["attrs"]] == [cols[j] for j in chosen]
    direct = VectorAssembler(inputCols=[cols[j] for j in chosen], outputCol="selected").transform(df)
    f2 = RandomForestClassifier(featuresCol="selected", labelCol="label_i", numTrees=5, maxDepth=6, seed=3).fit(direct)
    e1, e2 = forest._forest.export(), f2._forest.export()
    assert all(np.array_equal(e1[k], e2[k]) for k in e1)
    p1 = pipe.transform(out)._column_tensor("prediction")
    p2 = f2.transform(direct)._column_tensor("prediction")
    assert torch.equal(p1, p2)
    assert torch.equal(res._cols["selected"].data.to(torch.float64), x[:, chosen])

    vt = VarianceThresholdSelector(featuresCol="features", outputCol="v", varianceThreshold=0.5).fit(out)
    var = bs.variances(x)
    assert vt.selectedFeatures == [j for j in range(len(cols)) if var[j] > 0.5]
    dense = df._with(cols={"f": type(out._cols["features"])("vector", x, "f64", {}, None), "label_i": df._cols["label_i"]})
    vd = vt.copy({vt.featuresCol: "f"}).transform(dense)
    assert torch.equal(vd._cols["v"].data, x[:, vt.selectedFeatures]) and vd._cols["v"].prov is None
    cs = ChiSqSelector(numTopFeatures=2, featuresCol="cf", outputCol="c2", labelCol="label_i").fit(cat_df)
    assert cs.selectedFeatures == bs.select(chi.pValues.toArray(), "numTopFeatures", 2)
    fs = UnivariateFeatureSelector(featuresCol="features", outputCol="s", labelCol="label_i", selectionMode="fpr") \
        .setFeatureType("continuous").setLabelType("categorical").fit(out)
    assert fs.selectedFeatures == [j for j in range(len(cols)) if want.p_values[j] < 0.05]


def _wide_frame():
    from pyspark.sql import SparkSession
    import pandas as pd
    n = 10050
    return SparkSession.builder.getOrCreate().createDataFrame(pd.DataFrame({"src_bytes": np.arange(n, dtype=np.float64),
                                                                            "label": np.arange(n) % 2 * 1.0}))
