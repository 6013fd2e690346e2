"""NaiveBayes on the device: b200flow_nb_moments and b200flow_nb_raw through the C ABI at their edges, the four fits on KDD-
and CICIDS-shaped data against the numpy restatement bit for bit, the weighted paths against the unweighted ones, every
refusal, a CICIDS gaussian pipeline that keeps its negative features, and a CrossValidator over modelType x smoothing."""
import numpy as np
import pytest
import torch

import naive_bayes_oracle as nbo
import selection_oracle as so

pytestmark = pytest.mark.gpu

CANARY = -7.25


def _dev(a, dtype=torch.float64):
    return torch.from_numpy(np.ascontiguousarray(a)).to("cuda", dtype)


def _moments(x, ids, w, C, centers, row_offset):
    """b200flow_nb_moments into a buffer with a canary chunk on each side -> (partials, bad counts)."""
    from b200flow import naive_bayes as nb
    from b200flow._lib import call, ptr
    n, D = x.shape
    G, W = (C, D + 1) if centers is None else (C + 1, D)
    nc = len(so.chunks(n, row_offset))
    buf = torch.full((nc + 2, G, W), CANARY, dtype=torch.float64, device="cuda")
    bad = torch.zeros(5, dtype=torch.int64, device="cuda")
    p, code, ld = nb._rows(x)
    # every device input is held until the kernel has run: a dropped temporary's block goes back to torch's caching
    # allocator, and the next copy would overwrite it before the launch reads it
    ids_d, w_d, c_d = _dev(ids, torch.int32), _dev(w) if w is not None else None, _dev(centers) if centers is not None else None
    call("b200flow_nb_moments", p, code, n, D, ld, ptr(ids_d), ptr(w_d), C, ptr(c_d), row_offset, ptr(buf[1:nc + 1]), ptr(bad))
    got = buf.cpu().numpy()
    assert np.all(got[0] == CANARY) and np.all(got[-1] == CANARY)
    return got[1:-1], bad.cpu().numpy()


@pytest.mark.parametrize("n,D,C,row_offset,dtype,strided", [
    (5000, 1, 1, 0, torch.float64, False), (9000, 7, 2, 1234, torch.float32, True), (4096, 256, 3, 4096, torch.float64, True),
    (3000, 5, 256, 777, torch.float32, False), (1, 3, 2, 4095, torch.float64, False)])
def test_moments_kernel_edges(n, D, C, row_offset, dtype, strided):
    rng = np.random.default_rng(n + D + C)
    xh = np.round(rng.normal(size=(n, D)) * 4, 3)
    if dtype == torch.float32:
        xh = xh.astype(np.float32).astype(np.float64)
    ids = rng.integers(-1, C + 1, n)                       # some labels outside [0, C): left out and counted
    w = rng.uniform(0, 2, n)
    w[::7] = 0.0                                           # zero weights
    if C > 2:
        w[ids == 1] = 0.0                                  # a class present only with weight 0
    wide = _dev(np.concatenate([xh, np.full((n, 3), 99.0)], 1), dtype) if strided else _dev(xh, dtype)
    x = wide[:, :D]
    got, bad = _moments(x, ids, w, C, None, row_offset)
    want = nbo.moment_partials(xh, np.where((ids >= 0) & (ids < C), ids, -1), w, C, None, row_offset)
    assert got.tobytes() == want.tobytes()
    assert bad[4] == int(((ids < 0) | (ids >= C)).sum()) and bad[3] == 0
    assert bad[1] == int((xh < 0).sum()) and bad[2] == int(((xh != 0) & (xh != 1)).sum()) and bad[0] == 0
    centers = rng.normal(size=(C + 1, D))
    got, _ = _moments(x, ids, None, C, centers, row_offset)
    want = nbo.moment_partials(xh, np.where((ids >= 0) & (ids < C), ids, -1), None, C, centers, row_offset)
    assert got.tobytes() == want.tobytes()


def test_moments_kernel_counts_bad_inputs_and_takes_no_rows():
    x = np.array([[0.0, 1.0], [np.nan, 2.0], [np.inf, -1.0], [0.5, 0.0]])
    w = np.array([1.0, -1.0, np.nan, np.inf])
    _, bad = _moments(_dev(x), np.array([0, 1, 0, 1]), w, 2, None, 0)
    assert list(bad) == [2, 1, 5, 3, 0]
    from b200flow._lib import call, ptr
    xd = _dev(x)
    call("b200flow_nb_moments", ptr(xd), 1, 0, 2, 2, None, None, 2, None, 0, None, None)   # n = 0 on a rank: nothing


def _raw_kernel(f, x, model):
    from b200flow import naive_bayes as nb
    from b200flow._lib import call, ptr
    n, D = x.shape
    C = len(f.present)
    raw = torch.full((n + 1, C), CANARY, dtype=torch.float64, device="cuda")
    bad = torch.zeros(1, dtype=torch.int64, device="cuda")
    p, code, ld = nb._rows(x)
    a, c0, on = _dev(f.a), _dev(f.c0), _dev(f.present, torch.uint8)          # held until the kernel has run, as in _moments
    b, c1 = (_dev(f.b), _dev(f.c1)) if f.b is not None else (None, None)
    call("b200flow_nb_raw", p, code, n, D, ld, model, ptr(a), ptr(b), ptr(c0), ptr(c1), ptr(on), C, ptr(raw[:n]), ptr(bad))
    r = raw.cpu().numpy()
    assert np.all(r[n] == CANARY)
    return r[:n], int(bad.item())


@pytest.mark.parametrize("n,D,C,dtype,strided", [(100, 1, 1, torch.float64, False), (1000, 37, 2, torch.float32, True),
                                                 (300, 256, 40, torch.float64, True), (200, 9, 256, torch.float32, False),
                                                 (64, 256, 256, torch.float64, False)])
@pytest.mark.parametrize("mt", ["gaussian", "bernoulli", "complement"])
def test_raw_kernel_edges(n, D, C, dtype, strided, mt):
    rng = np.random.default_rng(n * D + C)
    m = max(2 * C, 50)
    xt = (rng.random((m, D)) < 0.4).astype(np.float64) if mt == "bernoulli" else np.round(rng.gamma(2.0, 2.0, (m, D)), 2)
    yt = np.arange(m) % max(C - 1, 1)                      # the last class is absent when C > 1
    f = nbo.fit(xt, yt, C, mt, 0.7)
    xh = (rng.random((n, D)) < 0.5).astype(np.float64) if mt == "bernoulli" else np.round(rng.gamma(2.0, 2.0, (n, D)), 2)
    if dtype == torch.float32:
        xh = xh.astype(np.float32).astype(np.float64)
    x = _dev(np.concatenate([xh, np.zeros((n, 2))], 1), dtype)[:, :D] if strided else _dev(xh, dtype)
    got, bad = _raw_kernel(f, x, 0 if mt == "gaussian" else 1)
    assert got.tobytes() == nbo.raw_sums(f, xh).tobytes()
    assert bad == int(((xh != 0) & (xh != 1)).sum())       # each value is counted once, whatever the model
    if mt == "complement":
        got, _ = _raw_kernel(f, x, 2)
        want = nbo.raw(f, xh)
        assert np.array_equal(np.isinf(got), np.isinf(want))
        np.testing.assert_allclose(got[np.isfinite(want)], want[np.isfinite(want)], rtol=1e-12, atol=1e-12)


def test_raw_kernel_counts_non_binary_values():
    f = nbo.fit(np.eye(3), np.arange(3), 3, "bernoulli")
    _, bad = _raw_kernel(f, _dev(np.array([[0.0, 1.0, 2.0], [0.5, 1.0, 0.0], [1.0, 1.0, 1.0]])), 1)
    assert bad == 2


# ------------------------------------------------------------------------------- whole fits
def _kdd(n, seed=5):
    """the 38 numeric KDD columns, the three categorical ones one-hot, the five binary flags, and the class label."""
    from b200flow import encode as enc, synth
    rec, dicts = synth.make_kdd(n, 5, seed=seed, device="cuda:0")
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


def _cicids(n, seed=6):
    from b200flow import encode as enc, synth
    rec, dicts = synth.make_cicids(n, 15, seed=seed, device="cuda:0")
    plan = enc.EncodePlan(synth.cicids_schema())
    for i in range(78):
        plan.add_numeric("f%02d" % i)
    plan.set_label("Label", np.arange(len(dicts["Label"]), dtype=np.int32))
    x, y, _ = plan.run(rec, torch.float32)
    return x, y.to(torch.float64), len(dicts["Label"])


def _check_fit(x, y, C, mt, lam, w=None):
    from b200flow import naive_bayes as nb
    fit = nb.nb_fit(x, y, C, mt, lam, weights=None if w is None else _dev(w))
    xh, yh = x.double().cpu().numpy(), y.cpu().numpy()
    f = nbo.fit(xh, yh, C, mt, lam, w)
    assert fit.pi.cpu().numpy().tobytes() == f.pi.tobytes(), mt
    assert fit.theta.cpu().numpy().tobytes() == f.theta.tobytes(), mt
    assert fit.sigma.cpu().numpy().tobytes() == f.sigma.tobytes(), mt
    assert fit.present.cpu().numpy().tolist() == f.present.tolist()
    if mt != "multinomial":
        got, _ = _raw_kernel(f, x[:3000], 0 if mt == "gaussian" else 1)
        assert got.tobytes() == nbo.raw_sums(f, xh[:3000]).tobytes(), mt
        r = nb.nb_raw(fit, x[:3000]).cpu().numpy()
        want = nbo.raw(f, xh[:3000])
        if mt == "complement":
            np.testing.assert_allclose(r[np.isfinite(want)], want[np.isfinite(want)], rtol=1e-12, atol=1e-12)
        else:
            assert r.tobytes() == want.tobytes(), mt
    return fit


@pytest.mark.parametrize("mt", ["multinomial", "complement", "bernoulli"])
def test_kdd_fits_equal_the_restatement(mt):
    xn, xb, y, C = _kdd(30000)
    x = xb if mt == "bernoulli" else xn
    w = np.random.default_rng(2).uniform(0.0, 3.0, x.shape[0])
    _check_fit(x, y, C, mt, 1.0)
    _check_fit(x, y, C, mt, 0.25, w)


def test_gaussian_fits_equal_the_restatement():
    x, y, C = _cicids(20000)
    _check_fit(x, y, C, "gaussian", 1.0)
    _check_fit(x, y, C, "gaussian", 1.0, np.random.default_rng(3).uniform(0.0, 2.0, x.shape[0]))
    xn, _, yk, Ck = _kdd(12000)
    _check_fit(xn, yk, Ck, "gaussian", 1.0)


def test_weights_of_one_equal_the_unweighted_fit():
    from b200flow import linear, naive_bayes as nb
    xn, _, y, C = _kdd(20000)
    a = linear.nb_fit(xn, y, C, 1.0)
    b = nb.nb_fit(xn, y, C, "multinomial", 1.0, weights=torch.ones(xn.shape[0], dtype=torch.float64, device="cuda"))
    np.testing.assert_allclose(b.pi.cpu().numpy(), a.pi.cpu().numpy(), rtol=1e-12)
    np.testing.assert_allclose(b.theta.cpu().numpy(), a.theta.cpu().numpy(), rtol=1e-12)


@pytest.mark.parametrize("mt", ["multinomial", "complement", "bernoulli", "gaussian"])
def test_integer_weights_equal_duplicated_rows(mt):
    from b200flow import naive_bayes as nb
    xn, xb, y, C = _kdd(8000)
    x = xb if mt == "bernoulli" else xn
    reps = torch.from_numpy(np.random.default_rng(4).integers(0, 4, x.shape[0])).cuda()
    a = nb.nb_fit(x, y, C, mt, 1.0, weights=reps.to(torch.float64))
    b = nb.nb_fit(torch.repeat_interleave(x, reps, 0), torch.repeat_interleave(y, reps), C, mt, 1.0)
    for name in ("pi", "theta", "sigma"):
        np.testing.assert_allclose(getattr(a, name).cpu().numpy(), getattr(b, name).cpu().numpy(), rtol=1e-12, atol=1e-300)


@pytest.mark.parametrize("mt,x,y,w,msg", [
    ("multinomial", [[1.0, -1.0], [0.0, 1.0]], [0, 1], [1.0, 1.0], "nonnegative feature values"),
    ("complement", [[1.0, -1.0], [0.0, 1.0]], [0, 1], None, "nonnegative feature values"),
    ("bernoulli", [[1.0, 0.5], [0.0, 1.0]], [0, 1], None, "0 or 1 feature values"),
    ("gaussian", [[1.0, np.nan], [0.0, 1.0]], [0, 1], None, "finite feature values"),
    ("gaussian", [[1.0, 2.0], [0.0, 1.0]], [0, 1], [1.0, -0.5], "weights must be finite and nonnegative"),
    ("complement", [[1.0, 2.0], [0.0, 1.0]], [0, 1], [np.inf, 1.0], "weights must be finite and nonnegative"),
    ("gaussian", [[1.0, 2.0], [1.0, 2.0]], [0, 1], None, "not constant"),
    ("bernoulli", [[1.0, 0.0], [0.0, 1.0]], [0, 1], [0.0, 0.0], "positive total weight")])
def test_fit_refusals(mt, x, y, w, msg):
    from pyspark.ml.classification import NaiveBayes
    from pyspark.ml.feature import IllegalArgumentException
    from pyspark.sql import ColumnData, DataFrame
    cols = {"features": ColumnData("vector", _dev(np.array(x)), "f64"), "label": ColumnData("numeric", _dev(np.array(y, float)), "f64")}
    if w is not None:
        cols["w"] = ColumnData("numeric", _dev(np.array(w)), "f64")
    with pytest.raises(IllegalArgumentException, match=msg):
        NaiveBayes(modelType=mt, weightCol="w" if w is not None else None).fit(DataFrame(len(y), None, None, {}, cols))


def test_library_refusals():
    from b200flow import _lib, naive_bayes as nb
    x = torch.ones((4, 257), dtype=torch.float64, device="cuda")
    y = torch.zeros(4, dtype=torch.float64, device="cuda")
    with pytest.raises(_lib.UnsupportedParamError):
        nb.nb_fit(x, y, 2, "gaussian")
    with pytest.raises(_lib.UnsupportedParamError):
        nb.nb_fit(x[:, :3], y, 257, "gaussian")
    with pytest.raises(ValueError, match="not integers"):
        nb.nb_fit(x[:, :3], torch.tensor([0.0, 1.5, 0.0, 1.0], dtype=torch.float64, device="cuda"), 2, "bernoulli")


def test_bernoulli_transform_refuses_non_binary_values():
    from pyspark.ml.classification import NaiveBayes
    from pyspark.ml.feature import IllegalArgumentException
    from pyspark.sql import ColumnData, DataFrame
    x, y = _dev(np.array([[1.0, 0.0], [0.0, 1.0]])), _dev(np.array([0.0, 1.0]))
    df = DataFrame(2, None, None, {}, {"features": ColumnData("vector", x, "f64"), "label": ColumnData("numeric", y, "f64")})
    m = NaiveBayes(modelType="bernoulli").fit(df)
    bad = DataFrame(1, None, None, {}, {"features": ColumnData("vector", _dev(np.array([[2.0, 0.0]])), "f64")})
    with pytest.raises(IllegalArgumentException, match="0 or 1 feature values"):
        m.transform(bad)


def test_known_answers_through_the_shim():
    from pyspark.ml.classification import NaiveBayes
    from pyspark.sql import ColumnData, DataFrame
    x = _dev(np.array([[0.0, 0.0], [0.0, 1.0], [1.0, 0.0]]))
    cols = {"features": ColumnData("vector", x, "f64"), "label": ColumnData("numeric", _dev(np.array([0.0, 0.0, 1.0])), "f64"),
            "w": ColumnData("numeric", _dev(np.array([0.1, 0.5, 1.0])), "f64")}
    df = DataFrame(3, None, None, {}, cols)
    pt = DataFrame(1, None, None, {}, {"features": ColumnData("vector", _dev(np.array([[1.0, 0.0]])), "f64")})
    for mt, wcol, prob in (("multinomial", "w", [0.324324, 0.675676]), ("complement", "w", [0.375, 0.625]),
                           ("bernoulli", None, [0.296703, 0.703297])):
        out = NaiveBayes(modelType=mt, weightCol=wcol).fit(df).transform(pt)
        np.testing.assert_allclose(out._column_tensor("probability").cpu().numpy()[0], prob, atol=1e-6)
        assert float(out._column_tensor("prediction")[0]) == 1.0
    m = NaiveBayes(modelType="gaussian").fit(df)
    eps = 1e-9 * 2.0 / 9.0
    np.testing.assert_allclose(m.sigma, [[eps, 0.25 + eps], [eps, eps]], rtol=1e-12)
    raw = m.transform(pt)._column_tensor("rawPrediction").cpu().numpy()[0]
    assert abs(raw[1] - 21.128731) < 1e-6 and np.argmax(raw) == 1
    assert NaiveBayes().fit(df).sigma.shape == (0, 0)


def test_cicids_gaussian_pipeline_keeps_negative_features():
    """the CICIDS2017 script's pipeline without its where-filters: negative flow features go straight into a gaussian fit"""
    from b200flow import synth
    from pyspark.ml import Pipeline
    from pyspark.ml.classification import NaiveBayes
    from pyspark.ml.evaluation import MulticlassClassificationEvaluator
    from pyspark.ml.feature import StringIndexer, VectorAssembler
    from pyspark.sql import DataFrame
    rec, dicts = synth.make_cicids(40000, 15, seed=9, device="cuda:0")
    f = rec.view(torch.float32)                            # 78 f32 fields and the label code per record
    f[:, 3] -= 5.0
    f[::3, 7] = -1.0
    df = DataFrame.fromRecords(rec, synth.cicids_schema(), dicts)
    feats = ["f%02d" % i for i in range(78)]
    pipe = Pipeline(stages=[StringIndexer(inputCol="Label", outputCol="label"), VectorAssembler(inputCols=feats, outputCol="features"),
                            NaiveBayes(modelType="gaussian")])
    model = pipe.fit(df)
    out = model.transform(df)
    assert MulticlassClassificationEvaluator(metricName="accuracy").evaluate(out) > 0.5
    nbm = model.stages[-1]
    x = out._column_tensor("features")
    want = nbo.fit(x.double().cpu().numpy(), out._column_tensor("label").cpu().numpy(), nbm.numClasses, "gaussian")
    assert float(x.min()) < 0.0
    assert nbm.theta.tobytes() == want.theta.tobytes() and nbm.sigma.tobytes() == want.sigma.tobytes()


def test_cross_validator_over_model_type_and_smoothing():
    from feature_helpers import kdd_frame
    from pyspark.ml.classification import NaiveBayes
    from pyspark.ml.evaluation import MulticlassClassificationEvaluator
    from pyspark.ml.feature import VectorAssembler
    from pyspark.ml.tuning import CrossValidator, ParamGridBuilder
    df, feats = kdd_frame(12000, 5, seed=13)
    vdf = VectorAssembler(inputCols=feats, outputCol="features").transform(df).select(["features", "label_num"])
    nb = NaiveBayes(labelCol="label_num")
    grid = ParamGridBuilder().addGrid(nb.modelType, ["multinomial", "complement", "gaussian"]).addGrid(nb.smoothing, [0.5, 1.0]).build()
    ev = MulticlassClassificationEvaluator(labelCol="label_num", metricName="accuracy")
    m = CrossValidator(estimator=nb, estimatorParamMaps=grid, evaluator=ev, numFolds=2, seed=7).fit(vdf)
    assert len(m.avgMetrics) == 6 and all(0.0 < v <= 1.0 for v in m.avgMetrics)
    assert m.avgMetrics[4] == m.avgMetrics[5]              # gaussian ignores smoothing
    assert m.bestModel.getOrDefault("modelType") in ("multinomial", "complement", "gaussian")
