"""FMClassifier and OneVsRest(FMClassifier) on the device: the fused DMMA factorization-machine kernel against the numpy
restatement (tests/fm_oracle.py), with and without the linear and intercept blocks and with a mini-batch; column
separability bit for bit (a K-column launch equals K one-column launches, for any subset and class block); feature dtypes
and chunk-order splits; canaries around every kernel output; fm_raw against the fit's arithmetic; the PySpark doctest
through createDataFrame; fits against the restatement's; the OneVsRest sub-models against standalone fits bit for bit; the
joint transform; the shim pipeline and the limits."""
import numpy as np
import pytest
import torch

import fm_oracle as fo

pytestmark = pytest.mark.gpu


def _problem(n, D, K, kf, seed, n_labels=None):
    rng = np.random.default_rng(seed)
    x = rng.normal(0.0, 1.0, (n, D)) * rng.uniform(0.3, 2.0, D) * (rng.random((n, D)) < 0.7)
    y = rng.integers(0, n_labels or max(K, 2), n).astype(np.int32)
    w = rng.normal(0.0, 0.6 / np.sqrt(D), (K, D * (kf + 1) + 1))
    w[:, -1] = rng.normal(0.0, 0.5, K)
    return np.ascontiguousarray(x), y, w


def _totals(x, y, pos, w, kf, fraction=1.0, seed=43):
    from b200flow import dist as bdist, fm as bfm
    xt = torch.as_tensor(x).cuda()
    sh = bdist.Shards(xt.shape[0], 0, None, xt.device)
    t = bfm.fm_loss_grad_totals(xt, torch.as_tensor(y).cuda(), torch.as_tensor(np.asarray(pos, np.int32)).cuda(),
                                torch.as_tensor(w).cuda().contiguous(), kf, fraction, seed, sh)
    return t.cpu().numpy()


def _spark_layout(t, w, D, kf, fl=True, fi=True):
    """(loss, count, gradient in Spark's layout) of one class's totals t and kernel weights w"""
    nv = D * kf
    parts = [t[2:2 + nv] - w[:nv] * np.repeat(t[3 + nv + D:3 + nv + 2 * D], kf)]
    if fl:
        parts.append(t[2 + nv:2 + nv + D])
    if fi:
        parts.append(t[2 + nv + D:3 + nv + D])
    return t[0], t[1], np.concatenate(parts)


def _oracle_w(w, D, kf, fl, fi):
    nv = D * kf
    return np.concatenate([w[:nv]] + ([w[nv:nv + D]] if fl else []) + ([w[-1:]] if fi else []))


def _check_against_the_restatement(got, x, y, w, D, kf, fl=True, fi=True, keep=None):
    keep = np.ones(x.shape[0], bool) if keep is None else keep
    for k in range(got.shape[0]):
        loss, cnt, g = _spark_layout(got[k], w[k], D, kf, fl, fi)
        want_loss, want_g = fo.sums(_oracle_w(w[k], D, kf, fl, fi), x[keep], (y[keep] == k).astype(np.float64), D, kf, fl, fi)
        assert cnt == keep.sum(), k
        assert abs(loss - want_loss) <= 1e-12 * abs(want_loss), k
        assert np.max(np.abs(g - want_g)) <= 1e-10 * max(1.0, np.max(np.abs(want_g))), k


SHAPES = [(5000, 5, 1, 4), (9001, 119, 23, 8), (4097, 41, 15, 3), (3000, 255, 3, 32), (777, 1, 2, 2), (2048, 64, 300, 8),
          (6000, 78, 9, 1)]


@pytest.mark.parametrize("n,D,K,kf", SHAPES)
def test_loss_grad_equals_the_restatement(n, D, K, kf):
    x, y, w = _problem(n, D, K, kf, 11)
    _check_against_the_restatement(_totals(x, y, range(K), w, kf), x, y, w, D, kf)


@pytest.mark.parametrize("fl,fi", [(False, True), (True, False), (False, False)])
def test_loss_grad_without_the_linear_or_intercept_block(fl, fi):
    D, kf = 30, 5
    x, y, w = _problem(5000, D, 4, kf, 12)
    if not fl:
        w[:, D * kf:D * kf + D] = 0.0
    if not fi:
        w[:, -1] = 0.0
    _check_against_the_restatement(_totals(x, y, range(4), w, kf), x, y, w, D, kf, fl, fi)


def _launch_totals(x, y, K, w, kf, fraction, seed, row_offset):
    """one launch at a global row offset that need not start a chunk, its partials chained in chunk order"""
    from b200flow import fm as bfm
    from b200flow._lib import call, ptr
    n, D = x.shape
    W = D * (kf + 1) + D + 3
    nc = (row_offset + n - 1) // 4096 - row_offset // 4096 + 1
    parts = torch.zeros((nc, K, W), dtype=torch.float64, device="cuda")
    bfm.loss_grad(torch.as_tensor(x).cuda(), torch.as_tensor(y).cuda(), torch.arange(K, dtype=torch.int32).cuda(),
                  torch.as_tensor(w).cuda(), kf, fraction, seed, row_offset, parts)
    tot = torch.zeros((K, W), dtype=torch.float64, device="cuda")
    call("b200flow_group_sums_chain", ptr(parts), nc, K, W, ptr(tot))
    return tot.cpu().numpy()


def test_mini_batch_partials_equal_the_restatement():
    D, kf, off = 20, 4, 1000
    x, y, w = _problem(9000, D, 3, kf, 13)
    for fraction, it in ((0.5, 1), (0.1, 7)):
        got = _launch_totals(x, y, 3, w, kf, fraction, 42 + it, off)
        keep = fo.batch_mask(x.shape[0], fraction, it, off)
        assert 0 < keep.sum() < x.shape[0]
        _check_against_the_restatement(got, x, y, w, D, kf, keep=keep)


@pytest.mark.parametrize("n,D,K,kf", SHAPES[1:])
def test_a_column_is_the_same_bits_in_any_launch(n, D, K, kf):
    """K columns at once, one at a time, a reversed subset, and with a column repeated so that it lands in another position
    and (for K = 300) another class block; with a mini-batch too"""
    x, y, w = _problem(n, D, K, kf, 14)
    for fraction in (1.0, 0.5):
        full = _totals(x, y, range(K), w, kf, fraction)
        for k in sorted({0, K - 1, K // 2, min(K - 1, 7), min(K - 1, 8)}):
            assert np.array_equal(_totals(x, y, [k], w[k:k + 1], kf, fraction), full[k:k + 1]), k
        sub = list(range(K - 1, -1, -3))
        assert np.array_equal(_totals(x, y, sub, w[sub], kf, fraction), full[sub])
        rep = [K - 1] * 9 + list(range(K))
        got = _totals(x, y, rep, w[rep], kf, fraction)
        assert np.array_equal(got[9:], full) and all(np.array_equal(got[i], full[K - 1]) for i in range(9))


def test_f32_features_equal_their_f64_copy_and_splits_chain_to_the_same_totals():
    from b200flow import selection, fm as bfm
    from b200flow._lib import call, ptr
    D, kf, K = 41, 6, 5
    W = D * (kf + 1) + D + 3
    x, y, w = _problem(20000, D, K, kf, 15)
    x32 = x.astype(np.float32)
    a = _totals(x32, y, range(K), w, kf)
    assert np.array_equal(a, _totals(x32.astype(np.float64), y, range(K), w, kf))
    assert np.array_equal(_totals(x32, y, range(K), w, kf, 0.5), _totals(x32.astype(np.float64), y, range(K), w, kf, 0.5))
    # two launches cut at a chunk boundary, chained, and the batched path of chunk_total
    xt, yt = torch.as_tensor(x32).cuda(), torch.as_tensor(y).cuda()
    pos, wt = torch.arange(K, dtype=torch.int32).cuda(), torch.as_tensor(w).cuda()
    parts = torch.zeros((5, K, W), dtype=torch.float64, device="cuda")
    bfm.loss_grad(xt[:8192], yt[:8192], pos, wt, kf, 1.0, 43, 0, parts[:2])
    bfm.loss_grad(xt[8192:], yt[8192:], pos, wt, kf, 1.0, 43, 8192, parts[2:])
    tot = torch.zeros((K, W), dtype=torch.float64, device="cuda")
    call("b200flow_group_sums_chain", ptr(parts), 5, K, W, ptr(tot))
    assert np.array_equal(tot.cpu().numpy(), a)
    old = selection.PARTIALS_BUDGET
    selection.PARTIALS_BUDGET = K * W * 8 * 2
    try:
        assert np.array_equal(_totals(x32, y, range(K), w, kf), a)
    finally:
        selection.PARTIALS_BUDGET = old
    # another global row offset moves the chunk boundaries: the same sums to rounding
    parts = torch.zeros((6, K, W), dtype=torch.float64, device="cuda")
    bfm.loss_grad(xt, yt, pos, wt, kf, 1.0, 43, 1000, parts)
    tot.zero_()
    call("b200flow_group_sums_chain", ptr(parts), 6, K, W, ptr(tot))
    assert np.max(np.abs(tot.cpu().numpy() - a)) <= 1e-9 * np.max(np.abs(a))


def test_canaries_around_the_kernel_outputs():
    from b200flow import fm as bfm
    from b200flow._lib import call, ptr
    D, kf, K, n = 30, 4, 11, 9000
    W = D * (kf + 1) + D + 3
    x, y, w = _problem(n, D, K, kf, 16)
    xt, yt = torch.as_tensor(x).cuda(), torch.as_tensor(y).cuda()
    pos, wt = torch.arange(K, dtype=torch.int32).cuda(), torch.as_tensor(w).cuda()
    buf = torch.full((3 * K * W + 2 * 64,), 777.0, dtype=torch.float64, device="cuda")
    bfm.loss_grad(xt, yt, pos, wt, kf, 1.0, 43, 0, buf[64:-64].view(3, K, W))
    h = buf.cpu().numpy()
    assert np.all(h[:64] == 777.0) and np.all(h[-64:] == 777.0) and not np.any(h[64:-64] == 777.0)
    raw = torch.full((n * K + 2 * 64,), 777.0, dtype=torch.float64, device="cuda")
    call("b200flow_fm_raw", ptr(xt), 1, n, D, D, kf, K, ptr(wt), ptr(raw[64:-64]))
    r = raw.cpu().numpy()
    assert np.all(r[:64] == 777.0) and np.all(r[-64:] == 777.0)
    want = np.stack([fo.raw(w[k], x, D, kf) for k in range(K)], 1)
    assert np.max(np.abs(r[64:-64].reshape(n, K) - want)) <= 1e-12 * np.max(np.abs(want))


def test_raw_is_the_fit_arithmetic_and_column_separable():
    """fm_raw shares the loss kernel's products and per-row arithmetic: a one-row loss launch gives g = sigmoid(r) - y and
    the loss of fm_raw's r, and its columns are the same bits in any launch, at any row offset and for f32 input"""
    from b200flow import fm as bfm
    D, kf, K = 119, 8, 23
    x, y, w = _problem(3000, D, K, kf, 17)
    xt = torch.as_tensor(x).cuda()
    full = bfm.fm_raw(xt, torch.as_tensor(w), kf).cpu().numpy()
    for k in (0, 9, 22):
        assert np.array_equal(bfm.fm_raw(xt, torch.as_tensor(w[k:k + 1]), kf).cpu().numpy()[:, 0], full[:, k])
    assert np.array_equal(bfm.fm_raw(xt[1234:], torch.as_tensor(w), kf).cpu().numpy(), full[1234:])
    assert np.array_equal(bfm.fm_raw(xt.float(), torch.as_tensor(w), kf).cpu().numpy(),
                          bfm.fm_raw(xt.float().double(), torch.as_tensor(w), kf).cpu().numpy())
    W = D * (kf + 1) + D + 3
    yt = torch.as_tensor(y).cuda()
    pos, wt = torch.arange(K, dtype=torch.int32).cuda(), torch.as_tensor(w).cuda()
    for i in (0, 1, 77, 2999):
        part = torch.zeros((1, K, W), dtype=torch.float64, device="cuda")
        bfm.loss_grad(xt[i:i + 1], yt[i:i + 1], pos, wt, kf, 1.0, 43, i, part)
        p = part.cpu().numpy()[0]
        r = full[i]
        lab = (np.arange(K) == y[i]).astype(np.float64)
        g = 1.0 / (1.0 + np.exp(-r)) - lab
        assert np.max(np.abs(p[:, 2 + D * kf + D] - g)) <= 1e-15, i
        assert np.max(np.abs(p[:, 0] - np.where(lab > 0, fo.log1p_exp(-r), fo.log1p_exp(r))) / p[:, 0]) <= 4e-15, i


def _spark():
    from pyspark.sql import SparkSession
    return SparkSession.builder.getOrCreate()


def test_the_pyspark_doctest_through_create_data_frame():
    from pyspark.ml.classification import FMClassifier
    from pyspark.ml.linalg import Vectors
    spark = _spark()
    df = spark.createDataFrame([(1.0, Vectors.dense(1.0)), (0.0, Vectors.dense(0.0))], ["label", "features"])
    fm = FMClassifier(factorSize=2)
    fm.setSeed(11)
    model = fm.fit(df)
    assert model.getFactorSize() == 2 and model.numFeatures == 1 and model.numClasses == 2
    d = fo.DOCTEST
    test0 = spark.createDataFrame([(Vectors.dense(-1.0),), (Vectors.dense(0.5),), (Vectors.dense(1.0),),
                                   (Vectors.dense(2.0),)], ["features"])
    out = model.transform(test0)
    prob = out._column_tensor("probability").cpu().numpy()
    assert np.max(np.abs(prob - np.array(d["probability"]))) <= 1e-12
    assert abs(model.intercept - d["intercept"]) <= 1e-12 * abs(d["intercept"])
    assert round(model.linear[0], 4) == d["linear"][0]
    r = fo.JavaRandom(11)
    assert model.factors.toArray().reshape(-1).tolist() == [r.next_gaussian() * 0.01, r.next_gaussian() * 0.01]
    assert np.round(model.factors.toArray().reshape(-1), 4).tolist() == d["factors"]
    raw = out._column_tensor("rawPrediction").cpu().numpy()
    assert np.array_equal(raw[:, 0], -raw[:, 1])
    assert out._column_tensor("prediction").cpu().numpy().tolist() == [0.0, 1.0, 1.0, 1.0]
    assert model.summary.totalIterations == len(model.summary.objectiveHistory) - 1 == 99


FIT_CASES = [("adamW", 0.0, 1.0, True, True), ("adamW", 0.05, 1.0, True, False), ("gd", 0.01, 1.0, True, True),
             ("gd", 0.0, 0.5, False, True), ("adamW", 0.0, 0.3, True, True)]


@pytest.mark.parametrize("solver,reg,fraction,fl,fi", FIT_CASES)
def test_fit_matches_the_restatement(solver, reg, fraction, fl, fi):
    """the same iterations as the numpy restatement, to the rounding of the device sums"""
    from b200flow import fm as bfm
    rng = np.random.default_rng(5)
    D, kf = 6, 3
    x = rng.normal(0.0, 1.0, (600, D))
    y = ((x[:, 0] * x[:, 1] + 0.5 * x[:, 2] + rng.normal(0, 0.5, 600)) > 0).astype(np.float64)
    step = 0.05 if solver == "adamW" else 0.5
    p = bfm.FMParams(factor_size=kf, fit_linear=fl, fit_intercept=fi, reg_param=reg, mini_batch_fraction=fraction,
                     init_std=0.1, max_iter=40, step_size=step, tol=1e-9, solver=solver, seed=3)
    fit = bfm.fm_fit_classes(torch.as_tensor(x).cuda(), torch.as_tensor(y).cuda(), [1], p)[0]
    w, hist, it = fo.fit(x, y, k=kf, fit_linear=fl, fit_intercept=fi, reg=reg, fraction=fraction, init_std=0.1,
                         max_iter=40, step=step, tol=1e-9, solver=solver, seed=3)
    V, lin, b = fo.split(w, D, kf, fl, fi)
    assert fit.iterations == it and len(fit.objective_history) == len(hist)
    assert np.max(np.abs(np.array(fit.objective_history) - hist)) <= 1e-10 * max(hist)
    for got, want in ((fit.factors, V), (fit.linear, lin), (np.array([fit.intercept]), np.array([b]))):
        assert np.max(np.abs(got - want)) <= 1e-9 * max(1.0, np.max(np.abs(want)))
    assert fl or not fit.linear.any()
    assert fi or fit.intercept == 0.0


def _frame(x, y, meta=None):
    from pyspark.sql import ColumnData, DataFrame
    from b200flow import synth
    rec, dicts = synth.make_kdd(x.shape[0], 2, seed=1, device="cuda:0")
    df = DataFrame.fromRecords(rec, synth.kdd_schema(), dicts).select("duration")
    cols = {"features": ColumnData("vector", torch.as_tensor(x).cuda(), "f64" if x.dtype == np.float64 else "f32"),
            "label": ColumnData("numeric", torch.as_tensor(np.asarray(y, np.float64)).cuda(), "f64", meta)}
    return df._with(cols=cols)


def _multiclass(n, D, K, absent, seed, dtype):
    rng = np.random.default_rng(seed)
    means = rng.normal(0.0, 1.0, (K, D))
    y = rng.integers(0, K, n)
    if absent is not None:
        y[y == absent] = (absent + 1) % K
    x = (means[y] + rng.normal(0.0, 1.0, (n, D))).astype(dtype)
    return np.ascontiguousarray(x), y.astype(np.float64)


@pytest.mark.parametrize("n,D,K,absent,dtype,extra", [(20000, 41, 23, 7, np.float32, {}),
                                                      (15000, 78, 15, None, np.float64,
                                                       {"solver": "gd", "miniBatchFraction": 0.5, "regParam": 0.01})])
def test_ovr_sub_models_equal_standalone_fits(n, D, K, absent, dtype, extra):
    from pyspark.ml.classification import FMClassifier, OneVsRest
    x, y = _multiclass(n, D, K, absent, 3, dtype)
    meta = {"ml_attr": {"type": "nominal", "vals": [str(float(k)) for k in range(K)]}}
    df = _frame(x, y, meta)
    fm = FMClassifier(factorSize=4, maxIter=12, stepSize=0.05, seed=5, tol=1e-4, **extra)
    ovr = OneVsRest(classifier=fm).fit(df)
    assert ovr.numClasses == K
    bin_meta = {"ml_attr": {"type": "nominal", "vals": ["0.0", "1.0"]}}
    for k in range(K):
        m = fm.fit(_frame(x, (y == k).astype(np.float64), bin_meta))
        sub = ovr.models[k]
        assert np.array_equal(sub.factors.toArray(), m.factors.toArray()), k
        assert np.array_equal(sub.linear.toArray(), m.linear.toArray()), k
        assert sub.intercept == m.intercept and sub.summary.objectiveHistory == m.summary.objectiveHistory, k
    if absent is not None:
        assert ovr.models[absent].intercept < 0
    out = ovr.transform(df)
    raw = out._column_tensor("rawPrediction").cpu().numpy()
    for k in range(K):
        assert np.array_equal(raw[:, k], ovr.models[k].transform(df)._column_tensor("rawPrediction").cpu().numpy()[:, 1]), k
    pred = out._column_tensor("prediction").cpu().numpy()
    assert np.array_equal(pred, raw.argmax(1).astype(np.float64)) and np.mean(pred == y) > 0.5


def _kdd_frame(n, seed):
    from b200flow import synth
    from pyspark.sql import DataFrame
    rec, dicts = synth.make_kdd(n, 5, seed=seed, device="cuda:0")
    return DataFrame.fromRecords(rec, synth.kdd_schema(), dicts)


def _stages():
    from b200flow import synth
    from pyspark.ml.feature import OneHotEncoder, StandardScaler, StringIndexer, VectorAssembler
    cats = synth.KDD_CATEGORICAL
    st = [StringIndexer(inputCol=c, outputCol=c + "_num") for c in cats + ["label"]]
    st.append(OneHotEncoder(inputCols=[c + "_num" for c in cats], outputCols=[c + "_oh" for c in cats]))
    nums = [c for c in synth.KDD_COLUMNS if c not in cats + ["label"]]
    st.append(VectorAssembler(inputCols=nums + [c + "_oh" for c in cats], outputCol="raw_features"))
    st.append(StandardScaler(inputCol="raw_features", outputCol="features", withMean=True, withStd=True))
    return st


def test_shim_pipeline_evaluators_and_cross_validation():
    from pyspark.ml import Pipeline
    from pyspark.ml.classification import FMClassifier, OneVsRest
    from pyspark.ml.evaluation import BinaryClassificationEvaluator, MulticlassClassificationEvaluator
    from pyspark.ml.tuning import CrossValidator, ParamGridBuilder, fold_frames
    from pyspark.sql import ColumnData
    df = _kdd_frame(20000, 7)
    model = Pipeline(stages=_stages() + [OneVsRest(classifier=FMClassifier(maxIter=20, stepSize=0.1), labelCol="label_num")]).fit(df)
    out = model.transform(df)
    acc = MulticlassClassificationEvaluator(labelCol="label_num", metricName="accuracy").evaluate(out)
    assert acc > 0.5
    feats = Pipeline(stages=_stages()).fit(df).transform(df).select("features", "label_num")
    cols = dict(feats._cols)
    cols["bin"] = ColumnData("numeric", (feats._column_tensor("label_num") > 0).to(torch.float64), "f64")
    two = feats._with(cols=cols)
    auc = BinaryClassificationEvaluator(labelCol="bin").evaluate(FMClassifier(labelCol="bin", maxIter=30, stepSize=0.1)
                                                                .fit(two).transform(two))
    assert 0.5 < auc <= 1.0
    fm = FMClassifier(maxIter=10, stepSize=0.1)
    ovr = OneVsRest(classifier=fm, labelCol="label_num")
    grid = ParamGridBuilder().addGrid(fm.factorSize, [2, 4]).addGrid(fm.regParam, [0.0, 0.01]).build()
    ev = MulticlassClassificationEvaluator(labelCol="label_num")
    cvm = CrossValidator(estimator=ovr, estimatorParamMaps=grid, evaluator=ev, numFolds=2, seed=9).fit(feats)
    want = [0.0] * len(grid)
    for train, val in fold_frames(feats, 2, 9):
        for i, pm in enumerate(grid):
            want[i] += ev.evaluate(ovr.fit(train, pm).transform(val))
    assert cvm.avgMetrics == [v / 2 for v in want]


def test_limits_and_refusals():
    from b200flow import _lib, fm as bfm
    from pyspark.ml.classification import FMClassifier
    from pyspark.ml.feature import IllegalArgumentException
    x = torch.zeros((10, 256), dtype=torch.float64, device="cuda")
    with pytest.raises(_lib.UnsupportedParamError):
        bfm.fm_fit_classes(x, torch.zeros(10, device="cuda"), [1], bfm.FMParams())
    with pytest.raises(_lib.UnsupportedParamError):
        bfm.fm_fit_classes(x[:, :255], torch.zeros(10, device="cuda"), [1], bfm.FMParams(factor_size=64))
    x = torch.ones((10, 3), dtype=torch.float64, device="cuda")
    y = torch.tensor([0, 1] * 5, dtype=torch.float64, device="cuda")
    with pytest.raises(ValueError, match="invalid label"):
        bfm.fm_fit_classes(x, y * 2, [1], bfm.FMParams())
    x[3, 1] = float("nan")
    with pytest.raises(ValueError, match="finite"):
        bfm.fm_fit_classes(x, y, [1], bfm.FMParams())
    assert _lib.fm_config(119, 8, 23)[:2] == (12, 2) and _lib.fm_config(255, 32, 1)[:2] == (1, 1)
    for D in (1, 64, 119, 200, 255):
        for kf in (1, 8, 32):
            _lib.fm_config(D, kf, 23)
    with pytest.raises(IllegalArgumentException):
        FMClassifier(factorSize=64).fit(_frame(np.zeros((10, 255)), [0, 1] * 5))
    m = FMClassifier(maxIter=0, seed=2).fit(_frame(np.ones((10, 3)), [0, 1] * 5))
    assert m.summary.objectiveHistory == [] and m.intercept == 0.0 and not m.linear.toArray().any()
