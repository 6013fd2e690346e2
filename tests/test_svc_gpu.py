"""LinearSVC and OneVsRest(LinearSVC) on the device: the fused DMMA hinge kernel against the numpy restatement
(tests/svc_oracle.py), column separability bit for bit (a K-column launch equals K one-column launches, for any subset and
class block), feature dtypes and chunk-order splits, fits against the QP optimum, the OneVsRest sub-models against
standalone fits bit for bit, the joint transform, canaries around every kernel output, and the pyspark shim."""
import numpy as np
import pytest
import torch

import svc_oracle as so
from test_svc import FIT_CASES, FIT_GAP

pytestmark = pytest.mark.gpu


def _problem(n, D, K, seed, n_labels=None):
    rng = np.random.default_rng(seed)
    x = rng.normal(0.0, 1.0, (n, D)) * rng.uniform(0.2, 4.0, D) + rng.normal(0, 3, D)
    y = rng.integers(0, n_labels or max(K, 2), n).astype(np.int32)
    w = rng.normal(0.0, 0.3, (K, D + 1))
    return np.ascontiguousarray(x), y, w


def _totals(x, y, pos, inv, w, row_offset=0):
    from b200flow import dist as bdist, svc as bsvc
    xt = torch.as_tensor(x).cuda()
    sh = bdist.Shards(xt.shape[0], row_offset, None, xt.device)
    t = bsvc.loss_grad_totals(xt, torch.as_tensor(y).cuda(), torch.as_tensor(np.asarray(pos, np.int32)).cuda(),
                              torch.as_tensor(inv).cuda(), torch.as_tensor(w).cuda().contiguous(), sh)
    return t.cpu().numpy()


SHAPES = [(5000, 5, 1), (9001, 119, 23), (4097, 41, 15), (3000, 255, 3), (777, 1, 2), (2048, 64, 300), (6000, 78, 9)]


@pytest.mark.parametrize("n,D,K", SHAPES)
def test_loss_grad_equals_the_restatement(n, D, K):
    x, y, w = _problem(n, D, K, 11)
    inv = so.inv_std(x)
    got = _totals(x, y, range(K), inv, w) / n
    xs = x * inv
    for k in range(K):
        loss, g = so.sums(w[k], xs, np.where(y == k, 1.0, -1.0))
        loss, g = loss / n, g / n
        assert abs(got[k, 0] - loss) <= 1e-12 * abs(loss), k
        assert np.max(np.abs(got[k, 1:] - g)) <= 1e-10 * max(1.0, np.max(np.abs(g))), k


@pytest.mark.parametrize("n,D,K", SHAPES[1:])
def test_a_column_is_the_same_bits_in_any_launch(n, D, K):
    """K columns at once, one at a time, a reversed subset, and with a column repeated so that it lands in another
    position and (for K = 300) another class block"""
    x, y, w = _problem(n, D, K, 12)
    inv = so.inv_std(x)
    full = _totals(x, y, range(K), inv, w)
    for k in sorted({0, K - 1, K // 2, min(K - 1, 7), min(K - 1, 8)}):
        assert np.array_equal(_totals(x, y, [k], inv, w[k:k + 1]), full[k:k + 1]), k
    sub = list(range(K - 1, -1, -3))
    assert np.array_equal(_totals(x, y, sub, inv, w[sub]), full[sub])
    rep = [K - 1] * 9 + list(range(K))
    got = _totals(x, y, rep, inv, w[rep])
    assert np.array_equal(got[9:], full) and all(np.array_equal(got[i], full[K - 1]) for i in range(9))


def test_f32_features_equal_their_f64_copy_and_splits_chain_to_the_same_totals():
    from b200flow import dist as bdist, selection, svc as bsvc
    from b200flow._lib import call, ptr
    x, y, w = _problem(20000, 41, 5, 13)
    x32 = x.astype(np.float32)
    inv = so.inv_std(x32.astype(np.float64))
    a = _totals(x32, y, range(5), inv, w)
    assert np.array_equal(a, _totals(x32.astype(np.float64), y, range(5), inv, w))
    assert np.array_equal(a, _totals(np.asfortranarray(x32).copy(order="C"), y, range(5), inv, w))
    # two launches cut at a chunk boundary, chained, and the batched path of chunk_total
    xt, yt = torch.as_tensor(x32).cuda(), torch.as_tensor(y).cuda()
    pos, it, wt = (torch.arange(5, dtype=torch.int32).cuda(), torch.as_tensor(inv).cuda(), torch.as_tensor(w).cuda())
    parts = torch.zeros((5, 5, 43), dtype=torch.float64, device="cuda")
    bsvc.loss_grad(xt[:8192], yt[:8192], pos, it, wt, 0, parts[:2])
    bsvc.loss_grad(xt[8192:], yt[8192:], pos, it, wt, 8192, parts[2:])
    tot = torch.zeros((5, 43), dtype=torch.float64, device="cuda")
    call("b200flow_group_sums_chain", ptr(parts), 5, 5, 43, ptr(tot))
    assert np.array_equal(tot.cpu().numpy(), a)
    old = selection.PARTIALS_BUDGET
    selection.PARTIALS_BUDGET = 5 * 43 * 8 * 2
    try:
        assert np.array_equal(_totals(x32, y, range(5), inv, w), a)
    finally:
        selection.PARTIALS_BUDGET = old
    # another global row offset moves the chunk boundaries: the same sums to rounding
    parts = torch.zeros((6, 5, 43), dtype=torch.float64, device="cuda")
    bsvc.loss_grad(xt, yt, pos, it, wt, 1000, parts)
    tot.zero_()
    call("b200flow_group_sums_chain", ptr(parts), 6, 5, 43, ptr(tot))
    assert np.max(np.abs(tot.cpu().numpy() - a)) <= 1e-9 * np.max(np.abs(a))


def test_canaries_around_the_kernel_outputs():
    from b200flow import svc as bsvc
    from b200flow._lib import call, ptr
    x, y, w = _problem(9000, 30, 11, 14)
    xt, yt = torch.as_tensor(x).cuda(), torch.as_tensor(y).cuda()
    inv = torch.as_tensor(so.inv_std(x)).cuda()
    pos = torch.arange(11, dtype=torch.int32).cuda()
    wt = torch.as_tensor(w).cuda()
    buf = torch.full((3 * 11 * 32 + 2 * 64,), 777.0, dtype=torch.float64, device="cuda")
    parts = buf[64:64 + 3 * 11 * 32].view(3, 11, 32)
    bsvc.loss_grad(xt, yt, pos, inv, wt, 0, parts)
    h = buf.cpu().numpy()
    assert np.all(h[:64] == 777.0) and np.all(h[-64:] == 777.0) and not np.any(h[64:-64] == 777.0)
    raw = torch.full((9000 * 11 + 2 * 64,), 777.0, dtype=torch.float64, device="cuda")
    call("b200flow_svc_margins", ptr(xt), 1, 9000, 30, 30, 11, ptr(wt), ptr(raw[64:64 + 9000 * 11]))
    r = raw.cpu().numpy()
    assert np.all(r[:64] == 777.0) and np.all(r[-64:] == 777.0)
    want = x @ w[:, :30].T + w[:, 30]
    assert np.max(np.abs(r[64:-64].reshape(9000, 11) - want)) <= 1e-12 * np.max(np.abs(want))


def test_margins_are_column_separable_and_position_free():
    from b200flow import svc as bsvc
    x, _, w = _problem(5000, 119, 23, 15)
    xt = torch.as_tensor(x).cuda()
    full = bsvc.svc_margins(xt, torch.as_tensor(w)).cpu().numpy()
    for k in (0, 9, 22):
        assert np.array_equal(bsvc.svc_margins(xt, torch.as_tensor(w[k:k + 1])).cpu().numpy()[:, 0], full[:, k])
    assert np.array_equal(bsvc.svc_margins(xt[1234:], torch.as_tensor(w)).cpu().numpy(), full[1234:])
    assert np.array_equal(bsvc.svc_margins(xt.float(), torch.as_tensor(w)).cpu().numpy(),
                          bsvc.svc_margins(xt.float().double(), torch.as_tensor(w)).cpu().numpy())


@pytest.mark.parametrize("gap,reg,st,fi", FIT_CASES)
def test_fit_reaches_the_qp_optimum(gap, reg, st, fi):
    """the objective at the fitted model is within FIT_GAP (tests/test_svc.py explains the figure) of the QP optimum, and
    the constant feature's coefficient stays exactly 0"""
    from b200flow import svc as bsvc
    x, y = so.blobs(200, 5, gap, 4, constant=2)
    _, fq = so.qp_solve(x, y, reg, st, fi)
    p = bsvc.SVCParams(max_iter=1000, reg_param=reg, tol=1e-12, fit_intercept=fi, standardization=st)
    fit = bsvc.svc_fit_classes(torch.as_tensor(x).cuda(), torch.as_tensor(y).cuda(), [1], p)[0]
    inv = so.inv_std(x)
    w = np.concatenate([np.where(inv > 0, fit.coef / np.where(inv > 0, inv, 1.0), 0.0), [fit.intercept]])
    f = so.objective(w, x, y, reg, st, fi)[0]
    assert -1e-9 <= (f - fq) / fq <= FIT_GAP, (f - fq) / fq
    assert fit.coef[2] == 0.0 and (fi or fit.intercept == 0.0)
    assert abs(fit.objective_history[-1] - f) <= 1e-12 * f and fit.iterations == len(fit.objective_history) - 1


def _frame(x, y, meta=None):
    from pyspark.sql import ColumnData, DataFrame
    from b200flow import synth
    rec, dicts = synth.make_kdd(x.shape[0], 2, seed=1, device="cuda:0")
    df = DataFrame.fromRecords(rec, synth.kdd_schema(), dicts).select("duration")
    cols = {"features": ColumnData("vector", torch.as_tensor(x).cuda(), "f64" if x.dtype == np.float64 else "f32"),
            "label": ColumnData("numeric", torch.as_tensor(np.asarray(y, np.float64)).cuda(), "f64", meta)}
    return df._with(cols=cols)


def test_predictions_raw_and_threshold():
    from pyspark.ml.classification import LinearSVC
    x, y = so.blobs(3000, 7, 0.8, 9)
    df = _frame(x, y)
    m = LinearSVC(regParam=0.01, maxIter=50).fit(df)
    assert m.numClasses == 2 and m.numFeatures == 7 and len(m.coefficients) == 7
    out = m.transform(df)
    raw = out._column_tensor("rawPrediction").cpu().numpy()
    mg = x @ m.coefficients.toArray() + m.intercept
    assert np.array_equal(raw[:, 0], -raw[:, 1]) and np.max(np.abs(raw[:, 1] - mg)) <= 1e-12 * np.max(np.abs(mg))
    assert np.array_equal(out._column_tensor("prediction").cpu().numpy(), (raw[:, 1] > 0.0).astype(np.float64))
    assert "probability" not in out._cols
    thr = float(np.median(raw[:, 1]))
    out2 = m.copy({"threshold": thr}).transform(df)
    assert np.array_equal(out2._column_tensor("prediction").cpu().numpy(), (raw[:, 1] > thr).astype(np.float64))
    assert m.summary.totalIterations == len(m.summary.objectiveHistory) - 1 <= 50


def _multiclass(n, D, K, absent, seed, dtype):
    rng = np.random.default_rng(seed)
    means = rng.normal(0.0, 2.0, (K, D))
    y = rng.integers(0, K, n)
    if absent is not None:
        y[y == absent] = (absent + 1) % K
    x = (means[y] + rng.normal(0.0, 1.0, (n, D))).astype(dtype)
    x[:, 3] = 1.5                                         # a constant column
    return np.ascontiguousarray(x), y.astype(np.float64)


@pytest.mark.parametrize("n,D,K,absent,dtype", [(20000, 41, 23, 7, np.float32), (15000, 78, 15, None, np.float64)])
def test_ovr_sub_models_equal_standalone_fits(n, D, K, absent, dtype):
    from pyspark.ml.classification import LinearSVC, OneVsRest
    x, y = _multiclass(n, D, K, absent, 3, dtype)
    meta = {"ml_attr": {"type": "nominal", "vals": [str(float(k)) for k in range(K)]}}
    df = _frame(x, y, meta)
    svc = LinearSVC(regParam=0.01, maxIter=12)
    ovr = OneVsRest(classifier=svc).fit(df)
    assert ovr.numClasses == K
    bin_meta = {"ml_attr": {"type": "nominal", "vals": ["0.0", "1.0"]}}
    for k in range(K):
        m = svc.fit(_frame(x, (y == k).astype(np.float64), bin_meta))
        sub = ovr.models[k]
        assert np.array_equal(sub.coefficients.toArray(), m.coefficients.toArray()), k
        assert sub.intercept == m.intercept and sub.summary.totalIterations == m.summary.totalIterations, k
        assert sub.summary.objectiveHistory == m.summary.objectiveHistory, k
        assert sub.coefficients[3] == 0.0
    if absent is not None:
        assert ovr.models[absent].intercept < 0
    out = ovr.transform(df)
    raw = out._column_tensor("rawPrediction").cpu().numpy()
    for k in range(K):
        assert np.array_equal(raw[:, k], ovr.models[k].transform(df)._column_tensor("rawPrediction").cpu().numpy()[:, 1]), k
    pred = out._column_tensor("prediction").cpu().numpy()
    assert np.array_equal(pred, raw.argmax(1).astype(np.float64)) and np.mean(pred == y) > 0.8


def _kdd_frame(n, seed):
    from b200flow import synth
    from pyspark.sql import DataFrame
    rec, dicts = synth.make_kdd(n, 5, seed=seed, device="cuda:0")
    return DataFrame.fromRecords(rec, synth.kdd_schema(), dicts)


def _stages(scale=True):
    from b200flow import synth
    from pyspark.ml.feature import StandardScaler, StringIndexer, VectorAssembler
    cats = synth.KDD_CATEGORICAL
    st = [StringIndexer(inputCol=c, outputCol=c + "_num") for c in cats + ["label"]]
    nums = [c for c in synth.KDD_COLUMNS if c not in cats + ["label"]]
    st.append(VectorAssembler(inputCols=nums + [c + "_num" for c in cats], outputCol="raw_features" if scale else "features"))
    if scale:
        st.append(StandardScaler(inputCol="raw_features", outputCol="features", withMean=True, withStd=True))
    return st


def test_shim_pipeline_evaluators_and_cross_validation():
    from pyspark.ml import Pipeline
    from pyspark.ml.classification import LinearSVC, OneVsRest
    from pyspark.ml.evaluation import BinaryClassificationEvaluator, MulticlassClassificationEvaluator
    from pyspark.ml.tuning import CrossValidator, ParamGridBuilder, fold_frames
    from pyspark.sql import ColumnData
    df = _kdd_frame(20000, 7)
    # a lazy VectorAssembler output straight into OneVsRest(LinearSVC)
    model = Pipeline(stages=_stages(scale=False) + [OneVsRest(classifier=LinearSVC(maxIter=20), labelCol="label_num")]).fit(df)
    out = model.transform(df)
    acc = MulticlassClassificationEvaluator(labelCol="label_num", metricName="accuracy").evaluate(out)
    assert acc > 0.5
    feats = Pipeline(stages=_stages()).fit(df).transform(df).select("features", "label_num")
    cols = dict(feats._cols)
    cols["bin"] = ColumnData("numeric", (feats._column_tensor("label_num") > 0).to(torch.float64), "f64")
    two = feats._with(cols=cols)
    auc = BinaryClassificationEvaluator(labelCol="bin").evaluate(LinearSVC(labelCol="bin", maxIter=30).fit(two).transform(two))
    assert 0.5 < auc <= 1.0
    svc = LinearSVC(maxIter=10)
    ovr = OneVsRest(classifier=svc, labelCol="label_num")
    grid = ParamGridBuilder().addGrid(svc.regParam, [0.0, 0.1]).build()
    ev = MulticlassClassificationEvaluator(labelCol="label_num")
    cvm = CrossValidator(estimator=ovr, estimatorParamMaps=grid, evaluator=ev, numFolds=2, seed=9).fit(feats)
    want = [0.0] * 2
    for train, val in fold_frames(feats, 2, 9):
        for i, pm in enumerate(grid):
            want[i] += ev.evaluate(ovr.fit(train, pm).transform(val))
    assert cvm.avgMetrics == [v / 2 for v in want]


def test_limits_and_refusals():
    from b200flow import _lib, svc as bsvc
    x = torch.zeros((10, 256), dtype=torch.float64, device="cuda")
    with pytest.raises(_lib.UnsupportedParamError):
        bsvc.svc_fit_classes(x, torch.zeros(10, device="cuda"), [1], bsvc.SVCParams())
    x = torch.ones((10, 3), dtype=torch.float64, device="cuda")
    y = torch.tensor([0, 1] * 5, dtype=torch.float64, device="cuda")
    with pytest.raises(ValueError, match="invalid label"):
        bsvc.svc_fit_classes(x, y * 2, [1], bsvc.SVCParams())
    x[3, 1] = float("nan")
    with pytest.raises(ValueError, match="finite"):
        bsvc.svc_fit_classes(x, y, [1], bsvc.SVCParams())
    assert _lib.svc_config(255, 1)[:2] == (8, 1) and _lib.svc_config(119, 23)[:2] == (24, 1)
    assert _lib.svc_config(64, 300)[1] == 2
