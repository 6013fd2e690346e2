"""MultilayerPerceptronClassifier on the device: the fused DMMA loss/gradient and forward kernels against the numpy
restatement (tests/mlp_oracle.py) within stated tolerances (exp and log are CUDA's, not libm's), bit-identity across
calls, feature dtypes and chunk-order splits, the optimisers, the limits, and the pyspark shim."""
import numpy as np
import pytest
import torch

import mlp_oracle as mo

pytestmark = pytest.mark.gpu


def _problem(layers, n, seed):
    rng = np.random.default_rng(seed)
    x = rng.normal(0.0, 1.0, (n, layers[0]))
    y = rng.integers(0, layers[-1], n).astype(np.int32)
    w = mo.init_weights(layers, seed) if sum(layers) < 200 else rng.uniform(-1, 1, sum((a + 1) * b for a, b in zip(layers[:-1], layers[1:]))) / np.sqrt(layers[0])
    return x, y, w


def _device_loss_grad(x, y, layers, w, row_offset=0):
    from b200flow import dist as bdist, mlp as bm
    xt, yt = torch.as_tensor(x).cuda(), torch.as_tensor(y).cuda()
    sh = bdist.Shards(xt.shape[0], row_offset, None, xt.device)
    t = bm.loss_grad_sums(xt, yt, layers, torch.as_tensor(w).cuda(), sh).cpu().numpy()
    return t


@pytest.mark.parametrize("layers,n", [([41, 64, 32, 5], 5000), ([41, 64, 32, 23], 4096), ([119, 64, 32, 5], 9001),
                                      ([78, 64, 32, 15], 3000), ([78, 100, 50, 15], 8192), ([41, 7, 3], 4097),
                                      ([1, 1, 2], 777), ([256, 8, 2], 2048)])
def test_loss_grad_equals_the_restatement(layers, n):
    x, y, w = _problem(layers, n, 11)
    got = _device_loss_grad(x, y, layers, w) / n
    loss, g = mo.loss_grad(w, layers, x, y)
    assert abs(got[0] - loss) <= 1e-12 * abs(loss)
    assert np.max(np.abs(got[1:] - g)) <= 1e-10 * max(1.0, np.max(np.abs(g)))


def test_loss_grad_is_the_same_bits_across_calls_dtypes_and_splits():
    from b200flow import dist as bdist
    layers, n = [41, 64, 32, 5], 3 * 4096 + 1001
    x, y, w = _problem(layers, n, 5)
    x32 = x.astype(np.float32)
    a = _device_loss_grad(x32.astype(np.float64), y, layers, w)
    assert np.array_equal(a, _device_loss_grad(x32.astype(np.float64), y, layers, w))
    assert np.array_equal(a.view(np.uint64), _device_loss_grad(x32, y, layers, w).view(np.uint64))
    # two calls split at row s (not a chunk boundary), chained as the ranks do: the first call also takes the rows of the
    # straddling chunk that lie past s
    s = 4096 + 1234
    t0 = 4096
    xt, yt, wt = torch.as_tensor(x32).cuda(), torch.as_tensor(y).cuda(), torch.as_tensor(w).cuda()
    la = np.array(layers, np.int32)
    P = w.size
    from b200flow._lib import call, ptr
    parts = torch.empty((4, P + 1), dtype=torch.float64, device="cuda")
    call("b200flow_mlp_loss_grad", ptr(xt[:t0 + 4096].contiguous()), 0, t0 + 4096, 41, ptr(yt[:t0 + 4096].contiguous()),
         la.ctypes.data, len(la), ptr(wt), 0, ptr(parts[:2]))
    rest = 2 * 4096
    call("b200flow_mlp_loss_grad", ptr(xt[rest:].contiguous()), 0, n - rest, 41, ptr(yt[rest:].contiguous()), la.ctypes.data,
         len(la), ptr(wt), rest, ptr(parts[2:]))
    sh = bdist.Shards(n, 0, None, xt.device)
    tot = bdist.chunk_chain(parts, 4, 1, P + 1, sh).reshape(-1).cpu().numpy()
    assert s > t0 and np.array_equal(tot.view(np.uint64), a.view(np.uint64))
    # a launch that starts at row s, inside chunk 1: its partials of the later chunks are the same bits
    p2 = torch.empty((3, P + 1), dtype=torch.float64, device="cuda")
    call("b200flow_mlp_loss_grad", ptr(xt[s:].contiguous()), 0, n - s, 41, ptr(yt[s:].contiguous()), la.ctypes.data, len(la),
         ptr(wt), s, ptr(p2))
    assert torch.equal(p2[1:], parts[2:])


@pytest.mark.parametrize("layers", [[41, 64, 32, 5], [78, 100, 50, 15], [41, 7, 3]])
def test_forward_equals_the_restatement(layers):
    from b200flow import mlp as bm
    x, _, w = _problem(layers, 1001, 3)
    got = bm.mlp_raw(torch.as_tensor(w).cuda(), layers, torch.as_tensor(x).cuda()).cpu().numpy()
    want = mo.raw(w, layers, x)
    assert np.max(np.abs(got - want)) <= 1e-12 * max(1.0, np.max(np.abs(want)))
    got32 = bm.mlp_raw(torch.as_tensor(w).cuda(), layers, torch.as_tensor(x.astype(np.float32)).cuda()).cpu().numpy()
    got64 = bm.mlp_raw(torch.as_tensor(w).cuda(), layers, torch.as_tensor(x.astype(np.float32).astype(np.float64)).cuda())
    assert np.array_equal(got32, got64.cpu().numpy())


def test_first_lbfgs_iterates_equal_the_restatement_driven_optimiser():
    from b200flow import linear, mlp as bm
    layers, n = [41, 16, 5], 6000
    x, y, _ = _problem(layers, n, 8)
    fit = bm.mlp_fit(torch.as_tensor(x).cuda(), torch.as_tensor(y).cuda(), layers, max_iter=3, seed=4)

    def fun(v):
        loss, g = mo.loss_grad(v.numpy(), layers, x, y)
        return torch.tensor(loss, dtype=torch.float64), torch.from_numpy(g)

    v, hist, it = linear.lbfgs(fun, torch.from_numpy(mo.init_weights(layers, 4)), 3, 1e-6)
    assert fit.iterations == it == 3
    assert np.max(np.abs(fit.weights.cpu().numpy() - v.numpy())) <= 1e-9 * max(1.0, float(v.abs().max()))
    assert np.allclose(fit.objective_history, hist, rtol=1e-9, atol=0)


def _blobs(n, seed):
    rng = np.random.default_rng(seed)
    centers = np.array([[4.0, 0.0, 0.0], [0.0, 4.0, 0.0], [0.0, 0.0, 4.0]])
    y = rng.integers(0, 3, n)
    return centers[y] + rng.normal(0.0, 0.5, (n, 3)), y


@pytest.mark.parametrize("solver,kw", [("l-bfgs", {}), ("gd", dict(step_size=2.0, max_iter=200))])
def test_fit_separates_blobs(solver, kw):
    from b200flow import mlp as bm
    x, y = _blobs(20000, 2)
    xt = torch.as_tensor(x).cuda()
    fit = bm.mlp_fit(xt, torch.as_tensor(y).cuda(), [3, 8, 3], solver=solver, seed=1, **kw)
    h = fit.objective_history
    assert all(b <= a for a, b in zip(h, h[1:])) and fit.iterations >= 1
    pred = bm.mlp_raw(fit.weights, [3, 8, 3], xt).argmax(1).cpu().numpy()
    assert (pred == y).mean() >= 0.99


def test_limits_and_bad_inputs_raise():
    from b200flow import _lib, mlp as bm
    x = torch.zeros((10, 119), dtype=torch.float64, device="cuda")
    y = torch.zeros(10, dtype=torch.int32, device="cuda")
    with pytest.raises(_lib.UnsupportedParamError):
        bm.mlp_fit(x, y, [119, 256, 5])
    with pytest.raises(_lib.UnsupportedParamError):
        bm.mlp_raw(torch.zeros(1, device="cuda"), [2] + [4] * 9 + [2], torch.zeros((1, 2), device="cuda"))
    with pytest.raises(ValueError):
        bm.mlp_fit(x, y, [118, 4, 5])
    with pytest.raises(ValueError):
        bm.mlp_fit(x, y + 5, [119, 4, 5])
    with pytest.raises(ValueError):
        bm.mlp_fit(x, y, [119, 4, 5], initial_weights=np.zeros(3))


def _kdd_frame(n, seed):
    from b200flow import synth
    from pyspark.sql import DataFrame
    rec, dicts = synth.make_kdd(n, 5, seed=seed, device="cuda:0")
    return DataFrame.fromRecords(rec, synth.kdd_schema(), dicts)


def _stages():
    from b200flow import synth
    from pyspark.ml.feature import StandardScaler, StringIndexer, VectorAssembler
    cats = synth.KDD_CATEGORICAL
    st = [StringIndexer(inputCol=c, outputCol=c + "_num") for c in cats + ["label"]]
    nums = [c for c in synth.KDD_COLUMNS if c not in cats + ["label"]]
    st.append(VectorAssembler(inputCols=nums + [c + "_num" for c in cats], outputCol="raw_features"))
    st.append(StandardScaler(inputCol="raw_features", outputCol="features", withMean=True, withStd=True))
    return st


def test_shim_pipeline_and_evaluators():
    from pyspark.ml import Pipeline
    from pyspark.ml.classification import MultilayerPerceptronClassifier
    from pyspark.ml.evaluation import BinaryClassificationEvaluator, MulticlassClassificationEvaluator
    from pyspark.ml.feature import IllegalArgumentException
    df = _kdd_frame(30000, 7)
    mlp = MultilayerPerceptronClassifier(layers=[41, 16, 5], labelCol="label_num", maxIter=30, seed=3)
    model = Pipeline(stages=_stages() + [mlp]).fit(df)
    out = model.transform(df)
    m = model.stages[-1]
    assert m.numFeatures == 41 and m.numClasses == 5 and m.layers == m.getLayers() == [41, 16, 5]
    assert len(m.weights) == 41 * 16 + 16 + 17 * 5 and m.summary.totalIterations <= 30
    x = out._cols["features"].data.to(torch.float64).cpu().numpy()
    raw = out._column_tensor("rawPrediction").cpu().numpy()
    assert np.max(np.abs(raw - mo.raw(m.weights.toArray(), [41, 16, 5], x))) <= 1e-10
    prob = out._column_tensor("probability").cpu().numpy()
    assert np.allclose(prob.sum(1), 1.0) and np.array_equal(out._column_tensor("prediction").cpu().numpy(), raw.argmax(1))
    acc = MulticlassClassificationEvaluator(labelCol="label_num", metricName="accuracy").evaluate(out)
    ll = MulticlassClassificationEvaluator(labelCol="label_num", metricName="logLoss").evaluate(out)
    lab = out._column_tensor("label_num").cpu().numpy().astype(np.int64)
    assert acc > 0.5 and abs(ll - np.mean(-np.log(np.clip(prob[np.arange(len(lab)), lab], 1e-15, 1 - 1e-15)))) <= 1e-9
    with pytest.raises(IllegalArgumentException):
        MultilayerPerceptronClassifier(layers=[40, 16, 5], labelCol="label_num").fit(out.select("features", "label_num"))
    with pytest.raises(IllegalArgumentException):
        MultilayerPerceptronClassifier(layers=[41, 16, 3], labelCol="label_num").fit(out.select("features", "label_num"))
    # two classes: the binary evaluator reads rawPrediction[1]
    from pyspark.sql import ColumnData
    two = out.select("features", "label_num")
    cols = dict(two._cols)
    cols["bin"] = ColumnData("numeric", (two._column_tensor("label_num") > 0).to(torch.float64), "f64")
    two = two._with(cols=cols)
    bm2 = MultilayerPerceptronClassifier(layers=[41, 8, 2], labelCol="bin", maxIter=20, seed=1).fit(two)
    auc = BinaryClassificationEvaluator(labelCol="bin").evaluate(bm2.transform(two))
    assert 0.5 < auc <= 1.0


def test_cross_validator_over_max_iter_and_layers():
    from pyspark.ml import Pipeline
    from pyspark.ml.classification import MultilayerPerceptronClassifier
    from pyspark.ml.evaluation import MulticlassClassificationEvaluator
    from pyspark.ml.tuning import CrossValidator, ParamGridBuilder, fold_frames
    df = _kdd_frame(12000, 4)
    feats = Pipeline(stages=_stages()).fit(df).transform(df).select("features", "label_num")
    mlp = MultilayerPerceptronClassifier(labelCol="label_num", seed=5)
    grid = ParamGridBuilder().addGrid(mlp.maxIter, [3, 10]).addGrid(mlp.layers, [[41, 8, 5], [41, 16, 8, 5]]).build()
    ev = MulticlassClassificationEvaluator(labelCol="label_num")
    cvm = CrossValidator(estimator=mlp, estimatorParamMaps=grid, evaluator=ev, numFolds=2, seed=9).fit(feats)
    want = [0.0] * 4
    for train, val in fold_frames(feats, 2, 9):
        for i, pm in enumerate(grid):
            want[i] += ev.evaluate(mlp.fit(train, pm).transform(val))
    assert cvm.avgMetrics == [v / 2 for v in want]
