"""KMeans and the silhouette on the GPU, bit for bit against the numpy restatement (tests/kmeans_oracle.py): the assign
kernel (KDD-shaped D = 41 and 119, k up to 300, duplicate centers), the grouped sums, the Philox draws, full fits with both
init modes (fewer distinct candidates than k, an empty cluster), the silhouette, and the shim pipeline
StringIndexer -> OneHotEncoder -> VectorAssembler -> StandardScaler -> KMeans -> ClusteringEvaluator with a CrossValidator
over k (DESIGN.md §5c)."""
import numpy as np
import pytest
import torch

import kmeans_oracle as ko

pytestmark = pytest.mark.gpu


def _kdd_like(n, D, seed):
    """flow-shaped features: heavy-tailed counts, rates in [0, 1], one-hot blocks, many repeated rows."""
    rng = np.random.default_rng(seed)
    n_num = min(D, 38)
    base = np.empty((n // 4 + 1, D))
    base[:, :n_num // 2] = np.floor(np.exp(rng.normal(2.0, 3.0, (base.shape[0], n_num // 2))))
    base[:, n_num // 2:n_num] = rng.integers(0, 101, (base.shape[0], n_num - n_num // 2)) / 100.0
    if D > n_num:
        base[:, n_num:] = 0.0
        hot = rng.integers(n_num, D, base.shape[0])
        base[np.arange(base.shape[0]), hot] = 1.0
    x = base[rng.integers(0, base.shape[0], n)]
    x[::7] = -x[::7] * 0.5
    return np.ascontiguousarray(x)


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.mark.parametrize("D", [41, 119])
@pytest.mark.parametrize("k", [2, 23, 100, 300])
def test_assign_equals_the_oracle(D, k):
    from b200flow import kmeans as bk
    x = _kdd_like(20011, D, D + k)
    rng = np.random.default_rng(k)
    centers = x[rng.choice(x.shape[0], k, replace=False)].copy()
    centers[k - 1] = centers[0]                            # a duplicate center: ties go to the lower index
    if k > 2:
        centers[1] = centers[k // 2]
    cl, d = bk.assign(_dev(x), _dev(centers))
    want_cl, want_d = ko.assign(x, centers)
    assert np.array_equal(cl.cpu().numpy(), want_cl)
    assert np.array_equal(d.cpu().numpy().view(np.int64), want_d.view(np.int64))
    assert (cl.cpu().numpy() != k - 1).all()


@pytest.mark.parametrize("G,W,n", [(1, 1, 10000), (23, 41, 30001), (300, 3, 9000), (4096, 2, 5000)])
def test_grouped_sum_equals_the_oracle(G, W, n):
    from b200flow import kmeans as bk
    rng = np.random.default_rng(G + W)
    v = rng.normal(size=(n, W)) * 10.0 ** rng.integers(-6, 6, (n, 1))
    v[::11] = -0.0
    ids = rng.integers(0, G, n).astype(np.int32) if G > 1 else None
    sh = bk._Shards(n, 0, None, "cuda")
    tot, cnt = bk.grouped_sum(_dev(v), _dev(ids) if ids is not None else None, G, sh)
    want, wcnt = ko.group_sums(v, ids, G)
    assert np.array_equal(tot.cpu().numpy().view(np.int64), want.view(np.int64))
    assert np.array_equal(cnt.cpu().numpy(), wcnt)


def test_device_philox_draws_equal_the_host():
    from b200flow import _lib, kmeans as bk
    n, off, seed = 50000, 2 ** 32 - 20000, 2019
    keys = torch.empty(n, dtype=torch.int64, device="cuda")
    _lib.call("b200flow_kmeans_row_keys", seed, off, n, _lib.ptr(keys))
    rows = np.arange(off, off + n, dtype=np.uint64)
    assert np.array_equal(keys.cpu().numpy(), ko.row_keys(seed, rows))
    assert [bk.row_key(seed, off + i) for i in (0, 1, 19999, 20000, n - 1)] == keys.cpu().numpy()[[0, 1, 19999, 20000, n - 1]].tolist()
    cost = np.random.default_rng(1).random(n) * 3.0
    flag = torch.empty(n, dtype=torch.uint8, device="cuda")
    _lib.call("b200flow_kmeans_select", seed, 0, n, 2, _lib.ptr(_dev(cost)), 23, 1000.0, _lib.ptr(flag))
    assert np.array_equal(flag.cpu().numpy().astype(bool), ko.select(seed, 2, cost, 23, 1000.0))


def _blobs(n, D, k, seed):
    rng = np.random.default_rng(seed)
    means = rng.normal(0.0, 3.0, (k, D))
    return np.ascontiguousarray(means[rng.integers(0, k, n)] + rng.normal(0.0, 1.0, (n, D)))


def _same_fit(res, want):
    assert np.array_equal(res.centers.cpu().numpy().view(np.int64), want["centers"].view(np.int64))
    assert res.num_iter == want["num_iter"]
    assert float(res.training_cost).hex() == float(want["training_cost"]).hex()
    assert np.array_equal(res.cluster_sizes, want["cluster_sizes"])


@pytest.mark.parametrize("init", ["k-means||", "random"])
@pytest.mark.parametrize("k,D,tol", [(5, 41, 1e-4), (23, 41, 0.0), (23, 119, 1e-4)])
def test_fit_equals_the_oracle(init, k, D, tol):
    from b200flow import kmeans as bk
    x = _blobs(30000, D, 8, k + D) if D == 41 else _kdd_like(30000, D, 5)
    res = bk.kmeans_fit(_dev(x), k, init=init, max_iter=12, tol=tol, seed=7)
    _same_fit(res, ko.fit(x, k, init=init, max_iter=12, tol=tol, seed=7))


def test_fit_with_fewer_distinct_candidates():
    from b200flow import kmeans as bk
    pts = np.array([[0.0, 0.0], [1.0, 0.0], [0.0, 5.0]])
    x = np.repeat(pts, 3000, axis=0)
    for init in ("k-means||", "random"):
        res = bk.kmeans_fit(_dev(x), 50, init=init, seed=3)
        want = ko.fit(x, 50, init=init, seed=3)
        _same_fit(res, want)
        assert res.centers.shape[0] == 3 and sorted(res.cluster_sizes.tolist()) == [3000, 3000, 3000]


def test_lloyd_keeps_an_empty_cluster():
    from b200flow import kmeans as bk
    x = _blobs(20000, 5, 3, 1)
    init = np.vstack([x[:3], np.full((1, 5), 1e6), x[3:4]])     # center 3 never wins a row
    sh = bk._Shards(x.shape[0], 0, None, "cuda")
    res = bk.lloyd(_dev(x), init, 10, 1e-4, sh)
    want = ko.lloyd(x, init, 10, 1e-4)
    _same_fit(res, want)
    assert res.cluster_sizes[3] == 0 and np.array_equal(res.centers.cpu().numpy()[3], init[3])


@pytest.mark.parametrize("k", [2, 23])
def test_silhouette_equals_the_oracle(k):
    from b200flow import kmeans as bk
    x = _blobs(20000, 41, k, k)
    cl = np.random.default_rng(k).integers(0, k + 2, x.shape[0]).astype(np.int32)
    cl[cl == k] = k + 1                                    # cluster k is absent
    cl[5] = k + 3                                          # a one-member cluster
    got = bk.silhouette(_dev(x), _dev(cl))
    assert got.hex() == float(ko.silhouette(x, cl)).hex()
    with pytest.raises(ValueError):
        bk.silhouette(_dev(x), torch.zeros(x.shape[0], dtype=torch.int32, device="cuda"))


def _kdd_frame(n, seed):
    from b200flow import synth
    from pyspark.sql import DataFrame
    rec, dicts = synth.make_kdd(n, 5, seed=seed, device="cuda:0")
    return DataFrame.fromRecords(rec, synth.kdd_schema(), dicts)


def _feature_pipeline():
    from b200flow import synth
    from pyspark.ml.feature import OneHotEncoder, StandardScaler, StringIndexer, VectorAssembler
    cats = synth.KDD_CATEGORICAL
    stages = [StringIndexer(inputCol=c, outputCol=c + "_num") for c in cats]
    stages.append(OneHotEncoder(inputCols=[c + "_num" for c in cats], outputCols=[c + "_oh" for c in cats]))
    nums = [c for c in synth.KDD_COLUMNS if c not in cats + ["label"]]
    stages.append(VectorAssembler(inputCols=nums + [c + "_oh" for c in cats], outputCol="raw_features"))
    stages.append(StandardScaler(inputCol="raw_features", outputCol="features", withMean=True, withStd=True))
    return stages


def test_shim_pipeline_kmeans_and_silhouette():
    from pyspark.ml import Pipeline
    from pyspark.ml.clustering import KMeans
    from pyspark.ml.evaluation import ClusteringEvaluator
    df = _kdd_frame(40000, 11)
    km = KMeans(k=6, seed=1, maxIter=10)
    model = Pipeline(stages=_feature_pipeline() + [km]).fit(df)
    out = model.transform(df)
    x = out._cols["features"].data.to(torch.float64).cpu().numpy()
    want = ko.fit(x, 6, max_iter=10, seed=1)
    kmm = model.stages[-1]
    assert np.array_equal(np.array(kmm.clusterCenters()), want["centers"])
    s = kmm.summary
    assert s.k == 6 and s.numIter == want["num_iter"] and s.trainingCost == want["training_cost"]
    assert s.clusterSizes == want["cluster_sizes"].tolist() and kmm.hasSummary
    pred = out._column_tensor("prediction").cpu().numpy()
    assert pred.dtype == np.int32 and np.array_equal(pred, ko.assign(x, want["centers"])[0])
    assert np.array_equal(s.cluster._column_tensor("prediction").cpu().numpy(), pred)
    sil = ClusteringEvaluator().evaluate(out)
    assert sil == ko.silhouette(x, pred)


def test_cross_validator_over_k_runs_the_generic_loop():
    from pyspark.ml import Pipeline
    from pyspark.ml.clustering import KMeans
    from pyspark.ml.evaluation import ClusteringEvaluator
    from pyspark.ml.tuning import CrossValidator, ParamGridBuilder, TrainValidationSplit, fold_frames
    df = _kdd_frame(20000, 4)
    feats = Pipeline(stages=_feature_pipeline()).fit(df).transform(df).select("features")
    km = KMeans(seed=5, maxIter=5)
    grid = ParamGridBuilder().addGrid(km.k, [2, 4, 7]).build()
    ev = ClusteringEvaluator()
    cvm = CrossValidator(estimator=km, estimatorParamMaps=grid, evaluator=ev, numFolds=2, seed=9).fit(feats)
    want = [0.0] * 3
    for train, val in fold_frames(feats, 2, 9):
        for i, m in enumerate(grid):
            want[i] += ev.evaluate(km.fit(train, m).transform(val))
    assert cvm.avgMetrics == [w / 2 for w in want]
    assert cvm.bestModel.summary.k == grid[int(np.argmax(want))][km.k]
    tvs = TrainValidationSplit(estimator=km, estimatorParamMaps=grid, evaluator=ev, seed=3).fit(feats)
    assert len(tvs.validationMetrics) == 3 and all(-1.0 <= v <= 1.0 for v in tvs.validationMetrics)
