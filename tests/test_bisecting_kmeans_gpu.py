"""BisectingKMeans on the GPU, bit for bit against the numpy restatement (tests/bisecting_kmeans_oracle.py): the split-assign
kernel (D = 41 and 119, 1 to 1024 dividing slots, duplicate children, absent children, non-dividing rows, dist_prev), the
tree-walk kernel (a random tree, one leaf, a deep chain, ties), full fits on blobs and KDD-shaped data with many repeated
rows, Spark's doctest through createDataFrame, and the shim pipeline StringIndexer -> OneHotEncoder -> VectorAssembler ->
StandardScaler -> BisectingKMeans -> ClusteringEvaluator with a CrossValidator over k (DESIGN.md §5t)."""
import numpy as np
import pytest
import torch

import bisecting_kmeans_oracle as bo
from test_kmeans_gpu import _feature_pipeline, _kdd_frame, _kdd_like

pytestmark = pytest.mark.gpu


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.int64)


def _blobs(n, D, k, seed):
    rng = np.random.default_rng(seed)
    means = rng.normal(0.0, 3.0, (k, D))
    return np.ascontiguousarray(means[rng.integers(0, k, n)] + rng.normal(0.0, 1.0, (n, D)))


@pytest.mark.parametrize("D", [41, 119])
@pytest.mark.parametrize("m", [1, 7, 300, 1024])
def test_assign_equals_the_oracle(D, m):
    from b200flow import bisecting_kmeans as bb
    rng = np.random.default_rng(D * m)
    n = 20011
    x = _kdd_like(n, D, m)
    num_nodes = m + 37
    slot_of_node = np.full(num_nodes, -1, np.int32)
    slot_of_node[rng.permutation(num_nodes)[:m]] = np.arange(m, dtype=np.int32)
    node = rng.integers(0, num_nodes, n).astype(np.int32)
    centers = x[rng.integers(0, n, 2 * m)] + rng.normal(0.0, 0.1, (2 * m, D))
    dup = rng.random(m) < 0.3                             # equal children: every row of the slot ties and goes left
    centers[1::2][dup] = centers[0::2][dup]
    present = np.ones(2 * m, np.uint8)
    gone = rng.random(2 * m) < 0.2
    present[gone] = 0
    present[:2][:] = (1, 0) if m > 1 else (1, 1)
    if m > 2:
        present[2:4] = 0                                   # slot 1 has no child at all: its rows get -1
    slot = {u: int(slot_of_node[u]) for u in range(num_nodes) if slot_of_node[u] >= 0}
    s_row = slot_of_node[node]
    side = rng.integers(0, 2, n)
    prev = np.where(s_row >= 0, 2 * s_row + side, -1).astype(np.int32)
    prev[rng.random(n) < 0.1] = -1
    d_args = (_dev(x), _dev(node), _dev(slot_of_node), _dev(centers), _dev(present))
    child, dp = bb.bkm_assign(*d_args)
    want, _ = bo.pair_assign(x, node, slot, centers, present.astype(bool))
    assert dp is None and np.array_equal(child.cpu().numpy(), want)
    child, dp = bb.bkm_assign(*d_args, prev=_dev(prev))
    want, want_dp = bo.pair_assign(x, node, slot, centers, present.astype(bool), prev=prev)
    assert np.array_equal(child.cpu().numpy(), want)
    assert np.array_equal(_bits(dp.cpu().numpy()), _bits(want_dp))
    got = child.cpu().numpy()
    assert (got[s_row < 0] == -1).all()
    for s in np.nonzero(dup)[0]:
        rows = s_row == s
        if present[2 * s] and present[2 * s + 1]:
            assert (got[rows] == 2 * s).all()


def _tree_arrays(clusters):
    from b200flow import bisecting_kmeans as bb
    return bb.build_tree(clusters, "cuda"), bo.build_tree(clusters)


def _random_clusters(rng, D, n_leaves, single=0.2):
    clusters = {1: (1, rng.normal(0.0, 3.0, D), 0.0)}
    leaves = [1]
    while len(leaves) < n_leaves:
        h = leaves.pop(rng.integers(0, len(leaves)))
        if h >= 1 << 40:
            leaves.append(h)
            continue
        kids = [2 * h] if rng.random() < single else [2 * h, 2 * h + 1]
        for c in kids:
            clusters[c] = (1, clusters[h][1] + rng.normal(0.0, 1.0, D), 0.0)
            leaves.append(c)
    return clusters


@pytest.mark.parametrize("D", [41, 119])
def test_predict_equals_the_oracle(D):
    from b200flow import bisecting_kmeans as bb
    rng = np.random.default_rng(D)
    x = _blobs(30011, D, 12, D) + 0.5
    cases = [_random_clusters(rng, D, 60), {1: (1, x[0], 0.0)}]
    chain = {1 << d: (1, rng.normal(0.0, 1.0, D), 0.0) for d in range(63)}                    # a 62-deep left chain
    chain.update({(1 << d) + 1: (1, rng.normal(0.0, 1.0, D), 0.0) for d in range(1, 63, 3)})   # with right siblings
    cases.append(chain)
    ties = _random_clusters(rng, D, 40, single=0.0)
    for h in list(ties):
        if h % 2 == 1 and h > 1 and rng.random() < 0.5:
            ties[h] = ties[h - 1]                          # equal siblings: every row goes to the left one
    cases.append(ties)
    for clusters in cases:
        tree, want_tree = _tree_arrays(clusters)
        assert tree.heap.tolist() == want_tree["heap"].tolist()
        leaf, d = bb.bkm_predict(_dev(x), tree)
        wl, wd = bo.predict_tree(x, want_tree)
        assert np.array_equal(leaf.cpu().numpy(), wl)
        assert np.array_equal(_bits(d.cpu().numpy()), _bits(wd))
    assert (leaf.cpu().numpy() >= 0).all()


def _same_fit(res, want, x):
    from b200flow import bisecting_kmeans as bb
    t, w = res.tree, want["tree"]
    for key in ("heap", "left", "right", "leaf", "size"):
        assert np.array_equal(getattr(t, key), w[key]), key
    assert np.array_equal(_bits(t.center), _bits(w["center"]))
    assert np.array_equal(_bits(t.cost), _bits(w["cost"]))
    assert float(res.training_cost).hex() == float(want["training_cost"]).hex()
    assert res.levels == want["levels"]
    wl, wd = bo.predict_tree(x, w)
    assert np.array_equal(res.leaf.cpu().numpy(), wl)
    assert np.array_equal(_bits(res.dist.cpu().numpy()), _bits(wd))
    assert bb.compute_cost(_dev(x), t).hex() == bo.compute_cost(x, w).hex()


@pytest.mark.parametrize("k,data,max_iter,mdcs", [(2, "blobs", 20, 1.0), (5, "kdd", 20, 1.0), (23, "blobs", 1, 1.0),
                                                   (23, "kdd", 20, 0.05), (100, "blobs", 5, 1.0), (100, "kdd", 20, 10.0),
                                                   (100, "kdd", 1, 0.001)])
def test_fit_equals_the_oracle(k, data, max_iter, mdcs):
    from b200flow import bisecting_kmeans as bb
    x = _blobs(20000, 41, 30, k) if data == "blobs" else _kdd_like(20000, 119, k)
    res = bb.bkm_fit(_dev(x), k, max_iter=max_iter, min_divisible=mdcs, seed=k + 1)
    want = bo.fit(x, k, max_iter=max_iter, min_divisible=mdcs, seed=k + 1)
    _same_fit(res, want, x)
    assert res.tree.num_leaves <= k


def test_fit_with_repeated_rows_has_fewer_leaves_than_k():
    from b200flow import bisecting_kmeans as bb
    pts = _kdd_like(40, 41, 3)
    x = np.ascontiguousarray(pts[np.random.default_rng(0).integers(0, 12, 30000)])   # 12 distinct rows at most
    res = bb.bkm_fit(_dev(x), 50, seed=4)
    want = bo.fit(x, 50, seed=4)
    _same_fit(res, want, x)
    assert res.tree.num_leaves <= 12 and res.tree.num_leaves < 50


def test_spark_doctest_through_create_data_frame():
    from pyspark.ml.clustering import BisectingKMeans
    from pyspark.ml.linalg import Vectors
    from pyspark.sql import SparkSession
    spark = SparkSession.builder.getOrCreate()
    data = [(Vectors.dense([0.0, 0.0]),), (Vectors.dense([1.0, 1.0]),), (Vectors.dense([9.0, 8.0]),),
            (Vectors.dense([8.0, 9.0]),)]
    df = spark.createDataFrame(data, ["features"])
    model = BisectingKMeans(k=2, minDivisibleClusterSize=1.0).fit(df)
    assert sorted(tuple(c) for c in model.clusterCenters()) == [(0.5, 0.5), (8.5, 8.5)]
    assert model.computeCost(df) == 2.0 and model.trainingCost == 2.0
    s = model.summary
    assert model.hasSummary and s.k == 2 and s.clusterSizes == [2, 2] and s.numIter == 20 and s.trainingCost == 2.0
    pred = model.transform(df)._column_tensor("prediction").cpu().numpy()
    assert pred.dtype == np.int32 and pred[0] == pred[1] != pred[2] == pred[3]
    assert model.predict(Vectors.dense([0.1, 0.2])) == pred[0] and model.predict([8.0, 8.0]) == pred[2]
    assert model.getK() == 2 and model.getMinDivisibleClusterSize() == 1.0


def test_shim_pipeline_and_cross_validator():
    """scaled without centring: a zero-mean root has no split noise (ℓ = 1e-4·‖μ‖ vanishes), so every row ties to the left
    child and the root only chains, in Spark as here."""
    from pyspark.ml import Pipeline
    from pyspark.ml.clustering import BisectingKMeans
    from pyspark.ml.evaluation import ClusteringEvaluator
    from pyspark.ml.feature import StandardScaler
    from pyspark.ml.tuning import CrossValidator, ParamGridBuilder
    df = _kdd_frame(30000, 12)
    bkm = BisectingKMeans(k=6, seed=2, maxIter=10)
    stages = _feature_pipeline()[:-1] + [StandardScaler(inputCol="raw_features", outputCol="features", withStd=True)]
    model = Pipeline(stages=stages + [bkm]).fit(df)
    out = model.transform(df)
    x = out._cols["features"].data.to(torch.float64).cpu().numpy()
    want = bo.fit(x, 6, max_iter=10, seed=2)
    m = model.stages[-1]
    wt = want["tree"]
    assert np.array_equal(_bits(np.array(m.clusterCenters())), _bits(wt["center"][wt["leaf_order"]]))
    pred = out._column_tensor("prediction").cpu().numpy()
    wl, _ = bo.predict_tree(x, wt)
    assert np.array_equal(pred, wl)
    s = m.summary
    assert np.array_equal(s.predictions._column_tensor("prediction").cpu().numpy(), pred)
    assert np.array_equal(s.cluster._column_tensor("prediction").cpu().numpy(), pred)
    assert s.k == 6 and s.numIter == 10 and s.trainingCost == want["training_cost"]
    assert s.clusterSizes == np.bincount(wl, minlength=6).tolist() and len(wt["leaf_order"]) == 6
    assert m.computeCost(out) == bo.compute_cost(x, wt)
    ev = ClusteringEvaluator()
    assert ev.evaluate(out) == ev.evaluate(s.predictions)
    feats = out.select("features")
    est = BisectingKMeans(seed=5, maxIter=5)
    grid = ParamGridBuilder().addGrid(est.k, [2, 4]).build()
    cvm = CrossValidator(estimator=est, estimatorParamMaps=grid, evaluator=ev, numFolds=2, seed=9).fit(feats)
    assert len(cvm.avgMetrics) == 2 and all(-1.0 <= v <= 1.0 for v in cvm.avgMetrics)
