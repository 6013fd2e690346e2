"""CPU checks of BisectingKMeans: the host split noise of b200flow.bisecting_kmeans against the numpy restatement
(tests/bisecting_kmeans_oracle.py) and the C oracle's Philox, the restatement on hand-made cases (duplicate-only data,
fractional minDivisibleClusterSize, the heap-index tie-break, an emptied child, the 63-level limit), the tree build, and the
shim's defaults and refusals (DESIGN.md §5t)."""
import numpy as np
import pytest

import bisecting_kmeans_oracle as bo
import kmeans_oracle as ko
import oracle
from b200flow import bisecting_kmeans as bb


def test_host_philox_matches_the_c_oracle():
    for seed in (0, 1, 2019, 0xFFFFFFFFFFFFFFFF):
        for heap in (1, 2, 3, 1 << 40, (1 << 62) + 5):
            for j in (0, 1, 118, 255):
                ctr = (heap & 0xFFFFFFFF, heap >> 32, j, 0)
                want = [int(v) for v in oracle.philox(seed, bb.PURPOSE_BKMS, *ctr)]
                assert bb.philox(seed, bb.PURPOSE_BKMS, *ctr) == want
                assert [int(v) for v in ko.philox(seed, bo.BKMS, *ctr)] == want
    assert bb.PURPOSE_BKMS == int.from_bytes(b"BKMS", "big") == bo.BKMS


@pytest.mark.parametrize("D", [1, 41, 119])
def test_split_noise_equals_the_restatement(D):
    rng = np.random.default_rng(D)
    center = rng.normal(0.0, 10.0, D) * 10.0 ** rng.integers(-5, 5, D)
    for heap in (1, 2, 7, 1 << 33, (1 << 62) + 1):
        for seed in (0, 42, 0xFFFFFFFFFFFFFFFF):
            got, want = bb.split_centers(center, heap, seed), bo.split(center, heap, seed)
            for g, w in zip(got, want):
                assert np.array_equal(g.view(np.int64), w.view(np.int64))
            z = (got[1] - center) / (1e-4 * np.sqrt(np.sum(center * center)))
            assert np.all(np.isfinite(z)) and np.all(np.abs(z) < 10.0)
    zero = np.zeros(D)                                   # ℓ = 0: both children are the center
    left, right = bb.split_centers(zero, 1, 3)
    assert np.array_equal(left, zero) and np.array_equal(right, zero)


def test_split_noise_is_standard_normal():
    z = []
    for heap in range(1, 200):
        left, right = bo.split(np.full(50, 1.0 / np.sqrt(50.0)), heap, 9)
        z.append((right - left) / 2e-4)
    z = np.concatenate(z)
    assert abs(z.mean()) < 0.05 and abs(z.std() - 1.0) < 0.05


def test_spark_doctest_answer():
    x = np.array([[0.0, 0.0], [1.0, 1.0], [9.0, 8.0], [8.0, 9.0]])
    for seed in (0, 1, 5):
        res = bo.fit(x, 2, seed=seed)
        t = res["tree"]
        centers = t["center"][t["leaf_order"]]
        assert sorted(map(tuple, centers)) == [(0.5, 0.5), (8.5, 8.5)]
        assert res["training_cost"] == 2.0 and bo.compute_cost(x, t) == 2.0
        leaf, _ = bo.predict_tree(x, t)
        assert leaf[0] == leaf[1] != leaf[2] == leaf[3]


def test_duplicate_only_block_is_never_split():
    x = np.repeat(np.array([[3.0, -1.0, 0.5]]), 500, axis=0)
    res = bo.fit(x, 5)
    assert res["levels"] == 0 and list(res["clusters"]) == [1] and res["training_cost"] == 0.0
    leaf, d = bo.predict_tree(x, res["tree"])
    assert (leaf == 0).all() and (d == 0.0).all()


def test_duplicate_blocks_stop_at_zero_cost():
    """three distinct points, many copies each: a leaf per point, fewer leaves than k, and each leaf costs 0."""
    pts = np.array([[0.0, 0.0], [10.0, 0.0], [0.0, 50.0]])
    x = np.repeat(pts, [400, 300, 200], axis=0)
    res = bo.fit(x, 10, seed=2)
    t = res["tree"]
    assert len(t["leaf_order"]) == 3 and res["training_cost"] == 0.0
    assert sorted(map(tuple, t["center"][t["leaf_order"]])) == sorted(map(tuple, pts))


def test_fractional_min_divisible_cluster_size():
    """root 1000 rows splits 600 / 400; with minDivisibleClusterSize 0.5 (= 500 rows) only the 600-row child may divide."""
    rng = np.random.default_rng(1)
    a = rng.normal(0.0, 1.0, (600, 2)) + [100.0, 0.0]
    b = rng.normal(0.0, 1.0, (400, 2)) + [-100.0, 0.0]
    x = np.vstack([a, b])
    res = bo.fit(x, 8, min_divisible=0.5, seed=3)
    cl = res["clusters"]
    big, small = (2, 3) if cl[2][0] == 600 else (3, 2)
    assert cl[big][0] == 600 and cl[small][0] == 400
    assert 2 * big in cl and 2 * small not in cl
    assert all(size >= 500 for h, (size, _, _) in cl.items() if 2 * h in cl)
    res = bo.fit(x, 8, min_divisible=601.0, seed=3)       # a count: nothing below 601 rows divides
    assert sorted(res["clusters"]) == [1, 2, 3]


def test_heap_index_breaks_ties_between_equal_sizes():
    """four equal, separated blobs: level 1 makes two 200-row clusters; with k = 3 only one of them may divide, the
    smaller heap index (2)."""
    rng = np.random.default_rng(4)
    cs = [[-50.0, -50.0], [-50.0, 50.0], [50.0, -50.0], [50.0, 50.0]]
    x = np.vstack([rng.normal(0.0, 1.0, (100, 2)) + c for c in cs])
    res = bo.fit(x, 3, seed=1)
    cl = res["clusters"]
    assert cl[2][0] == cl[3][0] == 200
    assert 4 in cl and 5 in cl and 6 not in cl and 7 not in cl
    assert len(res["tree"]["leaf_order"]) == 3


def test_emptied_child_and_the_level_limit():
    """a zero-mean cluster has ℓ = 0: both children start at its center, every row ties and goes left, and the right child
    disappears.  The cluster re-divides into one left child per level until the 63-level limit."""
    x = np.array([[1.0, 0.0], [-1.0, 0.0], [0.0, 2.0], [0.0, -2.0]])
    res = bo.fit(x, 100, max_iter=3)
    cl = res["clusters"]
    assert res["levels"] == bo.LEVEL_LIMIT - 1
    assert sorted(cl) == [1 << d for d in range(bo.LEVEL_LIMIT)]
    t = res["tree"]
    assert len(t["leaf_order"]) == 1 and (t["right"] == -1).all() and t["heap"][t["leaf_order"][0]] == 1 << 62
    assert all(c[0] == 4 and c[2] == 10.0 for c in cl.values()) and res["training_cost"] == 10.0
    leaf, d = bo.predict_tree(x, t)
    assert (leaf == 0).all() and d.tolist() == [1.0, 1.0, 4.0, 4.0]


def test_tree_build_matches_spark():
    """internal iff the left child exists; DFS leaf numbers left before right; a right-only cluster is a leaf."""
    c = {h: (1, np.zeros(1), 0.0) for h in (1, 2, 3, 4, 5, 7, 14, 15)}
    got, want = bb.build_tree(c, "cpu"), bo.build_tree(c)
    assert got.heap.tolist() == want["heap"].tolist() == [1, 2, 4, 5, 3]
    assert got.leaf.tolist() == want["leaf"].tolist() == [-1, -1, 0, 1, 2]
    assert got.left.tolist() == want["left"].tolist() and got.right.tolist() == want["right"].tolist() == [4, 3, -1, -1, -1]


def test_oracle_predict_walk_by_hand():
    center = np.array([[0.0], [-1.0], [1.0], [0.5], [1.5]])
    left, right, leaf = [1, -1, 3, -1, -1], [2, -1, 4, -1, -1], [-1, 0, -1, 1, 2]
    x = np.array([[-3.0], [0.0], [0.9], [1.0], [2.0]])
    got_leaf, got_d = bo.predict(x, left, right, leaf, center)
    assert got_leaf.tolist() == [0, 0, 1, 1, 2]             # 0.0 ties between -1 and 1 (left); 1.0 ties 0.5 / 1.5 (left)
    assert got_d.tolist() == [4.0, 1.0, 0.16000000000000003, 0.25, 0.25]


def test_shim_refusals_and_defaults():
    from pyspark.ml.clustering import BisectingKMeans
    from pyspark.ml.feature import IllegalArgumentException
    for bad in (dict(k=1), dict(k=2.5), dict(maxIter=0), dict(minDivisibleClusterSize=0.0), dict(distanceMeasure="cosine"),
                dict(distanceMeasure="manhattan"), dict(weightCol="w")):
        with pytest.raises(IllegalArgumentException):
            BisectingKMeans(**bad).fit(object())           # refused before the data is touched
    b = BisectingKMeans(seed=3)
    assert b.getK() == 4 and b.getMaxIter() == 20 and b.getMinDivisibleClusterSize() == 1.0
    assert b.getDistanceMeasure() == "euclidean" and b.getFeaturesCol() == "features" and b.getPredictionCol() == "prediction"


def test_validators_take_the_generic_loop():
    from pyspark.ml.clustering import BisectingKMeans
    from pyspark.ml.evaluation import ClusteringEvaluator
    from pyspark.ml.tuning import ParamGridBuilder, _grid_metrics
    b = BisectingKMeans()
    grid = ParamGridBuilder().addGrid(b.k, [2, 3]).build()
    assert _grid_metrics(b, grid, ClusteringEvaluator(), None, None) is None
