"""CPU checks of KMeans and the silhouette: the numpy restatement (tests/kmeans_oracle.py) against scikit-learn and hand-made
answers, the host Philox of b200flow.kmeans against the C oracle's, the shard bookkeeping of the grouped sum, and the
parameter refusals of the shim."""
import numpy as np
import pytest

import kmeans_oracle as ko
import oracle
from b200flow import kmeans as bk


def _blobs(n, D, k, seed, spread=0.3):
    rng = np.random.default_rng(seed)
    means = rng.normal(0.0, 4.0, (k, D))
    lab = rng.integers(0, k, n)
    return means[lab] + rng.normal(0.0, spread, (n, D)), lab, means


def test_oracle_lloyd_equals_sklearn():
    from sklearn.cluster import KMeans as SKMeans
    x, _, means = _blobs(3000, 5, 4, 1)
    init = means + 0.5
    want = SKMeans(n_clusters=4, init=init, n_init=1, algorithm="lloyd", max_iter=300, tol=0.0).fit(x)
    got = ko.lloyd(x, init, max_iter=300, tol=0.0)
    assert np.array_equal(ko.assign(x, got["centers"])[0], want.labels_)
    np.testing.assert_allclose(got["centers"], want.cluster_centers_, rtol=0, atol=1e-9)
    assert abs(got["training_cost"] - want.inertia_) <= 1e-9 * want.inertia_


@pytest.mark.parametrize("k", [2, 5])
def test_oracle_silhouette_equals_sklearn(k):
    from sklearn.metrics import silhouette_score
    x, lab, _ = _blobs(1500, 3, k, 2 + k, spread=1.5)
    lab[:3] = k + 1                                 # an absent cluster id (k) between present ones, and a one-member cluster
    lab[3] = k + 2
    want = silhouette_score(x, lab, metric="sqeuclidean")
    assert abs(ko.silhouette(x, lab) - want) <= 1e-9


def test_grouped_sum_is_chunked_and_sequential():
    rng = np.random.default_rng(3)
    v = rng.normal(size=(10000, 2)) * 10.0 ** rng.integers(-8, 8, (10000, 1))
    ids = rng.integers(0, 3, 10000)
    tot, cnt = ko.group_sums(v, ids, 4)
    for g in range(4):
        want = np.zeros(2)
        for s in range(0, 10000, 4096):
            part = np.zeros(2)
            for r in range(s, min(s + 4096, 10000)):
                if ids[r] == g:
                    part = part + v[r]
            want = want + part
        assert np.array_equal(tot[g], want)
    assert cnt.tolist() == np.bincount(ids, minlength=4).tolist()
    assert not np.signbit(ko.group_sums(np.array([[-0.0], [-0.0]]), None, 1)[0][0, 0])


def test_kmeans_parallel_with_fewer_distinct_candidates():
    """three distinct points, each three times, k = 50: round 1 keeps every row whose cost is non-zero (2·c·k/sumCost > 1),
    round 2 has sumCost 0 and keeps none; the distinct candidates (first center first) are the model."""
    pts = np.array([[0.0, 0.0], [1.0, 0.0], [0.0, 5.0]])
    x = np.repeat(pts, 3, axis=0)
    for seed in (0, 7, 2019):
        keys = ko.row_keys(seed, np.arange(9))
        first = x[np.argmin(keys)]
        centers = ko.init_parallel(x, 50, 2, seed)
        assert centers.shape == (3, 2) and np.array_equal(centers[0], first)
        assert sorted(map(tuple, centers)) == sorted(map(tuple, pts))
        res = ko.fit(x, 50, seed=seed)
        assert res["num_iter"] == 1 and res["training_cost"] == 0.0 and res["cluster_sizes"].tolist() == [3, 3, 3]


def test_random_init_takes_the_smallest_keys():
    x = np.arange(40.0).reshape(20, 2)
    keys = ko.row_keys(11, np.arange(20))
    got = ko.smallest_key_rows(x, 11, 4)
    assert np.array_equal(got, x[np.argsort(keys)[:4]])
    assert np.all(np.diff(keys[np.argsort(keys)[:4]]) > 0)


def test_host_philox_matches_the_c_oracle_and_the_restatement():
    for seed in (0, 1, 2019, 0xFFFFFFFFFFFFFFFF, 0x299F31D0A4093822):
        for purpose in (bk.PURPOSE_KMNS, bk.PURPOSE_KMPP, 0):
            for ctr in ((0, 0, 0, 0), (5, 0, 1, 0), (0xFFFFFFFF, 3, 2, 0), (123456789, 0, 0, 0)):
                want = [int(v) for v in oracle.philox(seed, purpose, *ctr)]
                assert bk.philox(seed, purpose, *ctr) == want
                assert [int(v) for v in ko.philox(seed, purpose, *ctr)] == want
    assert [hex(v) for v in bk.philox(0, 0, 0, 0, 0, 0)] == ["0x6627e8d5", "0xe169c58d", "0xbc57ac4c", "0x9b00dbd8"]
    rows = [0, 1, 4095, 4096, 2 ** 32 + 7]
    assert [bk.row_key(9, r) for r in rows] == ko.row_keys(9, rows).tolist()
    d, e = bk._Draws(3), ko._Draws(3)
    assert [d.next() for _ in range(5)] == [e.next() for _ in range(5)]


def test_local_kmeans_pp_equals_the_restatement():
    rng = np.random.default_rng(4)
    pts = np.concatenate([rng.normal(c, 0.2, (30, 3)) for c in (0.0, 3.0, 6.0, 9.0)])
    w = rng.integers(0, 9, pts.shape[0]).astype(np.float64)
    for k in (2, 4, 7):
        assert np.array_equal(bk._local_kmeans_pp(pts, w, k, 5), ko.local_kmeans_pp(pts, w, k, 5))


@pytest.mark.parametrize("offs_ns", [[(0, 5000)], [(0, 4096), (4096, 4096)], [(0, 100), (100, 50), (150, 9000)],
                                     [(0, 3000), (3000, 0), (3000, 6000)]])
def test_shard_bookkeeping(offs_ns):
    sh = bk._Shards.__new__(bk._Shards)
    sh.offs, sh.ns = [o for o, _ in offs_ns], [n for _, n in offs_ns]
    sh.lead = [min(m, (-o) % bk.CHUNK) for o, m in offs_ns]
    sh.owner = [sh._holder(bk.CHUNK * (o // bk.CHUNK)) if ld else -1 for o, ld in zip(sh.offs, sh.lead)]
    owned = []                                             # every global row is summed by exactly one rank, in chunks
    for r, (o, n) in enumerate(offs_ns):
        lead = sh.lead[r]
        rows = list(range(o + lead, o + n))
        for s in range(len(offs_ns)):
            if sh.owner[s] == r:
                rows += list(range(sh.offs[s], sh.offs[s] + sh.lead[s]))
        owned += rows
        if rows:
            assert rows[0] % bk.CHUNK == 0 and rows == list(range(rows[0], rows[0] + len(rows)))
    assert sorted(owned) == list(range(sum(sh.ns)))


def test_shim_refusals():
    from pyspark.ml.clustering import KMeans
    from pyspark.ml.evaluation import ClusteringEvaluator
    from pyspark.ml.feature import IllegalArgumentException
    for bad in (dict(k=1), dict(k=2.5), dict(initSteps=0), dict(initMode="kmeans++"), dict(maxIter=-1), dict(tol=-1.0),
                dict(distanceMeasure="cosine"), dict(distanceMeasure="manhattan"), dict(weightCol="w")):
        with pytest.raises(IllegalArgumentException):
            KMeans(**bad).fit(object())                    # refused before the data is touched
    for bad in (dict(distanceMeasure="cosine"), dict(weightCol="w"), dict(metricName="davies")):
        with pytest.raises(IllegalArgumentException):
            ClusteringEvaluator(**bad).evaluate(object())
    km = KMeans(k=7, seed=3)
    assert km.getK() == 7 and km.getInitMode() == "k-means||" and km.getInitSteps() == 2 and km.getTol() == 1e-4
    assert km.getMaxIter() == 20 and ClusteringEvaluator().isLargerBetter()


def test_validators_take_the_generic_loop_for_kmeans():
    from pyspark.ml.clustering import KMeans
    from pyspark.ml.evaluation import ClusteringEvaluator
    from pyspark.ml.tuning import ParamGridBuilder, _grid_metrics
    km = KMeans()
    grid = ParamGridBuilder().addGrid(km.k, [2, 3]).build()
    assert _grid_metrics(km, grid, ClusteringEvaluator(), None, None) is None
