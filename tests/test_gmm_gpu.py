"""GaussianMixture on the device: the E-step and moments kernels against the numpy restatement (tests/gmm_oracle.py) within
stated tolerances (DMMA rounds its four products once, exp and log are CUDA's), full fits on planted mixtures, the shapes
and limits, the batched partials, and the pyspark shim end to end."""
import math

import numpy as np
import pytest
import torch

import gmm_oracle as go

pytestmark = pytest.mark.gpu


def _dev(a):
    return torch.as_tensor(np.ascontiguousarray(a)).cuda()


# Densities must clear Spark's EPSILON floor for a test to see the kernels: with unit-scale data in tens of dimensions every
# logpdf is far below log EPSILON, every responsibility is 1/k and EM collapses all components onto one.  Tight clusters
# (spread 0.05, noise 0.0025) put the rows' densities far above it, and the tests assert that they do.
NOISE = 0.0025


def _planted(n, D, k, seed, spread=0.05):
    rng = np.random.default_rng(seed)
    centers = rng.normal(0.0, spread, (k, D))
    return np.ascontiguousarray(centers[rng.integers(0, k, n)] + rng.normal(0.0, NOISE, (n, D)))


def _params(x, k, seed):
    """a mixture with random full covariances of the clusters' scale around rows of x."""
    rng = np.random.default_rng(seed)
    D = x.shape[1]
    means = x[rng.integers(0, x.shape[0], k)] + rng.normal(0.0, 0.1 * NOISE, (k, D))
    covs = []
    for _ in range(k):
        a = rng.normal(0.0, 1.0, (D, D))
        covs.append(NOISE * NOISE * (a @ a.T / D + 0.5 * np.eye(D)))
    w = rng.uniform(0.5, 1.5, k)
    return w / w.sum(), means, np.stack(covs)


def _device_estep(x, w, means, covs, row_offset=0):
    from b200flow import gmm as bg
    n, D = x.shape
    k = w.shape[0]
    roots, u = bg.density_constants(covs)
    c = np.array([math.log(wi) + ui for wi, ui in zip(w, u)])
    prob = torch.empty((n, k), dtype=torch.float64, device="cuda")
    pred = torch.empty(n, dtype=torch.int32, device="cuda")
    nc = (row_offset + n - 1) // 4096 - row_offset // 4096 + 1
    parts = torch.full((nc, bg.width(k, D)), 7.0, dtype=torch.float64, device="cuda")
    bg.estep(_dev(x), _dev(means), _dev(roots), _dev(c), row_offset, resp=prob, pred=pred, partials=parts)
    return prob.cpu().numpy(), pred.cpu().numpy(), parts[:, 0].cpu().numpy()


def _close(got, want, rel):
    return np.max(np.abs(got - want) / np.maximum(1.0, np.abs(want))) <= rel


@pytest.mark.parametrize("n,D,k", [(1, 1, 2), (31, 41, 2), (4095, 78, 2), (4097, 119, 2), (8192, 256, 2), (1000, 41, 64),
                                   (300, 256, 64)])
def test_estep_equals_the_restatement(n, D, k):
    x = _planted(n, D, min(k, 8), n + D)
    w, means, covs = _params(x, k, D)
    prob, pred, ll = _device_estep(x, w, means, covs)
    r, lse = go.estep(x, w, means, covs)
    assert np.abs(r - 1.0 / k).max() > 0.1                       # the densities clear the EPSILON floor
    assert _close(prob, r, 1e-12)
    top = np.sort(r, 1)
    clear = top[:, -1] - top[:, -2] > 1e-9
    assert np.array_equal(pred[clear], r.argmax(1)[clear])
    want_ll = [float(sum(lse[c:c + 4096])) for c in range(0, n, 4096)]
    assert _close(ll, np.array(want_ll), 1e-12)
    for i in range(min(k, 2)):                                  # one component: the partial is the sum of logaddexp(log EPS, logpdf)
        _, _, l1 = _device_estep(x, np.array([1.0]), means[i:i + 1], covs[i:i + 1])
        t = np.logaddexp(math.log(go.EPSILON), go.logpdf(x, means[i], covs[i]))
        assert _close(l1, np.array([float(sum(t[c:c + 4096])) for c in range(0, n, 4096)]), 1e-12)


def test_estep_chunk_partials_follow_the_global_row_offset():
    x = _planted(5000, 41, 3, 1)
    w, means, covs = _params(x, 3, 2)
    _, lse = go.estep(x, w, means, covs)
    _, _, ll = _device_estep(x, w, means, covs, row_offset=4096 * 3 + 1000)
    assert ll.shape[0] == 2
    assert _close(ll, np.array([lse[:3096].sum(), lse[3096:].sum()]), 1e-12)


def _kdd_features(n):
    """KDD-shaped one-hot-encoded standardised features and labels (tools/bench_mlp.py's pipeline)."""
    import os
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
    from bench_mlp import features
    return features(n, 2019)


def _device_step(x, w, means, covs):
    from b200flow import dist as bdist, gmm as bg
    xt = _dev(x)
    sh = bdist.Shards(x.shape[0], 0, None, xt.device)
    roots, c, _ = bg._constants(covs, w, sh, xt.device)
    tot = bg.em_sums(xt, _dev(means), roots, c, sh).cpu().numpy()
    return (float(tot[0]),) + bg.m_step(tot, w.shape[0], x.shape[1])


def test_one_em_step_on_kdd_features_equals_the_restatement():
    xa, ya = _kdd_features(3673823)                              # every category present: D = 119
    x, y = xa[:9000].cpu().numpy(), ya[:9000].cpu().numpy()
    del xa, ya
    assert x.shape[1] == 119
    # standardised features in 119 dimensions put every density below EPSILON (the 2 pi factor alone is e^-109); scaled by
    # 0.01 the class densities clear it, while the rounding of every product and sum stays the same relative to the data
    x = x * 0.01
    # one component per class (its rows' mean and covariance, rank deficient where one-hot columns are constant within
    # the class), and one more with zero covariance, whose logpdf is the constant u
    cls = [c for c in range(int(y.max()) + 1) if (y == c).sum() > 1]
    means = np.stack([x[y == c].mean(0) for c in cls] + [x[0]])
    covs = np.stack([np.cov(x[y == c].T, bias=True) for c in cls] + [np.zeros((119, 119))])
    w = np.full(len(cls) + 1, 1.0 / (len(cls) + 1))
    r, _ = go.estep(x, w, means, covs)
    assert np.abs(r - 1.0 / w.shape[0]).max() > 0.1             # the densities clear the EPSILON floor
    got, want = _device_step(x, w, means, covs), go.em_step(x, w, means, covs)
    assert abs(got[0] - want[0]) <= 1e-10 * abs(want[0])
    for g, e in zip(got[1:], want[1:]):
        assert np.max(np.abs(g - e)) <= 1e-10 * np.max(np.abs(e))


@pytest.mark.parametrize("n,D,k", [(600, 256, 64), (5000, 1, 2), (4097, 119, 8)])
def test_one_em_step_at_the_moment_kernels_extreme_shapes(n, D, k):
    x = _planted(n, D, min(k, 8), D)
    w, means, covs = _params(x, k, D + 1)
    r, _ = go.estep(x, w, means, covs)
    assert np.abs(r - 1.0 / k).max() > 0.1
    got, want = _device_step(x, w, means, covs), go.em_step(x, w, means, covs)
    assert abs(got[0] - want[0]) <= 1e-10 * abs(want[0])
    for g, e in zip(got[1:], want[1:]):
        assert np.max(np.abs(g - e)) <= 1e-10 * np.max(np.abs(e))


@pytest.mark.parametrize("D,seed", [(41, 10), (78, 11)])
def test_full_fit_on_a_planted_mixture_equals_the_restatement(D, seed):
    from b200flow import gmm as bg
    x = _planted(12000, D, 4, D)
    fit = bg.gmm_fit(_dev(x), 4, max_iter=30, tol=0.01, seed=seed)
    w, m, c, ll, it = go.fit(x, 4, max_iter=30, tol=0.01, seed=seed)
    # EM really separates the four planted clusters: several iterations, no vanished component, distinct means
    assert it > 2 and w.min() > 0.2
    assert min(np.linalg.norm(m[i] - m[j]) for i in range(4) for j in range(i)) > 0.1
    assert fit.num_iter == it
    assert abs(fit.log_likelihood - ll) <= 1e-8 * abs(ll)
    for g, e in ((fit.weights, w), (fit.means, m), (fit.covariances, c)):
        assert np.max(np.abs(g - e)) <= 1e-8 * np.max(np.abs(e))
    r, pred = go.predict(x, w, m, c)
    top = np.sort(r, 1)
    clear = top[:, -1] - top[:, -2] > 1e-9
    assert clear.mean() > 0.99
    assert np.array_equal(fit.pred.cpu().numpy()[clear], pred[clear])
    assert fit.cluster_sizes.sum() == x.shape[0]


def test_loop_rules_on_the_device():
    from b200flow import gmm as bg
    x = _planted(3000, 5, 2, 3)
    f0 = bg.gmm_fit(_dev(x), 2, max_iter=0, seed=1)
    w, m, c = go.init(x, 2, 1)
    assert f0.num_iter == 0 and f0.log_likelihood == -1.7976931348623157e308
    assert np.array_equal(f0.means, m) and np.array_equal(f0.covariances, c)
    assert bg.gmm_fit(_dev(x), 2, max_iter=4, tol=1e300, seed=1).num_iter == 2


@pytest.mark.parametrize("n", [1, 31, 4095, 4097, 3 * 4096])
def test_fit_shapes_and_the_same_bits_as_the_transform(n):
    from b200flow import gmm as bg
    x = _planted(n, 7, 3, n)
    fit = bg.gmm_fit(_dev(x), 2, max_iter=3, seed=2) if n > 1 else None
    if fit is None:                                              # one row: every component sits on it with zero covariance
        fit = bg.gmm_fit(_dev(x), 2, max_iter=0, seed=2)
    prob, pred = bg.gmm_predict(_dev(x), fit)
    assert torch.equal(prob, fit.prob) and torch.equal(pred, fit.pred)
    assert np.allclose(prob.sum(1).cpu().numpy(), 1.0, rtol=0, atol=1e-12)


def test_limits_are_refused():
    from b200flow import _lib, gmm as bg
    with pytest.raises(_lib.UnsupportedParamError):
        bg.gmm_fit(_dev(np.zeros((10, 257))), 2)
    with pytest.raises(_lib.UnsupportedParamError):
        bg.gmm_fit(_dev(np.zeros((10, 3))), 65)
    with pytest.raises(ValueError):
        bg.gmm_fit(_dev(np.full((10, 3), np.nan)), 2)


def test_batched_partials_give_the_same_bits(monkeypatch):
    from b200flow import gmm as bg
    x = _dev(_planted(3 * 4096 + 77, 41, 4, 8))
    one = bg.gmm_fit(x, 4, max_iter=4, tol=0.0, seed=3)
    monkeypatch.setattr(bg, "PARTIALS_BUDGET", 1)               # one chunk per batch
    many = bg.gmm_fit(x, 4, max_iter=4, tol=0.0, seed=3)
    assert one.log_likelihood.hex() == many.log_likelihood.hex() and one.num_iter == many.num_iter
    for a, b in ((one.weights, many.weights), (one.means, many.means), (one.covariances, many.covariances)):
        assert a.tobytes() == b.tobytes()


def test_shim_pipeline_gaussian_mixture_and_silhouette():
    from b200flow import kmeans as bk
    from pyspark.ml import Pipeline
    from pyspark.ml.clustering import GaussianMixture
    from pyspark.ml.evaluation import ClusteringEvaluator
    from pyspark.ml.linalg import DenseMatrix, DenseVector
    from pyspark.ml.feature import StandardScaler, VectorAssembler
    from test_kmeans_gpu import _kdd_frame
    df = _kdd_frame(20000, 11)
    # six counters rather than the 115 one-hot columns, where every density would fall below EPSILON and all rows would
    # share one cluster (no silhouette)
    cols = ["src_bytes", "dst_bytes", "count", "srv_count", "dst_host_count", "dst_host_srv_count"]
    gm = GaussianMixture(k=3, seed=4, maxIter=3)
    model = Pipeline(stages=[VectorAssembler(inputCols=cols, outputCol="raw_features"),
                             StandardScaler(inputCol="raw_features", outputCol="features", withMean=True, withStd=True),
                             gm]).fit(df)
    out = model.transform(df)
    gmm = model.stages[-1]
    s = gmm.summary
    x = out._cols["features"].data.to(torch.float64).contiguous()
    from b200flow import gmm as bg
    want = bg.gmm_fit(x, 3, max_iter=3, seed=4)
    assert gmm.hasSummary and s.k == 3 and s.numIter == want.num_iter >= 2
    assert gmm.weights == want.weights.tolist() and s.logLikelihood == want.log_likelihood
    pred = out._column_tensor("prediction").cpu().numpy()
    assert pred.dtype == np.int32
    assert np.array_equal(s.cluster._column_tensor("prediction").cpu().numpy(), pred)
    prob = out._cols["probability"].data.cpu().numpy()
    assert np.array_equal(s.probability._cols["probability"].data.cpu().numpy(), prob)
    assert s.clusterSizes == np.bincount(pred, minlength=3).tolist()
    assert s.predictionCol == "prediction" and s.probabilityCol == "probability" and s.featuresCol == "features"
    assert math.isfinite(s.logLikelihood)
    D = out._cols["features"].data.shape[1]
    gs = gmm.gaussians
    assert len(gs) == 3 and np.array_equal(gs[0].mean.toArray(), gmm._fit_result.means[0])
    assert np.array_equal(gs[0].cov.toArray(), gmm._fit_result.covariances[0])
    rows = gmm.gaussiansDF.collect()
    assert len(rows) == 3 and isinstance(rows[1].mean, DenseVector) and isinstance(rows[1].cov, DenseMatrix)
    assert rows[1].cov.numRows == D and rows[1].cov == gs[1].cov
    sil = ClusteringEvaluator().evaluate(out)
    assert sil == bk.silhouette(x, torch.as_tensor(pred).cuda())
