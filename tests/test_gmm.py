"""GaussianMixture without a GPU: the numpy restatement (tests/gmm_oracle.py) against independent code — scipy's
multivariate normal, scikit-learn's EM step — the EM loop rules, the host half of b200flow/gmm.py against the restatement,
and the shim's parameter validation."""
import math

import numpy as np
import pytest
from scipy.stats import multivariate_normal

import gmm_oracle as go


def _spd(rng, D, scale=1.0):
    a = rng.normal(0.0, 1.0, (D, D))
    return scale * (a @ a.T / D + 0.5 * np.eye(D))


@pytest.mark.parametrize("D", [1, 3, 41, 119])
def test_logpdf_equals_scipy_for_full_rank(D):
    rng = np.random.default_rng(D)
    cov, mean = _spd(rng, D), rng.normal(0.0, 1.0, D)
    x = mean + rng.normal(0.0, 1.0, (200, D))
    want = multivariate_normal(mean, cov).logpdf(x)
    got = go.logpdf(x, mean, cov)
    assert np.max(np.abs(got - want) / np.abs(want)) <= 1e-12


def test_rank_deficient_logpdf_keeps_sparks_d_not_rank_constant():
    rng = np.random.default_rng(3)
    D, rank = 6, 4
    basis = np.linalg.qr(rng.normal(0.0, 1.0, (D, D)))[0][:, :rank]
    cov = basis @ np.diag([3.0, 2.0, 1.5, 0.5]) @ basis.T
    mean = rng.normal(0.0, 1.0, D)
    x = mean + rng.normal(0.0, 1.0, (50, rank)) @ basis.T          # on the support
    # scipy normalises by the rank; Spark's constant counts all D dimensions, 0.5 (D - rank) log 2 pi lower
    want = multivariate_normal(mean, cov, allow_singular=True).logpdf(x) - 0.5 * (D - rank) * math.log(2 * math.pi)
    got = go.logpdf(x, mean, cov)
    assert np.max(np.abs(got - want) / np.abs(want)) <= 1e-12


def test_zero_covariance_gives_a_constant_logpdf():
    D = 5
    x = np.random.default_rng(1).normal(0.0, 1.0, (20, D))
    got = go.logpdf(x, x[0], np.zeros((D, D)))
    assert np.all(got == -0.5 * D * math.log(2 * math.pi))


def test_one_em_step_equals_scikit_learn():
    from sklearn.mixture import GaussianMixture
    rng = np.random.default_rng(5)
    k, D, n = 3, 4, 3000
    centers = rng.normal(0.0, 1.0, (k, D))                          # tight clusters: every row's density dwarfs EPSILON
    x = centers[rng.integers(0, k, n)] + rng.normal(0.0, 0.05, (n, D))
    w = np.array([0.5, 0.3, 0.2])
    m = centers + rng.normal(0.0, 0.01, (k, D))
    c = np.stack([_spd(rng, D, 0.0025) for _ in range(k)])
    sk = GaussianMixture(k, covariance_type="full", reg_covar=0.0)
    sk.weights_, sk.means_, sk.covariances_ = w, m, c
    sk.precisions_cholesky_ = np.stack([np.linalg.cholesky(np.linalg.inv(ci)) for ci in c])
    lpn, log_resp = sk._e_step(x)
    sk._m_step(x, log_resp)
    ll, nw, nm, nc = go.em_step(x, w, m, c)
    assert abs(ll - lpn * n) <= 1e-9 * abs(ll)
    for got, want in ((nw, sk.weights_), (nm, sk.means_), (nc, sk.covariances_)):
        assert np.max(np.abs(got - want)) <= 1e-9 * np.max(np.abs(want))


def test_loop_rules():
    rng = np.random.default_rng(2)
    x = rng.normal(0.0, 1.0, (300, 3))
    w, m, c, ll, it = go.fit(x, 2, max_iter=0)
    assert ll == -1.7976931348623157e308 and it == 0
    assert np.array_equal((w, m, c)[1], go.init(x, 2, 0)[1])
    for mi in (2, 5):
        assert go.fit(x, 2, max_iter=mi, tol=1e300)[4] == 2         # two iterations whatever tol says
    assert go.fit(x, 2, max_iter=1, tol=0.0)[4] == 1


def test_host_half_equals_the_restatement():
    from b200flow import gmm as bg
    rng = np.random.default_rng(9)
    assert bg.sample_rows(77, 6, 1000) == list(go.sample_rows(77, 6, 1000))
    x = rng.normal(0.0, 1.0, (1000, 7))
    samples = x[bg.sample_rows(77, 6, 1000)]
    for got, want in zip(bg.init_params(samples, 6), go.init(x, 6, 77)):
        assert np.array_equal(got, want)
    covs = np.stack([_spd(rng, 7), np.zeros((7, 7)), np.diag([1.0, 0, 2, 0, 3, 0, 4])])
    roots, u = bg.density_constants(covs)
    for i in range(3):
        R, ui = go.constants(covs[i])
        assert np.array_equal(roots[i], R) and u[i] == ui


def test_m_step_from_packed_sums_equals_the_restatement():
    from b200flow import gmm as bg
    rng = np.random.default_rng(4)
    k, D, n = 3, 5, 400
    x = rng.normal(0.0, 1.0, (n, D))
    r = rng.dirichlet(np.ones(k), n)
    tot = [0.0]
    iu = np.triu_indices(D)
    for i in range(k):
        Q = (x * r[:, i:i + 1]).T @ x
        packed = np.empty(D * (D + 1) // 2)
        packed[iu[0] + iu[1] * (iu[1] + 1) // 2] = Q[iu]
        tot += [r[:, i].sum()] + list(r[:, i] @ x) + list(packed)
    tot = np.array(tot)
    assert tot.shape[0] == bg.width(k, D)
    w, m, c = bg.m_step(tot, k, D)
    sw = 0.0
    for i in range(k):
        sw = sw + r[:, i].sum()
    for i in range(k):
        W = r[:, i].sum()
        mean = (r[:, i] @ x) * (1.0 / W)
        Q = (x * r[:, i:i + 1]).T @ x
        cov = (Q + mean[:, None] * ((-W) * mean[None, :])) * (1.0 / W)
        assert w[i] == W / sw and np.array_equal(m[i], mean)
        assert np.array_equal(np.triu(c[i]), np.triu(cov)) and np.array_equal(c[i], c[i].T)
    bad = tot.copy()
    bad[1 + (1 + D + D * (D + 1) // 2)] = 0.0                        # component 1 lost all its responsibility
    with pytest.raises(ValueError, match="component 1"):
        bg.m_step(bad, k, D)


@pytest.mark.parametrize("kw", [{"k": 1}, {"k": 2.5}, {"maxIter": -1}, {"tol": -0.1}, {"aggregationDepth": 1},
                                {"weightCol": "w"}])
def test_shim_parameter_validation(kw):
    from pyspark.ml.clustering import GaussianMixture
    from pyspark.ml.feature import IllegalArgumentException
    with pytest.raises(IllegalArgumentException):
        GaussianMixture(**kw)._check()


def test_shim_defaults_and_dense_matrix():
    from pyspark.ml.clustering import GaussianMixture
    from pyspark.ml.linalg import DenseMatrix, Matrices
    g = GaussianMixture()
    g._check()
    assert [g.getOrDefault(p) for p in ("k", "maxIter", "tol", "aggregationDepth", "probabilityCol")] == \
        [2, 100, 0.01, 2, "probability"]
    m = Matrices.dense(2, 3, [1, 2, 3, 4, 5, 6])
    assert isinstance(m, DenseMatrix) and (m.numRows, m.numCols) == (2, 3)
    assert np.array_equal(m.toArray(), [[1, 3, 5], [2, 4, 6]])


def test_model_gaussians_and_gaussians_df_from_a_fit():
    from b200flow import gmm as bg
    from pyspark.ml.clustering import GaussianMixtureModel
    from pyspark.ml.linalg import DenseMatrix, DenseVector
    rng = np.random.default_rng(6)
    covs = np.stack([_spd(rng, 3), _spd(rng, 3)])
    fit = bg.GMMFit(np.array([0.25, 0.75]), rng.normal(0.0, 1.0, (2, 3)), covs, None, None, -12.5, 4)
    m = GaussianMixtureModel(fit)
    assert m.weights == [0.25, 0.75] and not m.hasSummary
    g = m.gaussians
    assert np.array_equal(g[1].mean.toArray(), fit.means[1]) and np.array_equal(g[1].cov.toArray(), covs[1])
    rows = m.gaussiansDF.collect()
    assert [type(r.mean) for r in rows] == [DenseVector] * 2 and [type(r.cov) for r in rows] == [DenseMatrix] * 2
    assert rows[0].cov == g[0].cov and rows[0].mean == g[0].mean
