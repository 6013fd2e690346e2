"""PCA and Pearson correlation on the CPU: the numpy restatement (tests/pca_oracle.py) against the PySpark doctest's known
answer, scikit-learn and numpy.corrcoef, its rules (signs, ties, constant features, k and n validation), and the host half
of b200flow/pca.py against the restatement bit for bit."""
import numpy as np
import pytest

import pca_oracle as po


def _sign_rule(cols):
    """every column's entry of largest magnitude made positive."""
    out = cols.copy()
    for j in range(out.shape[1]):
        if out[np.argmax(np.abs(out[:, j])), j] < 0:
            out[:, j] = -out[:, j]
    return out


def _spectrum_data(n, D, seed):
    """rows with a well-separated spectrum (variances 2^-j along a random rotation) around a non-zero mean."""
    rng = np.random.default_rng(seed)
    rot, _ = np.linalg.qr(rng.normal(size=(D, D)))
    return rng.normal(size=(n, D)) * (2.0 ** -np.arange(D)) @ rot.T + rng.normal(0.0, 5.0, D)


def test_known_answer_of_the_pyspark_doctest():
    x = np.array([[0.0, 1.0, 0.0, 7.0, 0.0], [2.0, 0.0, 3.0, 4.0, 5.0], [4.0, 0.0, 0.0, 6.0, 7.0]])
    pc, ev, _, _ = po.fit(x, 2)
    assert np.allclose(ev, [0.794393253, 0.205606747], rtol=0, atol=1e-9)
    y = po.transform(x, pc)
    # Spark prints [1.648..., -4.013...] for the first row.  A component's sign is LAPACK's there; here it is fixed by the
    # sign rule, so each column is compared up to its sign, and the rule's own signs are pinned below.
    assert np.allclose(np.abs(y[0]), [1.6485728230883807, 4.013282700516296], rtol=0, atol=1e-9)
    assert y[0, 0] < 0 and y[0, 1] < 0
    for j in range(2):
        assert pc[np.argmax(np.abs(pc[:, j])), j] > 0


@pytest.mark.parametrize("n,D,k", [(500, 6, 3), (2000, 12, 12), (5000, 9, 1)])
def test_restatement_equals_scikit_learn(n, D, k):
    from sklearn.decomposition import PCA
    x = _spectrum_data(n, D, n + D)
    pc, ev, mean, cov = po.fit(x, k)
    sk = PCA(n_components=k, svd_solver="full").fit(x)
    want = _sign_rule(sk.components_.T)
    assert np.max(np.abs(pc - want)) <= 1e-9
    assert np.max(np.abs(ev - sk.explained_variance_ratio_)) <= 1e-12
    assert np.allclose(mean, x.mean(0), rtol=0, atol=1e-12) and np.allclose(cov, np.cov(x.T), rtol=0, atol=1e-12)
    # Spark's transform does not subtract the mean: it is scikit-learn's plus the mean's projection
    assert np.max(np.abs(po.transform(x, pc) - ((x - sk.mean_) @ want + mean @ pc))) <= 1e-9


def test_pearson_equals_numpy_corrcoef():
    x = _spectrum_data(3000, 8, 5)
    x[:, 3] = x[:, 3] + 1e4                                           # a large mean does not hurt the two-pass form
    r = po.pearson(x)
    assert np.max(np.abs(r - np.corrcoef(x.T))) <= 1e-12
    assert np.array_equal(np.diag(r), np.ones(8))


def test_a_constant_feature_gives_nan_rows_and_columns():
    x = _spectrum_data(100, 5, 7)
    x[:, 2] = 3.25
    r = po.pearson(x)
    assert np.isnan(r[2]).all() and np.isnan(r[:, 2]).all()
    keep = [0, 1, 3, 4]
    assert np.isfinite(r[np.ix_(keep, keep)]).all()
    assert np.max(np.abs(r[np.ix_(keep, keep)] - np.corrcoef(x[:, keep].T))) <= 1e-12
    # every feature constant: the eigenvalues' sum is 0 and the ratios are NaN, as Spark's division gives
    _, ev, _, cov = po.fit(np.full((10, 3), 2.5), 2)
    assert np.array_equal(cov, np.zeros((3, 3))) and np.isnan(ev).all()


def test_sign_rule_on_equal_magnitudes(monkeypatch):
    from b200flow import pca as bp
    U = np.column_stack([[-0.5, 0.5, -0.5, 0.5], [0.5, 0.5, -0.5, -0.5], [0.0, -1.0, 0.0, 0.0], [0.5, -0.5, 0.5, -0.5]])
    monkeypatch.setattr(np.linalg, "eigh", lambda c: (np.array([1.0, 2.0, 3.0, 4.0]), U))
    for comp in (po.components, bp.components):
        pc, ev = comp(np.eye(4), 4)
        # eigh's columns reversed: the lowest index decides between equal magnitudes
        assert np.array_equal(pc[:, 0], [0.5, -0.5, 0.5, -0.5])       # first entry was positive: kept
        assert np.array_equal(pc[:, 1], [0.0, 1.0, 0.0, 0.0])         # -1 flipped
        assert np.array_equal(pc[:, 2], [0.5, 0.5, -0.5, -0.5])       # kept
        assert np.array_equal(pc[:, 3], [0.5, -0.5, 0.5, -0.5])       # first entry was negative: flipped
        assert np.array_equal(ev, np.array([4.0, 3.0, 2.0, 1.0]) / 10.0)


def test_negative_eigenvalues_are_ordered_by_magnitude():
    from b200flow import pca as bp
    c = np.diag([1.0, -3.0, 2.0])                                      # not a covariance: the SVD's s is |eigenvalue|
    for comp in (po.components, bp.components):
        pc, ev = comp(c, 3)
        assert np.array_equal(np.abs(pc), np.eye(3)[:, [1, 2, 0]])
        assert np.array_equal(ev, np.array([3.0, 2.0, 1.0]) / 6.0)


def test_k_and_n_validation():
    from b200flow import pca as bp
    x = _spectrum_data(20, 4, 1)
    for k in (0, 5, -1, 1.5, None):
        with pytest.raises(ValueError):
            po.fit(x, k)
        with pytest.raises(ValueError):
            bp.check_k(4, k)
    assert bp.check_k(4, 4) == 4 and bp.check_k(4, 1.0) == 1
    with pytest.raises(ValueError):
        po.fit(x[:1], 1)
    with pytest.raises(ValueError):
        po.pearson(x[:1])


@pytest.mark.parametrize("D,k", [(1, 1), (7, 3), (41, 41), (119, 8)])
def test_host_half_equals_the_restatement_bit_for_bit(D, k):
    from b200flow import pca as bp
    x = _spectrum_data(300, D, D) if D <= 41 else np.random.default_rng(D).normal(size=(300, D))
    x[:, 0] = x[:, 0] if D < 7 else 1.0                                # a constant feature from D = 7 up
    _, cov = po.covariance(x)
    got, want = bp.components(cov, k), po.components(cov, k)
    assert got[0].tobytes() == want[0].tobytes() and got[1].tobytes() == want[1].tobytes()
    assert bp.correlation(cov).tobytes() == po.pearson(x).tobytes()


def test_chunk_order_sums_and_packing():
    x = np.random.default_rng(3).normal(size=(5000, 3))
    assert po.chunks(5000, 4096 * 3 + 1000) == [(0, 3096), (3096, 5000)]
    assert po.chunks(1, 0) == [(0, 1)] and po.chunks(4097, 0) == [(0, 4096), (4096, 4097)]
    s = np.zeros(3)
    for r in x[:4096]:
        s = s + r
    t = np.zeros(3)
    for r in x[4096:]:
        t = t + r
    assert np.array_equal(po.column_sums(x), (np.zeros(3) + s) + t)
    q = np.arange(9.0).reshape(3, 3)
    assert np.array_equal(po.pack(q), [0.0, 1.0, 4.0, 2.0, 5.0, 8.0])
