"""PCA and Pearson correlation on the device: the centred-Gram and projection kernels against the numpy restatement
(tests/pca_oracle.py) within stated tolerances (DMMA rounds its four products once, so sums are not bit-equal to numpy's),
the projection's independence of a row's position, full fits, the large-mean case that the one-pass formula loses, the
batched partials, the limits, and the pyspark shim end to end."""
import numpy as np
import pytest
import torch

import pca_oracle as po

pytestmark = pytest.mark.gpu

CANARY = 7.0


def _dev(a):
    return torch.as_tensor(np.ascontiguousarray(a)).cuda()


def _rows(n, D, seed):
    rng = np.random.default_rng(seed)
    return np.ascontiguousarray(rng.normal(0.0, 1.0, (n, D)) * rng.uniform(0.1, 3.0, D) + rng.normal(0.0, 2.0, D))


def _planted(n, D, rank, seed):
    """low-rank signal with distinct strengths 2^-j along random directions, small noise, a non-zero mean."""
    rng = np.random.default_rng(seed)
    w = rng.normal(size=(rank, D)) * (4.0 * 2.0 ** -np.arange(rank))[:, None]
    return np.ascontiguousarray(rng.normal(size=(n, rank)) @ w + rng.normal(0.0, 0.01, (n, D)) + rng.normal(0.0, 3.0, D))


@pytest.mark.parametrize("shifted", [False, True])
@pytest.mark.parametrize("row_offset", [0, 4096 * 3 + 1000])
@pytest.mark.parametrize("n,D", [(1, 1), (31, 41), (4095, 78), (4097, 119), (8192, 256)])
def test_centered_gram_partials_equal_the_restatement(n, D, row_offset, shifted):
    from b200flow import pca as bp
    x = _rows(n, D, n + D)
    shift = x.mean(0) + 0.125 if shifted else None
    want = po.gram_partials(x, shift, row_offset)
    nc, P = len(want), D * (D + 1) // 2
    buf = torch.full((nc + 2, P), CANARY, dtype=torch.float64, device="cuda")
    bp.centered_gram(_dev(x), _dev(shift) if shifted else None, row_offset, buf[1:nc + 1])
    got = buf.cpu().numpy()
    assert np.all(got[0] == CANARY) and np.all(got[-1] == CANARY)     # nothing outside the chunks' rows is written
    assert not np.any(got[1:-1] == CANARY)                            # and every entry inside is
    for c, (q, scale) in enumerate(want):
        assert np.all(np.abs(got[1 + c] - po.pack(q)) <= 1e-12 * po.pack(scale) + 1e-300), (c, nc)


@pytest.mark.parametrize("n,D,ks", [(2500, 41, (1, 2, 8, 20, 41)), (1100, 119, (1, 8, 20, 32, 119)), (700, 256, (2, 72, 256)),
                                    (33, 1, (1,))])
def test_projection_equals_the_matrix_product(n, D, ks):
    from b200flow import pca as bp
    x = _rows(n, D, D)
    xt = _dev(x)
    for k in ks:
        pc = np.random.default_rng(k).normal(size=(D, k))
        got = bp.project(xt, _dev(pc)).cpu().numpy()
        assert got.shape == (n, k)
        assert np.all(np.abs(got - po.transform(x, pc)) <= 1e-12 * (np.abs(x) @ np.abs(pc)))


@pytest.mark.parametrize("D,k", [(119, 8), (256, 100), (41, 41)])
def test_a_rows_projection_does_not_depend_on_its_position(D, k):
    from b200flow import pca as bp
    x = _dev(_rows(3000, D, 9))
    pc = _dev(np.random.default_rng(k).normal(size=(D, k)))
    whole = bp.project(x, pc)
    assert torch.equal(torch.cat([bp.project(x[:1037].contiguous(), pc), bp.project(x[1037:].contiguous(), pc)]), whole)
    for i in (0, 31, 1024, 2999):
        assert torch.equal(bp.project(x[i:i + 1].contiguous(), pc), whole[i:i + 1])


def _assert_fit_equals_the_restatement(x, k):
    from b200flow import pca as bp
    fit = bp.pca_fit(_dev(x), k)
    pc, ev, mean, cov = po.fit(x, k)
    assert np.max(np.abs(fit.mean - mean)) <= 1e-10 * np.max(np.abs(mean))
    assert np.max(np.abs(fit.cov - cov)) <= 1e-10 * np.max(np.abs(cov))
    assert np.max(np.abs(fit.explained_variance - ev)) <= 1e-10
    # an eigenvector moves by the covariance's rounding over the gap to the next eigenvalue: the top k are separated
    s = np.sort(np.abs(np.linalg.eigvalsh(cov)))[::-1]
    gap = np.min(s[:k] - s[1:k + 1]) if k < x.shape[1] else np.min(s[:k - 1] - s[1:k])
    assert gap > 1e-6 * s[0]
    assert np.max(np.abs(fit.pc - pc)) <= max(1e-10, 1e-14 * s[0] / gap)      # the same order and the same signs
    got = bp.pca_transform(_dev(x), fit).cpu().numpy()
    assert np.all(np.abs(got - po.transform(x, pc)) <= 1e-9 * (np.abs(x) @ np.abs(pc)))
    r = bp.pearson(_dev(x))
    want_r = po.pearson(x)
    assert np.array_equal(np.isnan(r), np.isnan(want_r))
    assert np.max(np.abs(np.nan_to_num(r) - np.nan_to_num(want_r))) <= 1e-10
    return fit


@pytest.mark.parametrize("D", [41, 78])
def test_full_fit_on_planted_low_rank_data_equals_the_restatement(D):
    fit = _assert_fit_equals_the_restatement(_planted(12000, D, 5, D), 5)
    assert fit.explained_variance.sum() > 0.99                       # the five planted directions carry the variance


def test_full_fit_on_kdd_features_equals_the_restatement():
    import os
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
    from bench_mlp import features
    xa, _ = features(3673823, 2019)                                  # every category present: D = 119
    x = xa[:9000].cpu().numpy()
    del xa
    assert x.shape[1] == 119
    _assert_fit_equals_the_restatement(x, 8)


def test_two_passes_keep_a_small_variance_beside_a_large_mean():
    from b200flow import pca as bp
    rng = np.random.default_rng(4)
    x = rng.normal(size=(20000, 4))
    x[:, 0] = 1e9 + rng.normal(0.0, 1.0, 20000)                      # src_bytes-like: raw second moments reach 1e18
    fit = bp.pca_fit(_dev(x), 2)
    xl = x[:, 0].astype(np.longdouble)
    ref = float(((xl - xl.mean()) ** 2).sum() / (x.shape[0] - 1))
    assert abs(fit.cov[0, 0] - ref) <= 1e-9 * ref
    one_pass = (float((x[:, 0] * x[:, 0]).sum()) - x.shape[0] * float(x[:, 0].mean()) ** 2) / (x.shape[0] - 1)
    assert abs(one_pass - ref) > 1e-3 * ref                          # sum x^2 - n mean^2 in fp64 loses it


def test_batched_partials_give_the_same_bits(monkeypatch):
    from b200flow import pca as bp
    x = _dev(_planted(3 * 4096 + 77, 41, 4, 8))
    one = bp.pca_fit(x, 6)
    monkeypatch.setattr(bp, "PARTIALS_BUDGET", 1)                    # one chunk per batch
    many = bp.pca_fit(x, 6)
    for a, b in ((one.pc, many.pc), (one.explained_variance, many.explained_variance), (one.mean, many.mean),
                 (one.cov, many.cov)):
        assert a.tobytes() == b.tobytes()


def test_limits_are_refused():
    from b200flow import _lib, pca as bp
    with pytest.raises(_lib.UnsupportedParamError):
        bp.pca_fit(_dev(np.zeros((10, 257))), 2)
    for k in (0, 4, 1.5):
        with pytest.raises(ValueError):
            bp.pca_fit(_dev(_rows(10, 3, 1)), k)
    with pytest.raises(ValueError, match="<= 1 row"):
        bp.pca_fit(_dev(_rows(1, 3, 1)), 1)
    with pytest.raises(ValueError, match="finite"):
        bp.pca_fit(_dev(np.full((10, 3), np.nan)), 2)
    with pytest.raises(ValueError, match="<= 1 row"):
        bp.pearson(_dev(_rows(1, 3, 1)))
    with pytest.raises(_lib.B200FlowError):
        bp.pca_fit(torch.zeros((10, 3), dtype=torch.float32, device="cuda"), 2)
    with pytest.raises(_lib.B200FlowError):
        bp.pca_fit(torch.zeros((10, 3), dtype=torch.float64), 2)
    fit = bp.pca_fit(_dev(_rows(10, 3, 1)), 2)
    with pytest.raises(ValueError, match="does not match"):
        bp.pca_transform(_dev(_rows(10, 4, 1)), fit)
    # the entry points state their own limits
    wide = torch.zeros((10, 257), dtype=torch.float64, device="cuda")
    with pytest.raises(_lib.B200FlowError, match="1 <= D <= 256"):
        bp.centered_gram(wide, None, 0, torch.zeros((1, 257 * 258 // 2), dtype=torch.float64, device="cuda"))
    with pytest.raises(_lib.B200FlowError, match="1 <= D <= 256"):
        bp.project(wide, torch.zeros((257, 2), dtype=torch.float64, device="cuda"))


def test_shim_pipeline_pca_kmeans_and_correlation():
    from b200flow import pca as bp
    from pyspark.ml import Pipeline
    from pyspark.ml.clustering import KMeans
    from pyspark.ml.feature import PCA, IllegalArgumentException, StandardScaler, VectorAssembler
    from pyspark.ml.linalg import DenseMatrix, DenseVector
    from pyspark.ml.stat import Correlation
    from test_kmeans_gpu import _kdd_frame
    df = _kdd_frame(20000, 11)
    cols = ["src_bytes", "dst_bytes", "count", "srv_count", "dst_host_count", "dst_host_srv_count"]
    pca = PCA(k=3, inputCol="features", outputCol="pca")
    assert pca.getK() == 3 and pca.setK(3) is pca
    model = Pipeline(stages=[VectorAssembler(inputCols=cols, outputCol="raw_features"),
                             StandardScaler(inputCol="raw_features", outputCol="features", withMean=True, withStd=True),
                             pca, KMeans(k=3, seed=4, maxIter=5, featuresCol="pca")]).fit(df)
    out = model.transform(df)
    pm = model.stages[2]
    x = out._cols["features"].data.to(torch.float64).contiguous()
    want = bp.pca_fit(x, 3)
    assert isinstance(pm.pc, DenseMatrix) and (pm.pc.numRows, pm.pc.numCols) == (6, 3)
    assert np.array_equal(pm.pc.toArray(), want.pc)
    assert isinstance(pm.explainedVariance, DenseVector)
    ev = pm.explainedVariance.toArray()
    assert np.array_equal(ev, want.explained_variance) and np.all(np.diff(ev) <= 0) and 0 < ev.sum() <= 1 + 1e-12
    y = out._cols["pca"].data
    assert out._cols["pca"].kind == "vector" and y.dtype == torch.float64 and tuple(y.shape) == (20000, 3)
    assert torch.equal(y, bp.pca_transform(x, want))
    assert np.all(np.abs(y.cpu().numpy() - x.cpu().numpy() @ want.pc) <= 1e-12 * (np.abs(x.cpu().numpy()) @ np.abs(want.pc)))
    assert out._column_tensor("prediction").cpu().numpy().dtype == np.int32
    with pytest.raises(IllegalArgumentException, match="already exists"):
        pm.transform(out)
    with pytest.raises(IllegalArgumentException, match="does not match"):
        pm.copy({pm.inputCol: "pca", pm.outputCol: "again"}).transform(out)
    with pytest.raises(IllegalArgumentException, match="no less than k"):
        PCA(k=7, inputCol="features", outputCol="p").fit(out)
    corr = Correlation.corr(out, "features")
    assert corr.columns == ["pearson(features)"]
    m = corr.head()[0]
    assert isinstance(m, DenseMatrix) and m == corr.collect()[0][0] and (m.numRows, m.numCols) == (6, 6)
    r = m.toArray()
    assert np.array_equal(r, bp.pearson(x)) and np.array_equal(np.diag(r), np.ones(6)) and np.array_equal(r, r.T)
    assert np.max(np.abs(r - want.cov)) <= 1e-9                      # standardised features: covariance = correlation
    with pytest.raises(IllegalArgumentException, match="only 'pearson' is built"):
        Correlation.corr(out, "features", "spearman")
