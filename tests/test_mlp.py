"""MultilayerPerceptronClassifier without a GPU: the numpy restatement (tests/mlp_oracle.py) against finite differences and
scikit-learn, the MLPW draws, the L-BFGS extraction leaving LogisticRegression's iterates bit-identical, and the param
refusals of the shim."""
import hashlib

import numpy as np
import pytest
import torch

import mlp_oracle as mo


def _net(layers, seed):
    rng = np.random.default_rng(seed)
    P = sum((a + 1) * b for a, b in zip(layers[:-1], layers[1:]))
    x = rng.normal(0.0, 1.0, (37, layers[0]))
    y = rng.integers(0, layers[-1], 37)
    return rng.normal(0.0, 0.7, P), x, y


@pytest.mark.parametrize("layers", [[3, 2], [4, 5, 3], [5, 6, 4, 3], [2, 1, 2]])
def test_gradient_equals_central_differences(layers):
    w, x, y = _net(layers, 3)
    _, g = mo.loss_grad(w, layers, x, y)
    h = 1e-6
    fd = np.empty_like(w)
    for i in range(w.size):
        e = np.zeros_like(w); e[i] = h
        fd[i] = (mo.loss_grad(w + e, layers, x, y)[0] - mo.loss_grad(w - e, layers, x, y)[0]) / (2 * h)
    assert np.max(np.abs(fd - g)) <= 1e-7 * max(1.0, np.max(np.abs(g)))


@pytest.mark.parametrize("layers", [[6, 5, 3], [4, 7, 3, 5]])
def test_forward_equals_scikit_learn(layers):
    from sklearn.neural_network import MLPClassifier
    w, x, y = _net(layers, 9)
    y = np.arange(x.shape[0]) % layers[-1]
    clf = MLPClassifier(hidden_layer_sizes=tuple(layers[1:-1]), activation="logistic", max_iter=1)
    import warnings
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        clf.fit(x, y)
    params = mo.unpack(w, layers)
    clf.coefs_ = [W.T.copy() for W, _ in params]
    clf.intercepts_ = [b.copy() for _, b in params]
    want = clf.predict_proba(x)
    got = mo.softmax(mo.raw(w, layers, x))
    assert np.max(np.abs(got - want) / np.abs(want)) <= 1e-12


def test_layout_round_trips_and_matches_spark():
    layers = [3, 2, 2]
    w = np.arange(14, dtype=np.float64)
    (W1, b1), (W2, b2) = mo.unpack(w, layers)
    assert W1[1, 0] == 1.0 and W1[0, 1] == 2.0 and list(b1) == [6.0, 7.0]      # (o, i) at o + i*out, then b
    assert W2[0, 0] == 8.0 and list(b2) == [12.0, 13.0]
    assert np.array_equal(mo.pack(mo.unpack(w, layers)), w)


def test_host_mlpw_draws_equal_the_formula():
    from b200flow import kmeans as bk, mlp as bm
    layers = [5, 3, 2]
    got = bm.init_weights(layers, 77)
    assert np.array_equal(got, mo.init_weights(layers, 77))
    i = 19                                                  # the second layer's block: scale 1/sqrt(3)
    wds = bk.philox(77, 0x4D4C5057, i, 0)
    assert got[i] == (bk.uniform(wds[0], wds[1]) * 4.8 - 2.4) / np.sqrt(3.0)
    assert np.all(np.abs(got[:18]) <= 2.4 / np.sqrt(5.0)) and bm.n_params(layers) == got.size == 26
    assert not np.array_equal(got, bm.init_weights(layers, 78))


# sha256 of (coef, intercept, objective history) bytes, computed before linear.lbfgs was extracted from lr_fit
_LR_BITS = [
    (3, dict(reg_param=0.05, elastic_net=0.5), 13, "0afe62a47d12e1d06ad66a83ebb1ea24c88193f6678aecc5ef34f2ba341dc81e"),
    (3, dict(reg_param=0.0), 11, "3ccc5a542c5a0f7f88cbcd8e1906f58033830e4bcc8335deb7b17f68df0656b0"),
    (3, dict(reg_param=0.1, elastic_net=0.0, max_iter=7), 7, "439eab37544e7056b940925beef58e52c6a5d3aeb767b99b823d8d59e8ace890"),
    (2, dict(reg_param=0.02, elastic_net=1.0), 17, "613f260ce0b9af0001e41a48525d121fb57811a9ac8c96eae0484dc82ca7d9db"),
]


@pytest.mark.parametrize("case", range(len(_LR_BITS)))
def test_lr_fit_iterates_unchanged_by_the_lbfgs_extraction(case):
    from b200flow import linear
    C, kw, iters, digest = _LR_BITS[case]
    threads = torch.get_num_threads()
    torch.set_num_threads(1)
    try:
        rng = np.random.default_rng(5)
        x = torch.from_numpy(rng.normal(size=(300, 6)) * np.array([1, 2, 0.5, 3, 1, 1]) + np.array([0, 1, 0, 0, 2, 0]))
        y = torch.from_numpy(rng.integers(0, 3, 300))
        f = linear.lr_fit(x, y if C == 3 else (y > 0).long(), C, **kw)
    finally:
        torch.set_num_threads(threads)
    v = np.concatenate([f.coef.numpy().ravel(), f.intercept.numpy(), np.array(f.objective_history)])
    assert f.iterations == iters and hashlib.sha256(v.tobytes()).hexdigest() == digest


def test_plain_lbfgs_minimises_a_quadratic():
    from b200flow import linear
    A = torch.tensor([[3.0, 1.0], [1.0, 2.0]], dtype=torch.float64)
    c = torch.tensor([1.0, -1.0], dtype=torch.float64)
    v, hist, it = linear.lbfgs(lambda v: (0.5 * v @ A @ v - c @ v, A @ v - c), torch.zeros(2, dtype=torch.float64), 50, 1e-14)
    assert torch.allclose(v, torch.linalg.solve(A, c), atol=1e-8) and all(b <= a for a, b in zip(hist, hist[1:]))


@pytest.mark.parametrize("kw", [dict(layers=[4]), dict(layers=[4, 0, 2]), dict(layers=[4, 3, 2], maxIter=-1),
                                dict(layers=[4, 3, 2], blockSize=0), dict(layers=[4, 3, 2], stepSize=0.0),
                                dict(layers=[4, 3, 2], tol=-1e-6), dict(layers=[4, 3, 2], solver="adam"),
                                dict(layers=[4, 3, 1]), dict()])
def test_param_refusals(kw):
    from pyspark.ml.classification import MultilayerPerceptronClassifier
    from pyspark.ml.feature import IllegalArgumentException
    with pytest.raises(IllegalArgumentException):
        MultilayerPerceptronClassifier(**kw)._check()


def test_defaults_are_sparks():
    from pyspark.ml.classification import MultilayerPerceptronClassifier
    m = MultilayerPerceptronClassifier(layers=[4, 3, 2])
    assert (m.getMaxIter(), m.getTol(), m.getBlockSize(), m.getSolver(), m.getStepSize()) == (100, 1e-6, 128, "l-bfgs", 0.03)
    assert m.getLayers() == [4, 3, 2] and m._check() == [4, 3, 2]
