"""NaiveBayes without a GPU: the numpy restatement (tests/naive_bayes_oracle.py) against scikit-learn and against hand-worked
answers for the weighted multinomial, weighted complement, bernoulli and gaussian models, and the shim's param validation."""
import numpy as np
import pytest
import torch

import naive_bayes_oracle as nbo

# (label, weight, x): the three rows of the hand-worked answers (pyspark's NaiveBayes doctest data)
ROWS_Y = np.array([0.0, 0.0, 1.0])
ROWS_W = np.array([0.1, 0.5, 1.0])
ROWS_X = np.array([[0.0, 0.0], [0.0, 1.0], [1.0, 0.0]])
POINT = np.array([[1.0, 0.0]])


def _softmax(r):
    return nbo.probability(r)


@pytest.mark.parametrize("case", ["multinomial", "complement", "bernoulli"])
def test_discrete_known_answers(case):
    want = {
        "multinomial": ([-0.810930, -0.587787], [[-0.916291, -0.510826], [-0.405465, -1.098612]], [-1.727221, -0.993252],
                        [0.324324, 0.675676]),
        "complement": ([-0.810930, -0.587787], [[0.405465, 1.098612], [0.916291, 0.510826]], [-0.980829, -0.470004],
                       [0.375, 0.625]),
        "bernoulli": ([-0.510826, -0.916291], [[-1.386294, -0.693147], [-0.405465, -1.098612]], [-2.590267, -1.727221],
                      [0.296703, 0.703297]),
    }[case]
    f = nbo.fit(ROWS_X, ROWS_Y, 2, case, 1.0, w=None if case == "bernoulli" else ROWS_W)
    r = nbo.raw(f, POINT)
    np.testing.assert_allclose(f.pi, want[0], atol=1e-6)
    np.testing.assert_allclose(f.theta, want[1], atol=1e-6)
    np.testing.assert_allclose(r[0], want[2], atol=1e-6)
    np.testing.assert_allclose(_softmax(r)[0], want[3], atol=1e-6)
    assert int(np.argmax(r[0])) == 1


def test_gaussian_known_answer():
    f = nbo.fit(ROWS_X, ROWS_Y, 2, "gaussian")
    eps = 1e-9 * (2.0 / 9.0)
    np.testing.assert_allclose(f.pi, [-0.405465, -1.098612], atol=1e-6)
    np.testing.assert_array_equal(f.theta, [[0.0, 0.5], [1.0, 0.0]])
    np.testing.assert_allclose(f.sigma, [[eps, 0.25 + eps], [eps, eps]], rtol=1e-12)
    assert abs(eps - 2.2222e-10) < 1e-14
    r = nbo.raw(f, POINT)
    assert abs(r[0, 1] - 21.128731) < 1e-6
    assert int(np.argmax(r[0])) == 1


def _data(n=3000, D=6, C=4, seed=3, kind="counts"):
    rng = np.random.default_rng(seed)
    y = rng.integers(0, C, n)
    if kind == "binary":
        x = (rng.random((n, D)) < (0.2 + 0.15 * y[:, None] % 3)).astype(np.float64)
    elif kind == "normal":
        x = rng.normal(size=(n, D)) + y[:, None] * rng.uniform(-1, 1, D)
    else:
        x = rng.poisson(1.0 + y[:, None] * np.arange(1, D + 1) / D, (n, D)).astype(np.float64)
    return x, y.astype(np.float64)


def test_gaussian_against_sklearn():
    from sklearn.naive_bayes import GaussianNB
    x, y = _data(kind="normal")
    f = nbo.fit(x, y, 4, "gaussian")
    sk = GaussianNB(var_smoothing=1e-9).fit(x, y)
    np.testing.assert_allclose(f.theta, sk.theta_, rtol=1e-12, atol=1e-14)
    np.testing.assert_allclose(f.sigma, sk.var_, rtol=1e-10)
    np.testing.assert_allclose(nbo.probability(nbo.raw(f, x[:200])), sk.predict_proba(x[:200]), rtol=1e-8, atol=1e-12)


@pytest.mark.parametrize("lam", [1.0, 0.5])
def test_bernoulli_against_sklearn(lam):
    from sklearn.naive_bayes import BernoulliNB
    x, y = _data(kind="binary")
    f = nbo.fit(x, y, 4, "bernoulli", lam)
    sk = BernoulliNB(alpha=lam, binarize=None).fit(x, y)
    np.testing.assert_allclose(f.theta, sk.feature_log_prob_, rtol=1e-12)


@pytest.mark.parametrize("lam", [1.0, 0.5])
def test_complement_against_sklearn(lam):
    from sklearn.naive_bayes import ComplementNB
    x, y = _data(kind="counts")
    f = nbo.fit(x, y, 4, "complement", lam)
    sk = ComplementNB(alpha=lam, norm=False).fit(x, y)
    np.testing.assert_allclose(f.theta, sk.feature_log_prob_, rtol=1e-12)


def test_absent_class_is_never_predicted():
    x, y = _data(C=3)
    for mt in nbo.MODEL_TYPES:
        f = nbo.fit(x, y, 5, mt, 1.0)
        assert list(f.present) == [True, True, True, False, False]
        assert np.all(f.pi[3:] == -np.inf) and np.all(f.theta[3:] == 0.0)
        r = nbo.raw(f, x[:50])
        assert np.all(r[:, 3:] == -np.inf) and np.all(np.argmax(r, 1) < 3)


def _frame(weights=False):
    from pyspark.sql import ColumnData, DataFrame
    cols = {"features": ColumnData("vector", torch.from_numpy(ROWS_X), "f64"),
            "label": ColumnData("numeric", torch.from_numpy(ROWS_Y), "f64")}
    if weights:
        cols["w"] = ColumnData("numeric", torch.from_numpy(ROWS_W), "f64")
    return DataFrame(3, None, None, {}, cols)


def test_shim_params():
    from pyspark.ml.classification import NaiveBayes, NaiveBayesModel
    nb = NaiveBayes(modelType="gaussian", weightCol="w", smoothing=0.5)
    assert nb.getOrDefault("modelType") == "gaussian" and nb.getOrDefault("weightCol") == "w"
    assert NaiveBayes().getOrDefault("weightCol") is None
    assert NaiveBayesModel.hasParam(NaiveBayesModel, "modelType")


@pytest.mark.parametrize("kw,msg", [({"modelType": "poisson"}, "modelType must be one of"),
                                    ({"smoothing": -0.5}, "smoothing must be >= 0"),
                                    ({"smoothing": float("nan")}, "smoothing must be >= 0"),
                                    ({"weightCol": "missing"}, "Field \"missing\" does not exist")])
def test_shim_refusals(kw, msg):
    from pyspark.ml.classification import NaiveBayes
    from pyspark.ml.feature import IllegalArgumentException
    with pytest.raises(IllegalArgumentException, match=msg):
        NaiveBayes(**kw).fit(_frame(weights=True))
