"""GBTClassifier without a GPU: the shared exp (csrc/portable_exp.h, compiled for the host) against libm and the numpy
restatement, the restated regression tree against scikit-learn, a hand-worked two-iteration boost, and the shim's refusals."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

import gbt_oracle as go

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def pexp_host(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("pexp") / "libpexp.so")
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-std=c++17", "-ffp-contract=off", "-I",
                           os.path.join(ROOT, "spark-network-traffic-classifier_b200", "csrc"),
                           os.path.join(ROOT, "tests", "native", "portable_exp_host.cpp"), "-o", out])
    lib = C.CDLL(out)

    def run(x):
        x = np.ascontiguousarray(x, np.float64)
        y = np.empty_like(x)
        lib.pexp_batch(C.c_void_p(x.ctypes.data), C.c_int64(x.size), C.c_void_p(y.ctypes.data))
        return y
    return run


def _libm(v):
    try:
        return math.exp(v)
    except OverflowError:
        return math.inf


def test_exp_within_one_ulp_of_libm_and_equal_to_the_restatement(pexp_host):
    x = np.concatenate([np.linspace(-746.0, 710.0, 2_000_001), np.random.default_rng(3).uniform(-1.0, 1.0, 200_000),
                        2.0 ** -np.arange(1, 60), -(2.0 ** -np.arange(1, 60))])
    got = pexp_host(x)
    want = np.array([_libm(v) for v in x.tolist()])
    ulp = np.abs(got.view(np.int64) - want.view(np.int64))
    assert ulp.max() <= 1
    assert np.array_equal(got.view(np.int64), go.pexp(x).view(np.int64))


def test_exp_special_values_overflow_and_underflow(pexp_host):
    o = 7.09782712893383973096e+02
    u = -7.45133219101941108420e+02
    x = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, o, np.nextafter(o, np.inf), u, np.nextafter(u, -np.inf), -744.44, -708.5,
                  5e-324, -5e-324, 1e-300])
    got = pexp_host(x)
    assert got[0] == 1.0 and got[1] == 1.0 and got[2] == np.inf and got[3] == 0.0 and np.isnan(got[4])
    want = np.array([_libm(v) for v in x[5:].tolist()])
    assert np.array_equal(got[5:] == np.inf, want == np.inf) and np.array_equal(got[5:] == 0.0, want == 0.0)
    assert np.abs(got[5:].view(np.int64) - want.view(np.int64)).max() <= 1     # subnormal results: 1 ulp of the subnormal grid
    assert np.array_equal(got.view(np.int64)[~np.isnan(got)], go.pexp(x).view(np.int64)[~np.isnan(got)])


def test_residual_is_defined_for_infinite_and_nan_margins():
    y = np.array([1.0, 1.0, -1.0, -1.0, 1.0, -1.0])
    F = np.array([np.inf, -np.inf, np.inf, -np.inf, np.nan, np.nan])
    r = go.residual(y, F)
    q, q2 = go.to_grid(r, 40, 38)
    assert list(r[:4]) == [0.0, 4.0, -4.0, 0.0] or list(r[:4]) == [0.0, 4.0, -4.0, -0.0]
    assert list(q) == [0, 4 << 40, -(4 << 40), 0, 0, 0] and list(q2) == [0, 16 << 38, 16 << 38, 0, 0, 0]


def test_regression_tree_matches_scikit_learn():
    """one tree on real-valued targets: with integer-valued features (few distinct values, so MLlib's midpoint thresholds are
    scikit-learn's) the structure is the same and the leaf values agree to 1e-9"""
    from sklearn.tree import DecisionTreeRegressor
    rng = np.random.default_rng(5)
    n, F = 3000, 6
    x = rng.integers(0, 6, (n, F)).astype(np.float64)
    target = np.sin(x[:, 0]) + 0.5 * x[:, 1] * (x[:, 2] > 2) + 0.3 * rng.standard_normal(n)
    arity = np.zeros(F, np.int32)
    mpb, kind, m = 32, np.zeros(F, np.int32), F
    thr, n_thr, _ = __import__("oracle").find_splits(x, 0, 1 << 32, arity, mpb)
    tp, _ = __import__("oracle").bin_rows(x, thr, n_thr, arity, mpb)
    bins = tp[:, :F]
    feat_bins = (n_thr + 1).astype(np.int32)
    S, S2 = go.grid_shift(n)
    q, q2 = go.to_grid(target, S, S2)
    depth = 4
    nodes = go.grow_tree(0, bins, np.ones(n, np.int64), q, q2, feat_bins, kind, m, depth, 1, 0.0, 0, S, S2)
    sk = DecisionTreeRegressor(criterion="squared_error", max_depth=depth, random_state=0).fit(x, target).tree_

    def cmp(nid, k):
        nd = nodes[nid]
        if sk.children_left[k] < 0:
            assert nd["leaf"]
            assert abs(go.leaf_value(nd, 1.0, S) - sk.value[k].ravel()[0]) <= 1e-9
            return 1
        assert not nd["leaf"] and nd["feat"] == sk.feature[k] and thr[nd["feat"], nd["bin_thr"]] == sk.threshold[k]
        return cmp(2 * nid, sk.children_left[k]) + cmp(2 * nid + 1, sk.children_right[k])
    assert cmp(1, 0) == sum(1 for nd in nodes.values() if nd["leaf"]) and sk.node_count == len(nodes)


def test_two_iterations_by_hand():
    """x = [0, 0, 0, 1, 1, 1], labels [0, 0, 1, 1, 1, 0], maxDepth 1, stepSize 0.1"""
    bins = np.array([[0], [0], [0], [1], [1], [1]], np.uint8)
    labels = np.array([0, 0, 1, 1, 1, 0])
    trees, weights, Fm, S = go.boost(bins, labels, np.ones((1, 6), np.int64), np.array([2], np.int32), np.zeros(1, np.int32), 1,
                                     2, 0.1, 1, 1, 0.0, 0)
    assert weights == [1.0, 0.1] and S == 57
    t0, t1 = trees
    assert t0[1]["feat"] == 0 and t0[1]["bin_thr"] == 0 and abs(t0[2]["payload"] + 1 / 3) < 1e-15 and abs(t0[3]["payload"] - 1 / 3) < 1e-15
    a, b = 4.0 / (1.0 + math.exp(2.0 / 3.0)), 4.0 / (1.0 + math.exp(-2.0 / 3.0))   # |r| of the rows the first tree fits / misses
    left = (-2 * a + b) / 3                                                          # rows x=0: y = -1, -1, +1 at F = -1/3
    right = (2 * a - b) / 3                                                          # rows x=1: y = +1, +1, -1 at F = +1/3
    assert abs(t1[2]["payload"] - 0.1 * left) < 1e-15 and abs(t1[3]["payload"] - 0.1 * right) < 1e-15
    want = np.array([-1 / 3 + 0.1 * left] * 3 + [1 / 3 + 0.1 * right] * 3)
    assert np.max(np.abs(Fm - want)) < 1e-15
    y = np.where(labels > 0, 1.0, -1.0)
    r = go.residual(y, Fm)
    assert np.max(np.abs(r - 4 * y / (1 + np.exp(2 * y * want)))) < 1e-14
    mg, raw, prob, pred = go.predict(dict(trees=trees), bins)
    assert np.array_equal(mg, Fm) and list(pred) == [0, 0, 0, 1, 1, 1] and np.allclose(prob[:, 0], 1 / (1 + np.exp(2 * Fm)))


@pytest.mark.parametrize("kw", [dict(lossType="squared"), dict(impurity="gini"), dict(validationIndicatorCol="v"),
                                dict(weightCol="w"), dict(minWeightFractionPerNode=0.1), dict(maxIter=0), dict(stepSize=0.0),
                                dict(subsamplingRate=1.5)])
def test_param_refusals(kw):
    from pyspark.ml.classification import GBTClassifier
    from pyspark.ml.feature import IllegalArgumentException
    with pytest.raises(IllegalArgumentException):
        GBTClassifier(**kw)._params()


def test_defaults_are_sparks():
    from pyspark.ml.classification import GBTClassifier
    g = GBTClassifier()
    assert (g.getMaxIter(), g.getStepSize(), g.getMaxDepth(), g.getMaxBins(), g.getMinInstancesPerNode(), g.getMinInfoGain(),
            g.getSubsamplingRate(), g.getFeatureSubsetStrategy(), g.getLossType(), g.getImpurity()) == \
        (20, 0.1, 5, 32, 1, 0.0, 1.0, "all", "logistic", "variance")
    p = g.setSeed(3)._params()
    assert p.max_iter == 20 and p.seed == 3


def _cpu_frame(labels, meta=None):
    import torch
    from pyspark.sql import ColumnData, DataFrame
    y = torch.tensor(labels, dtype=torch.float64)
    x = torch.zeros((len(labels), 2), dtype=torch.float64)
    return DataFrame(len(labels), None, None, {}, {"features": ColumnData("vector", x, "f64"),
                                                   "label": ColumnData("numeric", y, "f64", meta=meta or {})})


@pytest.mark.parametrize("labels,meta", [([0, 1, 2, 1], None),                                    # a label 2
                                         ([0, 1, 1, 0], {"ml_attr": {"type": "nominal", "vals": ["a", "b", "c"]}})])  # 3 classes
def test_more_than_two_classes_are_refused(labels, meta):
    from pyspark.ml.classification import GBTClassifier
    from pyspark.ml.feature import IllegalArgumentException
    with pytest.raises(IllegalArgumentException, match="binary classification"):
        GBTClassifier().fit(_cpu_frame(labels, meta))
