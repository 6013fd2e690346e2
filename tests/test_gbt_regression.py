"""GBTRegressor without a GPU: the restated boosting loop against a loop of scikit-learn regression trees, a small
absolute-loss fit worked by hand, the residual-grid exponent at its edges, and the shim's params and refusals."""
import numpy as np
import pytest
import torch

import gbt_regression_oracle as gro
import regression_oracle as ro


def test_restated_boosting_matches_a_loop_of_scikit_learn_trees():
    """tree 0 fits y with weight 1.0, tree m fits 2 (y - F) with weight stepSize: on integer-valued features (MLlib's
    midpoint thresholds are then scikit-learn's, and the bins cover every distinct value) every tree has the same structure,
    its leaves agree within 1e-9, and so do the predictions"""
    from sklearn.tree import DecisionTreeRegressor
    rng = np.random.default_rng(11)
    n, F = 2500, 5
    x = rng.integers(0, 6, (n, F)).astype(np.float64)
    y = 40.0 * np.sin(x[:, 0]) + 7.0 * x[:, 1] * (x[:, 2] > 2) - 3.0 * x[:, 3] + 5.0 * rng.standard_normal(n) + 12.0
    depth, iters, step = 3, 5, 0.5
    model = gro.fit(x, y, np.zeros(F, np.int32), max_iter=iters, step_size=step, max_depth=depth)
    thr = model["thresholds"]
    Fm = np.zeros(n)
    for t in range(iters):
        target = y if t == 0 else 2.0 * (y - Fm)
        sk_tree = DecisionTreeRegressor(max_depth=depth, random_state=0).fit(x, target)
        sk = sk_tree.tree_
        nodes = model["trees"][t]

        def cmp(nid, k):
            nd = nodes[nid]
            if sk.children_left[k] < 0:
                v = sk.value[k].ravel()[0]
                assert nd["leaf"] and abs(nd["value"] - v) <= 1e-9 * max(1.0, abs(v)), (t, nid)
                return 1
            assert not nd["leaf"] and nd["feat"] == sk.feature[k] and thr[nd["feat"], nd["bin_thr"]] == sk.threshold[k], (t, nid)
            return cmp(2 * nid, sk.children_left[k]) + cmp(2 * nid + 1, sk.children_right[k])
        assert cmp(1, 0) == sum(1 for nd in nodes.values() if nd["leaf"]) and sk.node_count == len(nodes)
        Fm = Fm + (1.0 if t == 0 else step) * sk_tree.predict(x)
    assert np.max(np.abs(model["margin"] - Fm)) <= 1e-9 * np.max(np.abs(Fm))
    assert np.max(np.abs(gro.predict_x(model, x) - Fm)) <= 1e-9 * np.max(np.abs(Fm))
    assert model["weights"] == [1.0] + [step] * (iters - 1)
    assert len(set(model["E"])) > 1                  # the residuals' scale is not the labels'


def test_absolute_loss_by_hand():
    """x in {0, 1}, y = [1, 3, 4 | 10, 14, 15], depth 1, stepSize 0.5.  Tree 0 splits at 0.5 with leaves 8/3 and 13 (E_0 = 4,
    max |y| = 15).  y - F = [-5/3, 1/3, 4/3, -3, 1, 2] gives r = [-1, 1, 1, -1, 1, 1] (E_1 = 0): both sides have the root's
    mean 1/3 and variance 8/9, a gain of 0, so tree 1 is one leaf that keeps the mean 1/3 (not the median 1: Spark does not
    refit the leaves) and has payload 1/6."""
    x = np.array([[0.0], [0.0], [0.0], [1.0], [1.0], [1.0]])
    y = np.array([1.0, 3.0, 4.0, 10.0, 14.0, 15.0])
    model = gro.fit(x, y, [0], max_iter=2, step_size=0.5, max_depth=1, loss="absolute")
    t0, t1 = model["trees"]
    assert model["E"] == [4, 0] and model["thresholds"][0, 0] == 0.5
    assert not t0[1]["leaf"] and t0[2]["payload"] == 8.0 / 3.0 and t0[3]["payload"] == 13.0
    assert list(t1) == [1] and t1[1]["leaf"] and t1[1]["value"] == 1.0 / 3.0 and t1[1]["payload"] == 0.5 * (1.0 / 3.0)
    want = np.array([8.0 / 3.0] * 3 + [13.0] * 3) + 0.5 * (1.0 / 3.0)
    assert np.array_equal(model["margin"], want)
    assert np.array_equal(gro.residual(y, want, "absolute"), np.sign(y - want) + (y == want))


@pytest.mark.parametrize("M,E", [(0.0, 0), (1.0, 0), (2.0 ** 40, 40), (2.0 ** -40, -40), (3.0, 2), (2.0 ** -300, -300),
                                 (2.0 ** -301, -300), (5e-324, -300), (2.0 ** 300, 300)],
                         ids=["zero", "one", "2^40", "2^-40", "three", "2^-300", "2^-301", "denormal", "2^300"])
def test_residual_exponent_edges(M, E):
    from b200flow import gbt_regression as bgr
    assert bgr.residual_exponent(M) == gro.residual_exponent(M) == E
    if M > 0 and E > -300:
        assert M <= 2.0 ** E and M > 2.0 ** (E - 1)      # an exact power of two keeps its own exponent: |r'| <= 1 exactly


@pytest.mark.parametrize("M", [2.0 ** 301, 2.0 ** 300 * 1.0000001])
def test_residual_exponent_refuses_beyond_2_300(M):
    from b200flow import gbt_regression as bgr
    with pytest.raises(ValueError, match="residual"):
        bgr.residual_exponent(M)
    with pytest.raises(ValueError):
        gro.residual_exponent(M)


def test_grid_of_a_power_of_two_residual_sits_on_the_edge():
    E = gro.residual_exponent(2.0 ** 7)
    _, S, S2 = ro.label_grid(1.0, 1000)
    q, q2 = ro.to_grid(np.array([2.0 ** 7, -2.0 ** 7, 3.0]), E, S, S2)
    assert q[0] == 2 ** S and q[1] == -2 ** S and q2[0] == 2 ** S2


def test_constant_labels_leave_zero_residuals():
    rng = np.random.default_rng(1)
    x = rng.integers(0, 4, (400, 3)).astype(np.float64)
    model = gro.fit(x, np.full(400, 2.75), [0, 0, 0], max_iter=3, max_depth=2)
    assert model["E"] == [2, 0, 0] and np.array_equal(model["margin"], np.full(400, 2.75))
    assert all(nd["leaf"] for nodes in model["trees"] for nd in nodes.values())


def test_huge_residuals_are_refused_by_the_restatement():
    x = np.array([[0.0], [1.0]] * 4)
    y = np.array([0.9, -0.9] * 4) * 2.0 ** 300                         # depth 0: tree 0 is the mean 0, r = 2y > 2^300
    with pytest.raises(ValueError, match="residual"):
        gro.fit(x, y, [0], max_iter=2, max_depth=0)
    assert gro.fit(x, y, [0], max_iter=2, max_depth=0, loss="absolute")["E"] == [300, 0]


def test_param_defaults_and_auto_strategy():
    from pyspark.ml.regression import GBTRegressor
    from b200flow import gbt_regression as bgr
    g = GBTRegressor()
    want = dict(maxIter=20, stepSize=0.1, maxDepth=5, maxBins=32, minInstancesPerNode=1, minInfoGain=0.0, lossType="squared",
                subsamplingRate=1.0, impurity="variance", featureSubsetStrategy="all", validationTol=0.01,
                validationIndicatorCol=None, weightCol=None, minWeightFractionPerNode=0.0, leafCol="", maxMemoryInMB=256,
                cacheNodeIds=False, checkpointInterval=10, seed=None, labelCol="label", featuresCol="features",
                predictionCol="prediction")
    assert {k: g.getOrDefault(k) for k in want} == want
    assert not g.hasParam("varianceCol") and not g.hasParam("probabilityCol")
    p = GBTRegressor(featureSubsetStrategy="auto", seed=5, lossType="absolute")._params()
    assert p.feature_subset_strategy == "all" and p.loss == "absolute" and p.seed == 5
    assert GBTRegressor(featureSubsetStrategy="sqrt")._params().feature_subset_strategy == "sqrt"
    assert bgr.GBTRegressorParams() == bgr.GBTRegressorParams(max_iter=20, step_size=0.1, max_depth=5, max_bins=32, loss="squared")


@pytest.mark.parametrize("kw", [dict(lossType="huber"), dict(lossType="logistic"), dict(impurity="gini"),
                                dict(validationIndicatorCol="v"), dict(weightCol="w"), dict(minWeightFractionPerNode=0.1),
                                dict(maxIter=0), dict(stepSize=0.0), dict(stepSize=1.5), dict(subsamplingRate=0.0),
                                dict(maxBins=1), dict(maxDepth=-1)],
                         ids=lambda kw: "%s=%s" % next(iter(kw.items())))
def test_param_refusals(kw):
    from pyspark.ml.feature import IllegalArgumentException
    from pyspark.ml.regression import GBTRegressor
    with pytest.raises(IllegalArgumentException):
        GBTRegressor(**kw)._params()


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the refusal without a CUDA device")
def test_shim_raises_without_cuda():
    from b200flow._lib import B200FlowError
    from b200flow import gbt_regression as bgr
    from pyspark.ml.regression import GBTRegressor
    from pyspark.sql import ColumnData, DataFrame
    x = torch.zeros((4, 2), dtype=torch.float64)
    y = torch.tensor([0.0, 1.0, 2.5, -1.0], dtype=torch.float64)
    df = DataFrame(4, None, None, {}, {"features": ColumnData("vector", x, "f64"), "label": ColumnData("numeric", y, "f64")})
    with pytest.raises(B200FlowError):
        GBTRegressor().fit(df)
    with pytest.raises(B200FlowError):
        bgr.fit_gbt_regressor(x, y, [0, 0], bgr.GBTRegressorParams())
