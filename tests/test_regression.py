"""DecisionTreeRegressor / RandomForestRegressor and RegressionEvaluator without a GPU: the restated tree against
scikit-learn, the restated evaluator against sklearn.metrics, the label grid at its edges, and the shim's params and
refusals."""
import math

import numpy as np
import pytest
import torch

import oracle
import regression_oracle as ro


def test_restated_decision_tree_matches_scikit_learn():
    """one tree on real labels with integer-valued features (MLlib's midpoint thresholds are then scikit-learn's): the same
    structure, and leaf values within 1e-9"""
    from sklearn.tree import DecisionTreeRegressor
    rng = np.random.default_rng(5)
    n, F = 3000, 6
    x = rng.integers(0, 6, (n, F)).astype(np.float64)
    target = 1000.0 * (np.sin(x[:, 0]) + 0.5 * x[:, 1] * (x[:, 2] > 2) + 0.3 * rng.standard_normal(n)) - 250.0
    depth = 4
    model = ro.fit(x, target, np.zeros(F, np.int32), num_trees=1, max_depth=depth, bootstrap=False)
    assert model["E"] == 12 and model["m"] == F
    nodes, thr = model["trees"][0], model["thresholds"]
    sk = DecisionTreeRegressor(criterion="squared_error", max_depth=depth, random_state=0).fit(x, target).tree_

    def cmp(nid, k):
        nd = nodes[nid]
        if sk.children_left[k] < 0:
            assert nd["leaf"]
            assert abs(nd["payload"] - sk.value[k].ravel()[0]) <= 1e-9 * max(1.0, abs(sk.value[k].ravel()[0]))
            assert abs(nd["variance"] - sk.impurity[k]) <= 1e-9 * max(1.0, sk.impurity[k])
            return 1
        assert not nd["leaf"] and nd["feat"] == sk.feature[k] and thr[nd["feat"], nd["bin_thr"]] == sk.threshold[k]
        return cmp(2 * nid, sk.children_left[k]) + cmp(2 * nid + 1, sk.children_right[k])
    assert cmp(1, 0) == sum(1 for nd in nodes.values() if nd["leaf"]) and sk.node_count == len(nodes)
    pred, var = ro.predict_x(model, x)
    assert np.max(np.abs(pred - DecisionTreeRegressor(max_depth=depth, random_state=0).fit(x, target).predict(x))) < 1e-9


@pytest.mark.parametrize("seed", [0, 1])
def test_restated_metrics_match_sklearn(seed):
    from sklearn.metrics import explained_variance_score, mean_absolute_error, mean_squared_error, r2_score
    rng = np.random.default_rng(seed)
    n = 20000
    y = rng.standard_normal(n) * 50.0 + 7.0
    p = y + rng.standard_t(2, n) * 3.0                   # heavy-tailed errors
    got = ro.metrics(y, p)
    want = dict(mse=mean_squared_error(y, p), mae=mean_absolute_error(y, p), r2=r2_score(y, p))
    want["rmse"] = math.sqrt(want["mse"])
    want["var"] = float(np.mean((p - y.mean()) ** 2))
    for k, v in want.items():
        assert abs(got[k] - v) <= 1e-12 * abs(v), k
    assert abs(ro.metrics(y, p, through_origin=True)["r2"] - (1 - np.sum((y - p) ** 2) / np.sum(y * y))) < 1e-12
    assert explained_variance_score(y, p) <= 1.0


def test_metric_edge_cases():
    nan = ro.metrics(np.array([1.0, np.nan]), np.array([1.0, 2.0]))
    assert all(math.isnan(v) for v in nan.values())
    assert all(math.isnan(v) for v in ro.metrics(np.zeros(0), np.zeros(0)).values())
    const = ro.metrics(np.full(5, 3.0), np.full(5, 3.0))
    assert const["mse"] == 0.0 and math.isnan(const["r2"])
    assert ro.metrics(np.full(5, 3.0), np.full(5, 4.0))["r2"] == -math.inf


def test_exact_sum_is_exact_and_order_free():
    rng = np.random.default_rng(2)
    t = np.concatenate([rng.standard_normal(5000) * 1e6, [1e-3, -1e-3, 2.0 ** -30]])
    exact = ro.exact_sum(t, t.size)
    assert exact == ro.exact_sum(t[::-1], t.size) == ro.exact_sum(rng.permutation(t), t.size)
    from fractions import Fraction
    assert abs(exact - float(sum(Fraction(v) for v in t.tolist()))) <= abs(exact) * 2.0 ** -52


@pytest.mark.parametrize("ys", [np.zeros(7), np.array([4.0, -4.0, 1.0, 0.5]), np.array([-3.0, -1.5, -0.25]),
                                np.array([1e9, -9.99e8, 3.0, 1.0]), np.array([1e-9, -2e-9, 3e-10])],
                         ids=["zeros", "power_of_two", "negative", "1e9", "1e-9"])
@pytest.mark.parametrize("w_max", [1, 2, 4898431 * 3])
def test_label_grid_bound(ys, w_max):
    """|y'| <= 1, every cell sum stays below 2^62, the device formula equals the restatement, and the grid keeps the labels
    to 2^-S relative"""
    from b200flow import regression as br
    M = float(np.abs(ys).max())
    E, S, S2 = ro.label_grid(M, w_max)
    assert (E, S, S2) == br.label_grid(M, w_max)
    assert M <= 2.0 ** E and (M == 0.0 or M > 2.0 ** (E - 1))
    q, q2 = ro.to_grid(ys, E, S, S2)
    assert np.abs(q).max() <= 2 ** S and q2.max() <= 2 ** S2 and (q2 >= 0).all()
    assert w_max * (2 ** S) <= 2 ** 61 and w_max * (2 ** S2) <= 2 ** 61 and 2 * max(w_max, 2) * (2 ** S) > 2 ** 61
    back = q.astype(np.float64) * 2.0 ** -(S - E)
    assert np.all(np.abs(back - ys) <= 2.0 ** (E - S))
    if M > 0 and M == 2.0 ** E:                          # max |y| an exact power of two sits on the grid's edge, exactly
        assert np.abs(q).max() == 2 ** S


def test_label_grid_limits():
    from b200flow import regression as br
    assert br.label_grid(2.0 ** 300, 10)[0] == 300
    with pytest.raises(ValueError):
        br.label_grid(2.0 ** 300 * 1.5, 10)
    assert br.label_grid(5e-324, 10)[0] == br.E_MIN


def test_param_defaults_and_auto_strategy():
    from pyspark.ml.regression import DecisionTreeRegressor, RandomForestRegressor
    from b200flow import regression as br
    rf = RandomForestRegressor()
    assert (rf.getOrDefault("numTrees"), rf.getOrDefault("maxDepth"), rf.getOrDefault("maxBins"),
            rf.getOrDefault("minInstancesPerNode"), rf.getOrDefault("minInfoGain"), rf.getOrDefault("impurity"),
            rf.getOrDefault("featureSubsetStrategy"), rf.getOrDefault("subsamplingRate"), rf.getOrDefault("varianceCol")) == \
        (20, 5, 32, 1, 0.0, "variance", "auto", 1.0, None)
    dt = DecisionTreeRegressor()
    assert dt.getOrDefault("maxDepth") == 5 and dt.getOrDefault("impurity") == "variance" and not dt.hasParam("numTrees")
    assert br.resolve_strategy("auto", 20) == "onethird" and br.resolve_strategy("auto", 1) == "all"
    assert br.resolve_strategy("sqrt", 20) == "sqrt"
    mpb, kind, m = oracle.build_metadata(1000, 41, 2, [0] * 41, 32, 20, br.resolve_strategy("auto", 20))
    assert m == 14


@pytest.mark.parametrize("cls,kw", [("DecisionTreeRegressor", dict(impurity="gini")),
                                    ("RandomForestRegressor", dict(impurity="entropy")),
                                    ("RandomForestRegressor", dict(numTrees=0)),
                                    ("RandomForestRegressor", dict(subsamplingRate=0.0)),
                                    ("DecisionTreeRegressor", dict(maxBins=1))])
def test_param_refusals(cls, kw):
    import pyspark.ml.regression as R
    from pyspark.ml.feature import IllegalArgumentException
    est = getattr(R, cls)(**kw)
    with pytest.raises(IllegalArgumentException):
        est._params(est.getOrDefault("numTrees") if est.hasParam("numTrees") else 1, "all",
                    est.getOrDefault("subsamplingRate") if est.hasParam("subsamplingRate") else 1.0, True)


def test_evaluator_params():
    from pyspark.ml.evaluation import RegressionEvaluator
    ev = RegressionEvaluator()
    assert ev.getOrDefault("metricName") == "rmse" and ev.getOrDefault("throughOrigin") is False
    assert [RegressionEvaluator(metricName=m).isLargerBetter() for m in ("rmse", "mse", "r2", "mae", "var")] == \
        [False, False, True, False, True]
    with pytest.raises(ValueError):
        RegressionEvaluator(metricName="mape")._check()
    with pytest.raises(NotImplementedError):
        RegressionEvaluator(weightCol="w")._check()


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the refusal without a CUDA device")
def test_shim_raises_without_cuda():
    from b200flow._lib import B200FlowError
    from pyspark.ml.evaluation import RegressionEvaluator
    from pyspark.ml.regression import DecisionTreeRegressor, RandomForestRegressor
    from pyspark.sql import ColumnData, DataFrame
    x = torch.zeros((4, 2), dtype=torch.float64)
    y = torch.tensor([0.0, 1.0, 2.5, -1.0], dtype=torch.float64)
    df = DataFrame(4, None, None, {}, {"features": ColumnData("vector", x, "f64"), "label": ColumnData("numeric", y, "f64"),
                                       "prediction": ColumnData("numeric", y, "f64")})
    for est in (DecisionTreeRegressor(), RandomForestRegressor(numTrees=2)):
        with pytest.raises(B200FlowError):
            est.fit(df)
    with pytest.raises(B200FlowError):
        RegressionEvaluator().evaluate(df)
