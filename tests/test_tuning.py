"""Model selection without a GPU: Param objects and ParamGridBuilder of the pyspark.ml shim, the fit groups of
b200flow.tuning, and — on the CPU oracle — the premise of the one-fit-per-group fast path: the forest fitted with (T, d) is
the first T trees of the (T_max, d_max) forest cut at depth d (DESIGN.md §5a)."""
import numpy as np
import pytest

import oracle
from b200flow.tuning import fit_groups
from util import forests_equal


# ------------------------------------------------------------------ 1. Param objects and the grid builder
def test_param_objects_and_grid_builder_order():
    from pyspark.ml.classification import RandomForestClassifier, DecisionTreeClassifier
    from pyspark.ml.param import Param
    from pyspark.ml.tuning import ParamGridBuilder
    rf = RandomForestClassifier(labelCol="label_num", maxBins=70)
    assert isinstance(rf.numTrees, Param) and rf.numTrees.name == "numTrees" and rf.numTrees == rf.numTrees
    assert rf.numTrees != rf.maxDepth and rf.numTrees != RandomForestClassifier().numTrees
    with pytest.raises(AttributeError):
        rf.noSuchParam
    grid = (ParamGridBuilder().addGrid(rf.numTrees, [20, 50, 100]).addGrid(rf.maxDepth, [5, 10, 16])
            .baseOn({rf.maxBins: 64}).build())
    assert len(grid) == 9
    assert [(g[rf.numTrees], g[rf.maxDepth]) for g in grid] == [(t, d) for t in (20, 50, 100) for d in (5, 10, 16)]
    assert all(g[rf.maxBins] == 64 and len(g) == 3 for g in grid)
    assert ParamGridBuilder().baseOn((rf.seed, 3)).build() == [{rf.seed: 3}]
    assert ParamGridBuilder().build() == [{}]
    # Param-keyed maps carry the value; the original is untouched
    c = rf.copy({rf.numTrees: 5})
    assert c.getOrDefault("numTrees") == 5 and c.getOrDefault(c.numTrees) == 5 and c.isSet(rf.numTrees)
    assert rf.getOrDefault("numTrees") == 20 and not rf.isSet(rf.numTrees) and rf.getNumTrees() == 20
    assert c.uid == rf.uid
    with pytest.raises(ValueError):
        rf.getOrDefault(DecisionTreeClassifier().maxDepth)
    # name-keyed maps and the string setters / getters behave as before
    assert rf.copy({"maxDepth": 7}).getMaxDepth() == 7 and rf.getMaxDepth() == 5
    assert rf.setMaxDepth(9) is rf and rf.getOrDefault("maxDepth") == 9 and rf.isSet("maxDepth")
    assert rf.getLabelCol() == "label_num"
    with pytest.raises(TypeError):
        rf.copy({"noSuchParam": 1})


def test_fit_with_param_maps():
    from pyspark.ml import Estimator, Model, Pipeline
    from pyspark.ml.classification import RandomForestClassifier

    class Echo(Estimator):
        _defaults = {"k": 1, "tag": "x"}

        def _fit(self, df):
            m = Model()
            m.k, m.tag, m.df = self.getOrDefault("k"), self.getOrDefault("tag"), df
            return m

    e = Echo()
    m = e.fit("D", {e.k: 4})
    assert (m.k, m.tag, m.df) == (4, "x", "D") and e.getOrDefault("k") == 1
    ms = e.fit("D", [{e.k: 2}, {e.tag: "y"}, {"k": 3}])
    assert [(x.k, x.tag) for x in ms] == [(2, "x"), (1, "y"), (3, "x")]
    assert e.fit("D", ({e.k: 6},))[0].k == 6
    # a map of stage Params reaches the stage that owns it through Pipeline.copy; other stages ignore it
    rf, other = RandomForestClassifier(), Echo()
    p = Pipeline(stages=[other, rf]).copy({rf.numTrees: 7, other.k: 9})
    assert p.getStages()[1].getOrDefault("numTrees") == 7 and p.getStages()[0].getOrDefault("k") == 9
    assert rf.getOrDefault("numTrees") == 20 and other.getOrDefault("k") == 1


# ------------------------------------------------------------------ 2. fit groups
def _maps(points, **base):
    return [dict(base, numTrees=t, maxDepth=d) for t, d in points]


def test_fit_groups_full_grid():
    m = _maps([(t, d) for t in (20, 50, 100) for d in (5, 10, 16)], maxBins=32, seed=1)
    g = fit_groups(m)
    assert len(g) == 1
    T, d, members = g[0]
    assert (T, d) == (100, 16) and members == [(i, p["numTrees"], p["maxDepth"]) for i, p in enumerate(m)]


def test_fit_groups_split_out_numtrees_one_and_other_params():
    m = _maps([(1, 5), (1, 8), (10, 5), (10, 8)], maxBins=32) + _maps([(4, 3), (6, 2)], maxBins=64) + \
        _maps([(3, 9)], maxBins=32)
    g = fit_groups(m)
    assert g == [(1, 5, [(0, 1, 5)]), (1, 8, [(1, 1, 8)]),
                 (10, 9, [(2, 10, 5), (3, 10, 8), (6, 3, 9)]),
                 (6, 3, [(4, 4, 3), (5, 6, 2)])]


def test_fit_groups_ragged_grid_and_decision_tree():
    m = [dict(numTrees=5, maxDepth=2, seed=3), dict(numTrees=30, maxDepth=1, seed=3), dict(numTrees=2, maxDepth=7, seed=3),
         dict(numTrees=5, maxDepth=2, seed=4)]
    assert fit_groups(m) == [(30, 7, [(0, 5, 2), (1, 30, 1), (2, 2, 7)]), (5, 2, [(3, 5, 2)])]
    dt = [dict(maxDepth=d, maxBins=b) for d, b in ((3, 32), (0, 32), (6, 32), (4, 70))]
    assert fit_groups(dt, decision_tree=True) == [(1, 6, [(0, 1, 3), (1, 1, 0), (2, 1, 6)]), (1, 4, [(3, 1, 4)])]


# ------------------------------------------------------------------ 3. the premise on the CPU oracle
def cut_export(ex, T, d):
    """the first T trees of a canonical forest export, cut at depth d: nodes at depth d become leaves (their counts stay)."""
    ex = {k: np.asarray(v) for k, v in ex.items()}
    order = np.lexsort((ex["nid"], ex["tree"]))
    depth = np.floor(np.log2(ex["nid"][order].astype(np.float64))).astype(np.int64)
    sel = order[(ex["tree"][order] < T) & (depth <= d)]
    out = {k: v[sel].copy() for k, v in ex.items()}
    at = np.floor(np.log2(out["nid"].astype(np.float64))).astype(np.int64) == d
    out["is_leaf"][at] = 1
    out["feat"][at] = -1
    out["kind"][at] = 0
    out["bin_thr"][at] = 0
    out["mask"][at] = 0
    return out


def sorted_export(ex):
    ex = {k: np.asarray(v) for k, v in ex.items()}
    order = np.lexsort((ex["nid"], ex["tree"]))
    return {k: v[order] for k, v in ex.items()}


def _data(n, C, seed):
    """5 continuous features, a 3-value and a 4-value categorical (unordered for C > 2 at maxBins 32) and a 12-value one
    (ordered); labels depend on all of them, with noise, so the trees grow to full depth."""
    rng = np.random.default_rng(seed)
    cont = rng.standard_normal((n, 5))
    c3, c4, c12 = rng.integers(0, 3, n), rng.integers(0, 4, n), rng.integers(0, 12, n)
    x = np.column_stack([cont, c3, c12, c4]).astype(np.float64)
    score = cont[:, 0] * 2 + cont[:, 1] * cont[:, 2] + (c3 == 1) * 1.5 + c12 * 0.3 - (c4 == 2) + 0.5 * rng.standard_normal(n)
    y = np.clip(((score - score.min()) / (score.max() - score.min() + 1e-12) * C).astype(np.int32), 0, C - 1)
    return x, y, [0] * 5 + [3, 12, 4]


@pytest.mark.parametrize("C", [2, 5, 23])
def test_sub_forest_premise_on_the_oracle(C):
    x, y, arity = _data(3000, C, seed=C)
    big, _ = oracle.fit_forest(x, y, C, arity, num_trees=12, max_depth=6, seed=77)
    small, meta = oracle.fit_forest(x, y, C, arity, num_trees=5, max_depth=3, seed=77)
    if C > 2:
        assert {1, 2} <= set(meta["feat_kind"].tolist())              # ordered and unordered categorical splits both exist
    want = sorted_export(small.export())
    got = cut_export(big.export(), 5, 3)
    assert forests_equal(got, want) == []
    assert len(want["nid"]) > 5 * 7 and (want["is_leaf"] == 0).sum() > 5 * 3
    # the cut is not trivially the whole forest: the big forest goes deeper
    assert np.floor(np.log2(big.export()["nid"].max())) == 6


def test_sub_forest_premise_on_the_oracle_decision_tree():
    x, y, arity = _data(3000, 5, seed=11)
    big, _ = oracle.fit_forest(x, y, 5, arity, num_trees=1, max_depth=7, seed=5, strategy="all")
    for d in (0, 2, 4):
        small, _ = oracle.fit_forest(x, y, 5, arity, num_trees=1, max_depth=d, seed=5, strategy="all")
        assert forests_equal(cut_export(big.export(), 1, d), sorted_export(small.export())) == []
