"""pyspark.ml.regression shim: DecisionTreeRegressor, RandomForestRegressor and GBTRegressor on the device variance-tree
loop (b200flow/regression.py, b200flow/gbt_regression.py, csrc/regression.cu, DESIGN.md §5l, §5m).  Their models are the
same bits for any number of ranks.

Deviations from Spark: a NaN or infinite label raises IllegalArgumentException (Spark trains on it); labels (and GBT
residuals) beyond 2^300 in magnitude are refused; weightCol is not offered."""
import numpy as np
import torch

from b200flow import dist as bdist
from b200flow import forest as fr

from . import Estimator, Model
from ..sql import ColumnData
from .classification import _arity_from_attrs, _default_seed, _lazy_plan
from .feature import IllegalArgumentException

__all__ = ["DecisionTreeRegressionModel", "DecisionTreeRegressor", "GBTRegressionModel", "GBTRegressor",
           "RandomForestRegressionModel", "RandomForestRegressor"]


class _TreeRegressorParams:
    _defaults = {"featuresCol": "features", "labelCol": "label", "predictionCol": "prediction", "maxDepth": 5, "maxBins": 32,
                 "minInstancesPerNode": 1, "minInfoGain": 0.0, "maxMemoryInMB": 256, "cacheNodeIds": False,
                 "checkpointInterval": 10, "impurity": "variance", "seed": None, "varianceCol": None}


class _RandomForestRegressorParams(_TreeRegressorParams):
    _defaults = {"numTrees": 20, "featureSubsetStrategy": "auto", "subsamplingRate": 1.0}


class _TreeRegressorBase(Estimator):
    def _params(self, num_trees, strategy, subsampling, bootstrap):
        """Spark's param validators -> b200flow RegressorParams"""
        from b200flow import regression as br
        g = self.getOrDefault
        imp = str(g("impurity")).lower()
        if imp != "variance":
            raise IllegalArgumentException("%s impurity must be 'variance', got %r" % (type(self).__name__, g("impurity")))
        if int(g("maxBins")) < 2 or int(g("minInstancesPerNode")) < 1 or float(g("minInfoGain")) < 0.0 or int(g("maxDepth")) < 0:
            raise IllegalArgumentException("maxBins >= 2, minInstancesPerNode >= 1, minInfoGain >= 0 and maxDepth >= 0 are required")
        if int(num_trees) < 1:
            raise IllegalArgumentException("numTrees must be >= 1, got %r" % (num_trees,))
        if not 0.0 < float(subsampling) <= 1.0:
            raise IllegalArgumentException("subsamplingRate must be in (0, 1], got %r" % (subsampling,))
        seed = g("seed")
        return br.RegressorParams(num_trees=int(num_trees), max_depth=int(g("maxDepth")), max_bins=int(g("maxBins")),
                                  min_instances_per_node=int(g("minInstancesPerNode")), min_info_gain=float(g("minInfoGain")),
                                  feature_subset_strategy=str(strategy), subsampling_rate=float(subsampling),
                                  seed=_default_seed(self) if seed is None else int(seed), bootstrap=bootstrap)

    def _train(self, df, params, fit):
        fcol, lcol = self.getOrDefault("featuresCol"), self.getOrDefault("labelCol")
        for c in (fcol, lcol):
            if c not in df._cols:
                raise IllegalArgumentException("Field \"%s\" does not exist." % c)
        fc = df._cols[fcol]
        if fc.kind != "vector":
            raise IllegalArgumentException("Column %s must be of type vector" % fcol)
        x = fc.data                         # a lazy VectorAssembler column is assembled here, once
        y = df._column_tensor(lcol).to(torch.float64).reshape(-1).contiguous()
        try:
            grp = bdist.group()
            off, _ = bdist.global_offset(x.shape[0], x.device, grp)
            return fit(x, y, _arity_from_attrs(fc.meta.get("attrs"), x.shape[1]), params, row_offset=off, group=grp)
        except ValueError as e:        # includes b200flow's UnsupportedParamError; CUDA failures propagate as they are
            raise IllegalArgumentException(str(e))

    def _model(self, cls, reg):
        m = cls(reg)
        m._paramMap = {k: v for k, v in self._paramMap.items() if k in m._all_defaults()}
        return m


class DecisionTreeRegressor(_TreeRegressorBase, _TreeRegressorParams):
    """Spark 3's DecisionTreeRegressor: RandomForest.run with one tree, featureSubsetStrategy 'all', no bagging."""

    def __init__(self, featuresCol=None, labelCol=None, predictionCol=None, maxDepth=None, maxBins=None,
                 minInstancesPerNode=None, minInfoGain=None, maxMemoryInMB=None, cacheNodeIds=None, checkpointInterval=None,
                 impurity=None, seed=None, varianceCol=None):
        kw = dict(locals()); kw.pop("self"); kw.pop("__class__", None)
        super().__init__(**kw)

    def _fit(self, df):
        from b200flow import regression as br
        p = self._params(1, "all", 1.0, bootstrap=False)
        return self._model(DecisionTreeRegressionModel, self._train(df, p, br.fit_dt_regressor))


class RandomForestRegressor(_TreeRegressorBase, _RandomForestRegressorParams):
    """Spark 3's RandomForestRegressor: numTrees bagged regression trees; featureSubsetStrategy 'auto' is 'onethird' for
    more than one tree and 'all' for one."""

    def __init__(self, featuresCol=None, labelCol=None, predictionCol=None, maxDepth=None, maxBins=None,
                 minInstancesPerNode=None, minInfoGain=None, maxMemoryInMB=None, cacheNodeIds=None, checkpointInterval=None,
                 impurity=None, subsamplingRate=None, seed=None, numTrees=None, featureSubsetStrategy=None, varianceCol=None):
        kw = dict(locals()); kw.pop("self"); kw.pop("__class__", None)
        super().__init__(**kw)

    def _fit(self, df):
        from b200flow import regression as br
        T = self.getOrDefault("numTrees")
        if int(T) != T:
            raise IllegalArgumentException("numTrees must be an integer >= 1, got %r" % (T,))
        if self.getOrDefault("varianceCol"):
            raise IllegalArgumentException("varianceCol is only supported by DecisionTreeRegressor on the b200flow trainer")
        p = self._params(int(T), br.resolve_strategy(self.getOrDefault("featureSubsetStrategy"), int(T)),
                         self.getOrDefault("subsamplingRate"), bootstrap=True)
        return self._model(RandomForestRegressionModel, self._train(df, p, br.fit_rf_regressor))


class _RegressionModelBase(Model):
    def __init__(self, reg):
        super().__init__()
        self._reg = reg

    @property
    def numFeatures(self):
        return self._reg.F

    @property
    def totalNumNodes(self):
        return self._reg.n_nodes

    @property
    def featureImportances(self):
        from .linalg import DenseVector
        return DenseVector(self._reg.feature_importances())

    def _transform(self, df):
        fcol = self.getOrDefault("featuresCol")
        if fcol not in df._cols or df._cols[fcol].kind != "vector":
            raise IllegalArgumentException("Column %s must be of type vector" % fcol)
        vcol = self.getOrDefault("varianceCol") if self.hasParam("varianceCol") else None
        plan = _lazy_plan(df, fcol)
        fused = plan is not None and plan.n_out == self._reg.F      # lazy features: fused encode -> bins -> tree walk
        var = None
        from .feature import SparkException
        try:
            if vcol:
                if fused:
                    pred, var = self._reg.predict_with_variance(rec=df._rec, plan=plan,
                                                                on_invalid="error" if plan.check_nan else "ignore")
                else:
                    pred, var = self._reg.predict_with_variance(x=df._cols[fcol].data)
            elif fused:
                pred = self._reg.predict_records(df._rec, plan, on_invalid="error" if plan.check_nan else "ignore")
            else:
                pred = self._reg.predict(df._cols[fcol].data)
        except fr.InvalidRowsError as e:
            raise SparkException("Encountered NaN/null while assembling a row with handleInvalid = \"error\" (%s)" % e)
        cols = dict(df._cols)
        for name, val in ((self.getOrDefault("predictionCol"), pred), (vcol, var)):
            if name and val is not None:
                if name in cols:
                    raise IllegalArgumentException("Output column %s already exists." % name)
                cols[name] = ColumnData("numeric", val, "f64")
        return df._with(cols=cols)

    def _leaf_values(self, ex):
        """the value toDebugString prints for each exported node"""
        return ex["payload"]

    def _tree_lines(self, t):
        ex = self._reg.export()
        vals = self._leaf_values(ex)
        thr = self._reg.forest.thresholds.cpu().numpy()
        sel = np.nonzero(ex["tree"] == t)[0]
        idx = {int(ex["nid"][i]): i for i in sel}
        lines = []

        def rec(nid, depth):
            i = idx[nid]
            pad = " " * (depth + 1)
            if ex["is_leaf"][i]:
                lines.append("%sPredict: %r" % (pad, float(vals[i])))
                return
            f = int(ex["feat"][i])
            if ex["kind"][i] == 0:
                v = repr(float(thr[f, int(ex["bin_thr"][i])]))
                lines.append("%sIf (feature %d <= %s)" % (pad, f, v)); rec(nid * 2, depth + 1)
                lines.append("%sElse (feature %d > %s)" % (pad, f, v)); rec(nid * 2 + 1, depth + 1)
            else:
                cats = [c for c in range(256) if (int(ex["mask"][i][c >> 6]) >> (c & 63)) & 1]
                s = "{%s}" % ",".join("%.1f" % c for c in cats)
                lines.append("%sIf (feature %d in %s)" % (pad, f, s)); rec(nid * 2, depth + 1)
                lines.append("%sElse (feature %d not in %s)" % (pad, f, s)); rec(nid * 2 + 1, depth + 1)
        rec(1, 0)
        return len(sel), lines


class DecisionTreeRegressionModel(_RegressionModelBase, _TreeRegressorParams):
    @property
    def numNodes(self):
        return self._reg.n_nodes

    @property
    def depth(self):
        nid = self._reg.export()["nid"].astype(np.int64)
        return int(np.floor(np.log2(nid.max()))) if len(nid) else 0

    @property
    def toDebugString(self):
        nn, lines = self._tree_lines(0)
        return "DecisionTreeRegressionModel of depth %d with %d nodes\n%s\n" % (self.depth, nn, "\n".join(lines))

    def __repr__(self):
        return "DecisionTreeRegressionModel of depth %d with %d nodes" % (self.depth, self.numNodes)


class RandomForestRegressionModel(_RegressionModelBase, _RandomForestRegressorParams):
    @property
    def getNumTrees(self):
        return self._reg.T

    @property
    def treeWeights(self):
        return [1.0] * self._reg.T

    @property
    def toDebugString(self):
        parts = ["RandomForestRegressionModel with %d trees" % self._reg.T]
        for t in range(self._reg.T):
            parts.append("  Tree %d (weight 1.0):" % t)
            parts += ["  " + l for l in self._tree_lines(t)[1]]
        return "\n".join(parts) + "\n"

    def __repr__(self):
        return "RandomForestRegressionModel with %d trees" % self._reg.T


# ------------------------------------------------------------------------------- gradient-boosted trees
class _GBTRegressorParams:
    _defaults = {**{k: v for k, v in _TreeRegressorParams._defaults.items() if k != "varianceCol"},
                 "maxIter": 20, "stepSize": 0.1, "subsamplingRate": 1.0, "featureSubsetStrategy": "all", "lossType": "squared",
                 "validationTol": 0.01, "validationIndicatorCol": None, "weightCol": None, "minWeightFractionPerNode": 0.0,
                 "leafCol": ""}


class GBTRegressor(_TreeRegressorBase, _GBTRegressorParams):
    """Spark 3's GBTRegressor: boosting of regression trees under squared or absolute loss, trained on the device with a
    residual grid re-derived every iteration (b200flow/gbt_regression.py, DESIGN.md §5m); the model is the same bits for
    any number of ranks.  Under absolute loss the leaves keep the tree's mean, as Spark's do."""

    def __init__(self, featuresCol=None, labelCol=None, predictionCol=None, maxDepth=None, maxBins=None,
                 minInstancesPerNode=None, minInfoGain=None, maxMemoryInMB=None, cacheNodeIds=None, checkpointInterval=None,
                 lossType=None, maxIter=None, stepSize=None, seed=None, subsamplingRate=None, impurity=None,
                 featureSubsetStrategy=None, validationTol=None, validationIndicatorCol=None, leafCol=None,
                 minWeightFractionPerNode=None, weightCol=None):
        kw = dict(locals()); kw.pop("self"); kw.pop("__class__", None)
        super().__init__(**kw)

    def _params(self):
        """Spark's param validators, and the params the device trainer does not implement -> GBTRegressorParams"""
        from b200flow import gbt_regression as bgr
        g = self.getOrDefault
        loss = str(g("lossType")).lower()
        if loss not in bgr.LOSSES:
            raise IllegalArgumentException("GBTRegressor lossType must be 'squared' or 'absolute', got %r" % (g("lossType"),))
        if str(g("impurity")).lower() != "variance":
            raise IllegalArgumentException("GBTRegressor impurity must be 'variance', got %r" % (g("impurity"),))
        if g("validationIndicatorCol"):
            raise IllegalArgumentException("validationIndicatorCol (early stopping) is not supported by the b200flow GBT trainer")
        if g("weightCol"):
            raise IllegalArgumentException("weightCol is not supported by the b200flow GBT trainer")
        if float(g("minWeightFractionPerNode")) != 0.0:
            raise IllegalArgumentException("minWeightFractionPerNode must be 0.0 on the b200flow GBT trainer")
        it, step, rate = g("maxIter"), float(g("stepSize")), float(g("subsamplingRate"))
        if int(it) != it or int(it) < 1:
            raise IllegalArgumentException("maxIter must be an integer >= 1, got %r" % (it,))
        if not 0.0 < step <= 1.0:
            raise IllegalArgumentException("stepSize must be in (0, 1], got %r" % (step,))
        if not 0.0 < rate <= 1.0:
            raise IllegalArgumentException("subsamplingRate must be in (0, 1], got %r" % (rate,))
        if int(g("maxBins")) < 2 or int(g("minInstancesPerNode")) < 1 or float(g("minInfoGain")) < 0.0 or int(g("maxDepth")) < 0:
            raise IllegalArgumentException("maxBins >= 2, minInstancesPerNode >= 1, minInfoGain >= 0 and maxDepth >= 0 are required")
        strategy = str(g("featureSubsetStrategy"))
        seed = g("seed")
        return bgr.GBTRegressorParams(max_iter=int(it), step_size=step, max_depth=int(g("maxDepth")), max_bins=int(g("maxBins")),
                                      min_instances_per_node=int(g("minInstancesPerNode")), min_info_gain=float(g("minInfoGain")),
                                      subsampling_rate=rate, feature_subset_strategy="all" if strategy == "auto" else strategy,
                                      seed=_default_seed(self) if seed is None else int(seed), loss=loss)

    def _fit(self, df):
        from b200flow import gbt_regression as bgr
        return self._model(GBTRegressionModel, self._train(df, self._params(), bgr.fit_gbt_regressor))


class GBTRegressionModel(_RegressionModelBase, _GBTRegressorParams):
    @property
    def getNumTrees(self):
        return self._reg.T

    @property
    def treeWeights(self):
        return list(self._reg.tree_weights)

    def evaluateEachIteration(self, dataset, loss):
        """the mean loss ('squared' or 'absolute') of the model cut to its first m + 1 trees, for every m: RegressionEvaluator's
        mse / mae on each prefix model's predictions"""
        fcol, lcol = self.getOrDefault("featuresCol"), self.getOrDefault("labelCol")
        for c in (fcol, lcol):
            if c not in dataset._cols:
                raise IllegalArgumentException("Field \"%s\" does not exist." % c)
        if str(loss).lower() not in ("squared", "absolute"):
            raise IllegalArgumentException("loss must be 'squared' or 'absolute', got %r" % (loss,))
        y = dataset._column_tensor(lcol).to(torch.float64).reshape(-1).contiguous()
        return self._reg.evaluate_each_iteration(dataset._cols[fcol].data, y, str(loss).lower(), group=bdist.group())

    def _leaf_values(self, ex):
        return self._reg.leaf_values(ex)                 # unweighted, in label units, each tree on its own grid

    @property
    def toDebugString(self):
        parts = ["GBTRegressionModel with %d trees" % self._reg.T]
        for t in range(self._reg.T):
            parts.append("  Tree %d (weight %r):" % (t, self._reg.tree_weights[t]))
            parts += ["  " + l for l in self._tree_lines(t)[1]]
        return "\n".join(parts) + "\n"

    def __repr__(self):
        return "GBTRegressionModel with %d trees" % self._reg.T
