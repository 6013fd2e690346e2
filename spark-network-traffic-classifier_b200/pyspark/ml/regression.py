"""pyspark.ml.regression shim: DecisionTreeRegressor, RandomForestRegressor and GBTRegressor on the device variance-tree
loop (b200flow/regression.py, b200flow/gbt_regression.py, csrc/regression.cu, DESIGN.md §5l, §5m), and LinearRegression
on the normal equations and the fused least-squares / Huber kernel (b200flow/linreg.py, csrc/linreg.cu, DESIGN.md §5n),
GeneralizedLinearRegression by IRLS on the per-row GLM kernel and the weighted Gram kernel (b200flow/glm.py,
csrc/glm.cu, DESIGN.md §5o), IsotonicRegression on a device sort and a chunked pool-adjacent-violators merge
(b200flow/isotonic.py, csrc/isotonic.cu, DESIGN.md §5p), AFTSurvivalRegression on the Weibull instantiation of the
per-row linear-regression kernel (b200flow/aft.py, csrc/linreg.cu, DESIGN.md §5q), and FMRegressor on the squared-error
factorization-machine kernel (b200flow/fm.py, csrc/fm.cu, DESIGN.md §5r).
Their models are the same bits for any number of ranks.

Deviations from Spark: a NaN or infinite label raises IllegalArgumentException (Spark trains on it); labels (and GBT
residuals) beyond 2^300 in magnitude are refused; weightCol is not offered except by GeneralizedLinearRegression and
IsotonicRegression.  IsotonicRegression also refuses a non-finite feature or weight at fit time, and its empty model (every
weight 0) raises IllegalArgumentException where Spark throws NoSuchElementException."""
import numpy as np
import torch

from b200flow import dist as bdist
from b200flow import forest as fr

from . import Estimator, Model
from ..sql import ColumnData
from .classification import _arity_from_attrs, _default_seed, _lazy_plan
from .feature import IllegalArgumentException

__all__ = ["AFTSurvivalRegression", "AFTSurvivalRegressionModel", "DecisionTreeRegressionModel", "DecisionTreeRegressor",
           "FMRegressionModel", "FMRegressor", "GBTRegressionModel", "GBTRegressor",
           "GeneralizedLinearRegression", "GeneralizedLinearRegressionModel", "GeneralizedLinearRegressionSummary",
           "GeneralizedLinearRegressionTrainingSummary", "IsotonicRegression", "IsotonicRegressionModel",
           "LinearRegression", "LinearRegressionModel", "LinearRegressionSummary", "LinearRegressionTrainingSummary",
           "RandomForestRegressionModel", "RandomForestRegressor", "UnsupportedOperationException"]


class _TreeRegressorParams:
    _defaults = {"featuresCol": "features", "labelCol": "label", "predictionCol": "prediction", "maxDepth": 5, "maxBins": 32,
                 "minInstancesPerNode": 1, "minInfoGain": 0.0, "maxMemoryInMB": 256, "cacheNodeIds": False,
                 "checkpointInterval": 10, "impurity": "variance", "seed": None, "varianceCol": None}


class _RandomForestRegressorParams(_TreeRegressorParams):
    _defaults = {"numTrees": 20, "featureSubsetStrategy": "auto", "subsamplingRate": 1.0}


def _features_and_label(est, df):
    """(the features column, the label as a contiguous f64 tensor) of a regressor's input, after Spark's column checks"""
    fcol, lcol = est.getOrDefault("featuresCol"), est.getOrDefault("labelCol")
    for c in (fcol, lcol):
        if c not in df._cols:
            raise IllegalArgumentException("Field \"%s\" does not exist." % c)
    fc = df._cols[fcol]
    if fc.kind != "vector":
        raise IllegalArgumentException("Column %s must be of type vector" % fcol)
    return fc, df._column_tensor(lcol).to(torch.float64).reshape(-1).contiguous()


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
        fc, y = _features_and_label(self, df)
        x = fc.data                         # a lazy VectorAssembler column is assembled here, once
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


# ------------------------------------------------------------------------------- linear regression
class UnsupportedOperationException(RuntimeError):
    pass


class _LinearRegressionParams:
    _defaults = {"featuresCol": "features", "labelCol": "label", "predictionCol": "prediction", "maxIter": 100,
                 "regParam": 0.0, "elasticNetParam": 0.0, "tol": 1e-6, "fitIntercept": True, "standardization": True,
                 "solver": "auto", "loss": "squaredError", "epsilon": 1.35, "aggregationDepth": 2,
                 "maxBlockSizeInMB": 0.0, "weightCol": None}


class LinearRegression(Estimator, _LinearRegressionParams):
    """Spark 3's LinearRegression [recalled]: squared loss through the normal equations (solver auto or normal) or L-BFGS /
    OWL-QN, and Huber loss through L-BFGS, on the device (b200flow/linreg.py, DESIGN.md §5n).  aggregationDepth and
    maxBlockSizeInMB are validated but do not change the result: the sums have one fixed order.  weightCol raises."""

    def __init__(self, featuresCol=None, labelCol=None, predictionCol=None, maxIter=None, regParam=None,
                 elasticNetParam=None, tol=None, fitIntercept=None, standardization=None, solver=None, weightCol=None,
                 aggregationDepth=None, loss=None, epsilon=None, maxBlockSizeInMB=None):
        kw = dict(locals()); kw.pop("self"); kw.pop("__class__", None)
        super().__init__(**kw)

    def _check(self):
        """Spark's param validators, and the refusal of weightCol -> b200flow.linreg.LinRegParams"""
        from b200flow import linreg as blr
        g = self.getOrDefault
        it, depth = g("maxIter"), g("aggregationDepth")
        if isinstance(it, bool) or int(it) != it or int(it) < 0:
            raise IllegalArgumentException("maxIter must be an integer >= 0, got %r" % (it,))
        if isinstance(depth, bool) or int(depth) != depth or int(depth) < 2:
            raise IllegalArgumentException("aggregationDepth must be an integer >= 2, got %r" % (depth,))
        if not float(g("maxBlockSizeInMB")) >= 0:
            raise IllegalArgumentException("maxBlockSizeInMB must be >= 0, got %r" % (g("maxBlockSizeInMB"),))
        if g("weightCol"):
            raise IllegalArgumentException("weightCol is not supported by the b200flow LinearRegression")
        p = blr.LinRegParams(max_iter=int(it), reg_param=float(g("regParam")), elastic_net_param=float(g("elasticNetParam")),
                             tol=float(g("tol")), fit_intercept=bool(g("fitIntercept")),
                             standardization=bool(g("standardization")), solver=g("solver"), loss=g("loss"),
                             epsilon=float(g("epsilon")))
        try:
            blr.check_params(p)
        except ValueError as e:
            raise IllegalArgumentException(str(e))
        return p

    def _fit(self, df):
        from b200flow import linreg as blr
        p = self._check()
        fc, y = _features_and_label(self, df)
        x = fc.data
        try:
            grp = bdist.group()
            off, _ = bdist.global_offset(x.shape[0], x.device, grp)
            fit = blr.linreg_fit(x, y, p, row_offset=off, group=grp)
        except ValueError as e:        # includes b200flow's UnsupportedParamError; CUDA failures propagate as they are
            raise IllegalArgumentException(str(e))
        m = LinearRegressionModel(fit)
        m._paramMap = {k: v for k, v in self._paramMap.items() if k in m._all_defaults()}
        m._training = df
        return m


class LinearRegressionModel(Model, _LinearRegressionParams):
    """coefficients (original feature scale), intercept and scale (Huber's sigma, 1.0 for squared loss); prediction =
    x . coefficients + intercept."""

    def __init__(self, fit):
        super().__init__()
        self._fit_result = fit             # b200flow.linreg.LinRegFit
        self._training = None
        self._summary = None

    @property
    def coefficients(self):
        from .linalg import DenseVector
        return DenseVector(self._fit_result.coef.copy())

    @property
    def intercept(self):
        return self._fit_result.intercept

    @property
    def scale(self):
        return self._fit_result.scale

    @property
    def numFeatures(self):
        return int(self._fit_result.coef.shape[0])

    @property
    def hasSummary(self):
        return self._training is not None

    @property
    def summary(self):
        if self._training is None:
            raise RuntimeError("No training summary available for this LinearRegressionModel")
        if self._summary is None:
            self._summary = LinearRegressionTrainingSummary(self, self._training)
        return self._summary

    def evaluate(self, dataset):
        """a LinearRegressionSummary of the model on another dataset"""
        return LinearRegressionSummary(self, dataset)

    def _transform(self, df):
        from b200flow import linreg as blr
        fcol = self.getOrDefault("featuresCol")
        if fcol not in df._cols or df._cols[fcol].kind != "vector":
            raise IllegalArgumentException("Column %s must be of type vector" % fcol)
        pcol = self.getOrDefault("predictionCol")
        if not pcol:
            return df
        if pcol in df._cols:
            raise IllegalArgumentException("Output column %s already exists." % pcol)
        try:
            pred = blr.linreg_predict(df._cols[fcol].data, self._fit_result)
        except ValueError as e:
            raise IllegalArgumentException(str(e))
        cols = dict(df._cols)
        cols[pcol] = ColumnData("numeric", pred, "f64")
        return df._with(cols=cols)

    def __repr__(self):
        return "LinearRegressionModel: uid=%s, numFeatures=%d" % (self.uid, self.numFeatures)


class LinearRegressionSummary:
    """Spark 3's LinearRegressionSummary [recalled]: the metrics of RegressionMetrics (through the origin without an
    intercept), r2adj, residuals, degrees of freedom, the residual range, and the coefficient standard errors, t values
    and p values of the Cholesky path (the intercept last)."""

    def __init__(self, model, dataset):
        from b200flow import linreg as blr
        self._model = model
        self.predictionCol = model.getOrDefault("predictionCol") or "prediction"
        self.labelCol, self.featuresCol = model.getOrDefault("labelCol"), model.getOrDefault("featuresCol")
        fc, y = _features_and_label(model, dataset)
        fit = model._fit_result
        self._s = blr.summarize(fc.data, y, fit, bool(model.getOrDefault("fitIntercept")), group=bdist.group())
        cols = dict(dataset._cols)
        cols[self.predictionCol] = ColumnData("numeric", self._s.predictions, "f64")
        self.predictions = dataset._with(cols=cols)

    explainedVariance = property(lambda self: self._s.explained_variance)
    meanAbsoluteError = property(lambda self: self._s.mae)
    meanSquaredError = property(lambda self: self._s.mse)
    rootMeanSquaredError = property(lambda self: self._s.rmse)
    r2 = property(lambda self: self._s.r2)
    r2adj = property(lambda self: self._s.r2adj)
    numInstances = property(lambda self: self._s.num_instances)
    degreesOfFreedom = property(lambda self: self._s.degrees_of_freedom)
    devianceResiduals = property(lambda self: list(self._s.deviance_residuals))

    @property
    def residuals(self):
        """a frame with one column, residuals = label - prediction"""
        return self.predictions._with(cols={"residuals": ColumnData("numeric", self._s.residuals, "f64")})

    def _coefficient_stat(self, name):
        v = getattr(self._s, name)
        if v is None:
            raise UnsupportedOperationException("No Std. Error of coefficients available for this LinearRegressionModel")
        return [float(t) for t in v]

    coefficientStandardErrors = property(lambda self: self._coefficient_stat("std_errors"))
    tValues = property(lambda self: self._coefficient_stat("t_values"))
    pValues = property(lambda self: self._coefficient_stat("p_values"))


class LinearRegressionTrainingSummary(LinearRegressionSummary):
    """the summary of the training rows, with the optimiser's objective history"""

    @property
    def objectiveHistory(self):
        return list(self._model._fit_result.objective_history)

    @property
    def totalIterations(self):
        return len(self._model._fit_result.objective_history) - 1


# ------------------------------------------------------------------------------- generalized linear regression
class _GLRParams:
    _defaults = {"featuresCol": "features", "labelCol": "label", "predictionCol": "prediction", "family": "gaussian",
                 "link": None, "variancePower": 0.0, "linkPower": None, "fitIntercept": True, "maxIter": 25, "tol": 1e-6,
                 "regParam": 0.0, "solver": "irls", "aggregationDepth": 2, "weightCol": None, "offsetCol": None,
                 "linkPredictionCol": None}


def _glr_params(est):
    """Spark's param validators -> b200flow.glm.GLMParams"""
    from b200flow import glm as bg
    g = est.getOrDefault
    it, depth = g("maxIter"), g("aggregationDepth")
    if isinstance(it, bool) or int(it) != it or int(it) < 0:
        raise IllegalArgumentException("maxIter must be an integer >= 0, got %r" % (it,))
    if isinstance(depth, bool) or int(depth) != depth or int(depth) < 2:
        raise IllegalArgumentException("aggregationDepth must be an integer >= 2, got %r" % (depth,))
    p = bg.GLMParams(family=g("family"), link=g("link"), variance_power=float(g("variancePower")),
                     link_power=g("linkPower"), fit_intercept=bool(g("fitIntercept")), max_iter=int(it),
                     tol=float(g("tol")), reg_param=float(g("regParam")), solver=g("solver"))
    try:
        bg.check_params(p)
    except ValueError as e:
        raise IllegalArgumentException(str(e))
    return p


def _glr_columns(est, df):
    """(features, label, weight or None, offset or None) of a frame, after Spark's column checks"""
    fc, y = _features_and_label(est, df)
    extra = []
    for name in ("weightCol", "offsetCol"):
        c = est.getOrDefault(name)
        if c and c not in df._cols:
            raise IllegalArgumentException("Field \"%s\" does not exist." % c)
        extra.append(df._column_tensor(c).to(torch.float64).reshape(-1).contiguous() if c else None)
    return fc, y, extra[0], extra[1]


class GeneralizedLinearRegression(Estimator, _GLRParams):
    """Spark 3's GeneralizedLinearRegression [recalled]: gaussian, binomial, poisson, gamma and tweedie families fitted by
    IRLS on the device (b200flow/glm.py, csrc/glm.cu, DESIGN.md §5o).  aggregationDepth is validated but does not change
    the result: the sums have one fixed order."""

    def __init__(self, labelCol=None, featuresCol=None, predictionCol=None, family=None, link=None, fitIntercept=None,
                 maxIter=None, tol=None, regParam=None, weightCol=None, solver=None, linkPredictionCol=None,
                 variancePower=None, linkPower=None, offsetCol=None, aggregationDepth=None):
        kw = dict(locals()); kw.pop("self"); kw.pop("__class__", None)
        super().__init__(**kw)

    def _fit(self, df):
        from b200flow import glm as bg
        p = _glr_params(self)
        fc, y, w, off = _glr_columns(self, df)
        x = fc.data
        try:
            grp = bdist.group()
            ro, _ = bdist.global_offset(x.shape[0], x.device, grp)
            fit = bg.glm_fit(x, y, p, weight=w, offset=off, row_offset=ro, group=grp)
        except ValueError as e:        # includes b200flow's UnsupportedParamError; CUDA failures propagate as they are
            raise IllegalArgumentException(str(e))
        m = GeneralizedLinearRegressionModel(fit)
        m._paramMap = {k: v for k, v in self._paramMap.items() if k in m._all_defaults()}
        m._training = df
        return m


class GeneralizedLinearRegressionModel(Model, _GLRParams):
    """coefficients and intercept; prediction = linkInv(x . coefficients + intercept + offset), and with
    linkPredictionCol the linear predictor as well."""

    def __init__(self, fit):
        super().__init__()
        self._fit_result = fit             # b200flow.glm.GLMFit
        self._training = None
        self._summary = None

    @property
    def coefficients(self):
        from .linalg import DenseVector
        return DenseVector(self._fit_result.coef.copy())

    @property
    def intercept(self):
        return self._fit_result.intercept

    @property
    def numFeatures(self):
        return int(self._fit_result.coef.shape[0])

    @property
    def hasSummary(self):
        return self._training is not None

    @property
    def summary(self):
        if self._training is None:
            raise RuntimeError("No training summary available for this GeneralizedLinearRegressionModel")
        if self._summary is None:
            self._summary = GeneralizedLinearRegressionTrainingSummary(self, self._training)
        return self._summary

    def evaluate(self, dataset):
        """a GeneralizedLinearRegressionSummary of the model on another dataset"""
        return GeneralizedLinearRegressionSummary(self, dataset)

    def _transform(self, df):
        from b200flow import glm as bg
        fcol = self.getOrDefault("featuresCol")
        if fcol not in df._cols or df._cols[fcol].kind != "vector":
            raise IllegalArgumentException("Column %s must be of type vector" % fcol)
        pcol, lcol, ocol = (self.getOrDefault(k) for k in ("predictionCol", "linkPredictionCol", "offsetCol"))
        outs = [c for c in (pcol, lcol) if c]
        if not outs:
            return df
        for c in outs:
            if c in df._cols:
                raise IllegalArgumentException("Output column %s already exists." % c)
        if ocol and ocol not in df._cols:
            raise IllegalArgumentException("Field \"%s\" does not exist." % ocol)
        off = df._column_tensor(ocol).to(torch.float64).reshape(-1).contiguous() if ocol else None
        try:
            me = bg.glm_predict(df._cols[fcol].data, self._fit_result, off)
        except ValueError as e:
            raise IllegalArgumentException(str(e))
        cols = dict(df._cols)
        if pcol:
            cols[pcol] = ColumnData("numeric", me[:, 0].contiguous(), "f64")
        if lcol:
            cols[lcol] = ColumnData("numeric", me[:, 1].contiguous(), "f64")
        return df._with(cols=cols)

    def __repr__(self):
        return "GeneralizedLinearRegressionModel: uid=%s, family=%s, link=%s, numFeatures=%d" % (
            self.uid, self.getOrDefault("family"), self.getOrDefault("link"), self.numFeatures)


class GeneralizedLinearRegressionSummary:
    """Spark 3's GeneralizedLinearRegressionSummary [recalled]: predictions, counts and degrees of freedom, deviance,
    nullDeviance, dispersion, aic (tweedie raises) and residuals(residualsType)."""

    def __init__(self, model, dataset):
        from b200flow import glm as bg
        self._model = model
        self.predictionCol = model.getOrDefault("predictionCol") or "prediction"
        fc, y, w, off = _glr_columns(model, dataset)
        try:
            self._s = bg.summarize(fc.data, y, model._fit_result, _glr_params(model), weight=w, offset=off,
                                   group=bdist.group())
        except ValueError as e:
            raise IllegalArgumentException(str(e))
        cols = dict(dataset._cols)
        cols[self.predictionCol] = ColumnData("numeric", self._s.predictions[:, 0].contiguous(), "f64")
        lcol = model.getOrDefault("linkPredictionCol")
        if lcol:
            cols[lcol] = ColumnData("numeric", self._s.predictions[:, 1].contiguous(), "f64")
        self.predictions = dataset._with(cols=cols)

    numInstances = property(lambda self: self._s.num_instances)
    rank = property(lambda self: self._s.rank)
    degreesOfFreedom = property(lambda self: self._s.degrees_of_freedom)
    residualDegreeOfFreedom = property(lambda self: self._s.residual_dof)
    residualDegreeOfFreedomNull = property(lambda self: self._s.residual_dof_null)
    deviance = property(lambda self: self._s.deviance)
    nullDeviance = property(lambda self: self._s.null_deviance)
    dispersion = property(lambda self: self._s.dispersion)

    @property
    def aic(self):
        if self._s.aic is None:
            raise UnsupportedOperationException("No AIC available for the tweedie family")
        return self._s.aic

    def residuals(self, residualsType="deviance"):
        """a frame with one column, <type>Residuals"""
        from b200flow import glm as bg
        t = str(residualsType).lower()
        if t not in bg.RESIDUALS:
            raise IllegalArgumentException("residualsType must be one of %s, got %r" % (list(bg.RESIDUALS), residualsType))
        col = self._s.residuals[:, bg.RESIDUALS.index(t)].contiguous()
        return self.predictions._with(cols={t + "Residuals": ColumnData("numeric", col, "f64")})


class GeneralizedLinearRegressionTrainingSummary(GeneralizedLinearRegressionSummary):
    """the summary of the training rows, with the IRLS iteration count and the coefficient statistics"""

    numIterations = property(lambda self: self._model._fit_result.iterations)
    solver = property(lambda self: "irls")

    def _coefficient_stat(self, name):
        v = getattr(self._s, name)
        if v is None:
            raise UnsupportedOperationException("No Std. Error of coefficients available for this "
                                                "GeneralizedLinearRegressionModel")
        return [float(t) for t in v]

    coefficientStandardErrors = property(lambda self: self._coefficient_stat("std_errors"))
    tValues = property(lambda self: self._coefficient_stat("t_values"))
    pValues = property(lambda self: self._coefficient_stat("p_values"))


# ------------------------------------------------------------------------------- isotonic regression
class _IsotonicRegressionParams:
    _defaults = {"featuresCol": "features", "labelCol": "label", "predictionCol": "prediction", "weightCol": None,
                 "isotonic": True, "featureIndex": 0}


def _isotonic_feature(est, df):
    """the feature as one value per row: featuresCol itself when numeric, its element featureIndex when a vector (a strided
    view, f32 or f64)"""
    fcol = est.getOrDefault("featuresCol")
    if fcol not in df._cols:
        raise IllegalArgumentException("Field \"%s\" does not exist." % fcol)
    k = est.getOrDefault("featureIndex")
    if isinstance(k, bool) or int(k) != k or int(k) < 0:
        raise IllegalArgumentException("%s parameter featureIndex given invalid value %r." % (est.uid, k))
    c = df._cols[fcol]
    if c.kind == "vector":
        x = c.data
        if int(k) >= x.shape[1]:
            raise IllegalArgumentException("featureIndex %d is out of range for the %d-element vectors of column %s"
                                           % (int(k), x.shape[1], fcol))
        return x[:, int(k)]
    x = df._column_tensor(fcol)
    return x if x.dtype in (torch.float32, torch.float64) else x.to(torch.float64)


class IsotonicRegression(Estimator, _IsotonicRegressionParams):
    """Spark 3's IsotonicRegression [recalled]: the weighted isotonic (or antitonic) least-squares fit of the label on one
    feature by pool-adjacent-violators, on the device (b200flow/isotonic.py, csrc/isotonic.cu, DESIGN.md §5p).  The model
    is the same bits for any world size; it equals Spark's sequential PAV to rounding.  A NaN or infinite label, feature or
    weight raises IllegalArgumentException."""

    def __init__(self, featuresCol=None, labelCol=None, predictionCol=None, weightCol=None, isotonic=None,
                 featureIndex=None):
        kw = dict(locals()); kw.pop("self"); kw.pop("__class__", None)
        super().__init__(**kw)

    def _fit(self, df):
        from b200flow import isotonic as biso
        x = _isotonic_feature(self, df)
        lcol, wcol = self.getOrDefault("labelCol"), self.getOrDefault("weightCol")
        for c in (lcol, wcol):
            if c and c not in df._cols:
                raise IllegalArgumentException("Field \"%s\" does not exist." % c)
        y = df._column_tensor(lcol).to(torch.float64).reshape(-1)
        w = df._column_tensor(wcol).to(torch.float64).reshape(-1) if wcol else None
        try:
            fit = biso.isotonic_fit(x, y, w, isotonic=bool(self.getOrDefault("isotonic")), group=bdist.group())
        except ValueError as e:
            raise IllegalArgumentException(str(e))
        m = IsotonicRegressionModel(fit)
        m._paramMap = {k: v for k, v in self._paramMap.items() if k in m._all_defaults()}
        return m


class IsotonicRegressionModel(Model, _IsotonicRegressionParams):
    """boundaries (increasing) and predictions; predict(x) interpolates linearly between the boundaries around x and is
    constant outside them."""

    def __init__(self, fit):
        super().__init__()
        self._fit_result = fit             # b200flow.isotonic.IsotonicFit

    @property
    def boundaries(self):
        from .linalg import DenseVector
        return DenseVector(self._fit_result.boundaries.copy())

    @property
    def predictions(self):
        from .linalg import DenseVector
        return DenseVector(self._fit_result.predictions.copy())

    @property
    def numFeatures(self):
        return 1

    def predict(self, value):
        """the prediction at one feature value, on the host (the kernel's arithmetic, so the same bits)"""
        from b200flow import isotonic as biso
        try:
            return biso.predict_value(float(value), self._fit_result)
        except ValueError as e:
            raise IllegalArgumentException(str(e))

    def _transform(self, df):
        from b200flow import isotonic as biso
        x = _isotonic_feature(self, df)
        pcol = self.getOrDefault("predictionCol")
        if not pcol:
            return df
        if pcol in df._cols:
            raise IllegalArgumentException("Output column %s already exists." % pcol)
        try:
            pred = biso.isotonic_predict(x, self._fit_result)
        except ValueError as e:
            raise IllegalArgumentException(str(e))
        cols = dict(df._cols)
        cols[pcol] = ColumnData("numeric", pred, "f64")
        return df._with(cols=cols)

    def __repr__(self):
        return "IsotonicRegressionModel: uid=%s, numFeatures=1, boundaries=%d" % (self.uid, len(self._fit_result.boundaries))


# ------------------------------------------------------------------------------- survival regression
class _AFTSurvivalRegressionParams:
    _defaults = {"featuresCol": "features", "labelCol": "label", "predictionCol": "prediction", "censorCol": "censor",
                 "quantileProbabilities": [0.01, 0.05, 0.1, 0.25, 0.5, 0.75, 0.9, 0.95, 0.99], "quantilesCol": None,
                 "fitIntercept": True, "maxIter": 100, "tol": 1e-6, "aggregationDepth": 2, "maxBlockSizeInMB": 0.0}


class AFTSurvivalRegression(Estimator, _AFTSurvivalRegressionParams):
    """Spark 3's AFTSurvivalRegression [recalled]: the Weibull accelerated-failure-time model of a positive lifetime with
    right censoring (censor 1.0: the event was observed, 0.0: censored), fitted by L-BFGS on the device
    (b200flow/aft.py, DESIGN.md §5q).  aggregationDepth and maxBlockSizeInMB are validated but do not change the result:
    the sums have one fixed order."""

    def __init__(self, featuresCol=None, labelCol=None, predictionCol=None, fitIntercept=None, maxIter=None, tol=None,
                 censorCol=None, quantileProbabilities=None, quantilesCol=None, aggregationDepth=None,
                 maxBlockSizeInMB=None):
        kw = dict(locals()); kw.pop("self"); kw.pop("__class__", None)
        super().__init__(**kw)

    def _check(self):
        """Spark's param validators -> b200flow.aft.AFTParams"""
        from b200flow import aft as baft
        g = self.getOrDefault
        it, depth = g("maxIter"), g("aggregationDepth")
        if isinstance(it, bool) or int(it) != it or int(it) < 0:
            raise IllegalArgumentException("maxIter must be an integer >= 0, got %r" % (it,))
        if isinstance(depth, bool) or int(depth) != depth or int(depth) < 2:
            raise IllegalArgumentException("aggregationDepth must be an integer >= 2, got %r" % (depth,))
        if not float(g("maxBlockSizeInMB")) >= 0:
            raise IllegalArgumentException("maxBlockSizeInMB must be >= 0, got %r" % (g("maxBlockSizeInMB"),))
        try:
            p = baft.AFTParams(max_iter=int(it), tol=float(g("tol")), fit_intercept=bool(g("fitIntercept")),
                               quantile_probabilities=list(g("quantileProbabilities")))
            baft.check_params(p)
        except (TypeError, ValueError) as e:
            raise IllegalArgumentException(str(e))
        return p

    def _fit(self, df):
        from b200flow import aft as baft
        p = self._check()
        fc, y = _features_and_label(self, df)
        ccol = self.getOrDefault("censorCol")
        if ccol not in df._cols:
            raise IllegalArgumentException("Field \"%s\" does not exist." % ccol)
        c = df._column_tensor(ccol).to(torch.float64).reshape(-1).contiguous()
        x = fc.data
        try:
            grp = bdist.group()
            off, _ = bdist.global_offset(x.shape[0], x.device, grp)
            fit = baft.aft_fit(x, y, c, p, row_offset=off, group=grp)
        except ValueError as e:        # includes b200flow's UnsupportedParamError; CUDA failures propagate as they are
            raise IllegalArgumentException(str(e))
        m = AFTSurvivalRegressionModel(fit)
        m._paramMap = {k: v for k, v in self._paramMap.items() if k in m._all_defaults()}
        return m


class AFTSurvivalRegressionModel(Model, _AFTSurvivalRegressionParams):
    """coefficients (original feature scale), intercept and scale (the Weibull sigma); prediction = exp(x . coefficients +
    intercept), the quantiles lambda exp(log(-log1p(-p)) scale) for each p of quantileProbabilities.  Spark has no
    training summary for this model."""

    def __init__(self, fit):
        super().__init__()
        self._fit_result = fit             # b200flow.aft.AFTFit

    @property
    def coefficients(self):
        from .linalg import DenseVector
        return DenseVector(self._fit_result.coef.copy())

    @property
    def intercept(self):
        return self._fit_result.intercept

    @property
    def scale(self):
        return self._fit_result.scale

    @property
    def numFeatures(self):
        return int(self._fit_result.coef.shape[0])

    def _probs(self):
        from b200flow import aft as baft
        probs = list(self.getOrDefault("quantileProbabilities"))
        try:
            baft.check_quantiles(probs)
        except ValueError as e:
            raise IllegalArgumentException(str(e))
        return probs

    def _row(self, features):
        v = np.asarray(features.toArray() if hasattr(features, "toArray") else features, np.float64).reshape(1, -1)
        if v.shape[1] != self.numFeatures:
            raise IllegalArgumentException("the model has %d features, the vector %d" % (self.numFeatures, v.shape[1]))
        return torch.from_numpy(v).cuda()

    def predict(self, features):
        """the prediction for one feature vector: exp(features . coefficients + intercept), transform's arithmetic"""
        from b200flow import aft as baft
        return float(baft.aft_predict(self._row(features), self._fit_result)[0].item())

    def predictQuantiles(self, features):
        """DenseVector of the quantiles of one feature vector's lifetime at quantileProbabilities"""
        from b200flow import aft as baft
        from .linalg import DenseVector
        q = baft.aft_predict_quantiles(self._row(features), self._fit_result, self._probs())
        return DenseVector(q[0].cpu().numpy())

    def _transform(self, df):
        from b200flow import aft as baft
        fcol = self.getOrDefault("featuresCol")
        if fcol not in df._cols or df._cols[fcol].kind != "vector":
            raise IllegalArgumentException("Column %s must be of type vector" % fcol)
        pcol, qcol = self.getOrDefault("predictionCol"), self.getOrDefault("quantilesCol")
        outs = [c for c in (pcol, qcol) if c]
        if not outs:
            return df
        for c in outs:
            if c in df._cols:
                raise IllegalArgumentException("Output column %s already exists." % c)
        probs = self._probs() if qcol else None
        x = df._cols[fcol].data
        if x.shape[1] != self.numFeatures:
            raise IllegalArgumentException("the model has %d features, the input %d" % (self.numFeatures, x.shape[1]))
        lam = baft.aft_predict(x, self._fit_result)
        cols = dict(df._cols)
        if pcol:
            cols[pcol] = ColumnData("numeric", lam, "f64")
        if qcol:
            cols[qcol] = ColumnData("vector", baft.aft_predict_quantiles(x, self._fit_result, probs, lam=lam), "f64")
        return df._with(cols=cols)

    def __repr__(self):
        return "AFTSurvivalRegressionModel: uid=%s, numFeatures=%d" % (self.uid, self.numFeatures)


# ------------------------------------------------------------------------------- factorization machines
class _FMRegressorParams:
    _defaults = {"featuresCol": "features", "labelCol": "label", "predictionCol": "prediction", "factorSize": 8,
                 "fitIntercept": True, "fitLinear": True, "regParam": 0.0, "miniBatchFraction": 1.0, "initStd": 0.01,
                 "maxIter": 100, "stepSize": 1.0, "tol": 1e-6, "solver": "adamW", "seed": None, "weightCol": None}


class FMRegressor(Estimator, _FMRegressorParams):
    """Spark 3's FMRegressor [recalled]: a factorization machine with the squared error, trained by mllib's mini-batch
    gradient descent with the adamW or gd updater, on the device (b200flow/fm.py, csrc/fm.cu, DESIGN.md §5r).  Features
    and labels are not scaled.  weightCol raises."""

    def __init__(self, featuresCol=None, labelCol=None, predictionCol=None, factorSize=None, fitIntercept=None,
                 fitLinear=None, regParam=None, miniBatchFraction=None, initStd=None, maxIter=None, stepSize=None, tol=None,
                 solver=None, seed=None, weightCol=None):
        kw = dict(locals()); kw.pop("self"); kw.pop("__class__", None)
        super().__init__(**kw)

    def _check(self):
        """Spark's param validators, and the refusal of weightCol -> b200flow.fm.FMParams (FMClassifier's rules)"""
        from b200flow import fm as bfm
        g = self.getOrDefault
        fs, it = g("factorSize"), g("maxIter")
        if isinstance(fs, bool) or int(fs) != fs or int(fs) < 1:
            raise IllegalArgumentException("factorSize must be an integer >= 1, got %r" % (fs,))
        if isinstance(it, bool) or int(it) != it or int(it) < 0:
            raise IllegalArgumentException("maxIter must be an integer >= 0, got %r" % (it,))
        for name in ("regParam", "initStd", "tol"):
            if not float(g(name)) >= 0:
                raise IllegalArgumentException("%s must be >= 0, got %r" % (name, g(name)))
        if not float(g("stepSize")) > 0:
            raise IllegalArgumentException("stepSize must be > 0, got %r" % (g("stepSize"),))
        if not 0.0 < float(g("miniBatchFraction")) <= 1.0:
            raise IllegalArgumentException("miniBatchFraction must be in (0, 1], got %r" % (g("miniBatchFraction"),))
        if g("solver") not in bfm.SOLVERS:
            raise IllegalArgumentException("solver must be 'gd' or 'adamW', got %r" % (g("solver"),))
        if g("weightCol"):
            raise IllegalArgumentException("weightCol is not supported by the b200flow FMRegressor (out of scope)")
        seed = g("seed")
        return bfm.FMParams(factor_size=int(fs), fit_intercept=bool(g("fitIntercept")), fit_linear=bool(g("fitLinear")),
                            reg_param=float(g("regParam")), mini_batch_fraction=float(g("miniBatchFraction")),
                            init_std=float(g("initStd")), max_iter=int(it), step_size=float(g("stepSize")),
                            tol=float(g("tol")), solver=g("solver"), seed=_default_seed(self) if seed is None else int(seed))

    def _fit(self, df):
        from b200flow import fm as bfm
        params = self._check()
        fc, y = _features_and_label(self, df)
        try:
            fit = bfm.fm_regression_fit(fc.data, y, params, group=bdist.group())
        except ValueError as e:        # includes b200flow's UnsupportedParamError
            raise IllegalArgumentException(str(e))
        m = FMRegressionModel(fit)
        m._paramMap = {k: v for k, v in self._paramMap.items() if k in m._all_defaults()}
        return m


class FMRegressionModel(Model, _FMRegressorParams):
    """intercept, linear (DenseVector [D]), factors (DenseMatrix D x k); prediction = r, the factorization machine's raw
    value.  Spark has no training summary for this model."""

    def __init__(self, fit):
        super().__init__()
        self._fit_result = fit             # b200flow.fm.FMFit

    @property
    def intercept(self):
        return self._fit_result.intercept

    @property
    def linear(self):
        from .linalg import DenseVector
        return DenseVector(self._fit_result.linear.copy())

    @property
    def factors(self):
        from .linalg import DenseMatrix
        f = self._fit_result.factors
        return DenseMatrix(f.shape[0], f.shape[1], f.T.reshape(-1))

    @property
    def numFeatures(self):
        return int(self._fit_result.factors.shape[0])

    def _weights(self):
        """[1, D (k + 1) + 1] f64 host: [V (row-major) | w | b], fm_raw's layout"""
        f = self._fit_result
        return torch.from_numpy(np.concatenate([f.factors.reshape(-1), f.linear, [f.intercept]])).reshape(1, -1)

    def _raw(self, x):
        from b200flow import fm as bfm
        try:
            return bfm.fm_raw(x, self._weights(), self._fit_result.factors.shape[1])[:, 0].contiguous()
        except ValueError as e:
            raise IllegalArgumentException(str(e))

    def predict(self, features):
        """the prediction for one feature vector, transform's arithmetic"""
        v = np.asarray(features.toArray() if hasattr(features, "toArray") else features, np.float64).reshape(1, -1)
        return float(self._raw(torch.from_numpy(v).cuda())[0].item())

    def _transform(self, df):
        fcol = self.getOrDefault("featuresCol")
        if fcol not in df._cols or df._cols[fcol].kind != "vector":
            raise IllegalArgumentException("Column %s must be of type vector" % fcol)
        pcol = self.getOrDefault("predictionCol")
        if not pcol:
            return df
        if pcol in df._cols:
            raise IllegalArgumentException("Output column %s already exists." % pcol)
        cols = dict(df._cols)
        cols[pcol] = ColumnData("numeric", self._raw(df._cols[fcol].data), "f64")
        return df._with(cols=cols)

    def __repr__(self):
        return "FMRegressionModel: uid=%s, numFeatures=%d, factorSize=%d" % (self.uid, self.numFeatures,
                                                                              self._fit_result.factors.shape[1])
