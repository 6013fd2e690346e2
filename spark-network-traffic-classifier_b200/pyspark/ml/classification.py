"""pyspark.ml.classification shim.

RandomForestClassifier / DecisionTreeClassifier (kdd99.py:61,64; cicids17.py:65,68) are the hot path and run
entirely on the b200flow CUDA kernels (histogram build, Gini split scoring, batch predict).
GBTClassifier (binary) runs on the variance-histogram level loop of csrc/gbt.cu (b200flow/gbt.py, DESIGN.md §5e); its
model is the same bits for any number of ranks.
MultilayerPerceptronClassifier runs on the fused fp64 tensor-core loss/gradient and forward kernels (b200flow/mlp.py,
csrc/mlp.cu, DESIGN.md §5d); its model is the same bits for any number of ranks.
OneVsRest reduces a K-class problem to K binary ones; OneVsRest(GBTClassifier) trains the K boosted models together in one
level loop on the device (b200flow.gbt.fit_gbt_ovr, DESIGN.md §5f), each the same bits as its standalone fit.
LinearSVC runs on the fused fp64 tensor-core hinge kernel (b200flow/svc.py, csrc/svc.cu, DESIGN.md §5j);
OneVsRest(LinearSVC) trains its K models together, one kernel pass per optimiser round, each the same bits as its standalone
fit, and its transform computes the K margins in one launch.  Both are the same bits for any number of ranks.
FMClassifier runs on the fused fp64 tensor-core factorization-machine kernel (b200flow/fm.py, csrc/fm.cu, DESIGN.md §5k);
OneVsRest(FMClassifier) trains its K models together, one kernel pass per gradient-descent iteration, each the same bits
as its standalone fit, and its transform computes the K raw values in one launch.  Both are the same bits for any number
of ranks.
LogisticRegression and NaiveBayes (kdd99.py:57,67; cicids17.py:61,71) are OUT of the kernel scope (SURVEY.md
§8f rank 4): torch fp64 implementations of MLlib's statistics / objective (b200flow/linear.py), checked against a numpy
restatement and scikit-learn in tests/test_linear_models.py.
"""
import zlib

import numpy as np
import torch

from b200flow import dist as bdist
from b200flow import forest as fr
from b200flow import fm as _fm
from b200flow import linear as _linear
from b200flow import mlp as _mlp
from b200flow import svc as _svc

from . import Estimator, Model, Pipeline
from .param import Param
from ..sql import ColumnData
from .feature import IllegalArgumentException, _materialize


def _default_seed(obj):
    # pyspark uses hash(type(self).__name__), which Python 3 randomises per process; a stable hash is used instead
    return zlib.crc32(type(obj).__name__.encode())


def _features_and_labels(df, est):
    fcol, lcol = est.getOrDefault("featuresCol"), est.getOrDefault("labelCol")
    for c in (fcol, lcol):
        if c not in df._cols:
            raise IllegalArgumentException("Field \"%s\" does not exist." % c)
    fc = df._cols[fcol]
    if fc.kind != "vector":
        raise IllegalArgumentException("Column %s must be of type vector" % fcol)
    x = fc.data
    y = df._column_tensor(lcol)
    lab_meta = df._cols[lcol].meta.get("ml_attr", {})
    if lab_meta.get("type") == "nominal":
        num_classes = len(lab_meta["vals"])
    else:
        if bool(((y < 0) | (y != torch.floor(y))).any().item()):
            raise IllegalArgumentException("Classifier was given dataset with invalid label. Labels must be integers in [0, numClasses).")
        num_classes = int(y.max().item()) + 1 if y.numel() else 0
    return x, y, num_classes, fc.meta.get("attrs")


def _arity_from_attrs(attrs, F):
    if not attrs or len(attrs) != F:
        return [0] * F
    return [int(a.get("arity", 0)) if a.get("type") in ("nominal", "binary") else 0 for a in attrs]


def _lazy_plan(df, fcol):
    """(encode plan, emulate-f32 flag) when the features column is still lazy — VectorAssembler over raw record fields whose
    kernel has not run — so that trees can be trained / applied straight from the records (fused encode -> bins); else None."""
    fc = df._cols.get(fcol)
    if fc is None or fc.kind != "vector" or not fc.lazy or fc.prov is None or fc.prov[0] != "plan" or df._rec is None:
        return None
    return fc.prov[1]


def _records_fit_inputs(df, est):
    """-> (records, plan with the label column set, num_classes, per-slot attrs) for the fused record path, or None."""
    import copy
    fcol, lcol = est.getOrDefault("featuresCol"), est.getOrDefault("labelCol")
    plan = _lazy_plan(df, fcol)
    lc = df._cols.get(lcol)
    if plan is None or lc is None or lc.prov is None or lc.prov[0] != "index" or not lc.lazy:
        return None
    lab_meta = lc.meta.get("ml_attr", {})
    if lab_meta.get("type") != "nominal":
        return None
    p2 = copy.copy(plan); p2.slots = list(plan.slots); p2.luts = list(plan.luts); p2._dev = None
    p2.set_label(lc.prov[1], lc.prov[2])
    return df._rec, p2, len(lab_meta["vals"]), df._cols[fcol].meta.get("attrs")


class _TreeParams:
    _defaults = {"featuresCol": "features", "labelCol": "label", "predictionCol": "prediction",
                 "probabilityCol": "probability", "rawPredictionCol": "rawPrediction", "maxDepth": 5, "maxBins": 32,
                 "minInstancesPerNode": 1, "minInfoGain": 0.0, "maxMemoryInMB": 256, "cacheNodeIds": False,
                 "checkpointInterval": 10, "impurity": "gini", "seed": None}


class _TreeClassifierBase(Estimator, _TreeParams):
    def _forest_params(self, num_trees, strategy, subsampling, bootstrap):
        imp = str(self.getOrDefault("impurity")).lower()
        if imp not in ("gini", "entropy"):
            raise IllegalArgumentException("impurity must be gini or entropy, got %r" % imp)
        if imp == "entropy":       # log is not bit-reproducible between libm and CUDA: not offered on the CUDA path (DESIGN.md)
            raise IllegalArgumentException("impurity='entropy' is not supported by the b200flow tree trainer; use 'gini' "
                                           "(the reference scripts take the default, kdd99.py:64 / cicids17.py:68)")
        seed = self.getOrDefault("seed")
        return fr.ForestParams(num_trees=int(num_trees), max_depth=int(self.getOrDefault("maxDepth")),
                               max_bins=int(self.getOrDefault("maxBins")),
                               min_instances_per_node=int(self.getOrDefault("minInstancesPerNode")),
                               min_info_gain=float(self.getOrDefault("minInfoGain")), feature_subset_strategy=str(strategy),
                               subsampling_rate=float(subsampling), impurity=imp,
                               seed=_default_seed(self) if seed is None else int(seed), bootstrap=bootstrap)

    def _train(self, df, params):
        from .feature import SparkException
        fused = _records_fit_inputs(df, self)
        try:
            grp = bdist.group()
            if fused is not None:                           # lazy VectorAssembler output: bin straight from the raw records
                rec, plan, C, attrs = fused
                if C > 100:
                    raise IllegalArgumentException("Classifier inferred %d classes; maximum is 100" % C)
                off, _ = bdist.global_offset(rec.shape[0], rec.device, grp)
                return fr.fit_forest_records(rec, plan, C, _arity_from_attrs(attrs, plan.n_out), params, row_offset=off, group=grp)
            x, y, C, attrs = _features_and_labels(df, self)
            if C > 100:
                raise IllegalArgumentException("Classifier inferred %d classes; maximum is 100" % C)
            off, _ = bdist.global_offset(x.shape[0], x.device, grp)
            forest = fr.fit_forest(x, y.to(torch.int32), C, _arity_from_attrs(attrs, x.shape[1]), params,
                                   row_offset=off, group=grp)
        except fr.InvalidRowsError as e:                    # NaN / null under handleInvalid="error": surfaces at the action, as in Spark
            raise SparkException("Encountered NaN/null while assembling a row with handleInvalid = \"error\" (%s)" % e)
        except ValueError as e:        # includes b200flow's UnsupportedParamError; CUDA failures propagate as they are
            raise IllegalArgumentException(str(e))
        return forest


class RandomForestClassifier(_TreeClassifierBase):
    _defaults = {"numTrees": 20, "featureSubsetStrategy": "auto", "subsamplingRate": 1.0}

    def __init__(self, featuresCol=None, labelCol=None, predictionCol=None, probabilityCol=None, rawPredictionCol=None,
                 maxDepth=None, maxBins=None, minInstancesPerNode=None, minInfoGain=None, maxMemoryInMB=None,
                 cacheNodeIds=None, checkpointInterval=None, impurity=None, numTrees=None, featureSubsetStrategy=None,
                 seed=None, subsamplingRate=None):
        kw = dict(locals()); kw.pop("self"); kw.pop("__class__", None)
        super().__init__(**kw)

    def _fit(self, df):
        p = self._forest_params(self.getOrDefault("numTrees"), self.getOrDefault("featureSubsetStrategy"),
                                self.getOrDefault("subsamplingRate"), bootstrap=True)
        m = RandomForestClassificationModel(self._train(df, p))
        m._paramMap = {k: v for k, v in self._paramMap.items() if k in m._all_defaults()}
        return m


class DecisionTreeClassifier(_TreeClassifierBase):
    """MLlib trains it as RandomForest.run(numTrees=1, featureSubsetStrategy='all'), no bagging."""

    def __init__(self, featuresCol=None, labelCol=None, predictionCol=None, probabilityCol=None, rawPredictionCol=None,
                 maxDepth=None, maxBins=None, minInstancesPerNode=None, minInfoGain=None, maxMemoryInMB=None,
                 cacheNodeIds=None, checkpointInterval=None, impurity=None, seed=None):
        kw = dict(locals()); kw.pop("self"); kw.pop("__class__", None)
        super().__init__(**kw)

    def _fit(self, df):
        p = self._forest_params(1, "all", 1.0, bootstrap=False)
        m = DecisionTreeClassificationModel(self._train(df, p))
        m._paramMap = {k: v for k, v in self._paramMap.items() if k in m._all_defaults()}
        return m


class _ForestModelBase(Model, _TreeParams):
    def __init__(self, forest):
        super().__init__()
        self._forest = forest

    @property
    def numClasses(self):
        return self._forest.C

    @property
    def numFeatures(self):
        return self._forest.F

    @property
    def totalNumNodes(self):
        return self._forest.n_nodes

    @property
    def featureImportances(self):
        from .linalg import DenseVector
        return DenseVector(self._forest.feature_importances())

    def _transform(self, df):
        fcol = self.getOrDefault("featuresCol")
        if fcol not in df._cols or df._cols[fcol].kind != "vector":
            raise IllegalArgumentException("Column %s must be of type vector" % fcol)
        plan = _lazy_plan(df, fcol)
        if plan is not None and plan.n_out == self._forest.F:   # lazy features: fused encode -> bins -> tree walk, no dense matrix
            from .feature import SparkException
            try:
                raw, prob, pred, _ = self._forest.predict_records(df._rec, plan, on_invalid="error" if plan.check_nan else "ignore")
            except fr.InvalidRowsError as e:
                raise SparkException("Encountered NaN/null while assembling a row with handleInvalid = \"error\" (%s)" % e)
        else:
            x = df._cols[fcol].data
            raw, prob, pred = self._forest.predict(x)          # R9: bin + walk all trees on the GPU
        cols = dict(df._cols)
        for name, key, kind in ((self.getOrDefault("rawPredictionCol"), raw, "vector"),
                                (self.getOrDefault("probabilityCol"), prob, "vector"),
                                (self.getOrDefault("predictionCol"), pred, "numeric")):
            if name:
                if name in cols:
                    raise IllegalArgumentException("Output column %s already exists." % name)
                cols[name] = ColumnData(kind, key, "f64")
        return df._with(cols=cols)

    def _tree_strings(self):
        ex = self._forest.export()
        thr = self._forest.thresholds.cpu().numpy()
        out = []
        for t in range(self._forest.T):
            sel = np.nonzero(ex["tree"] == t)[0]
            idx = {int(ex["nid"][i]): i for i in sel}
            lines = []

            def rec(nid, depth):
                i = idx[nid]
                pad = " " * (depth + 1)
                if ex["is_leaf"][i]:
                    lines.append("%sPredict: %.1f" % (pad, float(np.argmax(ex["counts"][i]))))
                    return
                f = int(ex["feat"][i])
                if ex["kind"][i] == 0:
                    v = thr[f, int(ex["bin_thr"][i])]
                    lines.append("%sIf (feature %d <= %s)" % (pad, f, repr(float(v)))); rec(nid * 2, depth + 1)
                    lines.append("%sElse (feature %d > %s)" % (pad, f, repr(float(v)))); rec(nid * 2 + 1, depth + 1)
                else:
                    cats = [c for c in range(256) if (int(ex["mask"][i][c >> 6]) >> (c & 63)) & 1]
                    s = "{%s}" % ",".join("%.1f" % c for c in cats)
                    lines.append("%sIf (feature %d in %s)" % (pad, f, s)); rec(nid * 2, depth + 1)
                    lines.append("%sElse (feature %d not in %s)" % (pad, f, s)); rec(nid * 2 + 1, depth + 1)
            rec(1, 0)
            out.append((len(sel), lines))
        return out


class RandomForestClassificationModel(_ForestModelBase):
    _defaults = {"numTrees": 20, "featureSubsetStrategy": "auto", "subsamplingRate": 1.0}

    @property
    def getNumTrees(self):
        return self._forest.T

    @property
    def treeWeights(self):
        return [1.0] * self._forest.T

    @property
    def toDebugString(self):
        parts = ["RandomForestClassificationModel with %d trees" % self._forest.T]
        for t, (nn, lines) in enumerate(self._tree_strings()):
            parts.append("  Tree %d (weight 1.0):" % t)
            parts += ["  " + l for l in lines]
        return "\n".join(parts) + "\n"

    def __repr__(self):
        return "RandomForestClassificationModel with %d trees" % self._forest.T


class DecisionTreeClassificationModel(_ForestModelBase):
    @property
    def numNodes(self):
        return self._forest.n_nodes

    @property
    def depth(self):
        nid = self._forest.export()["nid"].astype(np.int64)
        return int(np.floor(np.log2(nid.max()))) if len(nid) else 0

    @property
    def toDebugString(self):
        nn, lines = self._tree_strings()[0]
        return "DecisionTreeClassificationModel of depth %d with %d nodes\n%s\n" % (self.depth, nn, "\n".join(lines))

    def __repr__(self):
        return "DecisionTreeClassificationModel of depth %d with %d nodes" % (self.depth, self.numNodes)


# ------------------------------------------------------------------------------- out-of-scope models (torch)
class _ProbModel(Model):
    _defaults = {"featuresCol": "features", "labelCol": "label", "predictionCol": "prediction",
                 "probabilityCol": "probability", "rawPredictionCol": "rawPrediction"}

    def _emit(self, df, raw, prob):
        pred = torch.argmax(raw, 1).to(torch.float64)
        cols = dict(df._cols)
        cols[self.getOrDefault("rawPredictionCol")] = ColumnData("vector", raw, "f64")
        cols[self.getOrDefault("probabilityCol")] = ColumnData("vector", prob, "f64")
        cols[self.getOrDefault("predictionCol")] = ColumnData("numeric", pred, "f64")
        return df._with(cols=cols)


class LogisticRegression(Estimator):
    """Multinomial / binomial elastic-net logistic regression with MLlib's objective (standardised features, unpenalised
    intercepts), minimised by OWL-QN: b200flow/linear.py (kdd99.py:57-58, cicids17.py:61-62)."""
    _defaults = dict(_ProbModel._defaults, maxIter=100, regParam=0.0, elasticNetParam=0.0, tol=1e-6, fitIntercept=True,
                     standardization=True, family="auto", threshold=0.5)

    def __init__(self, featuresCol=None, labelCol=None, predictionCol=None, maxIter=None, regParam=None,
                 elasticNetParam=None, tol=None, fitIntercept=None, threshold=None, probabilityCol=None,
                 rawPredictionCol=None, standardization=None, family=None):
        kw = dict(locals()); kw.pop("self"); kw.pop("__class__", None)
        super().__init__(**kw)

    def _fit(self, df):
        x, y, C, _ = _features_and_labels(df, self)
        g = self.getOrDefault
        if g("family") not in ("auto", "binomial", "multinomial"):
            raise IllegalArgumentException("family must be auto, binomial or multinomial")
        try:
            fit = _linear.lr_fit(x, y, C, max_iter=int(g("maxIter")), reg_param=float(g("regParam")), elastic_net=float(g("elasticNetParam")),
                                 tol=float(g("tol")), fit_intercept=bool(g("fitIntercept")), standardization=bool(g("standardization")),
                                 family=g("family"), group=bdist.group())
        except ValueError as e:
            raise IllegalArgumentException(str(e))
        m = LogisticRegressionModel(fit, C)
        m._paramMap = {k: v for k, v in self._paramMap.items() if k in m._all_defaults()}
        return m


class _TrainingSummary:
    def __init__(self, hist, iterations):
        self.objectiveHistory, self.totalIterations = list(hist), int(iterations)


class LogisticRegressionModel(_ProbModel):
    def __init__(self, fit, C):
        super().__init__()
        self._fit_result, self.numClasses = fit, C
        self.summary = _TrainingSummary(fit.objective_history, fit.iterations)

    @property
    def coefficientMatrix(self):
        return self._fit_result.coef.cpu().numpy()

    @property
    def interceptVector(self):
        return self._fit_result.intercept.cpu().numpy()

    def _transform(self, df):
        raw = _linear.lr_raw(self._fit_result, df._cols[self.getOrDefault("featuresCol")].data)
        return self._emit(df, raw, _linear.lr_probability(self._fit_result, raw))


class NaiveBayes(Estimator):
    """Multinomial naive Bayes with MLlib's smoothed prior and likelihood (b200flow/linear.py; kdd99.py:67, cicids17.py:71);
    rejects negative features as MLlib does (the reason for the where-filters at cicids17.py:30-35)."""
    _defaults = dict(_ProbModel._defaults, smoothing=1.0, modelType="multinomial")

    def __init__(self, featuresCol=None, labelCol=None, predictionCol=None, probabilityCol=None, rawPredictionCol=None,
                 smoothing=None, modelType=None):
        kw = dict(locals()); kw.pop("self"); kw.pop("__class__", None)
        super().__init__(**kw)

    def _fit(self, df):
        if self.getOrDefault("modelType") != "multinomial":
            raise IllegalArgumentException("only modelType='multinomial' is implemented")
        x, y, C, _ = _features_and_labels(df, self)
        try:
            fit = _linear.nb_fit(x, y, C, float(self.getOrDefault("smoothing")), group=bdist.group())
        except ValueError as e:
            raise IllegalArgumentException(str(e))
        m = NaiveBayesModel(fit, C)
        m._paramMap = {k: v for k, v in self._paramMap.items() if k in m._all_defaults()}
        return m


class NaiveBayesModel(_ProbModel):
    def __init__(self, fit, C):
        super().__init__()
        self._fit_result, self.numClasses = fit, C

    @property
    def pi(self):
        return self._fit_result.pi.cpu().numpy()

    @property
    def theta(self):
        return self._fit_result.theta.cpu().numpy()

    def _transform(self, df):
        raw = _linear.nb_raw(self._fit_result, df._cols[self.getOrDefault("featuresCol")].data)
        return self._emit(df, raw, torch.softmax(raw, 1))


# ------------------------------------------------------------------------------- multilayer perceptron (CUDA)
class _MLPParams:
    _defaults = dict(_ProbModel._defaults, layers=None, maxIter=100, tol=1e-6, blockSize=128, solver="l-bfgs", stepSize=0.03,
                     seed=None, initialWeights=None)


class MultilayerPerceptronClassifier(Estimator, _MLPParams):
    """Spark's feed-forward classifier: sigmoid hidden layers, softmax output, trained in fp64 by L-BFGS or gradient
    descent on the device (b200flow/mlp.py).  blockSize is validated but does not change the result (DESIGN.md §5d)."""

    def __init__(self, featuresCol=None, labelCol=None, predictionCol=None, maxIter=None, tol=None, seed=None, layers=None,
                 blockSize=None, stepSize=None, solver=None, initialWeights=None, probabilityCol=None, rawPredictionCol=None):
        kw = dict(locals()); kw.pop("self"); kw.pop("__class__", None)
        super().__init__(**kw)

    def _check(self):
        """Spark's param validators."""
        g = self.getOrDefault
        layers = g("layers")
        if layers is None:
            raise IllegalArgumentException("MultilayerPerceptronClassifier needs the layers param")
        if len(layers) < 2 or any(int(v) != v or int(v) <= 0 for v in layers):
            raise IllegalArgumentException("layers must have at least 2 entries, all integers > 0, got %r" % (list(layers),))
        if int(layers[-1]) < 2:
            raise IllegalArgumentException("the output layer needs at least 2 classes, got %r" % (layers[-1],))
        it, bs = g("maxIter"), g("blockSize")
        if int(it) != it or int(it) < 0:
            raise IllegalArgumentException("maxIter must be an integer >= 0, got %r" % (it,))
        if int(bs) != bs or int(bs) <= 0:
            raise IllegalArgumentException("blockSize must be an integer > 0, got %r" % (bs,))
        for name in ("stepSize", "tol"):
            if not float(g(name)) > 0:
                raise IllegalArgumentException("%s must be > 0, got %r" % (name, g(name)))
        if g("solver") not in ("l-bfgs", "gd"):
            raise IllegalArgumentException("solver must be 'l-bfgs' or 'gd', got %r" % (g("solver"),))
        return [int(v) for v in layers]

    def _fit(self, df):
        layers = self._check()
        g = self.getOrDefault
        x, y, _, _ = _features_and_labels(df, self)
        seed = _default_seed(self) if g("seed") is None else int(g("seed"))
        iw = g("initialWeights")
        if iw is not None and hasattr(iw, "toArray"):
            iw = iw.toArray()
        try:
            fit = _mlp.mlp_fit(x, y, layers, solver=g("solver"), max_iter=int(g("maxIter")), tol=float(g("tol")),
                               step_size=float(g("stepSize")), seed=seed, initial_weights=iw, group=bdist.group())
        except ValueError as e:        # includes b200flow's UnsupportedParamError
            raise IllegalArgumentException(str(e))
        m = MultilayerPerceptronClassificationModel(layers, fit)
        m._paramMap = {k: v for k, v in self._paramMap.items() if k in m._all_defaults()}
        m._paramMap["layers"] = list(layers)
        return m


class MultilayerPerceptronClassificationModel(_ProbModel, _MLPParams):
    def __init__(self, layers, fit):
        super().__init__()
        self._layers, self._weights = list(layers), fit.weights
        self.summary = _TrainingSummary(fit.objective_history, fit.iterations)

    @property
    def layers(self):
        return list(self._layers)

    @property
    def weights(self):
        from .linalg import DenseVector
        return DenseVector(self._weights.cpu().numpy())

    @property
    def numFeatures(self):
        return self._layers[0]

    @property
    def numClasses(self):
        return self._layers[-1]

    def _transform(self, df):
        fcol = self.getOrDefault("featuresCol")
        if fcol not in df._cols or df._cols[fcol].kind != "vector":
            raise IllegalArgumentException("Column %s must be of type vector" % fcol)
        try:
            raw = _mlp.mlp_raw(self._weights, self._layers, df._cols[fcol].data)
        except ValueError as e:
            raise IllegalArgumentException(str(e))
        return self._emit(df, raw, torch.softmax(raw, 1))


# ------------------------------------------------------------------------------- linear SVM (CUDA)
class _LinearSVCParams:
    _defaults = {"featuresCol": "features", "labelCol": "label", "predictionCol": "prediction",
                 "rawPredictionCol": "rawPrediction", "maxIter": 100, "regParam": 0.0, "tol": 1e-6, "fitIntercept": True,
                 "standardization": True, "threshold": 0.0, "aggregationDepth": 2, "maxBlockSizeInMB": 0.0,
                 "weightCol": None}


class LinearSVC(Estimator, _LinearSVCParams):
    """Spark 3's binary LinearSVC [recalled]: the hinge loss plus an L2 penalty on standardised (not centred) features,
    minimised by OWL-QN with a zero L1 weight, on the device (b200flow/svc.py).  aggregationDepth and maxBlockSizeInMB are
    validated but do not change the result: the sums have one fixed order (DESIGN.md §5j)."""

    def __init__(self, featuresCol=None, labelCol=None, predictionCol=None, maxIter=None, regParam=None, tol=None,
                 rawPredictionCol=None, fitIntercept=None, standardization=None, threshold=None, weightCol=None,
                 aggregationDepth=None, maxBlockSizeInMB=None):
        kw = dict(locals()); kw.pop("self"); kw.pop("__class__", None)
        super().__init__(**kw)

    def _check(self):
        """Spark's param validators, and the refusal of weightCol -> b200flow.svc.SVCParams."""
        g = self.getOrDefault
        it, depth = g("maxIter"), g("aggregationDepth")
        if isinstance(it, bool) or int(it) != it or int(it) < 0:
            raise IllegalArgumentException("maxIter must be an integer >= 0, got %r" % (it,))
        if isinstance(depth, bool) or int(depth) != depth or int(depth) < 2:
            raise IllegalArgumentException("aggregationDepth must be an integer >= 2, got %r" % (depth,))
        for name in ("regParam", "tol", "maxBlockSizeInMB"):
            if not float(g(name)) >= 0:
                raise IllegalArgumentException("%s must be >= 0, got %r" % (name, g(name)))
        if g("weightCol"):
            raise IllegalArgumentException("weightCol is not supported by the b200flow LinearSVC (out of scope)")
        return _svc.SVCParams(max_iter=int(it), reg_param=float(g("regParam")), tol=float(g("tol")),
                              fit_intercept=bool(g("fitIntercept")), standardization=bool(g("standardization")))

    def _fit(self, df):
        params = self._check()
        fcol, lcol = self.getOrDefault("featuresCol"), self.getOrDefault("labelCol")
        for c in (fcol, lcol):
            if c not in df._cols:
                raise IllegalArgumentException("Field \"%s\" does not exist." % c)
        if df._cols[fcol].kind != "vector":
            raise IllegalArgumentException("Column %s must be of type vector" % fcol)
        # numClasses and the invalid-label check from values reduced over every rank, so that a rank whose shard is empty
        # or lacks label 1 decides as the others do, and every rank raises or none does
        C = _ovr_num_classes(df, lcol)
        if C != 2:
            raise IllegalArgumentException("LinearSVC only supports binary classification. %d classes detected in %s"
                                           % (C, lcol))
        try:
            fit = _svc.svc_fit_classes(df._cols[fcol].data, df._column_tensor(lcol), [1], params, group=bdist.group())[0]
        except ValueError as e:        # includes b200flow's UnsupportedParamError
            raise IllegalArgumentException(str(e))
        return _svc_model(fit, self._paramMap)


def _svc_model(fit, param_map):
    m = LinearSVCModel(fit)
    m._paramMap = {k: v for k, v in param_map.items() if k in m._all_defaults()}
    return m


class LinearSVCModel(Model, _LinearSVCParams):
    """coefficients (original feature scale), intercept; rawPrediction = [-m, m] with m = x . coefficients + intercept,
    prediction = 1.0 iff m > threshold; no probability column [recalled]."""

    def __init__(self, fit):
        super().__init__()
        self._fit_result = fit             # b200flow.svc.SVCFit
        self.summary = _TrainingSummary(fit.objective_history, fit.iterations)

    @property
    def coefficients(self):
        from .linalg import DenseVector
        return DenseVector(self._fit_result.coef.copy())

    @property
    def intercept(self):
        return self._fit_result.intercept

    @property
    def numClasses(self):
        return 2

    @property
    def numFeatures(self):
        return int(self._fit_result.coef.shape[0])

    def _weights(self):
        """[D + 1] f64 host: the coefficients, then the intercept"""
        return np.concatenate([self._fit_result.coef, [self._fit_result.intercept]])

    def _transform(self, df):
        fcol = self.getOrDefault("featuresCol")
        if fcol not in df._cols or df._cols[fcol].kind != "vector":
            raise IllegalArgumentException("Column %s must be of type vector" % fcol)
        try:
            m = _svc.svc_margins(df._cols[fcol].data, torch.from_numpy(self._weights()).reshape(1, -1))
        except ValueError as e:
            raise IllegalArgumentException(str(e))
        cols = dict(df._cols)
        rcol, pcol = self.getOrDefault("rawPredictionCol"), self.getOrDefault("predictionCol")
        if rcol:
            cols[rcol] = ColumnData("vector", torch.cat([-m, m], 1), "f64")
        if pcol:
            cols[pcol] = ColumnData("numeric", (m[:, 0] > float(self.getOrDefault("threshold"))).to(torch.float64), "f64")
        return df._with(cols=cols)


class _OvRSVCJoint:
    """the K LinearSVC models of a OneVsRest fit as one weight matrix: the K margins of a row in one launch"""

    def __init__(self, models):
        self.weights = torch.from_numpy(np.stack([m._weights() for m in models]))     # [K, D + 1] f64 host

    def predict(self, x):
        raw = _svc.svc_margins(x, self.weights)
        return raw, _first_argmax(raw)


# ------------------------------------------------------------------------------- factorization machines (CUDA)
class _FMParams:
    _defaults = dict(_ProbModel._defaults, factorSize=8, fitIntercept=True, fitLinear=True, regParam=0.0,
                     miniBatchFraction=1.0, initStd=0.01, maxIter=100, stepSize=1.0, tol=1e-6, solver="adamW",
                     thresholds=None, seed=None, weightCol=None)


class FMClassifier(Estimator, _FMParams):
    """Spark 3's binary FMClassifier [recalled]: a factorization machine with the logistic loss, trained by mllib's
    mini-batch gradient descent with the adamW or gd updater, on the device (b200flow/fm.py, csrc/fm.cu, DESIGN.md §5k).
    Features are not standardised."""

    def __init__(self, featuresCol=None, labelCol=None, predictionCol=None, probabilityCol=None, rawPredictionCol=None,
                 factorSize=None, fitIntercept=None, fitLinear=None, regParam=None, miniBatchFraction=None, initStd=None,
                 maxIter=None, stepSize=None, tol=None, solver=None, thresholds=None, seed=None, weightCol=None):
        kw = dict(locals()); kw.pop("self"); kw.pop("__class__", None)
        super().__init__(**kw)

    def _check(self):
        """Spark's param validators, and the refusals of weightCol and thresholds -> b200flow.fm.FMParams."""
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
        if g("solver") not in _fm.SOLVERS:
            raise IllegalArgumentException("solver must be 'gd' or 'adamW', got %r" % (g("solver"),))
        if g("weightCol"):
            raise IllegalArgumentException("weightCol is not supported by the b200flow FMClassifier (out of scope)")
        if g("thresholds") is not None:
            raise IllegalArgumentException("thresholds is not supported by the b200flow FMClassifier")
        seed = g("seed")
        return _fm.FMParams(factor_size=int(fs), fit_intercept=bool(g("fitIntercept")), fit_linear=bool(g("fitLinear")),
                            reg_param=float(g("regParam")), mini_batch_fraction=float(g("miniBatchFraction")),
                            init_std=float(g("initStd")), max_iter=int(it), step_size=float(g("stepSize")),
                            tol=float(g("tol")), solver=g("solver"), seed=_default_seed(self) if seed is None else int(seed))

    def _fit(self, df):
        params = self._check()
        fcol, lcol = self.getOrDefault("featuresCol"), self.getOrDefault("labelCol")
        for c in (fcol, lcol):
            if c not in df._cols:
                raise IllegalArgumentException("Field \"%s\" does not exist." % c)
        if df._cols[fcol].kind != "vector":
            raise IllegalArgumentException("Column %s must be of type vector" % fcol)
        # numClasses from values reduced over every rank, as LinearSVC
        C = _ovr_num_classes(df, lcol)
        if C != 2:
            raise IllegalArgumentException("FMClassifier only supports binary classification. %d classes detected in %s"
                                           % (C, lcol))
        try:
            fit = _fm.fm_fit_classes(df._cols[fcol].data, df._column_tensor(lcol), [1], params, group=bdist.group())[0]
        except ValueError as e:        # includes b200flow's UnsupportedParamError
            raise IllegalArgumentException(str(e))
        return _fm_model(fit, self._paramMap)


def _fm_model(fit, param_map):
    m = FMClassificationModel(fit)
    m._paramMap = {k: v for k, v in param_map.items() if k in m._all_defaults()}
    return m


class FMClassificationModel(_ProbModel, _FMParams):
    """intercept, linear (DenseVector [D]), factors (DenseMatrix D x k); rawPrediction = [-r, r], probability =
    [1 - sigmoid(r), sigmoid(r)], prediction = the first argmax of rawPrediction (1.0 iff r > 0) [recalled]."""

    def __init__(self, fit):
        super().__init__()
        self._fit_result = fit             # b200flow.fm.FMFit
        # Spark's TrainingSummary: totalIterations = objectiveHistory.length - 1
        self.summary = _TrainingSummary(fit.objective_history, max(len(fit.objective_history) - 1, 0))

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
    def numClasses(self):
        return 2

    @property
    def numFeatures(self):
        return int(self._fit_result.factors.shape[0])

    def _weights(self):
        """[D (k + 1) + 1] f64 host: [V (row-major) | w | b], fm_raw's layout"""
        f = self._fit_result
        return np.concatenate([f.factors.reshape(-1), f.linear, [f.intercept]])

    def _transform(self, df):
        fcol = self.getOrDefault("featuresCol")
        if fcol not in df._cols or df._cols[fcol].kind != "vector":
            raise IllegalArgumentException("Column %s must be of type vector" % fcol)
        try:
            r = _fm.fm_raw(df._cols[fcol].data, torch.from_numpy(self._weights()).reshape(1, -1),
                           self._fit_result.factors.shape[1])
        except ValueError as e:
            raise IllegalArgumentException(str(e))
        raw = torch.cat([-r, r], 1)
        p1 = 1.0 / (1.0 + torch.exp(-r))
        cols = dict(df._cols)
        for name, val, kind in ((self.getOrDefault("rawPredictionCol"), raw, "vector"),
                                (self.getOrDefault("probabilityCol"), torch.cat([1.0 - p1, p1], 1), "vector"),
                                (self.getOrDefault("predictionCol"), _first_argmax(raw), "numeric")):
            if name:
                cols[name] = ColumnData(kind, val, "f64")
        return df._with(cols=cols)


class _OvRFMJoint:
    """the K FMClassifier models of a OneVsRest fit as one weight matrix: the K raw values of a row in one launch"""

    def __init__(self, models):
        self.factor_size = models[0]._fit_result.factors.shape[1]
        self.weights = torch.from_numpy(np.stack([m._weights() for m in models]))     # [K, D (k + 1) + 1] f64 host

    def predict(self, x):
        raw = _fm.fm_raw(x, self.weights, self.factor_size)
        return raw, _first_argmax(raw)


# ------------------------------------------------------------------------------- gradient-boosted trees (CUDA)
class _GBTParams(_TreeParams):
    _defaults = {"impurity": "variance", "maxIter": 20, "stepSize": 0.1, "subsamplingRate": 1.0, "featureSubsetStrategy": "all",
                 "lossType": "logistic", "validationTol": 0.01, "validationIndicatorCol": None, "weightCol": None,
                 "minWeightFractionPerNode": 0.0, "leafCol": ""}


class GBTClassifier(Estimator, _GBTParams):
    """Spark 3's GBTClassifier: binary LogLoss boosting of regression trees (variance impurity), trained on the device with
    exact fixed-point histograms (b200flow/gbt.py, csrc/gbt.cu, DESIGN.md §5e); the model is the same bits for any number
    of ranks."""

    def __init__(self, featuresCol=None, labelCol=None, predictionCol=None, maxDepth=None, maxBins=None, minInstancesPerNode=None,
                 minInfoGain=None, maxMemoryInMB=None, cacheNodeIds=None, checkpointInterval=None, lossType=None, maxIter=None,
                 stepSize=None, seed=None, subsamplingRate=None, impurity=None, featureSubsetStrategy=None, validationTol=None,
                 validationIndicatorCol=None, leafCol=None, minWeightFractionPerNode=None, weightCol=None, probabilityCol=None,
                 rawPredictionCol=None):
        kw = dict(locals()); kw.pop("self"); kw.pop("__class__", None)
        super().__init__(**kw)

    def _params(self):
        """Spark's param validators, and the params the device trainer does not implement."""
        from b200flow import gbt as _gbt
        g = self.getOrDefault
        if str(g("lossType")).lower() != "logistic":
            raise IllegalArgumentException("GBTClassifier lossType must be 'logistic', got %r" % (g("lossType"),))
        if str(g("impurity")).lower() != "variance":
            raise IllegalArgumentException("GBTClassifier trains regression trees: impurity must be 'variance', got %r" % (g("impurity"),))
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
        seed = g("seed")
        return _gbt.GBTParams(max_iter=int(it), step_size=step, max_depth=int(g("maxDepth")), max_bins=int(g("maxBins")),
                              min_instances_per_node=int(g("minInstancesPerNode")), min_info_gain=float(g("minInfoGain")),
                              subsampling_rate=rate, feature_subset_strategy=str(g("featureSubsetStrategy")),
                              seed=_default_seed(self) if seed is None else int(seed))

    def _fit(self, df):
        from b200flow import gbt as _gbt
        from .feature import SparkException
        p = self._params()
        binary_only = "GBTClassifier currently only supports binary classification, but %d classes were found"
        fused = _records_fit_inputs(df, self)
        try:
            grp = bdist.group()
            if fused is not None:                           # lazy VectorAssembler output: bin straight from the raw records
                rec, plan, C, attrs = fused
                if C > 2:
                    raise IllegalArgumentException(binary_only % C)
                off, _ = bdist.global_offset(rec.shape[0], rec.device, grp)
                model = _gbt.fit_gbt_records(rec, plan, _arity_from_attrs(attrs, plan.n_out), p, row_offset=off, group=grp)
            else:
                x, y, C, attrs = _features_and_labels(df, self)
                if C > 2:
                    raise IllegalArgumentException(binary_only % C)
                off, _ = bdist.global_offset(x.shape[0], x.device, grp)
                model = _gbt.fit_gbt(x, y.to(torch.int32), _arity_from_attrs(attrs, x.shape[1]), p, row_offset=off, group=grp)
        except fr.InvalidRowsError as e:
            raise SparkException("Encountered NaN/null while assembling a row with handleInvalid = \"error\" (%s)" % e)
        except ValueError as e:        # includes b200flow's UnsupportedParamError; CUDA failures propagate as they are
            raise IllegalArgumentException(str(e))
        m = GBTClassificationModel(model)
        m._paramMap = {k: v for k, v in self._paramMap.items() if k in m._all_defaults()}
        return m


class GBTClassificationModel(Model, _GBTParams):
    def __init__(self, gbt):
        super().__init__()
        self._gbt = gbt

    @property
    def numClasses(self):
        return 2

    @property
    def numFeatures(self):
        return self._gbt.F

    @property
    def getNumTrees(self):
        return self._gbt.T

    @property
    def treeWeights(self):
        return list(self._gbt.tree_weights)

    @property
    def totalNumNodes(self):
        return self._gbt.n_nodes

    @property
    def featureImportances(self):
        from .linalg import DenseVector
        return DenseVector(self._gbt.feature_importances())

    def _transform(self, df):
        fcol = self.getOrDefault("featuresCol")
        if fcol not in df._cols or df._cols[fcol].kind != "vector":
            raise IllegalArgumentException("Column %s must be of type vector" % fcol)
        plan = _lazy_plan(df, fcol)
        if plan is not None and plan.n_out == self._gbt.F:      # lazy features: fused encode -> bins -> tree walk
            from .feature import SparkException
            try:
                raw, prob, pred = self._gbt.predict_records(df._rec, plan, on_invalid="error" if plan.check_nan else "ignore")
            except fr.InvalidRowsError as e:
                raise SparkException("Encountered NaN/null while assembling a row with handleInvalid = \"error\" (%s)" % e)
        else:
            raw, prob, pred = self._gbt.predict(df._cols[fcol].data)
        cols = dict(df._cols)
        for name, val, kind in ((self.getOrDefault("rawPredictionCol"), raw, "vector"),
                                (self.getOrDefault("probabilityCol"), prob, "vector"),
                                (self.getOrDefault("predictionCol"), pred, "numeric")):
            if name:
                if name in cols:
                    raise IllegalArgumentException("Output column %s already exists." % name)
                cols[name] = ColumnData(kind, val, "f64")
        return df._with(cols=cols)

    @property
    def toDebugString(self):
        ex = self._gbt.export()
        thr = self._gbt.forest.thresholds.cpu().numpy()
        parts = ["GBTClassificationModel with %d trees" % self._gbt.T]
        for t in range(self._gbt.T):
            sel = np.nonzero(ex["tree"] == t)[0]
            idx = {int(ex["nid"][i]): i for i in sel}
            parts.append("  Tree %d (weight %r):" % (t, self._gbt.tree_weights[t]))

            def rec(nid, depth):
                i = idx[nid]
                pad = "  " + " " * (depth + 1)
                if ex["is_leaf"][i]:
                    st = ex["stats"][i]
                    parts.append("%sPredict: %r" % (pad, float(st[1]) * 2.0 ** -self._gbt.S / float(st[0])))
                    return
                f = int(ex["feat"][i])
                if ex["kind"][i] == 0:
                    v = repr(float(thr[f, int(ex["bin_thr"][i])]))
                    parts.append("%sIf (feature %d <= %s)" % (pad, f, v)); rec(nid * 2, depth + 1)
                    parts.append("%sElse (feature %d > %s)" % (pad, f, v)); rec(nid * 2 + 1, depth + 1)
                else:
                    cats = [c for c in range(256) if (int(ex["mask"][i][c >> 6]) >> (c & 63)) & 1]
                    s = "{%s}" % ",".join("%.1f" % c for c in cats)
                    parts.append("%sIf (feature %d in %s)" % (pad, f, s)); rec(nid * 2, depth + 1)
                    parts.append("%sElse (feature %d not in %s)" % (pad, f, s)); rec(nid * 2 + 1, depth + 1)
            rec(1, 0)
        return "\n".join(parts) + "\n"

    def __repr__(self):
        return "GBTClassificationModel with %d trees" % self._gbt.T


# ------------------------------------------------------------------------------- one-vs-rest
def _first_argmax(raw):
    """Spark's Vector.argmax per row of raw [n, K]: start at index 0 and move only on a strict `>`.  So a tie keeps the first
    index, -0.0 does not beat +0.0, and a NaN is never chosen unless it sits at index 0 (where nothing beats it); torch.argmax
    treats NaN as the maximum instead."""
    n, K = raw.shape
    arg = torch.zeros(n, dtype=torch.float64, device=raw.device)
    if K == 0:
        return arg
    best = raw[:, 0]
    for k in range(1, K):
        v = raw[:, k]
        gt = v > best
        best = torch.where(gt, v, best)
        arg = torch.where(gt, torch.full_like(arg, float(k)), arg)
    return arg


def _ovr_num_classes(df, lcol):
    """MetadataUtils.getNumClasses of the label column, else max label + 1 (over every rank) [recalled]; invalid labels raise
    as in _features_and_labels."""
    lab_meta = df._cols[lcol].meta.get("ml_attr", {})
    if lab_meta.get("type") == "nominal":
        return len(lab_meta["vals"])
    y = df._column_tensor(lcol).to(torch.float64)
    bad = ((y < 0) | (y != torch.floor(y))).any().reshape(1).to(torch.float64)
    mx = (y.max() if y.numel() else torch.full((), -1.0, dtype=torch.float64, device=y.device)).reshape(1)
    grp = bdist.group()
    if grp is not None:
        import torch.distributed as dist
        bdist.all_reduce_(bad, grp, op=dist.ReduceOp.MAX)
        bdist.all_reduce_(mx, grp, op=dist.ReduceOp.MAX)
    if bool(bad.item()):
        raise IllegalArgumentException("Classifier was given dataset with invalid label. Labels must be integers in [0, numClasses).")
    return int(mx.item()) + 1


class _OneVsRestParams:
    _defaults = {"classifier": None, "featuresCol": "features", "labelCol": "label", "predictionCol": "prediction",
                 "rawPredictionCol": "rawPrediction", "weightCol": None, "parallelism": 1}


class OneVsRest(Estimator, _OneVsRestParams):
    """Spark 3's OneVsRest [recalled]: one binary model per class k, fitted on the label (label == k ? 1.0 : 0.0), which
    carries two-value nominal metadata; the prediction is the first argmax of the models' rawPrediction[1].  A GBTClassifier
    with at most 256 classes (the label byte of a binned record) is trained as ONE class-batched boosting run on the device
    (DESIGN.md §5f), whose K models equal the K separate fits bit for bit; a LinearSVC trains its K models in lockstep on one
    kernel pass per optimiser round (DESIGN.md §5j), each equal to its separate fit bit for bit; an FMClassifier trains its K
    models in lockstep on one kernel pass per gradient-descent iteration (DESIGN.md §5k), each equal to its separate fit bit
    for bit; every other classifier, and
    GBT with more classes, take the generic loop.  parallelism is validated but only orders host work, so it does not change the result (DESIGN.md §6)."""
    GBT_MAX_CLASSES = 256

    def __init__(self, featuresCol=None, labelCol=None, predictionCol=None, rawPredictionCol=None, classifier=None,
                 weightCol=None, parallelism=None):
        kw = dict(locals()); kw.pop("self"); kw.pop("__class__", None)
        super().__init__(**kw)

    def copy(self, extra=None):
        """as in pyspark, the param map also reaches the classifier (fit(df, {gbt.maxDepth: 3}), ParamGridBuilder grids)."""
        c = super().copy(extra)
        staged = {k: v for k, v in (extra or {}).items() if isinstance(k, Param)}
        if staged and c.getOrDefault("classifier") is not None:
            c._paramMap["classifier"] = c.getOrDefault("classifier").copy(staged)
        return c

    def _check(self):
        g = self.getOrDefault
        clf = g("classifier")
        if clf is None:
            raise IllegalArgumentException("OneVsRest needs the classifier param")
        if not isinstance(clf, Estimator) or isinstance(clf, (OneVsRest, Pipeline)):
            raise IllegalArgumentException("OneVsRest classifier must be a classifier Estimator, got %s" % type(clf).__name__)
        if g("weightCol"):
            raise IllegalArgumentException("weightCol is not supported by OneVsRest in this shim")
        par = g("parallelism")
        if isinstance(par, bool) or int(par) != par or int(par) < 1:
            raise IllegalArgumentException("parallelism must be an integer >= 1, got %r" % (par,))
        return clf

    def _binary_copy(self, clf, label_col):
        """the classifier as OneVsRest fits it for one class: its labelCol the relabelled column, its featuresCol and
        predictionCol the OneVsRest's [recalled]"""
        g = self.getOrDefault
        return clf.copy({"labelCol": label_col, "featuresCol": g("featuresCol"), "predictionCol": g("predictionCol")})

    def _fit(self, df):
        clf = self._check()
        fcol, lcol = self.getOrDefault("featuresCol"), self.getOrDefault("labelCol")
        for c in (fcol, lcol):
            if c not in df._cols:
                raise IllegalArgumentException("Field \"%s\" does not exist." % c)
        if df._cols[fcol].kind != "vector":
            raise IllegalArgumentException("Column %s must be of type vector" % fcol)
        K = _ovr_num_classes(df, lcol)
        if K < 1:
            raise IllegalArgumentException("OneVsRest needs at least one class, the label column has none")
        tmp = _ovr_temp_name(df, "ovr_binary_label")
        if type(clf) is GBTClassifier and K <= self.GBT_MAX_CLASSES:
            models, joint = self._fit_gbt(clf, df, K, tmp)
        elif type(clf) is LinearSVC:
            models, joint = self._fit_svc(clf, df, K, tmp)
        elif type(clf) is FMClassifier:
            models, joint = self._fit_fm(clf, df, K, tmp)
        else:
            models, joint = self._fit_generic(clf, df, K, tmp), None
        m = OneVsRestModel(models, joint)
        m._paramMap = {k: v for k, v in self._paramMap.items() if k in m._all_defaults()}
        return m

    def _fit_generic(self, clf, df, K, tmp):
        """K fits of the classifier, one per relabelled frame"""
        y = df._column_tensor(self.getOrDefault("labelCol"))
        out = []
        for k in range(K):
            cols = dict(df._cols)
            cols[tmp] = ColumnData("numeric", (y == k).to(torch.float64), "f64", _BINARY_LABEL_META)
            out.append(self._binary_copy(clf, tmp).fit(df._with(cols=cols)))
        return out

    def _fit_gbt(self, clf, df, K, tmp):
        """the class-batched device trainer -> (K GBTClassificationModels, the joint model)"""
        from b200flow import gbt as _gbt
        from .feature import SparkException
        binary = self._binary_copy(clf, tmp)
        p = binary._params()
        fcol, lcol = self.getOrDefault("featuresCol"), self.getOrDefault("labelCol")
        fused = _records_fit_inputs(df, clf.copy({"featuresCol": fcol, "labelCol": lcol}))
        try:
            grp = bdist.group()
            if fused is not None:                           # lazy VectorAssembler output: bin straight from the raw records
                rec, plan, _, attrs = fused
                off, _ = bdist.global_offset(rec.shape[0], rec.device, grp)
                joint = _gbt.fit_gbt_ovr_records(rec, plan, K, _arity_from_attrs(attrs, plan.n_out), p, row_offset=off, group=grp)
            else:
                fc = df._cols[fcol]
                x, y = fc.data, df._column_tensor(lcol)
                off, _ = bdist.global_offset(x.shape[0], x.device, grp)
                joint = _gbt.fit_gbt_ovr(x, y.to(torch.int32), K, _arity_from_attrs(fc.meta.get("attrs"), x.shape[1]), p,
                                         row_offset=off, group=grp)
        except fr.InvalidRowsError as e:
            raise SparkException("Encountered NaN/null while assembling a row with handleInvalid = \"error\" (%s)" % e)
        except ValueError as e:        # includes b200flow's UnsupportedParamError; CUDA failures propagate as they are
            raise IllegalArgumentException(str(e))
        models = []
        for sub in joint.models:
            m = GBTClassificationModel(sub)
            m._paramMap = {k: v for k, v in binary._paramMap.items() if k in m._all_defaults()}
            models.append(m)
        return models, joint

    def _fit_svc(self, clf, df, K, tmp):
        """the K LinearSVC fits in lockstep on the device (b200flow.svc.svc_fit_classes with positives 0..K-1) -> (K
        LinearSVCModels, the joint model).  A class absent from the rows still gets its model, as its all-0 relabelled
        column carries two-value metadata."""
        binary = self._binary_copy(clf, tmp)
        params = binary._check()
        fcol = df._cols[self.getOrDefault("featuresCol")]
        y = df._column_tensor(self.getOrDefault("labelCol"))
        try:
            fits = _svc.svc_fit_classes(fcol.data, y, range(K), params, group=bdist.group())
        except ValueError as e:        # includes b200flow's UnsupportedParamError
            raise IllegalArgumentException(str(e))
        models = [_svc_model(f, binary._paramMap) for f in fits]
        return models, _OvRSVCJoint(models)

    def _fit_fm(self, clf, df, K, tmp):
        """the K FMClassifier fits in lockstep on the device (b200flow.fm.fm_fit_classes with positives 0..K-1) -> (K
        FMClassificationModels, the joint model).  A class absent from the rows still gets its model."""
        binary = self._binary_copy(clf, tmp)
        params = binary._check()
        fcol = df._cols[self.getOrDefault("featuresCol")]
        y = df._column_tensor(self.getOrDefault("labelCol"))
        try:
            fits = _fm.fm_fit_classes(fcol.data, y, range(K), params, group=bdist.group())
        except ValueError as e:        # includes b200flow's UnsupportedParamError
            raise IllegalArgumentException(str(e))
        models = [_fm_model(f, binary._paramMap) for f in fits]
        return models, _OvRFMJoint(models)


_BINARY_LABEL_META = {"ml_attr": {"type": "nominal", "vals": ["0.0", "1.0"]}}


def _ovr_temp_name(df, base):
    name = base
    while name in df._cols:
        name = "_" + name
    return name


class OneVsRestModel(Model, _OneVsRestParams):
    """models[k]: class k's binary model.  rawPrediction = each model's rawPrediction[1], prediction = the first argmax
    (_first_argmax); no probability column [recalled]."""

    def __init__(self, models, joint=None):
        super().__init__()
        self.models = list(models)
        self._joint = joint                   # b200flow.gbt.OvRGBTModel of a class-batched GBT fit, _OvRSVCJoint, _OvRFMJoint or None

    @property
    def numClasses(self):
        return len(self.models)

    def _transform(self, df):
        fcol = self.getOrDefault("featuresCol")
        if fcol not in df._cols or df._cols[fcol].kind != "vector":
            raise IllegalArgumentException("Column %s must be of type vector" % fcol)
        rcol, pcol = self.getOrDefault("rawPredictionCol"), self.getOrDefault("predictionCol")
        for name in (rcol, pcol):
            if name and name in df._cols:
                raise IllegalArgumentException("Output column %s already exists." % name)
        if self._joint is not None:
            raw, pred = self._joint_predict(df, fcol)
        else:
            tmp = _ovr_temp_name(df, "ovr_raw")
            cols = []
            for m in self.models:
                out = m.copy({"rawPredictionCol": tmp, "predictionCol": "", "probabilityCol": ""}).transform(df)
                cols.append(out._column_tensor(tmp)[:, 1].to(torch.float64))
            raw = torch.stack(cols, 1) if cols else torch.zeros((df.count(), 0), dtype=torch.float64, device=df._device())
            pred = _first_argmax(raw)
        cols = dict(df._cols)
        if rcol:
            cols[rcol] = ColumnData("vector", raw, "f64")
        if pcol:
            cols[pcol] = ColumnData("numeric", pred, "f64")
        return df._with(cols=cols)

    def _joint_predict(self, df, fcol):
        """one tree walk over the K·T trees (b200flow_predict_forest with C = K): the margins and the `>` argmax in one kernel"""
        j = self._joint
        if isinstance(j, (_OvRSVCJoint, _OvRFMJoint)):
            try:
                return j.predict(df._cols[fcol].data)
            except ValueError as e:
                raise IllegalArgumentException(str(e))
        plan = _lazy_plan(df, fcol)
        if plan is not None and plan.n_out == j.F:          # lazy features: fused encode -> bins -> tree walk
            from .feature import SparkException
            try:
                return j.predict_records(df._rec, plan, on_invalid="error" if plan.check_nan else "ignore")
            except fr.InvalidRowsError as e:
                raise SparkException("Encountered NaN/null while assembling a row with handleInvalid = \"error\" (%s)" % e)
        return j.predict(df._cols[fcol].data)
