"""pyspark.ml.clustering shim: KMeans / KMeansModel on the b200flow k-means kernels (b200flow/kmeans.py, DESIGN.md §5c),
BisectingKMeans / BisectingKMeansModel on the split-assign and tree-walk kernels (b200flow/bisecting_kmeans.py, DESIGN.md
§5t) and GaussianMixture / GaussianMixtureModel on the EM kernels (b200flow/gmm.py, DESIGN.md §5g).

The models are the same bits for any number of ranks.  Deviations from Spark: KMeans and BisectingKMeans distances are
exact (no fastSquaredDistance bound), the random draws are this project's Philox streams, distanceMeasure="cosine" and
weightCol are refused; BisectingKMeans' cluster costs are exact two-pass sums, children are compared on squared distances
and equally large divisible clusters are chosen by heap index (b200flow/bisecting_kmeans.py); GaussianMixture's
deviations are listed in b200flow/gmm.py."""
import numpy as np
import torch

from b200flow import bisecting_kmeans as _bkm
from b200flow import dist as bdist
from b200flow import gmm as _gm
from b200flow import kmeans as _km

from . import Estimator, Model
from ..sql import ColumnData, LocalFrame
from .classification import _default_seed
from .feature import IllegalArgumentException, _materialize
from .linalg import DenseMatrix, DenseVector
from .stat import MultivariateGaussian


def _features(df, fcol):
    """the features column as a CUDA f64 [n, D] matrix (a lazy assembled / scaled column runs the fused encode kernel once)."""
    c = df._cols.get(fcol)
    if c is None:
        raise IllegalArgumentException("Field \"%s\" does not exist." % fcol)
    if c.kind != "vector":
        raise IllegalArgumentException("Column %s must be of type vector" % fcol)
    return _materialize(df, fcol)


class _KMeansParams:
    _defaults = {"featuresCol": "features", "predictionCol": "prediction", "k": 2, "initMode": "k-means||", "initSteps": 2,
                 "maxIter": 20, "tol": 1e-4, "seed": None, "distanceMeasure": "euclidean", "weightCol": None}


class KMeans(Estimator, _KMeansParams):
    def __init__(self, featuresCol=None, predictionCol=None, k=None, initMode=None, initSteps=None, tol=None, maxIter=None,
                 seed=None, distanceMeasure=None, weightCol=None):
        kw = dict(locals()); kw.pop("self"); kw.pop("__class__", None)
        super().__init__(**kw)

    def _check(self):
        """Spark's param validators, and the refusals of this implementation."""
        g = self.getOrDefault
        k, steps, it, tol = g("k"), g("initSteps"), g("maxIter"), g("tol")
        if int(k) != k or int(k) <= 1:
            raise IllegalArgumentException("KMeans parameter k given invalid value %r: it must be an integer > 1" % (k,))
        if g("initMode") not in ("random", "k-means||"):
            raise IllegalArgumentException("initMode must be 'random' or 'k-means||', got %r" % (g("initMode"),))
        if int(steps) != steps or int(steps) <= 0:
            raise IllegalArgumentException("initSteps must be an integer > 0, got %r" % (steps,))
        if int(it) != it or int(it) < 0:
            raise IllegalArgumentException("maxIter must be an integer >= 0, got %r" % (it,))
        if not float(tol) >= 0:
            raise IllegalArgumentException("tol must be >= 0, got %r" % (tol,))
        dm = g("distanceMeasure")
        if dm == "cosine":
            raise IllegalArgumentException("distanceMeasure='cosine' is not supported by the b200flow KMeans (out of scope); use "
                                           "'euclidean'")
        if dm != "euclidean":
            raise IllegalArgumentException("distanceMeasure must be 'euclidean' or 'cosine', got %r" % (dm,))
        if g("weightCol"):
            raise IllegalArgumentException("weightCol is not supported by the b200flow KMeans (out of scope)")

    def _fit(self, df):
        self._check()
        g = self.getOrDefault
        x = _features(df, g("featuresCol"))
        seed = _default_seed(self) if g("seed") is None else int(g("seed"))
        try:
            res = _km.kmeans_fit(x, int(g("k")), init=g("initMode"), init_steps=int(g("initSteps")), max_iter=int(g("maxIter")),
                                 tol=float(g("tol")), seed=seed, group=bdist.group())
        except ValueError as e:        # includes b200flow's UnsupportedParamError
            raise IllegalArgumentException(str(e))
        m = KMeansModel(res.centers)
        m._paramMap = {k: v for k, v in self._paramMap.items() if k in m._all_defaults()}
        m._summary = KMeansSummary(m._with_prediction(df, res.cluster), res, g("featuresCol"), g("predictionCol"))
        return m


class KMeansModel(Model, _KMeansParams):
    def __init__(self, centers):
        super().__init__()
        self._centers = centers            # CUDA f64 [k, D]
        self._summary = None

    def clusterCenters(self):
        return [r for r in self._centers.cpu().numpy()]

    @property
    def hasSummary(self):
        return self._summary is not None

    @property
    def summary(self):
        if self._summary is None:
            raise RuntimeError("No training summary available for this KMeansModel")
        return self._summary

    def _with_prediction(self, df, cluster):
        name = self.getOrDefault("predictionCol")
        if name in df._cols:
            raise IllegalArgumentException("Output column %s already exists." % name)
        cols = dict(df._cols)
        cols[name] = ColumnData("numeric", cluster.to(torch.int32).contiguous(), "i32")
        return df._with(cols=cols)

    def _transform(self, df):
        cl, _ = _km.kmeans_predict(_features(df, self.getOrDefault("featuresCol")), self._centers)
        return self._with_prediction(df, cl)


class KMeansSummary:
    def __init__(self, predictions, res, featuresCol, predictionCol):
        self.predictions, self.featuresCol, self.predictionCol = predictions, featuresCol, predictionCol
        self.k = int(res.centers.shape[0])
        self.clusterSizes = [int(v) for v in np.asarray(res.cluster_sizes)]
        self.trainingCost = float(res.training_cost)
        self.numIter = int(res.num_iter)

    @property
    def cluster(self):
        return self.predictions.select(self.predictionCol)


class _BisectingKMeansParams:
    _defaults = {"featuresCol": "features", "predictionCol": "prediction", "k": 4, "maxIter": 20, "seed": None,
                 "minDivisibleClusterSize": 1.0, "distanceMeasure": "euclidean", "weightCol": None}


class BisectingKMeans(Estimator, _BisectingKMeansParams):
    """Spark 3's BisectingKMeans (DESIGN.md §5t).  maxIter = 0, which Spark's validator accepts but its fit cannot run, is
    refused here; so are distanceMeasure="cosine", weightCol, more than 256 features and k > 2048."""

    def __init__(self, featuresCol=None, predictionCol=None, maxIter=None, seed=None, k=None, minDivisibleClusterSize=None,
                 distanceMeasure=None, weightCol=None):
        kw = dict(locals()); kw.pop("self"); kw.pop("__class__", None)
        super().__init__(**kw)

    def _check(self):
        """Spark's param validators, and the refusals of this implementation."""
        g = self.getOrDefault
        k, it, mdcs = g("k"), g("maxIter"), g("minDivisibleClusterSize")
        if int(k) != k or int(k) <= 1:
            raise IllegalArgumentException("BisectingKMeans parameter k given invalid value %r: it must be an integer > 1"
                                           % (k,))
        if int(it) != it or int(it) < 1:
            raise IllegalArgumentException("maxIter must be an integer >= 1 for BisectingKMeans, got %r" % (it,))
        if not float(mdcs) > 0.0:
            raise IllegalArgumentException("minDivisibleClusterSize must be > 0, got %r" % (mdcs,))
        dm = g("distanceMeasure")
        if dm == "cosine":
            raise IllegalArgumentException("distanceMeasure='cosine' is not supported by the b200flow BisectingKMeans (out of "
                                           "scope); use 'euclidean'")
        if dm != "euclidean":
            raise IllegalArgumentException("distanceMeasure must be 'euclidean' or 'cosine', got %r" % (dm,))
        if g("weightCol"):
            raise IllegalArgumentException("weightCol is not supported by the b200flow BisectingKMeans (out of scope)")

    def _fit(self, df):
        self._check()
        g = self.getOrDefault
        x = _features(df, g("featuresCol"))
        seed = _default_seed(self) if g("seed") is None else int(g("seed"))
        try:
            res = _bkm.bkm_fit(x, int(g("k")), max_iter=int(g("maxIter")), min_divisible=float(g("minDivisibleClusterSize")),
                               seed=seed, group=bdist.group())
        except ValueError as e:        # includes b200flow's UnsupportedParamError
            raise IllegalArgumentException(str(e))
        m = BisectingKMeansModel(res.tree, res.training_cost)
        m._paramMap = {k: v for k, v in self._paramMap.items() if k in m._all_defaults()}
        m._summary = BisectingKMeansSummary(m._with_prediction(df, res.leaf), res, int(g("k")), int(g("maxIter")),
                                            g("featuresCol"), g("predictionCol"))
        return m


class BisectingKMeansModel(Model, _BisectingKMeansParams):
    def __init__(self, tree, training_cost):
        super().__init__()
        self._tree = tree                  # b200flow.bisecting_kmeans.Tree
        self._training_cost = float(training_cost)
        self._summary = None

    def clusterCenters(self):
        return [r.copy() for r in self._tree.center[self._tree.leaf_nodes()]]

    @property
    def trainingCost(self):
        return self._training_cost

    @property
    def hasSummary(self):
        return self._summary is not None

    @property
    def summary(self):
        if self._summary is None:
            raise RuntimeError("No training summary available for this BisectingKMeansModel")
        return self._summary

    def _check_width(self, x):
        if x.shape[1] != self._tree.center.shape[1]:
            raise IllegalArgumentException("the model has %d features, the data %d" % (self._tree.center.shape[1], x.shape[1]))
        return x

    def predict(self, features):
        """the leaf index of one feature vector, the walk transform takes"""
        v = np.asarray(features.toArray() if hasattr(features, "toArray") else features, np.float64).reshape(1, -1)
        leaf, _ = _bkm.bkm_predict(self._check_width(torch.from_numpy(v).cuda()), self._tree)
        return int(leaf[0].item())

    def computeCost(self, dataset):
        """the sum of squared distances of the rows to the leaf centers they reach (deprecated in Spark 3, still there)"""
        x = self._check_width(_features(dataset, self.getOrDefault("featuresCol")))
        return _bkm.compute_cost(x, self._tree, group=bdist.group())

    def _with_prediction(self, df, leaf):
        name = self.getOrDefault("predictionCol")
        if name in df._cols:
            raise IllegalArgumentException("Output column %s already exists." % name)
        cols = dict(df._cols)
        cols[name] = ColumnData("numeric", leaf.to(torch.int32).contiguous(), "i32")
        return df._with(cols=cols)

    def _transform(self, df):
        x = self._check_width(_features(df, self.getOrDefault("featuresCol")))
        leaf, _ = _bkm.bkm_predict(x, self._tree)
        return self._with_prediction(df, leaf)


class BisectingKMeansSummary:
    def __init__(self, predictions, res, k, max_iter, featuresCol, predictionCol):
        self.predictions, self.featuresCol, self.predictionCol = predictions, featuresCol, predictionCol
        self.k = k
        self.clusterSizes = [int(v) for v in _bkm.cluster_sizes(res.leaf, k)]
        self.trainingCost = float(res.training_cost)
        self.numIter = max_iter

    @property
    def cluster(self):
        return self.predictions.select(self.predictionCol)


class _GaussianMixtureParams:
    _defaults = {"featuresCol": "features", "predictionCol": "prediction", "probabilityCol": "probability", "k": 2,
                 "maxIter": 100, "tol": 0.01, "seed": None, "aggregationDepth": 2, "weightCol": None}


class GaussianMixture(Estimator, _GaussianMixtureParams):
    def __init__(self, featuresCol=None, predictionCol=None, k=None, probabilityCol=None, tol=None, maxIter=None, seed=None,
                 aggregationDepth=None, weightCol=None):
        kw = dict(locals()); kw.pop("self"); kw.pop("__class__", None)
        super().__init__(**kw)

    def _check(self):
        """Spark's param validators, and the refusals of this implementation (aggregationDepth is validated but has no
        effect: the sums have one fixed order)."""
        g = self.getOrDefault
        k, it, tol, depth = g("k"), g("maxIter"), g("tol"), g("aggregationDepth")
        if int(k) != k or int(k) <= 1:
            raise IllegalArgumentException("GaussianMixture parameter k given invalid value %r: it must be an integer > 1"
                                           % (k,))
        if int(it) != it or int(it) < 0:
            raise IllegalArgumentException("maxIter must be an integer >= 0, got %r" % (it,))
        if not float(tol) >= 0:
            raise IllegalArgumentException("tol must be >= 0, got %r" % (tol,))
        if int(depth) != depth or int(depth) < 2:
            raise IllegalArgumentException("aggregationDepth must be an integer >= 2, got %r" % (depth,))
        if g("weightCol"):
            raise IllegalArgumentException("weightCol is not supported by the b200flow GaussianMixture (out of scope)")

    def _fit(self, df):
        self._check()
        g = self.getOrDefault
        x = _features(df, g("featuresCol"))
        seed = _default_seed(self) if g("seed") is None else int(g("seed"))
        try:
            fit = _gm.gmm_fit(x, int(g("k")), max_iter=int(g("maxIter")), tol=float(g("tol")), seed=seed, group=bdist.group())
        except ValueError as e:        # includes b200flow's UnsupportedParamError
            raise IllegalArgumentException(str(e))
        m = GaussianMixtureModel(fit)
        m._paramMap = {k: v for k, v in self._paramMap.items() if k in m._all_defaults()}
        m._summary = GaussianMixtureSummary(m._with_outputs(df, fit.prob, fit.pred), fit, g("featuresCol"), g("predictionCol"),
                                            g("probabilityCol"))
        return m


class GaussianMixtureModel(Model, _GaussianMixtureParams):
    def __init__(self, fit):
        super().__init__()
        self._fit_result = fit             # b200flow.gmm.GMMFit
        self._summary = None

    @property
    def weights(self):
        return [float(v) for v in self._fit_result.weights]

    @property
    def gaussians(self):
        f = self._fit_result
        D = f.means.shape[1]
        return [MultivariateGaussian(DenseVector(m.copy()), DenseMatrix(D, D, c.T.ravel()))
                for m, c in zip(f.means, f.covariances)]

    @property
    def gaussiansDF(self):
        import pandas as pd
        gs = self.gaussians
        return LocalFrame(pd.DataFrame({"mean": [g.mean for g in gs], "cov": [g.cov for g in gs]}))

    @property
    def hasSummary(self):
        return self._summary is not None

    @property
    def summary(self):
        if self._summary is None:
            raise RuntimeError("No training summary available for this GaussianMixtureModel")
        return self._summary

    def _with_outputs(self, df, prob, pred):
        names = [self.getOrDefault("probabilityCol"), self.getOrDefault("predictionCol")]
        for name in names:
            if name in df._cols:
                raise IllegalArgumentException("Output column %s already exists." % name)
        cols = dict(df._cols)
        cols[names[0]] = ColumnData("vector", prob, "f64")
        cols[names[1]] = ColumnData("numeric", pred.to(torch.int32).contiguous(), "i32")
        return df._with(cols=cols)

    def _transform(self, df):
        try:
            prob, pred = _gm.gmm_predict(_features(df, self.getOrDefault("featuresCol")), self._fit_result)
        except ValueError as e:
            raise IllegalArgumentException(str(e))
        return self._with_outputs(df, prob, pred)


class GaussianMixtureSummary:
    def __init__(self, predictions, fit, featuresCol, predictionCol, probabilityCol):
        self.predictions, self.featuresCol = predictions, featuresCol
        self.predictionCol, self.probabilityCol = predictionCol, probabilityCol
        self.k = int(fit.weights.shape[0])
        self.clusterSizes = [int(v) for v in np.asarray(fit.cluster_sizes)]
        self.logLikelihood = float(fit.log_likelihood)
        self.numIter = int(fit.num_iter)

    @property
    def cluster(self):
        return self.predictions.select(self.predictionCol)

    @property
    def probability(self):
        return self.predictions.select(self.probabilityCol)
