"""pyspark.ml.clustering shim: KMeans / KMeansModel on the b200flow k-means kernels (b200flow/kmeans.py, DESIGN.md §5c) and
GaussianMixture / GaussianMixtureModel on the EM kernels (b200flow/gmm.py, DESIGN.md §5g).

The models are the same bits for any number of ranks.  Deviations from Spark: KMeans distances are exact (no
fastSquaredDistance bound), the random draws are this project's Philox streams, distanceMeasure="cosine" and weightCol are
refused; GaussianMixture's deviations are listed in b200flow/gmm.py."""
import numpy as np
import torch

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
