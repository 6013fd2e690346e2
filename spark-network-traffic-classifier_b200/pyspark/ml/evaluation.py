"""pyspark.ml.evaluation (kdd99.py:86-91; cicids17.py:90-95).

MulticlassClassificationEvaluator: confusion counts by the b200flow kernel (R10), metrics per MulticlassMetrics (A.8) +
macro-F1; logLoss from the probability column.  BinaryClassificationEvaluator: areaUnderROC / areaUnderPR by the device
sort-and-scan of b200flow.metrics (DESIGN.md §5b).  ClusteringEvaluator: the silhouette of b200flow.kmeans (DESIGN.md §5c).
RegressionEvaluator: exact fixed-point sums of b200flow.metrics.regression_metrics (DESIGN.md §5l)."""
import math

import torch

from b200flow import dist as bdist
from b200flow import forest as fr
from b200flow import metrics as bm

from .feature import IllegalArgumentException, _materialize
from .param import Params

__all__ = ["BinaryClassificationEvaluator", "ClusteringEvaluator", "MulticlassClassificationEvaluator", "RegressionEvaluator"]


class MulticlassClassificationEvaluator(Params):
    _defaults = {"predictionCol": "prediction", "labelCol": "label", "metricName": "f1", "metricLabel": 0.0, "beta": 1.0,
                 "eps": 1e-15, "probabilityCol": "probability", "weightCol": None}
    _metrics = ("f1", "accuracy", "weightedPrecision", "weightedRecall", "macroF1",
                "weightedTruePositiveRate", "weightedFalsePositiveRate", "weightedFMeasure",
                "truePositiveRateByLabel", "falsePositiveRateByLabel", "precisionByLabel", "recallByLabel", "fMeasureByLabel",
                "hammingLoss", "logLoss")
    _smaller_is_better = ("hammingLoss", "logLoss")

    def __init__(self, predictionCol=None, labelCol=None, metricName=None, weightCol=None, metricLabel=None, beta=None,
                 probabilityCol=None, eps=None):
        super().__init__(predictionCol=predictionCol, labelCol=labelCol, metricName=metricName, weightCol=weightCol,
                         metricLabel=metricLabel, beta=beta, probabilityCol=probabilityCol, eps=eps)

    def _check(self):
        """-> the metric name, after the checks Spark makes on the params."""
        name = self.getOrDefault("metricName")
        if name not in self._metrics:
            raise ValueError("metricName must be one of %s, got %r" % (list(self._metrics), name))
        if self.getOrDefault("weightCol"):
            raise IllegalArgumentException("weightCol is not supported by this evaluator (integer counts keep the metrics exact)")
        if not float(self.getOrDefault("beta")) > 0:
            raise IllegalArgumentException("beta must be > 0, got %r" % (self.getOrDefault("beta"),))
        ml = float(self.getOrDefault("metricLabel"))
        if not (math.isfinite(ml) and ml >= 0):
            raise IllegalArgumentException("metricLabel must be a finite number >= 0, got %r" % (self.getOrDefault("metricLabel"),))
        eps = float(self.getOrDefault("eps"))
        if not 0 < eps < 0.5:
            raise IllegalArgumentException("eps must be in range (0, 0.5), got %r" % (eps,))
        return name

    def confusionMatrix(self, dataset):
        pred = dataset._column_tensor(self.getOrDefault("predictionCol")).to(torch.float64).contiguous()
        lab = dataset._column_tensor(self.getOrDefault("labelCol")).to(torch.float64).contiguous()
        # an empty local shard still takes part in both collectives (every rank issues the same sequence)
        mx = (torch.maximum(pred.max(), lab.max()) if pred.numel() else torch.zeros((), dtype=torch.float64, device=pred.device)).reshape(1)
        if bdist.group() is not None:
            import torch.distributed as dist
            bdist.all_reduce_(mx, bdist.group(), op=dist.ReduceOp.MAX)
        C = int(mx.item()) + 1
        return bdist.all_reduce_sum_(fr.confusion_matrix(pred, lab, C)).cpu()

    def _metric_from_confusion(self, cm, name):
        """one confusion-derived metric of the C x C counts (also what the tuning fast path applies to each grid point)."""
        m = fr.metrics_from_confusion(cm, metric_label=float(self.getOrDefault("metricLabel")),
                                      beta=float(self.getOrDefault("beta")))
        if name not in m:
            raise IllegalArgumentException("metricLabel %r is not a label of the dataset" % (self.getOrDefault("metricLabel"),))
        return m[name]

    def _log_loss(self, dataset):
        """mean over the rows of -log(probability[label]), clipped to [eps, 1 - eps] as Spark does; fp64 torch on the device,
        the sum and the count all-reduced over the ranks."""
        prob = dataset._column_tensor(self.getOrDefault("probabilityCol")).to(torch.float64)
        lab = dataset._column_tensor(self.getOrDefault("labelCol")).to(torch.float64)
        eps = float(self.getOrDefault("eps"))
        li = lab.to(torch.int64)
        bad = ((li.to(torch.float64) != lab) | (li < 0) | (li >= prob.shape[1])).sum().reshape(1) if lab.numel() else \
            torch.zeros(1, dtype=torch.int64, device=lab.device)
        p = prob.gather(1, li.clamp(0, max(prob.shape[1] - 1, 0)).reshape(-1, 1)).reshape(-1) if lab.numel() else prob.new_zeros(0)
        loss = torch.where(p < eps, -math.log(eps), torch.where(p > 1 - eps, -math.log1p(-eps), -torch.log(p)))
        acc = torch.stack([loss.sum(), torch.tensor(float(lab.numel()), dtype=torch.float64, device=loss.device),
                           bad.to(torch.float64).reshape(())])
        bdist.all_reduce_sum_(acc)
        s, n, nbad = acc.cpu().tolist()
        if nbad:
            raise IllegalArgumentException("logLoss: %d labels are not integers in [0, %d)" % (int(nbad), prob.shape[1]))
        if n == 0:
            raise IllegalArgumentException("logLoss: the dataset is empty")
        return s / n

    def evaluate(self, dataset, params=None):
        ev = self.copy(params) if params else self
        name = ev._check()
        if name == "logLoss":
            return ev._log_loss(dataset)
        return ev._metric_from_confusion(ev.confusionMatrix(dataset).numpy(), name)

    def isLargerBetter(self):
        return self.getOrDefault("metricName") not in self._smaller_is_better


class BinaryClassificationEvaluator(Params):
    """areaUnderROC (default) / areaUnderPR of BinaryClassificationMetrics(score, label, numBins).  The score is element 1
    of a vector rawPredictionCol, or the column itself when it is numeric; a row is positive iff label > 0.5.  Deviations
    from Spark: a NaN score and an empty dataset raise IllegalArgumentException; weightCol is not supported."""
    _defaults = {"rawPredictionCol": "rawPrediction", "labelCol": "label", "metricName": "areaUnderROC", "numBins": 1000,
                 "weightCol": None}
    _metrics = ("areaUnderROC", "areaUnderPR")

    def __init__(self, rawPredictionCol=None, labelCol=None, metricName=None, weightCol=None, numBins=None):
        super().__init__(rawPredictionCol=rawPredictionCol, labelCol=labelCol, metricName=metricName, weightCol=weightCol,
                         numBins=numBins)

    def _check(self):
        name = self.getOrDefault("metricName")
        if name not in self._metrics:
            raise ValueError("metricName must be one of %s, got %r" % (list(self._metrics), name))
        if self.getOrDefault("weightCol"):
            raise IllegalArgumentException("weightCol is not supported by this evaluator (integer counts keep the areas exact)")
        nb = self.getOrDefault("numBins")
        if int(nb) != nb or int(nb) < 0:
            raise IllegalArgumentException("numBins must be an integer >= 0, got %r" % (nb,))
        return name

    def _scores(self, dataset):
        col = self.getOrDefault("rawPredictionCol")
        c = dataset._cols.get(col)
        if c is None:
            raise ValueError("cannot resolve '%s' given input columns: %s" % (col, list(dataset._cols)))
        t = dataset._column_tensor(col)
        if c.kind == "vector":
            if t.shape[1] < 2:
                raise IllegalArgumentException("rawPredictionCol %s has %d elements; the score is element 1" % (col, t.shape[1]))
            t = t[:, 1]
        return t.to(torch.float64).contiguous()

    def evaluate(self, dataset, params=None):
        ev = self.copy(params) if params else self
        name = ev._check()
        scores = ev._scores(dataset)
        labels = dataset._column_tensor(ev.getOrDefault("labelCol")).to(torch.float64).contiguous()
        try:
            return bm.binary_metrics(scores, labels, num_bins=int(ev.getOrDefault("numBins")))[name]
        except bm.InvalidScoresError as e:
            raise IllegalArgumentException(str(e)) from None

    def isLargerBetter(self):
        return True


class ClusteringEvaluator(Params):
    """silhouette with the squared Euclidean distance (Spark's SquaredEuclideanSilhouette), by b200flow.kmeans.silhouette:
    the cluster statistics come from one grouped sum, so the value is the same bits for any world size.  Deviations from
    Spark: distanceMeasure="cosine" and weightCol are not supported."""
    _defaults = {"featuresCol": "features", "predictionCol": "prediction", "metricName": "silhouette",
                 "distanceMeasure": "squaredEuclidean", "weightCol": None}

    def __init__(self, predictionCol=None, featuresCol=None, metricName=None, distanceMeasure=None, weightCol=None):
        super().__init__(predictionCol=predictionCol, featuresCol=featuresCol, metricName=metricName,
                         distanceMeasure=distanceMeasure, weightCol=weightCol)

    def _check(self):
        if self.getOrDefault("metricName") != "silhouette":
            raise IllegalArgumentException("metricName must be 'silhouette', got %r" % (self.getOrDefault("metricName"),))
        dm = self.getOrDefault("distanceMeasure")
        if dm == "cosine":
            raise IllegalArgumentException("distanceMeasure='cosine' is not supported by this evaluator (out of scope); use "
                                           "'squaredEuclidean'")
        if dm != "squaredEuclidean":
            raise IllegalArgumentException("distanceMeasure must be 'squaredEuclidean' or 'cosine', got %r" % (dm,))
        if self.getOrDefault("weightCol"):
            raise IllegalArgumentException("weightCol is not supported by this evaluator (out of scope)")

    def evaluate(self, dataset, params=None):
        from b200flow import kmeans as bk
        ev = self.copy(params) if params else self
        ev._check()
        fcol = ev.getOrDefault("featuresCol")
        if fcol not in dataset._cols or dataset._cols[fcol].kind != "vector":
            raise IllegalArgumentException("Column %s must be of type vector" % fcol)
        x = _materialize(dataset, fcol)
        cl = dataset._column_tensor(ev.getOrDefault("predictionCol"))
        try:
            return bk.silhouette(x, cl)
        except ValueError as e:
            raise IllegalArgumentException(str(e)) from None

    def isLargerBetter(self):
        return True


class RegressionEvaluator(Params):
    """rmse (default) / mse / r2 / mae / var of RegressionMetrics(prediction, label), from sums that are exact in 128-bit
    fixed point on the device: the same bits for any world size or shard layout.  A non-finite label or prediction makes
    the metric NaN, and so does an empty dataset.  Deviation from Spark: weightCol is not supported."""
    _defaults = {"predictionCol": "prediction", "labelCol": "label", "metricName": "rmse", "weightCol": None,
                 "throughOrigin": False}
    _metrics = ("rmse", "mse", "r2", "mae", "var")

    def __init__(self, predictionCol=None, labelCol=None, metricName=None, weightCol=None, throughOrigin=None):
        super().__init__(predictionCol=predictionCol, labelCol=labelCol, metricName=metricName, weightCol=weightCol,
                         throughOrigin=throughOrigin)

    def _check(self):
        name = self.getOrDefault("metricName")
        if name not in self._metrics:
            raise ValueError("metricName must be one of %s, got %r" % (list(self._metrics), name))
        if self.getOrDefault("weightCol"):
            raise NotImplementedError("weightCol is not supported by RegressionEvaluator")
        return name

    def evaluate(self, dataset, params=None):
        ev = self.copy(params) if params else self
        name = ev._check()
        for c in (ev.getOrDefault("labelCol"), ev.getOrDefault("predictionCol")):
            if c not in dataset._cols:
                raise IllegalArgumentException("Field \"%s\" does not exist." % c)
        pred = dataset._column_tensor(ev.getOrDefault("predictionCol"))
        lab = dataset._column_tensor(ev.getOrDefault("labelCol"))
        return bm.regression_metrics(lab, pred, through_origin=bool(ev.getOrDefault("throughOrigin")))[name]

    def isLargerBetter(self):
        return self.getOrDefault("metricName") in ("r2", "var")
