"""pyspark.ml.tuning shim: ParamGridBuilder, CrossValidator and TrainValidationSplit.

A RandomForestClassifier / DecisionTreeClassifier scored by a MulticlassClassificationEvaluator on the estimator's own label
and prediction columns, with any metric derived from the confusion matrix (every metric but logLoss; by-label metrics with
the evaluator's metricLabel and beta), takes the fast path: per fold and per fit group (b200flow.tuning.fit_groups) ONE
forest fit at (T_max, d_max), then ONE ForestModel.grid_confusion pass that yields the confusion matrix of every
(numTrees, maxDepth) point.  A BinaryClassificationEvaluator on the estimator's label and rawPrediction columns takes the
same path through ForestModel.grid_binary_metrics (the score of every grid point per distinct validation record, then the
device sort-and-scan over the I·J segments).  Each point's metric equals what fitting that point on its own and evaluating
it would give, bit for bit (DESIGN.md §5a, §5b).  Every other estimator / evaluator (logLoss, and collectSubModels=True)
runs the generic loop: fit, transform, evaluate per map.
"""
import itertools

import numpy as np
import torch

from b200flow import dist as bdist
from b200flow import tuning as _tuning

from . import Estimator, Model
from .classification import (DecisionTreeClassifier, RandomForestClassifier, _default_seed, _lazy_plan,
                             _records_fit_inputs)
from .evaluation import BinaryClassificationEvaluator, MulticlassClassificationEvaluator
from .param import Param


class ParamGridBuilder:
    """the cartesian product of the grids added, in pyspark's order: the first grid added varies slowest."""

    def __init__(self):
        self._param_grid = {}

    def addGrid(self, param, values):
        if not isinstance(param, Param):
            raise TypeError("addGrid expects a Param (est.numTrees), got %r" % (param,))
        self._param_grid[param] = list(values)
        return self

    def baseOn(self, *args):
        """fixed values for every map: baseOn({p: v, ...}) or baseOn((p, v), ...)"""
        if len(args) == 1 and isinstance(args[0], dict):
            return self.baseOn(*args[0].items())
        for param, value in args:
            self.addGrid(param, [value])
        return self

    def build(self):
        keys = list(self._param_grid)
        return [dict(zip(keys, prod)) for prod in itertools.product(*[self._param_grid[k] for k in keys])]


class _ValidatorParams:
    _defaults = {"estimator": None, "estimatorParamMaps": None, "evaluator": None, "seed": None, "parallelism": 1,
                 "collectSubModels": False}

    def _seed(self):
        s = self.getOrDefault("seed")
        return _default_seed(self) if s is None else int(s)

    def _parts(self):
        est, maps, ev = self.getOrDefault("estimator"), self.getOrDefault("estimatorParamMaps"), self.getOrDefault("evaluator")
        if est is None or ev is None or not maps:
            raise ValueError("%s needs an estimator, a non-empty estimatorParamMaps and an evaluator" % type(self).__name__)
        return est, list(maps), ev

    def _score(self, est, maps, ev, train, val):
        """-> (metric per map on val for models fitted on train, the fitted models or None)"""
        if not self.getOrDefault("collectSubModels"):
            fast = _grid_metrics(est, maps, ev, train, val)
            if fast is not None:
                return fast, None
        models = [est.fit(train, m) for m in maps]
        return [ev.evaluate(m.transform(val)) for m in models], models

    def _best(self, ev, metrics):
        return int(np.argmax(metrics)) if ev.isLargerBetter() else int(np.argmin(metrics))


def _grid_metrics(est, maps, ev, train, val):
    """the fast path (module docstring) -> list of metrics, or None when the inputs do not qualify."""
    binary = type(ev) is BinaryClassificationEvaluator
    if type(est) not in (RandomForestClassifier, DecisionTreeClassifier) or \
            (type(ev) is not MulticlassClassificationEvaluator and not binary):
        return None
    name = ev._check()
    if name == "logLoss":                                  # reads the probability column: no confusion matrix gives it
        return None
    resolved = [est.copy(m) for m in maps]
    values = [{k: e.getOrDefault(k) for k in e._all_defaults()} for e in resolved]
    lcol = ev.getOrDefault("labelCol")
    ocol, key = ("rawPredictionCol", "rawPredictionCol") if binary else ("predictionCol", "predictionCol")
    if any(v["labelCol"] != lcol or v[key] != ev.getOrDefault(ocol) for v in values):
        return None
    dt = type(est) is DecisionTreeClassifier
    out = [None] * len(maps)
    for T_max, d_max, members in _tuning.fit_groups(values, decision_tree=dt):
        rep = resolved[members[0][0]]
        rep = rep.copy({"maxDepth": d_max} if dt else {"numTrees": T_max, "maxDepth": d_max})
        forest = rep.fit(train)._forest
        tree_cuts = sorted({t for _, t, _ in members})
        depth_cuts = sorted({d for _, _, d in members})
        if binary:
            if forest.C < 2:                               # no rawPrediction[1]: the generic loop raises as evaluate does
                return None
            auc = _grid_on_val(forest, rep, val, tree_cuts, depth_cuts, int(ev.getOrDefault("numBins")))
            col = 0 if name == "areaUnderROC" else 1
            for i, t, d in members:
                out[i] = float(auc[tree_cuts.index(t), depth_cuts.index(d), col])
            continue
        cm = _grid_on_val(forest, rep, val, tree_cuts, depth_cuts).numpy()
        for i, t, d in members:
            c = cm[tree_cuts.index(t), depth_cuts.index(d)]
            nz = np.nonzero(c)
            side = int(max(nz[0].max(), nz[1].max())) + 1 if nz[0].size else 1     # the evaluator's max(label, prediction) + 1
            out[i] = ev._metric_from_confusion(c[:side, :side], name)
    return out


def _grid_on_val(forest, est, val, tree_cuts, depth_cuts, num_bins=None):
    """grid_confusion (num_bins None) or grid_binary_metrics on the validation frame, through the path model.transform would
    take (raw records or the dense vector)."""
    fcol, lcol = est.getOrDefault("featuresCol"), est.getOrDefault("labelCol")
    grp = bdist.group()
    plan = _lazy_plan(val, fcol)
    fused = _records_fit_inputs(val, est) if plan is not None and plan.n_out == forest.F else None
    if fused is not None:                                  # lazy features and indexed label: fused encode -> bins, labels < C
        rec, plan_l, _, _ = fused
        if num_bins is not None:
            return forest.grid_binary_metrics(rec, tree_cuts, depth_cuts, plan=plan_l, num_bins=num_bins, group=grp)
        return forest.grid_confusion(rec, tree_cuts, depth_cuts, plan=plan_l, group=grp)
    x = val._cols[fcol].data
    y = val._column_tensor(lcol).to(torch.float64)
    if num_bins is not None:
        return forest.grid_binary_metrics(x, tree_cuts, depth_cuts, labels=y.to(torch.int32), num_bins=num_bins, group=grp)
    mx = (y.max() if y.numel() else torch.zeros((), dtype=torch.float64, device=y.device)).reshape(1)
    if grp is not None:
        import torch.distributed as dist
        bdist.all_reduce_(mx, grp, op=dist.ReduceOp.MAX)
    return forest.grid_confusion(x, tree_cuts, depth_cuts, labels=y.to(torch.int32), cm_side=int(mx.item()) + 1, group=grp)


def fold_frames(dataset, k, seed):
    """the k (training, validation) frames of a k-fold split: fold ids from random_split_ids(n, [1] * k, seed, global row
    offset) (DESIGN.md §5), fold i = the two stable compactions of the frame by id != i / id == i.  A generator: one fold's
    frames exist at a time."""
    from b200flow.rows import random_split_ids
    dev = dataset._device()
    off, _ = bdist.global_offset(dataset.count(), dev)
    fid = random_split_ids(dataset.count(), [1.0] * k, seed, off, dev)
    for i in range(k):
        yield dataset._compact(fid != i), dataset._compact(fid == i)


class CrossValidator(Estimator, _ValidatorParams):
    _defaults = {"numFolds": 3, "foldCol": ""}

    def __init__(self, estimator=None, estimatorParamMaps=None, evaluator=None, numFolds=None, seed=None, parallelism=None,
                 collectSubModels=None, foldCol=None):
        kw = dict(locals()); kw.pop("self"); kw.pop("__class__", None)
        super().__init__(**kw)

    def _fit(self, dataset):
        est, maps, ev = self._parts()
        k = int(self.getOrDefault("numFolds"))
        if k < 2:
            raise ValueError("numFolds must be >= 2, got %d" % k)
        if self.getOrDefault("foldCol"):
            raise NotImplementedError("foldCol is not supported by this shim")
        sums = [0.0] * len(maps)
        sub = [] if self.getOrDefault("collectSubModels") else None
        for train, val in fold_frames(dataset, k, self._seed()):
            metrics, models = self._score(est, maps, ev, train, val)
            sums = [s + m for s, m in zip(sums, metrics)]
            if sub is not None:
                sub.append(models)
        avg = [s / k for s in sums]
        best = est.fit(dataset, maps[self._best(ev, avg)])
        return CrossValidatorModel(best, avg, sub)


class CrossValidatorModel(Model):
    def __init__(self, bestModel, avgMetrics=None, subModels=None):
        super().__init__()
        self.bestModel, self.avgMetrics, self.subModels = bestModel, list(avgMetrics or []), subModels

    def _transform(self, dataset):
        return self.bestModel.transform(dataset)


class TrainValidationSplit(Estimator, _ValidatorParams):
    _defaults = {"trainRatio": 0.75}

    def __init__(self, estimator=None, estimatorParamMaps=None, evaluator=None, trainRatio=None, seed=None, parallelism=None,
                 collectSubModels=None):
        kw = dict(locals()); kw.pop("self"); kw.pop("__class__", None)
        super().__init__(**kw)

    def _fit(self, dataset):
        est, maps, ev = self._parts()
        r = float(self.getOrDefault("trainRatio"))
        train, val = dataset.randomSplit([r, 1.0 - r], seed=self._seed())
        metrics, models = self._score(est, maps, ev, train, val)
        best = est.fit(dataset, maps[self._best(ev, metrics)])
        return TrainValidationSplitModel(best, metrics, models)


class TrainValidationSplitModel(Model):
    def __init__(self, bestModel, validationMetrics=None, subModels=None):
        super().__init__()
        self.bestModel, self.validationMetrics, self.subModels = bestModel, list(validationMetrics or []), subModels

    def _transform(self, dataset):
        return self.bestModel.transform(dataset)
