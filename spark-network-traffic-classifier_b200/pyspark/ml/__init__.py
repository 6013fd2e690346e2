"""pyspark.ml shim: Estimator / Transformer / Model / Pipeline (kdd99.py:36-37)."""
from .param import Param, Params


class Transformer(Params):
    def transform(self, dataset, params=None):
        return (self.copy(params) if params else self)._transform(dataset)


class Estimator(Params):
    def fit(self, dataset, params=None):
        """params: a param map (keyed by names or Params) applied to a copy, or a list / tuple of maps -> one model each."""
        if isinstance(params, (list, tuple)):
            return [self.fit(dataset, p) for p in params]
        return (self.copy(params) if params else self)._fit(dataset)


class Model(Transformer):
    pass


class Pipeline(Estimator):
    """Pipeline(stages=[...]).fit(df): fit estimators in order, transforming the data between them."""
    _defaults = {"stages": None}

    def __init__(self, stages=None):
        super().__init__(stages=stages)

    def getStages(self):
        return list(self.getOrDefault("stages") or [])

    def copy(self, extra=None):
        """as in pyspark, the Params of a map reach the stages that own them (fit(df, {rf.numTrees: 50}) on a pipeline)."""
        c = super().copy(extra)
        staged = {k: v for k, v in (extra or {}).items() if isinstance(k, Param)}
        if staged and c.getOrDefault("stages") is not None:
            c._paramMap["stages"] = [s.copy(staged) for s in c.getStages()]
        return c

    def _fit(self, dataset):
        stages = self.getStages()
        for s in stages:
            if not isinstance(s, (Estimator, Transformer)):
                raise TypeError("Cannot recognize a pipeline stage of type %s." % type(s))
        last_est = max([i for i, s in enumerate(stages) if isinstance(s, Estimator)], default=-1)
        from .feature import StringIndexer, _prefetch_category_counts
        if hasattr(dataset, "_cat_counts"):                # ONE count pass for every StringIndexer stage, before the first host read
            _prefetch_category_counts(dataset, [s.getOrDefault("inputCol") for s in stages if isinstance(s, StringIndexer)])
        fitted, cur = [], dataset
        for i, s in enumerate(stages):
            if isinstance(s, Estimator):
                m = s.fit(cur)
                fitted.append(m)
                if i < last_est:
                    cur = m.transform(cur)
            else:
                fitted.append(s)
                if i < last_est:
                    cur = s.transform(cur)
        return PipelineModel(fitted)


class PipelineModel(Model):
    def __init__(self, stages):
        super().__init__()
        self.stages = list(stages)

    def _transform(self, dataset):
        for s in self.stages:
            dataset = s.transform(dataset)
        return dataset
