"""pyspark.ml.feature shim: StringIndexer, VectorAssembler (used by the reference scripts: kdd99.py:34-35,45-46;
cicids17.py:41-46) and OneHotEncoder, StandardScaler (named by the north star) — all executed by the fused
b200flow encode kernel — PCA on the PCA kernels (b200flow/pca.py), and the feature selectors (UnivariateFeatureSelector,
ChiSqSelector, VarianceThresholdSelector) on the selection kernels (b200flow/selection.py), and the imputer, scalers and
discretizers (Imputer, RobustScaler, MinMaxScaler, MaxAbsScaler, QuantileDiscretizer, Bucketizer) on the quantile kernels
(b200flow/quantile.py).  Each output column remembers how it derives from the raw record fields
(ColumnData.prov), so VectorAssembler / StandardScaler re-run ONE fused kernel over the raw AoS records
instead of chaining per-stage passes (StringIndexer lookup + one-hot expand + scale + assemble).
"""
import copy

import numpy as np
import torch

from b200flow import dist as bdist
from b200flow import encode as enc
from b200flow import pca as _pca
from b200flow import quantile as _q
from b200flow import selection as _sel
from b200flow._lib import SRC_F32, SRC_INDEX, SRC_ONEHOT, B200FlowError
from b200flow.encode import EncodePlan, RecordSchema

from . import Estimator, Model, Transformer
from ..sql import ColumnData, DataFrame, LocalFrame
from .linalg import DenseMatrix, DenseVector


class SparkException(Exception):
    pass


class IllegalArgumentException(ValueError):
    pass


def _check_handle_invalid(v, allowed=("error", "skip", "keep")):
    if v not in allowed:
        raise IllegalArgumentException("handleInvalid must be one of %s, got %r" % (list(allowed), v))
    return v


def _dense_schema(D):
    return RecordSchema([("v%d" % i, "f64") for i in range(D)])


def _materialize(df, name):
    """numeric/vector value of a column as a contiguous f64 [n, k] CUDA tensor."""
    c = df._cols[name]
    if c.kind == "field":
        return df._field_values(name).to(torch.float64).reshape(-1, 1).contiguous()
    d = c.data
    return (d.reshape(d.shape[0], -1) if d.dim() == 1 else d).to(torch.float64).contiguous()


def _peek(df, name):
    """like _materialize, but a lazy column's values are computed without being kept: the column stays lazy, so a tree
    trainer downstream still bins straight from the raw records."""
    c = df._cols[name]
    if c.kind != "field" and c.lazy and c._maker is not None and df._rec is not None:
        d = c._maker(df._rec)
        return (d.reshape(d.shape[0], -1) if d.dim() == 1 else d).to(torch.float64).contiguous()
    return _materialize(df, name)


def _prefetch_category_counts(df, col):
    """enqueue the count kernel of a raw code field without waiting for it (Pipeline.fit does this for every
    StringIndexer stage up front, so the four fits of kdd99.py:34-37 cost one host sync instead of four)."""
    cols = [col] if isinstance(col, str) else list(col)
    cols = [c for c in dict.fromkeys(cols) if df._rec is not None and c in df._cols and c not in df._cat_counts and
            df._cols[c].kind == "field" and df._schema.type_of[c] == "code"]
    for i in range(0, len(cols), 8):                                   # raw code fields: one pass per 8 columns
        part = cols[i:i + 8]
        for c, cnt in zip(part, enc.category_counts_multi(df._rec, df._schema, part, [len(df._dicts[c]) for c in part])):
            df._cat_counts[c] = bdist.all_reduce_sum_(cnt)             # ranks share the dictionaries


def _category_counts(df, col):
    """global category counts of a raw code field as a host array (cached per record buffer)."""
    _prefetch_category_counts(df, col)
    if torch.is_tensor(df._cat_counts[col]):                              # fetch every pending column in ONE device->host copy
        pend = [k for k, v in df._cat_counts.items() if torch.is_tensor(v)]
        host = torch.cat([df._cat_counts[k].reshape(-1) for k in pend]).cpu().numpy()
        o = 0
        for k in pend:
            nk = df._cat_counts[k].numel()
            df._cat_counts[k] = host[o:o + nk][:len(df._dicts[k])]; o += nk
    return df._cat_counts[col]


# ----------------------------------------------------------------------------------- StringIndexer
class StringIndexer(Estimator):
    _defaults = {"inputCol": None, "outputCol": None, "handleInvalid": "error", "stringOrderType": "frequencyDesc"}

    def __init__(self, inputCol=None, outputCol=None, handleInvalid=None, stringOrderType=None):
        super().__init__(inputCol=inputCol, outputCol=outputCol, handleInvalid=handleInvalid, stringOrderType=stringOrderType)

    def _fit(self, df):
        col = self.getOrDefault("inputCol")
        if col not in df._cols:
            raise IllegalArgumentException("Field \"%s\" does not exist." % col)
        c = df._cols[col]
        order = self.getOrDefault("stringOrderType")
        if c.kind == "field" and df._schema.type_of[col] == "code":
            strings = df._dicts[col]
            counts = _category_counts(df, col)
        else:                                              # numeric column: cast to string like Spark does
            vals, cnt = torch.unique(_materialize(df, col)[:, 0], return_counts=True)
            keep = ~torch.isnan(vals)
            strings = [repr(float(v)) for v in vals[keep].cpu().numpy()]
            counts = cnt[keep].cpu().numpy()
        idx = [i for i in range(len(strings)) if counts[i] > 0]
        if order == "frequencyDesc":                        # ties alphabetical (Spark >= 3.0; 2.4 unspecified)
            idx.sort(key=lambda i: (-int(counts[i]), strings[i]))
        elif order == "frequencyAsc":
            idx.sort(key=lambda i: (int(counts[i]), strings[i]))
        elif order == "alphabetDesc":
            idx.sort(key=lambda i: strings[i], reverse=True)
        elif order == "alphabetAsc":
            idx.sort(key=lambda i: strings[i])
        else:
            raise IllegalArgumentException("unsupported stringOrderType %r" % order)
        m = StringIndexerModel([strings[i] for i in idx])
        m._paramMap = dict(self._paramMap)
        return m


class StringIndexerModel(Model):
    _defaults = dict(StringIndexer._defaults)

    def __init__(self, labels):
        super().__init__()
        self.labels = list(labels)

    def _transform(self, df):
        col, out = self.getOrDefault("inputCol"), self.getOrDefault("outputCol")
        hi = _check_handle_invalid(self.getOrDefault("handleInvalid"))
        if col not in df._cols:
            raise IllegalArgumentException("Field \"%s\" does not exist." % col)
        if out in df._cols:
            raise IllegalArgumentException("Output column %s already exists." % out)
        c = df._cols[col]
        K = len(self.labels)
        rank_of = {s: i for i, s in enumerate(self.labels)}
        if c.kind == "field" and df._schema.type_of[col] == "code":
            rec, schema, field = df._rec, df._schema, col
            strings = df._dicts[col]
            prov_ok = True
        else:                                              # numeric input: dictionary-encode on the fly (host dictionary)
            vals = _materialize(df, col)[:, 0]
            uniq, inv = torch.unique(vals, return_inverse=True)
            strings = [repr(float(v)) for v in uniq.cpu().numpy()]
            schema, field = RecordSchema([("c", "code")]), "c"
            rec = inv.to(torch.int32).contiguous().view(torch.uint8).reshape(-1, 4)
            prov_ok = False
        lut = np.array([rank_of.get(s, K if hi == "keep" else -1) for s in strings] or [0], np.int32)
        plan = EncodePlan(schema).add_index(field, lut)
        labels = self.labels + (["__unknown"] if hi == "keep" else [])
        if prov_ok and col in df._cat_counts and (hi == "keep" or
                                                  int(np.asarray(_category_counts(df, col))[lut[:len(strings)] < 0].sum()) == 0):
            # every row's label is known (the counts of this very record buffer say so): nothing to check, nothing to drop.
            # The index column is fully described by its provenance, so its kernel is deferred until the values are read —
            # VectorAssembler fuses the lookup into the one encode pass instead (SURVEY 8a R2+R3).
            mk = lambda r: plan.run(r, torch.float64, want_valid=False)[0].view(-1)     # noqa: E731
            newc = ColumnData("numeric", None, "f64", {"ml_attr": {"type": "nominal", "vals": labels}},
                              ("index", field, lut, labels), thunk=lambda: mk(rec), maker=mk)
            cols = dict(df._cols); cols[out] = newc
            return df._with(cols=cols)
        vals, _, valid = plan.run(rec, torch.float64)
        newc = ColumnData("numeric", vals.view(-1), "f64", {"ml_attr": {"type": "nominal", "vals": labels}},
                          ("index", field, lut, labels) if prov_ok else None)
        cols = dict(df._cols); cols[out] = newc
        res = df._with(cols=cols)
        if hi != "keep":
            n_bad = int((valid == 0).sum().item())
            if n_bad:
                if hi == "error":
                    raise SparkException("Unseen label in column %s (%d rows). To handle unseen labels, set Param "
                                         "handleInvalid to keep." % (col, n_bad))
                res = res._compact(valid)
        return res


# ----------------------------------------------------------------------------------- VectorAssembler
class VectorAssembler(Transformer):
    _defaults = {"inputCols": None, "outputCol": None, "handleInvalid": "error"}

    def __init__(self, inputCols=None, outputCol=None, handleInvalid=None):
        super().__init__(inputCols=inputCols, outputCol=outputCol, handleInvalid=handleInvalid)

    def _transform(self, df):
        cols_in, out = list(self.getOrDefault("inputCols") or []), self.getOrDefault("outputCol")
        hi = _check_handle_invalid(self.getOrDefault("handleInvalid"))
        if out in df._cols:
            raise IllegalArgumentException("Output column %s already exists." % out)
        for c in cols_in:
            if c not in df._cols:
                raise IllegalArgumentException("Field \"%s\" does not exist." % c)
        fused = df._rec is not None and all(df._cols[c].prov is not None for c in cols_in)
        attrs = []
        if fused:
            plan = EncodePlan(df._schema)
            for name in cols_in:
                c = df._cols[name]
                p = c.prov
                if p[0] == "field":
                    if df._schema.type_of[name] == "code":
                        raise IllegalArgumentException("Data type string of column %s is not supported." % name)
                    plan.add_numeric(name); attrs.append({"type": "numeric", "name": name})
                elif p[0] == "index":
                    plan.add_index(p[1], p[2]); attrs.append({"type": "nominal", "name": name, "arity": len(p[3])})
                elif p[0] == "onehot":
                    width = p[3] - 1 if p[4] else p[3]
                    plan.add_onehot(p[1], p[2], p[3], drop_last=p[4])
                    attrs += [{"type": "binary", "name": "%s_%d" % (name, k), "arity": 2} for k in range(width)]
                elif p[0] == "plan":
                    sub = p[1]
                    for s in sub.slots:
                        lo = s[2]
                        if s[0] >= 3:                        # re-home the slot's LUT in this plan's pool
                            lo, _ = plan._add_lut(sub.lut_array()[s[2]:s[2] + s[3]])
                        plan.slots.append((s[0], s[1], lo, s[3], s[4], s[5], s[6]))
                    attrs += list(c.meta.get("attrs", [{"type": "numeric"}] * sub.n_out))
                else:
                    raise B200FlowError("unknown provenance %r" % (p,))
            plan.check_nan = 1
            # f32 record fields, index ranks and one-hot flags are exact in f32: keep the vector in f32 (half the bytes through
            # assemble, randomSplit and binning); values widen to the same doubles whenever they are read as f64
            exact32 = all(s[0] in (SRC_F32, SRC_INDEX, SRC_ONEHOT) and s[5] == 0.0 and s[6] == 1.0 for s in plan.slots)
            vdtype = torch.float32 if exact32 else torch.float64
            prov = ("plan", plan)
            if hi != "skip":
                # No row can disappear ("error" raises, "keep" keeps): the vector is fully described by the plan, so nothing is
                # computed here.  A tree trainer / model downstream bins straight from the records (fused encode -> bins, the
                # dense matrix never exists); anything else that reads the values runs the fused encode kernel then.  Like
                # Spark's lazy transform, a NaN under handleInvalid="error" surfaces at the action that consumes the column.
                plan.check_nan = 1 if hi == "error" else 0

                def mk(r, plan=plan, vdtype=vdtype, hi=hi):
                    feats, _, valid = plan.run(r, vdtype, want_valid=(hi == "error"))
                    if hi == "error" and r.shape[0] and int((valid == 0).sum().item()):
                        raise SparkException("Encountered NaN/null while assembling a row with handleInvalid = \"error\". Consider "
                                             "removing NaNs from dataset or using handleInvalid = \"keep\" or \"skip\".")
                    return feats
                rec0 = df._rec
                newc = ColumnData("vector", None, "f32" if exact32 else "f64", {"attrs": attrs}, prov, thunk=lambda: mk(rec0), maker=mk)
                cols = dict(df._cols); cols[out] = newc
                return df._with(cols=cols)
            feats, _, valid = plan.run(df._rec, vdtype)
        else:                                               # columns without raw provenance: concatenate, then one pass
            parts = [_materialize(df, c) for c in cols_in]
            for name, part in zip(cols_in, parts):
                meta = df._cols[name].meta
                if "attrs" in meta:
                    attrs += list(meta["attrs"])
                elif meta.get("ml_attr", {}).get("type") == "nominal":
                    attrs.append({"type": "nominal", "name": name, "arity": len(meta["ml_attr"]["vals"])})
                else:
                    attrs += [{"type": "numeric", "name": name}] * part.shape[1]
            dense = torch.cat(parts, 1).contiguous()
            plan = EncodePlan(_dense_schema(dense.shape[1]))
            for i in range(dense.shape[1]):
                plan.add_numeric("v%d" % i)
            plan.check_nan = 1
            feats, _, valid = plan.run(dense.view(torch.uint8).reshape(dense.shape[0], -1), torch.float64)
            prov = None
        newc = ColumnData("vector", feats, "f32" if feats.dtype == torch.float32 else "f64", {"attrs": attrs}, prov)
        cols = dict(df._cols); cols[out] = newc
        res = df._with(cols=cols)
        if hi != "keep":
            n_bad = int((valid == 0).sum().item()) if df._n else 0
            if n_bad:
                if hi == "error":
                    raise SparkException("Encountered NaN/null while assembling a row with handleInvalid = \"error\". Consider "
                                         "removing NaNs from dataset or using handleInvalid = \"keep\" or \"skip\".")
                res = res._compact(valid)
        return res


# ----------------------------------------------------------------------------------- OneHotEncoder
class OneHotEncoder(Estimator):
    """Spark >= 3.0 OneHotEncoder / 2.3-2.4 OneHotEncoderEstimator (inputCols/outputCols, or single inputCol/outputCol)."""
    _defaults = {"inputCols": None, "outputCols": None, "inputCol": None, "outputCol": None, "dropLast": True,
                 "handleInvalid": "error"}

    def __init__(self, inputCols=None, outputCols=None, inputCol=None, outputCol=None, dropLast=None, handleInvalid=None):
        super().__init__(inputCols=inputCols, outputCols=outputCols, inputCol=inputCol, outputCol=outputCol,
                         dropLast=dropLast, handleInvalid=handleInvalid)

    def _io(self):
        if self.getOrDefault("inputCols"):
            return list(self.getOrDefault("inputCols")), list(self.getOrDefault("outputCols"))
        return [self.getOrDefault("inputCol")], [self.getOrDefault("outputCol")]

    def _fit(self, df):
        ins, outs = self._io()
        if len(ins) != len(outs):
            raise IllegalArgumentException("The number of input and output columns must match")
        sizes = []
        for name in ins:
            c = df._cols[name]
            vals = c.meta.get("ml_attr", {}).get("vals")
            if vals is not None:
                sizes.append(len(vals))
            else:
                v = _materialize(df, name)[:, 0]
                if bool(((v < 0) | (v != torch.floor(v))).any().item()):
                    raise SparkException("Values to encode must be non-negative integers")
                sizes.append(int(v.max().item()) + 1 if v.numel() else 0)
        m = OneHotEncoderModel(sizes)
        m._paramMap = dict(self._paramMap)
        return m


OneHotEncoderEstimator = OneHotEncoder


class OneHotEncoderModel(Model):
    _defaults = dict(OneHotEncoder._defaults)

    def __init__(self, categorySizes):
        super().__init__()
        self.categorySizes = list(categorySizes)

    def _transform(self, df):
        ins, outs = OneHotEncoder._io(self)
        drop = bool(self.getOrDefault("dropLast"))
        hi = _check_handle_invalid(self.getOrDefault("handleInvalid"), ("error", "keep"))
        cols = dict(df._cols)
        for name, out, K in zip(ins, outs, self.categorySizes):
            if out in cols:
                raise IllegalArgumentException("Output column %s already exists." % out)
            c = df._cols[name]
            ncat = K + 1 if hi == "keep" else K           # 'keep': one extra category for invalid values
            if c.prov is not None and c.prov[0] == "index" and df._rec is not None:
                field, lut = c.prov[1], c.prov[2].copy()
                lut[lut >= K] = K if hi == "keep" else -1
                rec, schema, prov_ok = df._rec, df._schema, True
            else:
                v = _materialize(df, name)[:, 0]
                rec = v.to(torch.int32).contiguous().view(torch.uint8).reshape(-1, 4)
                schema, field, prov_ok = RecordSchema([("c", "code")]), "c", False
                lut = np.arange(K, dtype=np.int32)
            plan = EncodePlan(schema).add_onehot(field, lut, ncat, drop_last=drop)
            if plan.n_out == 0:
                raise IllegalArgumentException("column %s has a single category; nothing to encode with dropLast" % name)
            vec, _, valid = plan.run(rec, torch.float64)
            if hi == "error" and df._n and int((valid == 0).sum().item()):
                raise SparkException("Unseen value in column %s. To handle unseen values, set Param handleInvalid to keep." % name)
            width = plan.n_out
            cols[out] = ColumnData("vector", vec, "f64", {"attrs": [{"type": "binary", "name": "%s_%d" % (out, k), "arity": 2}
                                                                      for k in range(width)]},
                                   ("onehot", field, lut, ncat, drop) if prov_ok else None)
        return df._with(cols=cols)


# ----------------------------------------------------------------------------------- StandardScaler
class StandardScaler(Estimator):
    _defaults = {"inputCol": None, "outputCol": None, "withMean": False, "withStd": True}

    def __init__(self, withMean=None, withStd=None, inputCol=None, outputCol=None):
        super().__init__(withMean=withMean, withStd=withStd, inputCol=inputCol, outputCol=outputCol)

    def _fit(self, df):
        x = _materialize(df, self.getOrDefault("inputCol"))
        mean, std = enc.column_moments(x, bdist.group())   # R3c: corrected two-pass, unbiased (n-1)
        m = StandardScalerModel(mean.cpu().numpy(), std.cpu().numpy())
        m._paramMap = dict(self._paramMap)
        return m


class StandardScalerModel(Model):
    _defaults = dict(StandardScaler._defaults)

    def __init__(self, mean, std):
        super().__init__()
        self.mean, self.std = np.asarray(mean, np.float64), np.asarray(std, np.float64)

    def _transform(self, df):
        D = len(self.mean)
        mean = self.mean if self.getOrDefault("withMean") else np.zeros(D)
        scale = (np.where(self.std != 0, 1.0 / np.where(self.std != 0, self.std, 1.0), 0.0)
                 if self.getOrDefault("withStd") else np.ones(D))
        return _scale_column(df, self.getOrDefault("inputCol"), self.getOrDefault("outputCol"), mean, scale)


def _scale_column(df, name, out, mean, scale):
    """df with column `out` = (x - mean) * scale of the vector column `name` (StandardScalerModel, RobustScalerModel,
    MaxAbsScalerModel).  A column with raw-record provenance is re-encoded from the records with the scaling fused into
    the plan, and keeps that provenance; otherwise the encode kernel scales the dense vector."""
    if out in df._cols:
        raise IllegalArgumentException("Output column %s already exists." % out)
    c = df._cols[name]
    D = len(mean)
    plan = None
    if c.prov is not None and c.prov[0] == "plan" and df._rec is not None:
        src = c.prov[1]
        if src.n_out == D and all(s[5] == 0.0 and s[6] == 1.0 for s in src.slots):
            plan = copy.copy(src); plan.slots = list(src.slots); plan.luts = list(src.luts); plan._dev = None
            plan.label = None
            plan.set_scaling(mean, scale)              # fused: index + one-hot + scale + assemble from raw records
            vec, _, _ = plan.run(df._rec, torch.float64, want_valid=False)
    if plan is None:
        x = _materialize(df, name)
        if x.shape[1] != D:
            raise IllegalArgumentException("vector size %d does not match the fitted size %d" % (x.shape[1], D))
        plan = EncodePlan(_dense_schema(D))
        for i in range(D):
            plan.add_numeric("v%d" % i, mean[i], scale[i])
        vec, _, _ = plan.run(x.view(torch.uint8).reshape(x.shape[0], -1), torch.float64, want_valid=False)
        plan = None
    cols = dict(df._cols)
    cols[out] = ColumnData("vector", vec, "f64", {"attrs": [{"type": "numeric"}] * D}, ("plan", plan) if plan else None)
    return df._with(cols=cols)


# ----------------------------------------------------------------------------------- PCA
class PCA(Estimator):
    """pyspark.ml.feature.PCA on the b200flow PCA kernels (b200flow/pca.py, DESIGN.md §5h).  The model is the same bits for
    any number of ranks; each principal component's sign is fixed so that its entry of largest magnitude is positive."""
    _defaults = {"k": None, "inputCol": None, "outputCol": None}

    def __init__(self, k=None, inputCol=None, outputCol=None):
        super().__init__(k=k, inputCol=inputCol, outputCol=outputCol)

    def _fit(self, df):
        name = self.getOrDefault("inputCol")
        if name not in df._cols:
            raise IllegalArgumentException("Field \"%s\" does not exist." % name)
        try:
            fit = _pca.pca_fit(_materialize(df, name), self.getOrDefault("k"), group=bdist.group())
        except ValueError as e:        # includes b200flow's UnsupportedParamError
            raise IllegalArgumentException(str(e))
        m = PCAModel(fit)
        m._paramMap = dict(self._paramMap)
        return m


class PCAModel(Model):
    _defaults = dict(PCA._defaults)

    def __init__(self, fit):
        super().__init__()
        self._fit_result = fit             # b200flow.pca.PCAFit

    @property
    def pc(self):
        p = self._fit_result.pc
        return DenseMatrix(p.shape[0], p.shape[1], p.T.ravel())

    @property
    def explainedVariance(self):
        return DenseVector(self._fit_result.explained_variance.copy())

    def _transform(self, df):
        name, out = self.getOrDefault("inputCol"), self.getOrDefault("outputCol")
        if out in df._cols:
            raise IllegalArgumentException("Output column %s already exists." % out)
        if name not in df._cols:
            raise IllegalArgumentException("Field \"%s\" does not exist." % name)
        try:
            vec = _pca.pca_transform(_materialize(df, name), self._fit_result)
        except ValueError as e:
            raise IllegalArgumentException(str(e))
        cols = dict(df._cols)
        cols[out] = ColumnData("vector", vec, "f64", {"attrs": [{"type": "numeric"}] * vec.shape[1]}, None)
        return df._with(cols=cols)


# ----------------------------------------------------------------------------------- feature selection
_SELECTION_MODES = ("numTopFeatures", "percentile", "fpr", "fdr", "fwe")
_DEFAULT_THRESHOLD = {"numTopFeatures": 50, "percentile": 0.1, "fpr": 0.05, "fdr": 0.05, "fwe": 0.05}


def _check_selection(mode, threshold):
    if mode not in _SELECTION_MODES:
        raise IllegalArgumentException("selectionMode must be one of %s, got %r" % (list(_SELECTION_MODES), mode))
    if mode == "numTopFeatures":
        if not threshold >= 1:
            raise IllegalArgumentException("numTopFeatures must be >= 1, got %r" % (threshold,))
    elif not 0.0 <= threshold <= 1.0:
        raise IllegalArgumentException("%s must be in [0, 1], got %r" % (mode, threshold))
    return float(threshold)


def _select_column(df, name, out, sel):
    """df with column `out` = the slots `sel` (ascending) of the vector column `name`, keeping their per-slot attrs.  A
    column with raw-record provenance stays a plan over the selected slots (lazy when the input is lazy), so a tree trainer
    downstream still bins straight from the records; otherwise the encode kernel gathers the slots from the dense vector."""
    if name not in df._cols:
        raise IllegalArgumentException("Field \"%s\" does not exist." % name)
    if out in df._cols:
        raise IllegalArgumentException("Output column %s already exists." % out)
    c = df._cols[name]
    if c.kind != "vector":
        raise IllegalArgumentException("Column %s must be of type vector" % name)
    attrs_in = c.meta.get("attrs")
    plan_in = c.prov[1] if c.prov is not None and c.prov[0] == "plan" and df._rec is not None else None
    x = None if plan_in is not None else _materialize(df, name)         # the only read of a dense input
    D = plan_in.n_out if plan_in is not None else x.shape[1]
    if sel and sel[-1] >= D:
        raise IllegalArgumentException("vector size %d does not hold the selected feature %d" % (D, sel[-1]))
    attrs = [attrs_in[i] for i in sel] if attrs_in and len(attrs_in) == D else [{"type": "numeric"}] * len(sel)
    cols = dict(df._cols)
    if not sel:
        cols[out] = ColumnData("vector", torch.empty((df._n, 0), dtype=torch.float64, device=df._device()), "f64",
                               {"attrs": []}, None)
    elif plan_in is not None:
        plan = copy.copy(plan_in); plan.slots = [plan_in.slots[i] for i in sel]; plan.luts = list(plan_in.luts)
        plan._dev = None
        plan.label = None
        vdtype = torch.float32 if c.dtype == "f32" else torch.float64
        if c.lazy:
            def mk(r, plan=plan, vdtype=vdtype):
                feats, _, valid = plan.run(r, vdtype, want_valid=bool(plan.check_nan))
                if plan.check_nan and r.shape[0] and int((valid == 0).sum().item()):
                    raise SparkException("Encountered NaN/null while assembling a row with handleInvalid = \"error\". Consider "
                                         "removing NaNs from dataset or using handleInvalid = \"keep\" or \"skip\".")
                return feats
            rec0 = df._rec
            cols[out] = ColumnData("vector", None, c.dtype, {"attrs": attrs}, ("plan", plan), thunk=lambda: mk(rec0), maker=mk)
        else:
            vec, _, _ = plan.run(df._rec, vdtype, want_valid=False)
            cols[out] = ColumnData("vector", vec, c.dtype, {"attrs": attrs}, ("plan", plan))
    else:
        plan = EncodePlan(_dense_schema(D))
        for i in sel:
            plan.add_numeric("v%d" % i)
        vec, _, _ = plan.run(x.view(torch.uint8).reshape(x.shape[0], -1), torch.float64, want_valid=False)
        cols[out] = ColumnData("vector", vec, "f64", {"attrs": attrs}, None)
    return df._with(cols=cols)


class _SelectorModel(Model):
    """selectedFeatures (ascending indices); transform keeps those slots of featuresCol."""

    def __init__(self, selectedFeatures):
        super().__init__()
        self.selectedFeatures = [int(j) for j in selectedFeatures]

    def _transform(self, df):
        out = self.getOrDefault("outputCol") or "%s__output" % self.uid
        return _select_column(df, self.getOrDefault("featuresCol"), out, self.selectedFeatures)


def _statistical_selection(est, df, test, mode, threshold):
    from .stat import _run_test
    res = _run_test(test, df, est.getOrDefault("featuresCol"), est.getOrDefault("labelCol"))
    return _sel.select(res.p_values, mode, threshold)


class UnivariateFeatureSelector(Estimator):
    """pyspark.ml.feature.UnivariateFeatureSelector (Spark 3.1): chi-square (categorical features and label), ANOVA
    (continuous features, categorical label) or F-value (continuous features and label) p-values, then one of five
    selection rules (b200flow/selection.py, DESIGN.md §5i).  The model is the same for any number of ranks."""
    _defaults = {"featuresCol": "features", "outputCol": None, "labelCol": "label", "featureType": None, "labelType": None,
                 "selectionMode": "numTopFeatures", "selectionThreshold": None}

    def __init__(self, featuresCol=None, outputCol=None, labelCol=None, selectionMode=None):
        super().__init__(featuresCol=featuresCol, outputCol=outputCol, labelCol=labelCol, selectionMode=selectionMode)

    def _fit(self, df):
        ft, lt = self.getOrDefault("featureType"), self.getOrDefault("labelType")
        for v, what in ((ft, "featureType"), (lt, "labelType")):
            if v not in ("categorical", "continuous"):
                raise IllegalArgumentException("%s must be 'categorical' or 'continuous', got %r" % (what, v))
        test = {("categorical", "categorical"): _sel.chi_square_test, ("continuous", "categorical"): _sel.anova_test,
                ("continuous", "continuous"): _sel.f_value_test}.get((ft, lt))
        if test is None:
            raise IllegalArgumentException("Unsupported combination: featureType=%s, labelType=%s" % (ft, lt))
        mode = self.getOrDefault("selectionMode")
        thr = self.getOrDefault("selectionThreshold")
        thr = _check_selection(mode, _DEFAULT_THRESHOLD.get(mode, 0.0) if thr is None else thr)
        m = UnivariateFeatureSelectorModel(_statistical_selection(self, df, test, mode, thr))
        m._paramMap = dict(self._paramMap)
        return m


class UnivariateFeatureSelectorModel(_SelectorModel):
    _defaults = dict(UnivariateFeatureSelector._defaults)


class ChiSqSelector(Estimator):
    """pyspark.ml.feature.ChiSqSelector: the chi-square test of every categorical feature against the label, then
    selectorType's rule (numTopFeatures, percentile, fpr, fdr, fwe)."""
    _defaults = {"numTopFeatures": 50, "featuresCol": "features", "outputCol": None, "labelCol": "label",
                 "selectorType": "numTopFeatures", "percentile": 0.1, "fpr": 0.05, "fdr": 0.05, "fwe": 0.05}

    def __init__(self, numTopFeatures=None, featuresCol=None, outputCol=None, labelCol=None, selectorType=None,
                 percentile=None, fpr=None, fdr=None, fwe=None):
        super().__init__(numTopFeatures=numTopFeatures, featuresCol=featuresCol, outputCol=outputCol, labelCol=labelCol,
                         selectorType=selectorType, percentile=percentile, fpr=fpr, fdr=fdr, fwe=fwe)

    def _fit(self, df):
        mode = self.getOrDefault("selectorType")
        if mode not in _SELECTION_MODES:
            raise IllegalArgumentException("selectorType must be one of %s, got %r" % (list(_SELECTION_MODES), mode))
        for k in _SELECTION_MODES:                       # every threshold is validated, as Spark's param validators do
            _check_selection(k, self.getOrDefault(k))
        thr = float(self.getOrDefault(mode))
        m = ChiSqSelectorModel(_statistical_selection(self, df, _sel.chi_square_test, mode, thr))
        m._paramMap = dict(self._paramMap)
        return m


class ChiSqSelectorModel(_SelectorModel):
    _defaults = dict(ChiSqSelector._defaults)


class VarianceThresholdSelector(Estimator):
    """pyspark.ml.feature.VarianceThresholdSelector: keeps the features whose unbiased variance is > varianceThreshold."""
    _defaults = {"featuresCol": "features", "outputCol": None, "varianceThreshold": 0.0}

    def __init__(self, featuresCol=None, outputCol=None, varianceThreshold=None):
        super().__init__(featuresCol=featuresCol, outputCol=outputCol, varianceThreshold=varianceThreshold)

    def _fit(self, df):
        t = self.getOrDefault("varianceThreshold")
        if not t >= 0.0:
            raise IllegalArgumentException("varianceThreshold must be >= 0, got %r" % (t,))
        name = self.getOrDefault("featuresCol")
        if name not in df._cols:
            raise IllegalArgumentException("Field \"%s\" does not exist." % name)
        try:
            var = _sel.variances(_peek(df, name), group=bdist.group())
        except ValueError as e:        # includes b200flow's UnsupportedParamError
            raise IllegalArgumentException(str(e))
        m = VarianceThresholdSelectorModel([j for j in range(len(var)) if var[j] > t])
        m._paramMap = dict(self._paramMap)
        return m


class VarianceThresholdSelectorModel(_SelectorModel):
    _defaults = dict(VarianceThresholdSelector._defaults)


# ----------------------------------------------------------------------------------- imputer, scalers, discretizers
def _check_relative_error(v):
    if not 0.0 <= v <= 1.0:
        raise IllegalArgumentException("relativeError must be in [0, 1], got %r" % (v,))
    return float(v)


def _io_cols(stage, single_in="inputCol", multi_in="inputCols", single_out="outputCol", multi_out="outputCols"):
    """(input columns, output columns) of a stage with inputCol(s) / outputCol(s)"""
    if stage.getOrDefault(multi_in):
        if stage.getOrDefault(single_in):
            raise IllegalArgumentException("%s and %s cannot both be set" % (single_in, multi_in))
        ins, outs = list(stage.getOrDefault(multi_in)), list(stage.getOrDefault(multi_out) or [])
    else:
        ins = [stage.getOrDefault(single_in)] if stage.getOrDefault(single_in) else []
        outs = [stage.getOrDefault(single_out)] if stage.getOrDefault(single_out) else []
    if not ins:
        raise IllegalArgumentException("%s or %s must be set" % (single_in, multi_in))
    if len(ins) != len(outs):
        raise IllegalArgumentException("The number of input and output columns must match (%d vs %d)" % (len(ins), len(outs)))
    return ins, outs


def _check_numeric(df, names):
    for c in names:
        if c not in df._cols:
            raise IllegalArgumentException("Field \"%s\" does not exist." % c)
        col = df._cols[c]
        if col.kind == "vector" or (col.kind == "field" and df._schema.type_of[c] == "code"):
            raise IllegalArgumentException("Column %s must be of a numeric type" % c)


def _numeric_columns(df, names):
    """the numeric columns `names` as one Columns: raw record fields read in place through their offsets, one derived
    column as its tensor; a mix is stacked as f64, which widens exactly, so this serves fits and outputs that are f64
    whatever the input type (statistics, quantiles, buckets).  Transforms that keep each input's type use _column_groups."""
    _check_numeric(df, names)
    if df._rec is not None and all(df._cols[c].kind == "field" for c in names):
        return _q.record_columns(df._rec, df._schema, names)
    if len(names) == 1:
        return _q.columns(df._column_tensor(names[0]))
    return _q.columns(torch.stack([_materialize(df, c)[:, 0] for c in names], 1))


def _column_groups(df, names):
    """the numeric columns `names` as [(positions in names, Columns)], each column in its own type: every raw record field
    in one Columns over the records, every derived column in a Columns of its own tensor"""
    _check_numeric(df, names)
    fields = [i for i, c in enumerate(names) if df._rec is not None and df._cols[c].kind == "field"]
    groups = [(fields, _q.record_columns(df._rec, df._schema, [names[i] for i in fields]))] if fields else []
    for i, c in enumerate(names):
        if i not in fields:
            t = df._column_tensor(c)
            groups.append(([i], _q.columns(t if t.dtype in (torch.float32, torch.float64, torch.int32) else t.to(torch.float64))))
    return groups


def _vector_input(df, name):
    """a vector column's values [n, D] for a fit: a lazy column is computed without being kept (_peek)"""
    if name not in df._cols:
        raise IllegalArgumentException("Field \"%s\" does not exist." % name)
    c = df._cols[name]
    if c.kind != "vector":
        raise IllegalArgumentException("Column %s must be of type vector" % name)
    if not c.lazy and c.data is not None and c.data.dtype in (torch.float32, torch.float64):
        return c.data
    return _peek(df, name)


class Imputer(Estimator):
    """pyspark.ml.feature.Imputer (b200flow/quantile.py, DESIGN.md §5s): mean, median or mode surrogates of numeric columns
    computed from the values that are neither NaN nor missingValue; the model is the same for any number of ranks."""
    _defaults = {"inputCol": None, "inputCols": None, "outputCol": None, "outputCols": None, "strategy": "mean",
                 "missingValue": float("nan"), "relativeError": 0.001}

    def __init__(self, strategy=None, missingValue=None, inputCols=None, outputCols=None, inputCol=None, outputCol=None,
                 relativeError=None):
        super().__init__(strategy=strategy, missingValue=missingValue, inputCols=inputCols, outputCols=outputCols,
                         inputCol=inputCol, outputCol=outputCol, relativeError=relativeError)

    def _fit(self, df):
        ins, _ = _io_cols(self)
        strategy = self.getOrDefault("strategy")
        if strategy not in ("mean", "median", "mode"):
            raise IllegalArgumentException("strategy must be one of ['mean', 'median', 'mode'], got %r" % (strategy,))
        _check_relative_error(self.getOrDefault("relativeError"))
        mv = float(self.getOrDefault("missingValue"))
        cs = _numeric_columns(df, ins)
        grp = bdist.group()
        if strategy == "mean":
            st = _q.column_stats(cs, mv, grp, with_mean=True)
            count, sur = st.count, st.mean
        elif strategy == "median":
            count = _q.column_stats(cs, mv, grp).count
            q = _q.select_ranks(cs, [[_q.target_rank(0.5, count[c])] if count[c] else [] for c in range(cs.D)], mv, grp)
            sur = np.array([v[0] if len(v) else np.nan for v in q])
        else:
            sur = _q.mode(cs, mv, grp)
            count = np.where(np.isnan(sur), 0, 1)
        for c, name in enumerate(ins):
            if count[c] == 0:
                raise SparkException("surrogate cannot be computed. All the values in %s are Null, Nan or missingValue(%r)"
                                     % (name, mv))
        m = ImputerModel(dict(zip(ins, (float(v) for v in sur))))
        m._paramMap = dict(self._paramMap)
        return m


class ImputerModel(Model):
    _defaults = dict(Imputer._defaults)

    def __init__(self, surrogates):
        super().__init__()
        self._surrogates = dict(surrogates)            # input column -> surrogate (f64, before the cast to the column type)

    @property
    def surrogateDF(self):
        import pandas as pd
        return LocalFrame(pd.DataFrame({k: [v] for k, v in self._surrogates.items()}))

    def _transform(self, df):
        ins, outs = _io_cols(self)
        for o in outs:
            if o in df._cols:
                raise IllegalArgumentException("Output column %s already exists." % o)
        names = {_q.F32: "f32", _q.F64: "f64", _q.I32: "i32"}
        mv = float(self.getOrDefault("missingValue"))
        cols = dict(df._cols)
        for pos, cs in _column_groups(df, ins):            # one launch per group; every output keeps its input's type
            filled = _q.fill(cs, [self._surrogates[ins[i]] for i in pos], mv)
            for i, t, code in zip(pos, filled, cs.dtypes):
                cols[outs[i]] = ColumnData("numeric", t, names[code], {}, None)
        return df._with(cols=cols)


class RobustScaler(Estimator):
    """pyspark.ml.feature.RobustScaler (Spark 3.0): per feature the median and the range q(upper) - q(lower) of its
    non-NaN values, exact quantiles (b200flow/quantile.py); the transform is (x - median) * (1 / range) on the encode plan."""
    _defaults = {"inputCol": None, "outputCol": None, "lower": 0.25, "upper": 0.75, "withCentering": False,
                 "withScaling": True, "relativeError": 0.001}

    def __init__(self, lower=None, upper=None, withCentering=None, withScaling=None, inputCol=None, outputCol=None,
                 relativeError=None):
        super().__init__(lower=lower, upper=upper, withCentering=withCentering, withScaling=withScaling, inputCol=inputCol,
                         outputCol=outputCol, relativeError=relativeError)

    def _fit(self, df):
        lo, hi = self.getOrDefault("lower"), self.getOrDefault("upper")
        if not 0.0 <= lo <= 1.0 or not 0.0 <= hi <= 1.0:
            raise IllegalArgumentException("lower and upper must be in [0, 1], got %r and %r" % (lo, hi))
        if not lo < hi:
            raise IllegalArgumentException("lower must be less than upper, got %r and %r" % (lo, hi))
        _check_relative_error(self.getOrDefault("relativeError"))
        q = _q.quantiles(_vector_input(df, self.getOrDefault("inputCol")), [lo, 0.5, hi], group=bdist.group())
        median = np.array([v[1] if len(v) else np.nan for v in q])
        rng = np.array([v[2] - v[0] if len(v) else np.nan for v in q])
        m = RobustScalerModel(median, rng)
        m._paramMap = dict(self._paramMap)
        return m


class RobustScalerModel(Model):
    _defaults = dict(RobustScaler._defaults)

    def __init__(self, median, range_):
        super().__init__()
        self._median, self._range = np.asarray(median, np.float64), np.asarray(range_, np.float64)

    @property
    def median(self):
        return DenseVector(self._median.copy())

    @property
    def range(self):
        return DenseVector(self._range.copy())

    def _transform(self, df):
        D = len(self._median)
        shift = self._median if self.getOrDefault("withCentering") else np.zeros(D)
        if self.getOrDefault("withScaling"):
            scale = np.array([0.0 if v == 0.0 else 1.0 / v for v in self._range])
        else:
            scale = np.ones(D)
        return _scale_column(df, self.getOrDefault("inputCol"), self.getOrDefault("outputCol"), shift, scale)


class MaxAbsScaler(Estimator):
    """pyspark.ml.feature.MaxAbsScaler: x * (1 / max |x|) per feature (1 for a feature whose max |x| is 0), NaN skipped by
    the fit; the transform runs on the encode plan."""
    _defaults = {"inputCol": None, "outputCol": None}

    def __init__(self, inputCol=None, outputCol=None):
        super().__init__(inputCol=inputCol, outputCol=outputCol)

    def _fit(self, df):
        st = _q.column_stats(_vector_input(df, self.getOrDefault("inputCol")), group=bdist.group())
        m = MaxAbsScalerModel(st.max_abs)
        m._paramMap = dict(self._paramMap)
        return m


class MaxAbsScalerModel(Model):
    _defaults = dict(MaxAbsScaler._defaults)

    def __init__(self, max_abs):
        super().__init__()
        self._max_abs = np.asarray(max_abs, np.float64)

    @property
    def maxAbs(self):
        return DenseVector(self._max_abs.copy())

    def _transform(self, df):
        scale = np.array([1.0 if v == 0.0 else 1.0 / v for v in self._max_abs])
        return _scale_column(df, self.getOrDefault("inputCol"), self.getOrDefault("outputCol"), np.zeros(len(scale)), scale)


class MinMaxScaler(Estimator):
    """pyspark.ml.feature.MinMaxScaler: (x - E_min) * (max - min) / (E_max - E_min) + min per feature, NaN skipped by the fit
    and kept by the transform (b200flow_min_max)."""
    _defaults = {"min": 0.0, "max": 1.0, "inputCol": None, "outputCol": None}

    def __init__(self, min=None, max=None, inputCol=None, outputCol=None):      # noqa: A002 (Spark's parameter names)
        super().__init__(min=min, max=max, inputCol=inputCol, outputCol=outputCol)

    def _fit(self, df):
        lo, hi = self.getOrDefault("min"), self.getOrDefault("max")
        if not lo < hi:
            raise IllegalArgumentException("min (%r) must be less than max (%r)" % (lo, hi))
        st = _q.column_stats(_vector_input(df, self.getOrDefault("inputCol")), group=bdist.group())
        m = MinMaxScalerModel(st.min, st.max)
        m._paramMap = dict(self._paramMap)
        return m


class MinMaxScalerModel(Model):
    _defaults = dict(MinMaxScaler._defaults)

    def __init__(self, original_min, original_max):
        super().__init__()
        self._omin, self._omax = np.asarray(original_min, np.float64), np.asarray(original_max, np.float64)

    @property
    def originalMin(self):
        return DenseVector(self._omin.copy())

    @property
    def originalMax(self):
        return DenseVector(self._omax.copy())

    def _transform(self, df):
        name, out = self.getOrDefault("inputCol"), self.getOrDefault("outputCol")
        if out in df._cols:
            raise IllegalArgumentException("Output column %s already exists." % out)
        lo, hi = float(self.getOrDefault("min")), float(self.getOrDefault("max"))
        x = _vector_input(df, name)
        if x.shape[1] != len(self._omin):
            raise IllegalArgumentException("vector size %d does not match the fitted size %d" % (x.shape[1], len(self._omin)))
        span = hi - lo
        rng = self._omax - self._omin
        scale = np.array([span / r if r != 0.0 else 0.0 for r in rng])
        vec = _q.min_max(x, self._omin, scale, lo, 0.5 * span + lo)
        cols = dict(df._cols)
        cols[out] = ColumnData("vector", vec, "f64", {"attrs": [{"type": "numeric"}] * vec.shape[1]}, None)
        return df._with(cols=cols)


def _check_splits(splits):
    s = [float(v) for v in splits]
    if len(s) < 3:
        raise IllegalArgumentException("Bucketizer splits should have at least 3 split points, got %d" % len(s))
    if not all(a < b for a, b in zip(s, s[1:])):
        raise IllegalArgumentException("Bucketizer splits should be strictly increasing, got %r" % (s,))
    return s


class Bucketizer(Transformer):
    """pyspark.ml.feature.Bucketizer: Spark's binarySearchForBuckets per value (b200flow_bucketize), one launch over every
    input column.  NaN raises (error), gets index len(splits) - 1 (keep) or drops the row (skip); a value outside the splits
    raises under every handleInvalid."""
    _defaults = {"splits": None, "splitsArray": None, "inputCol": None, "inputCols": None, "outputCol": None,
                 "outputCols": None, "handleInvalid": "error"}

    def __init__(self, splits=None, inputCol=None, outputCol=None, handleInvalid=None, splitsArray=None, inputCols=None,
                 outputCols=None):
        super().__init__(splits=splits, inputCol=inputCol, outputCol=outputCol, handleInvalid=handleInvalid,
                         splitsArray=splitsArray, inputCols=inputCols, outputCols=outputCols)

    def _splits(self, n_in):
        if self.getOrDefault("inputCols"):
            arr = self.getOrDefault("splitsArray")
            if arr is None or len(arr) != n_in:
                raise IllegalArgumentException("splitsArray must hold one split list per input column")
            return [_check_splits(s) for s in arr]
        if self.getOrDefault("splits") is None:
            raise IllegalArgumentException("splits must be set")
        return [_check_splits(self.getOrDefault("splits"))]

    def _transform(self, df):
        ins, outs = _io_cols(self)
        splits = self._splits(len(ins))
        hi = _check_handle_invalid(self.getOrDefault("handleInvalid"))
        for o in outs:
            if o in df._cols:
                raise IllegalArgumentException("Output column %s already exists." % o)
        out, flags, nan, oob = _q.bucketize(_numeric_columns(df, ins), splits)
        if oob:
            raise SparkException("Feature value out of Bucketizer bounds (%d values). Check your features, or loosen the "
                                 "lower/upper bound constraints." % oob)
        if nan and hi == "error":
            raise SparkException("Bucketizer encountered NaN value. To handle or skip NaNs, try setting "
                                 "Bucketizer.handleInvalid.")
        cols = dict(df._cols)
        for c, o in enumerate(outs):
            cols[o] = ColumnData("numeric", out[:, c].contiguous(), "f64", {}, None)
        res = df._with(cols=cols)
        return res._compact(flags) if nan and hi == "skip" else res


class QuantileDiscretizer(Estimator):
    """pyspark.ml.feature.QuantileDiscretizer: splits at the exact i / numBuckets quantiles of the non-NaN values, the ends
    replaced by -inf / +inf, -0.0 normalised to 0.0 and duplicates removed (getDistinctSplits); fit returns a Bucketizer."""
    _defaults = {"numBuckets": 2, "numBucketsArray": None, "inputCol": None, "inputCols": None, "outputCol": None,
                 "outputCols": None, "relativeError": 0.001, "handleInvalid": "error"}

    def __init__(self, numBuckets=None, inputCol=None, outputCol=None, relativeError=None, handleInvalid=None,
                 numBucketsArray=None, inputCols=None, outputCols=None):
        super().__init__(numBuckets=numBuckets, inputCol=inputCol, outputCol=outputCol, relativeError=relativeError,
                         handleInvalid=handleInvalid, numBucketsArray=numBucketsArray, inputCols=inputCols,
                         outputCols=outputCols)

    def _fit(self, df):
        ins, outs = _io_cols(self)
        hi = _check_handle_invalid(self.getOrDefault("handleInvalid"))
        _check_relative_error(self.getOrDefault("relativeError"))
        if self.getOrDefault("inputCols") and self.getOrDefault("numBucketsArray") is not None:
            nb = [int(v) for v in self.getOrDefault("numBucketsArray")]
            if len(nb) != len(ins):
                raise IllegalArgumentException("numBucketsArray must hold one value per input column")
        else:
            nb = [int(self.getOrDefault("numBuckets"))] * len(ins)
        for k in nb:
            if k < 2:
                raise IllegalArgumentException("numBuckets must be >= 2, got %d" % k)
        q = _q.quantiles(_numeric_columns(df, ins), [[i / k for i in range(1, k)] for k in nb], group=bdist.group())
        splits = []
        for name, v in zip(ins, q):
            if len(v) == 0:
                raise SparkException("QuantileDiscretizer: column %s has no non-NaN value to compute splits from" % name)
            try:                                          # an all +-inf column leaves only [-inf, +inf]
                splits.append(_check_splits(distinct_splits([-np.inf] + list(v) + [np.inf])))
            except IllegalArgumentException as e:
                raise IllegalArgumentException("QuantileDiscretizer: the splits of column %s are invalid: %s" % (name, e))
        b = Bucketizer(handleInvalid=hi)
        if self.getOrDefault("inputCols"):
            b._set(inputCols=ins, outputCols=outs, splitsArray=splits)
        else:
            b._set(inputCol=ins[0], outputCol=outs[0], splits=splits[0])
        return b


def distinct_splits(splits):
    """Spark's QuantileDiscretizer.getDistinctSplits: ends -inf / +inf, -0.0 -> 0.0, duplicates removed in order"""
    s = [float(v) for v in splits]
    s[0], s[-1] = -np.inf, np.inf
    return list(dict.fromkeys(0.0 if v == 0.0 else v for v in s))
