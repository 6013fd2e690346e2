"""pyspark.sql shim: SparkSession + a columnar DataFrame whose base columns live in ONE row-major
(AoS) device buffer of raw flow records — the layout the fused encode kernel streams — plus derived
device columns produced by pyspark.ml transformers.

Covers exactly what the reference scripts call (SURVEY.md §2.2): read.csv, toDF, withColumn(regexp_replace),
count, columns, select, where(col > x), randomSplit, cache, printSchema, groupBy().count().orderBy().show(),
distinct, orderBy, rdd.flatMap(...).collect().  Row filtering (where / randomSplit / handleInvalid="skip")
runs the b200flow compaction kernel; everything else here is host-side bookkeeping, not the hot path.
"""
import glob as _glob
import os
import re

import numpy as np
import torch

from b200flow import _lib
from b200flow._lib import call, ptr
from b200flow.encode import RecordSchema


# ----------------------------------------------------------------------------------- columns
class AnalysisException(Exception):
    """pyspark.sql.utils.AnalysisException: what spark.read raises for input it cannot load"""


class ColumnData:
    """One DataFrame column.  kind: 'field' (lives in the record buffer), 'numeric' ([n] tensor),
    'vector' ([n, D] tensor).  meta carries ML attributes (nominal values / per-slot attrs);
    prov records how the column derives from raw record fields so later stages can fuse."""

    def __init__(self, kind, data=None, dtype=None, meta=None, prov=None, thunk=None, maker=None):
        self.kind, self._data, self.dtype, self.meta, self.prov = kind, data, dtype, dict(meta or {}), prov
        self._thunk = thunk                    # lazy column: () -> tensor, run on first access of .data
        self._maker = maker                    # lazy column derived from the record buffer: (records) -> tensor; lets row
        #                                        filters (where / randomSplit) move the RECORDS only and re-bind the column

    @property
    def lazy(self):
        """True while the column exists only as its provenance (no kernel has produced its values yet)."""
        return self._data is None and (self._thunk is not None or self._maker is not None)

    def rebound(self, rec):
        """the same lazy column over another (filtered) record buffer."""
        mk = self._maker
        return ColumnData(self.kind, None, self.dtype, self.meta, self.prov, thunk=lambda: mk(rec), maker=mk)

    @property
    def data(self):
        """the column's tensor.  A transformer whose output is fully described by `prov` (StringIndexerModel on a raw code field,
        VectorAssembler over raw fields) defers its kernel until somebody reads the values — a later VectorAssembler fuses the
        lookup, and the tree trainer bins straight from the records (fused encode -> bins) without the vector ever existing."""
        if self._data is None and self._thunk is not None:
            self._data, self._thunk = self._thunk(), None
        return self._data

    @data.setter
    def data(self, v):
        self._data, self._thunk, self._maker = v, None, None


class Column:
    """Column expression (pyspark.sql.Column): only comparisons against a literal are needed."""

    def __init__(self, name, op=None, value=None):
        self.name, self.op, self.value = name, op, value

    def _cmp(self, op, v):
        return Column(self.name, op, v)

    def __gt__(self, v): return self._cmp("gt", v)
    def __ge__(self, v): return self._cmp("ge", v)
    def __lt__(self, v): return self._cmp("lt", v)
    def __le__(self, v): return self._cmp("le", v)
    def __eq__(self, v): return self._cmp("eq", v)      # noqa: E704
    def __ne__(self, v): return self._cmp("ne", v)      # noqa: E704
    __hash__ = None


class _RegexpReplace:
    def __init__(self, col, pattern, replacement):
        self.col, self.pattern, self.replacement = col, pattern, replacement


class Row(tuple):
    def __new__(cls, values, names):
        r = tuple.__new__(cls, values)
        r._names = list(names)
        return r

    def __getattr__(self, k):
        if k.startswith("_"):
            raise AttributeError(k)
        return self[self._names.index(k)]

    def asDict(self):
        return dict(zip(self._names, self))


class _RDD:
    def __init__(self, rows):
        self._rows = rows

    def flatMap(self, f):
        out = []
        for r in self._rows:
            out.extend(f(r))
        return _RDD(out)

    def map(self, f):
        return _RDD([f(r) for r in self._rows])

    def collect(self):
        return list(self._rows)

    def count(self):
        return len(self._rows)


class LocalFrame:
    """Small host-side result (distinct / groupBy().count()) over a pandas frame."""

    def __init__(self, pdf):
        self._pdf = pdf

    @property
    def columns(self):
        return list(self._pdf.columns)

    def orderBy(self, *cols, ascending=True):
        cols = [c for cc in cols for c in (cc if isinstance(cc, (list, tuple)) else [cc])]
        return LocalFrame(self._pdf.sort_values(cols, ascending=ascending, kind="stable").reset_index(drop=True))

    sort = orderBy

    def select(self, *cols):
        cols = [c for cc in cols for c in (cc if isinstance(cc, (list, tuple)) else [cc])]
        return LocalFrame(self._pdf[cols])

    def distinct(self):
        return LocalFrame(self._pdf.drop_duplicates().reset_index(drop=True))

    def count(self):
        return len(self._pdf)

    def collect(self):
        names = list(self._pdf.columns)
        return [Row([_py(v) for v in rec], names) for rec in self._pdf.itertuples(index=False, name=None)]

    def head(self, n=None):
        rows = LocalFrame(self._pdf.head(1 if n is None else n)).collect()
        return (rows[0] if rows else None) if n is None else rows

    @property
    def rdd(self):
        return _RDD(self.collect())

    def show(self, n=20, truncate=True):
        print(_format_table(self._pdf.head(n), truncate))
        if len(self._pdf) > n:
            print("only showing top %d rows\n" % n)

    def toPandas(self):
        return self._pdf.copy()


def _py(v):
    if isinstance(v, (np.floating,)):
        return float(v)
    if isinstance(v, (np.integer,)):
        return int(v)
    return v


def _format_table(pdf, truncate=True):
    cells = [[str(c) for c in pdf.columns]] + [[("null" if v is None else str(_py(v))) for v in row]
                                               for row in pdf.itertuples(index=False, name=None)]
    if truncate:
        cells = [[c if len(c) <= 20 else c[:17] + "..." for c in row] for row in cells]
    w = [max(len(r[i]) for r in cells) for i in range(len(cells[0]))]
    bar = "+" + "+".join("-" * x for x in w) + "+"
    lines = [bar, "|" + "|".join(c.rjust(x) for c, x in zip(cells[0], w)) + "|", bar]
    lines += ["|" + "|".join(c.rjust(x) for c, x in zip(r, w)) + "|" for r in cells[1:]]
    lines.append(bar + "\n")
    return "\n".join(lines)


class _GroupedData:
    def __init__(self, df, cols):
        self._df, self._cols = df, cols

    def count(self):
        import pandas as pd
        df, c = self._df, self._cols
        if len(c) == 1 and c[0] in df._cols and df._cols[c[0]].kind == "field" and df._schema.type_of[c[0]] == "code":
            from b200flow.encode import category_counts
            labels = df._dicts[c[0]]
            cnt = category_counts(df._rec, df._schema, c[0], len(labels)).cpu().numpy()
            keep = cnt > 0
            return LocalFrame(pd.DataFrame({c[0]: [l for l, k in zip(labels, keep) if k], "count": cnt[keep]}))
        pdf = df.select(*c).toPandas()
        return LocalFrame(pdf.groupby(c, sort=False).size().reset_index(name="count"))


# ----------------------------------------------------------------------------------- DataFrame
class DataFrame:
    def __init__(self, n, rec, schema, dicts, cols, session=None, cat_counts=None):
        self._n = int(n)
        # per-record-buffer cache of category counts of raw code fields (device tensor while pending, numpy once read):
        # shared by every DataFrame that views the same record buffer, dropped when rows are filtered
        self._cat_counts = cat_counts if cat_counts is not None else {}
        self._rec, self._schema, self._dicts = rec, schema, dict(dicts or {})
        self._cols = cols                      # ordered: name -> ColumnData
        self._session = session
        self.is_cached = False

    # ---- construction helpers
    @staticmethod
    def fromRecords(records, schema, dicts, session=None):
        """b200flow extension: DataFrame over already-parsed AoS flow records (uint8 [n, row_bytes] torch tensor,
        host or device; host buffers are copied to the current CUDA device), a RecordSchema and the string
        dictionaries of its 'code' fields — the entry point that skips CSV parsing."""
        _lib.require_cuda()
        if not records.is_cuda:
            records = records.to(torch.device("cuda", torch.cuda.current_device()), non_blocking=True)
        return DataFrame._from_records(records, schema, dicts, session)

    @staticmethod
    def _from_records(rec, schema, dicts, session=None):
        cols = {name: ColumnData("field", dtype=schema.type_of[name], prov=("field", name)) for name in schema.names}
        return DataFrame(rec.shape[0], rec, schema, dicts, cols, session)

    def _with(self, cols=None, n=None, rec="same", dicts=None):
        same = isinstance(rec, str) and n is None and dicts is None
        cols = dict(self._cols) if cols is None else cols
        if not isinstance(rec, str) and rec is not None:    # another record buffer: still-lazy derived columns follow it
            cols = {k: (c.rebound(rec) if (c.kind != "field" and c.lazy and c._maker is not None) else c) for k, c in cols.items()}
        return DataFrame(self._n if n is None else n, self._rec if isinstance(rec, str) else rec, self._schema,
                         self._dicts if dicts is None else dicts, cols, self._session,
                         self._cat_counts if same else None)

    def _device(self):
        if self._rec is not None:
            return self._rec.device
        for c in self._cols.values():
            if c._data is not None:
                return c._data.device
        return torch.device("cuda")

    # ---- basic API
    @property
    def columns(self):
        return list(self._cols)

    def count(self):
        return self._n

    def cache(self):
        self.is_cached = True
        return self

    persist = cache

    def unpersist(self):
        self.is_cached = False
        return self

    def toDF(self, *names):
        if len(names) != len(self._cols):
            raise ValueError("toDF: expected %d column names, got %d" % (len(self._cols), len(names)))
        old = list(self._cols)
        ren = dict(zip(old, names))
        schema = RecordSchema([(ren[f], t) for f, t in zip(self._schema.names, self._schema.types)]) if self._schema else None
        dicts = {ren[k]: v for k, v in self._dicts.items()}
        cols = {}
        for o in old:
            c = self._cols[o]
            cols[ren[o]] = ColumnData(c.kind, c.data, c.dtype, c.meta, ("field", ren[o]) if c.kind == "field" else c.prov)
        return DataFrame(self._n, self._rec, schema, dicts, cols, self._session)

    def printSchema(self):
        print("root")
        names = {"f32": "float", "f64": "double", "i32": "integer", "code": "string"}
        for name, c in self._cols.items():
            t = names.get(c.dtype, "vector" if c.kind == "vector" else "double")
            print(" |-- %s: %s (nullable = true)" % (name, t))
        print()

    def select(self, *cols):
        cols = [c for cc in cols for c in (cc if isinstance(cc, (list, tuple)) else [cc])]
        cols = [c.name if isinstance(c, Column) else c for c in cols]
        for c in cols:
            if c not in self._cols:
                raise ValueError("cannot resolve '%s' given input columns: %s" % (c, list(self._cols)))
        return self._with(cols={c: self._cols[c] for c in cols})

    def drop(self, *cols):
        return self._with(cols={k: v for k, v in self._cols.items() if k not in cols})

    def withColumn(self, name, expr):
        if isinstance(expr, _RegexpReplace):
            return self._regexp_replace(name, expr)
        raise NotImplementedError("withColumn supports regexp_replace(...) only in this shim")

    def _regexp_replace(self, name, e):
        src = e.col.name if isinstance(e.col, Column) else e.col
        c = self._cols.get(src)
        if c is None or c.kind != "field" or self._schema.type_of[src] != "code":
            raise NotImplementedError("regexp_replace needs a string column")
        if name != src:
            raise NotImplementedError("regexp_replace into a new column name is not supported by this shim")
        pat = re.compile(e.pattern)
        new_vals = [pat.sub(_java_repl(e.replacement), s) for s in self._dicts[src]]
        uniq, remap = [], []
        for v in new_vals:                                   # merge dictionary entries that became equal
            if v not in uniq:
                uniq.append(v)
            remap.append(uniq.index(v))
        rec = self._rec
        if len(uniq) != len(new_vals):
            rec = rec.clone()
            j = self._schema.offsets[src] // 4
            lut = torch.tensor(remap + [-1], dtype=torch.int32, device=rec.device)
            codes = rec.view(torch.int32)[:, j].long()
            rec.view(torch.int32)[:, j] = lut[torch.where(codes < 0, torch.full_like(codes, len(remap)), codes)]
        dicts = dict(self._dicts); dicts[src] = uniq
        return self._with(rec=rec, dicts=dicts)

    # ---- row filtering (where / randomSplit / handleInvalid='skip'): stable compaction kernel
    def _field_values(self, name):
        """device view of one base field as a typed strided tensor (no copy)."""
        off, t = self._schema.offsets[name], self._schema.type_of[name]
        if t == "f64":
            if off % 8 or self._schema.row_bytes % 8:
                lo = self._rec.view(torch.int32)[:, off // 4].to(torch.int64) & 0xFFFFFFFF
                hi = self._rec.view(torch.int32)[:, off // 4 + 1].to(torch.int64)
                return ((hi << 32) | lo).view(torch.float64)
            return self._rec.view(torch.float64)[:, off // 8]
        v = self._rec.view(torch.int32)[:, off // 4]
        return v.view(torch.float32) if t == "f32" else v

    def _column_tensor(self, name):
        c = self._cols[name]
        if c.kind == "field":
            if self._schema.type_of[name] == "code":
                raise NotImplementedError("string column %s has no numeric value" % name)
            return self._field_values(name)
        return c.data

    def _compact_bufs(self):
        """buffers a row filter has to move: the record buffer (when a base field or a still-lazy derived column needs it) and
        every MATERIALISED derived column.  Lazy columns with a maker are not computed: they are re-bound to the filtered records."""
        lazy = [k for k, c in self._cols.items() if c.kind != "field" and c.lazy and c._maker is not None and self._rec is not None]
        needs_rec = self._rec is not None and (any(c.kind == "field" for c in self._cols.values()) or bool(lazy))
        names = [k for k, c in self._cols.items() if c.kind != "field" and k not in lazy]
        return needs_rec, names, ([self._rec] if needs_rec else []) + [self._cols[k].data for k in names]

    def _compact(self, flag):
        """keep rows with flag != 0 in every column (order preserved) — b200flow compaction kernel."""
        from b200flow.rows import compact_many
        needs_rec, names, bufs = self._compact_bufs()
        outs, k = compact_many(bufs, flag)
        return self._from_compacted(needs_rec, names, outs, k)

    def _from_compacted(self, needs_rec, names, outs, k):
        rec = outs[0] if needs_rec else None
        outs = outs[1:] if needs_rec else outs
        cols = {}
        for name, c in self._cols.items():
            if c.kind == "field":
                cols[name] = c
            elif name in names:
                cols[name] = ColumnData(c.kind, outs[names.index(name)], c.dtype, c.meta, c.prov if rec is not None else None)
            else:                                            # still lazy: the same provenance over the filtered records
                cols[name] = c.rebound(rec)
        return DataFrame(k, rec, self._schema if rec is not None else None, self._dicts if rec is not None else {}, cols,
                         self._session)

    def where(self, cond):
        if not isinstance(cond, Column) or cond.op is None:
            raise NotImplementedError("where() supports `col(name) <op> literal` only in this shim")
        v = self._column_tensor(cond.name)
        ops = {"gt": torch.gt, "ge": torch.ge, "lt": torch.lt, "le": torch.le, "eq": torch.eq, "ne": torch.ne}
        flag = ops[cond.op](v, cond.value)               # NaN compares false, like SQL null/NaN > x
        return self._compact(flag)

    filter = where

    def randomSplit(self, weights, seed=None):
        """Bernoulli split keyed by (seed, global row index) (A.9 build rule; Spark's own draw is irreproducible).
        Under torch.distributed the row index is global over the ranks' shards."""
        from b200flow import dist as bdist
        from b200flow.rows import random_split_ids
        if seed is None:
            seed = int.from_bytes(os.urandom(8), "little")
        dev = self._device()
        off, _ = bdist.global_offset(self._n, dev)
        sid = random_split_ids(self._n, weights, seed, off, dev)
        from b200flow.rows import split_many
        needs_rec, names, bufs = self._compact_bufs()          # every split is enqueued, then ONE host sync for the row counts
        return [self._from_compacted(needs_rec, names, outs, k) for outs, k in split_many(bufs, sid, len(weights))]

    def groupBy(self, *cols):
        cols = [c for cc in cols for c in (cc if isinstance(cc, (list, tuple)) else [cc])]
        return _GroupedData(self, cols)

    groupby = groupBy

    def distinct(self):
        return LocalFrame(self.toPandas()).distinct()

    def orderBy(self, *cols, ascending=True):
        return LocalFrame(self.toPandas()).orderBy(*cols, ascending=ascending)

    def toPandas(self):
        import pandas as pd
        out = {}
        for name, c in self._cols.items():
            if c.kind == "field":
                if self._schema.type_of[name] == "code":
                    codes = self._field_values(name).cpu().numpy()
                    d = np.asarray(self._dicts[name] + [None], dtype=object)
                    out[name] = d[np.where(codes < 0, len(d) - 1, codes)]
                else:
                    out[name] = self._field_values(name).cpu().numpy()
            elif c.kind == "vector":
                out[name] = list(c.data.cpu().numpy())
            else:
                out[name] = c.data.cpu().numpy()
        return pd.DataFrame(out)

    def collect(self):
        return LocalFrame(self.toPandas()).collect()

    def take(self, n):
        return self.limit(n).collect()

    def limit(self, n):
        n = min(n, self._n)
        cols = {k: (c if c.kind == "field" else ColumnData(c.kind, c.data[:n], c.dtype, c.meta, None)) for k, c in self._cols.items()}
        return DataFrame(n, self._rec[:n] if self._rec is not None else None, self._schema, self._dicts, cols, self._session)

    def show(self, n=20, truncate=True):
        LocalFrame(self.limit(n).toPandas()).show(n, truncate)

    @property
    def rdd(self):
        return _RDD(self.collect())

    def approxQuantile(self, col, probabilities, relativeError):
        """DataFrameStatFunctions.approxQuantile over numeric columns (b200flow/quantile.py): the exact element of rank
        ceil(q n) among the non-NaN values, which is within any relativeError of the target; [] for a column without a
        value.  col: a name (-> list of floats) or a list of names (-> one list per column)."""
        from b200flow import dist as bdist
        from b200flow import quantile as q
        if not relativeError >= 0.0:
            raise ValueError("Relative Error must be non-negative but got %r" % (relativeError,))
        names = [col] if isinstance(col, str) else list(col)
        probs = q.check_probabilities(probabilities)
        for c in names:
            if c not in self._cols or self._cols[c].kind == "vector" or \
                    (self._cols[c].kind == "field" and self._schema.type_of[c] == "code"):
                raise ValueError("approxQuantile needs numeric columns, got %r" % c)
        if self._rec is not None and all(self._cols[c].kind == "field" for c in names):
            cs = q.record_columns(self._rec, self._schema, names)
        else:
            cs = q.columns(torch.stack([self._column_tensor(c).to(torch.float64) for c in names], 1))
        res = [[float(v) for v in r] for r in q.quantiles(cs, probs, group=bdist.group())]
        return res[0] if isinstance(col, str) else res

    @property
    def stat(self):
        return _StatFunctions(self)


class _StatFunctions:
    """df.stat (pyspark.sql.DataFrameStatFunctions): approxQuantile"""

    def __init__(self, df):
        self._df = df

    def approxQuantile(self, col, probabilities, relativeError):
        return self._df.approxQuantile(col, probabilities, relativeError)


def _java_repl(r):
    return re.sub(r"\$(\d+)", r"\\\1", r)


# ----------------------------------------------------------------------------------- CSV ingest
def _dedup_names(names):
    low = [n.lower() for n in names]
    return [n + str(i) if low.count(n.lower()) > 1 else n for i, n in enumerate(names)]


def _read_csv(paths, header, inferSchema, strip_lead, strip_trail, device):
    import pandas as pd
    frames = []
    for p in paths:
        pdf = pd.read_csv(p, header=0 if header else None, skipinitialspace=bool(strip_lead), low_memory=False,
                          dtype=None if inferSchema else str, keep_default_na=True, encoding="utf-8", encoding_errors="replace",
                          float_precision="round_trip")
        if header:
            cols = [str(c) for c in pdf.columns]
            cols = [c.strip() if (strip_lead or strip_trail) else c for c in cols]
            # pandas de-duplicates as 'name.1'; Spark appends the positional index to every duplicate
            cols = [re.sub(r"\.\d+$", "", c) if re.sub(r"\.\d+$", "", c) in cols else c for c in cols]
            pdf.columns = _dedup_names(cols)
        else:
            pdf.columns = ["_c%d" % i for i in range(pdf.shape[1])]
        frames.append(pdf)
    pdf = frames[0] if len(frames) == 1 else pd.concat(frames, ignore_index=True)
    fields, arrays, dicts = [], {}, {}
    for name in pdf.columns:
        s = pdf[name]
        if _is_str(s):
            if strip_trail or strip_lead:
                s = s.str.strip() if strip_trail and strip_lead else (s.str.rstrip() if strip_trail else s.str.lstrip())
            codes, uniques = pd.factorize(s, sort=False)           # null -> -1
            fields.append((name, "code")); arrays[name] = codes.astype(np.int32); dicts[name] = [str(u) for u in uniques]
        elif np.issubdtype(s.dtype, np.integer) and len(s) and s.min() >= -2 ** 31 and s.max() < 2 ** 31:
            fields.append((name, "i32")); arrays[name] = s.to_numpy(np.int32)
        elif np.issubdtype(s.dtype, np.bool_):
            fields.append((name, "i32")); arrays[name] = s.to_numpy(np.int32)
        else:
            fields.append((name, "f64")); arrays[name] = s.to_numpy(np.float64)
    schema = RecordSchema(fields)
    host = np.zeros(len(pdf), schema.numpy_dtype())
    for name in pdf.columns:
        host[name] = arrays[name]
    rec = torch.from_numpy(host.view(np.uint8).reshape(len(pdf), schema.row_bytes))
    if torch.cuda.is_available():
        rec = rec.pin_memory().to(device, non_blocking=True)
    return rec, schema, dicts


class DataFrameReader:
    def __init__(self, session):
        self._session = session
        self._opts = {}

    def option(self, k, v):
        self._opts[k] = v
        return self

    def options(self, **kw):
        self._opts.update(kw)
        return self

    def csv(self, path, schema=None, sep=None, header=None, inferSchema=None, multiLine=None,
            ignoreLeadingWhiteSpace=None, ignoreTrailingWhiteSpace=None, **kw):
        """spark.read.csv (kdd99.py:25, cicids17.py:19-20): path or glob -> DataFrame of AoS device records."""
        _lib.require_cuda()
        o = self._opts
        header = _truthy(header if header is not None else o.get("header", False))
        infer = _truthy(inferSchema if inferSchema is not None else o.get("inferSchema", False))
        paths = []
        for p in (path if isinstance(path, (list, tuple)) else [path]):
            hits = sorted(_glob.glob(p)) if any(ch in p for ch in "*?[") else [p]
            paths.extend(hits)
        if not paths:
            raise FileNotFoundError("Path does not exist: %s" % path)
        lead = _truthy(ignoreLeadingWhiteSpace if ignoreLeadingWhiteSpace is not None else o.get("ignoreLeadingWhiteSpace", False))
        trail = _truthy(ignoreTrailingWhiteSpace if ignoreTrailingWhiteSpace is not None else o.get("ignoreTrailingWhiteSpace", False))
        dev = torch.device("cuda", torch.cuda.current_device())
        engine = str(o.get("b200flow.csvEngine", "device")).lower()
        import torch.distributed as tdist
        from b200flow.dist import group, shard_bounds
        shard = (tdist.get_rank(), tdist.get_world_size()) if group() is not None else None   # one process per GPU: a row block each
        if engine == "device":                                   # csrc/csv.cu: index, inference, dictionaries and parsing on the GPU
            from b200flow import csvio
            try:
                rec, rschema, dicts = csvio.read_csv(paths, header, infer, lead, trail, dev, shard=shard)
            except csvio.CsvFormatError as e:
                raise AnalysisException(str(e))
        elif engine == "host":                                   # explicit opt-in (quoted fields): pandas on the host, then one H2D copy
            rec, rschema, dicts = _read_csv(paths, header, infer, lead, trail, dev)
            if shard is not None:
                lo, hi = shard_bounds(rec.shape[0], *shard)
                rec = rec[lo:hi].contiguous()
        else:
            raise ValueError("b200flow.csvEngine must be 'device' or 'host'")
        return DataFrame._from_records(rec, rschema, dicts, self._session)


def _vector_column(s, name):
    """a column of DenseVector / number lists -> f64 [n, D]; every row must have the same length."""
    rows = [np.asarray(v.toArray() if hasattr(v, "toArray") else v, np.float64) for v in s]
    if any(r.ndim != 1 for r in rows) or len({r.shape[0] for r in rows}) != 1:
        raise NotImplementedError("createDataFrame: column %s must hold DenseVectors or number lists of one length" % name)
    return np.ascontiguousarray(np.stack(rows))


def _is_str(s):
    import pandas as pd
    return s.dtype == object or pd.api.types.is_string_dtype(s.dtype)


def _truthy(v):
    return str(v).lower() == "true" if isinstance(v, str) else bool(v)


# ----------------------------------------------------------------------------------- session
class _Conf:
    def __init__(self, d):
        self._d = d

    def get(self, k, default=None):
        return self._d.get(k, default)

    def set(self, k, v):
        self._d[k] = v


class _SparkContext:
    def __init__(self, conf):
        self._conf = conf

    def setLogLevel(self, level):
        self._conf["spark.log.level"] = level

    @property
    def appName(self):
        return self._conf.get("spark.app.name")


class SparkSession:
    _active = None

    class Builder:
        def __init__(self):
            self._conf = {}

        def appName(self, name):
            self._conf["spark.app.name"] = name
            return self

        def master(self, m):
            self._conf["spark.master"] = m
            return self

        def config(self, k=None, v=None, **kw):
            if k is not None:
                self._conf[k] = v
            return self

        def getOrCreate(self):
            if SparkSession._active is None:
                SparkSession._active = SparkSession(dict(self._conf))
            else:
                SparkSession._active._confd.update(self._conf)
            return SparkSession._active

    builder = None   # set below (a fresh Builder per access, like pyspark's classproperty)

    def __init__(self, conf):
        self._confd = conf
        self.conf = _Conf(conf)
        self.sparkContext = _SparkContext(conf)

    @property
    def read(self):
        return DataFrameReader(self)

    def createDataFrame(self, data, schema=None):
        """host rows / pandas frame -> DataFrame (numeric columns as f64 fields, strings as dictionary codes, DenseVector or
        equal-length number-list columns as f64 vector columns)."""
        import pandas as pd
        _lib.require_cuda()
        pdf = data if isinstance(data, pd.DataFrame) else pd.DataFrame(list(data), columns=list(schema) if schema else None)
        fields, dicts = [], {}
        host_cols, vectors = {}, {}
        for name in pdf.columns:
            s = pdf[name]
            if s.dtype == object and len(s) and not isinstance(s.iloc[0], str):
                vectors[str(name)] = _vector_column(s, name)
                continue
            if _is_str(s):
                codes, uniq = pd.factorize(s, sort=False)
                fields.append((str(name), "code")); host_cols[str(name)] = codes.astype(np.int32); dicts[str(name)] = [str(u) for u in uniq]
            else:
                fields.append((str(name), "f64")); host_cols[str(name)] = s.to_numpy(np.float64)
        rs = RecordSchema(fields)
        host = np.zeros(len(pdf), rs.numpy_dtype())
        for k, v in host_cols.items():
            host[k] = v
        rec = torch.from_numpy(host.view(np.uint8).reshape(len(pdf), rs.row_bytes)).to("cuda")
        df = DataFrame._from_records(rec, rs, dicts, self)
        if vectors:                                          # keep the frame's column order
            cols = {str(k): (ColumnData("vector", torch.from_numpy(vectors[str(k)]).to("cuda"), "f64") if str(k) in vectors
                             else df._cols[str(k)]) for k in pdf.columns}
            df = df._with(cols=cols)
        return df

    def stop(self):
        SparkSession._active = None


class _BuilderDescriptor:
    def __get__(self, obj, owner):
        return SparkSession.Builder()


SparkSession.builder = _BuilderDescriptor()
