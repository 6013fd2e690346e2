"""The preprocessing stages on the device (DESIGN.md §5s) against the numpy restatement (tests/quantile_oracle.py), bit
for bit: column statistics, quantiles (shared-memory and global-memory histograms), Imputer surrogates and fills, Bucketizer
and QuantileDiscretizer splits and buckets, MinMaxScaler, over f32 / f64 / i32 columns read contiguous, strided and as raw
record fields, on random, 90 %-zero, all-equal and NaN / Infinity-laden columns; the scalers' plan provenance; a Pipeline
and a CrossValidator."""
import math

import numpy as np
import pytest
import torch

import quantile_oracle as qo

pytestmark = pytest.mark.gpu

NAN, INF = float("nan"), float("inf")
KINDS = ("random", "zeros", "equal", "naninf")


def _col(kind, n, seed, dtype=np.float64):
    rng = np.random.default_rng(seed)
    if kind == "random":
        v = rng.normal(0.0, 1e3, n)
    elif kind == "zeros":
        v = np.where(rng.random(n) < 0.9, 0.0, np.round(rng.exponential(50.0, n)))
        v[rng.random(n) < 0.01] = -0.0
    elif kind == "equal":
        v = np.full(n, 2.5)
    else:
        v = rng.normal(0.0, 1.0, n)
        r = rng.random(n)
        v[r < 0.05] = NAN
        v[(r >= 0.05) & (r < 0.06)] = INF
        v[(r >= 0.06) & (r < 0.07)] = -INF
    if dtype == np.int32:
        v = np.nan_to_num(v, nan=0, posinf=7, neginf=-7).astype(np.int32)
    return v.astype(dtype)


def _hex(a):
    return [float(v).hex() for v in np.asarray(a, np.float64).reshape(-1)]


def _matrix(n, seed, dtype):
    return np.stack([_col(k, n, seed + i, dtype) for i, k in enumerate(KINDS)], 1)


PROBS = [0.0, 0.001, 0.14, 0.25, 0.5, 0.7, 0.75, 0.999, 1.0]


@pytest.mark.parametrize("n", [20000, 1000000])
@pytest.mark.parametrize("dtype", [np.float32, np.float64, np.int32])
@pytest.mark.parametrize("layout", ["contiguous", "strided"])
def test_stats_and_quantiles_equal_oracle(n, dtype, layout):
    from b200flow import quantile as q
    m = _matrix(n, 3, dtype)
    t = torch.from_numpy(m).cuda()
    if layout == "strided":                                # every other column of a wider matrix, every row
        w = torch.zeros((n, 2 * m.shape[1]), dtype=t.dtype, device="cuda")
        w[:, ::2] = t
        t = w[:, ::2]
    x64 = m.astype(np.float64)
    st = q.column_stats(t, with_mean=True)
    got = q.quantiles(t, PROBS)
    for j in range(m.shape[1]):
        v = qo.valid(x64[:, j])
        assert st.count[j] == v.shape[0]
        s = qo.sorted_values(x64[:, j])
        assert _hex([st.min[j], st.max[j]]) == _hex([s[0], s[-1]])
        assert _hex([st.mean[j]]) == _hex([qo.mean(x64[:, j])])
        assert _hex(got[j]) == _hex(qo.quantiles(x64[:, j], PROBS)), (j, KINDS[j])


def test_global_memory_histograms_and_many_targets():
    """199 targets on one column: the group bound passes the shared-memory limit after the first pass"""
    from b200flow import quantile as q
    n = 1000000
    for kind in ("random", "zeros"):
        v = _col(kind, n, 9)
        probs = [i / 200 for i in range(1, 200)]
        assert len(probs) > q.SMEM_GROUPS
        got = q.quantiles(torch.from_numpy(v).cuda(), probs)[0]
        assert _hex(got) == _hex(qo.quantiles(v, probs))
        # several columns at once, each with its own probabilities
        two = torch.from_numpy(np.stack([v, _col("random", n, 10)], 1)).cuda()
        got2 = q.quantiles(two, [probs, [0.5]])
        assert _hex(got2[0]) == _hex(qo.quantiles(v, probs)) and _hex(got2[1]) == _hex(qo.quantiles(_col("random", n, 10), [0.5]))


def test_kdd_sized_columns_and_mode():
    from b200flow import quantile as q
    n = 4898431
    for kind in ("zeros", "naninf"):
        v = _col(kind, n, 21).astype(np.float32)
        t = torch.from_numpy(v).cuda()
        assert _hex(q.quantiles(t, PROBS)[0]) == _hex(qo.quantiles(v.astype(np.float64), PROBS))
        assert _hex(q.mode(t)) == _hex([qo.mode(v.astype(np.float64))])
    v = np.round(np.random.default_rng(2).normal(0, 3, 100000))
    v[:7] = NAN
    assert q.mode(torch.from_numpy(v).cuda())[0] == qo.mode(v)
    assert q.mode(torch.from_numpy(np.array([3.0, 3.0, 1.0, 1.0, 2.0])).cuda())[0] == 1.0
    assert math.isnan(q.mode(torch.from_numpy(np.array([NAN, NAN])).cuda())[0])


def _records_frame(n, seed):
    """a CICIDS-shaped frame: raw f64 'Flow Bytes/s' with NaN and Infinity, an f32 field, an i32 field"""
    from pyspark.sql import DataFrame
    from b200flow.encode import RecordSchema
    schema = RecordSchema([("Destination Port", "i32"), ("Flow Bytes/s", "f64"), ("Fwd IAT", "f32"), ("label", "code")])
    host = np.zeros(n, schema.numpy_dtype())
    rng = np.random.default_rng(seed)
    host["Destination Port"] = rng.integers(0, 6, n) * 80
    fb = rng.exponential(1e5, n)
    fb[rng.random(n) < 0.03] = NAN
    fb[rng.random(n) < 0.01] = INF
    host["Flow Bytes/s"] = fb
    host["Fwd IAT"] = np.where(rng.random(n) < 0.9, 0.0, rng.exponential(10.0, n)).astype(np.float32)
    host["label"] = rng.integers(0, 2, n)
    rec = torch.from_numpy(host.view(np.uint8).reshape(n, schema.row_bytes)).cuda()
    return DataFrame.fromRecords(rec, schema, {"label": ["BENIGN", "DDoS"]}), host


def test_imputer_on_raw_record_fields():
    from pyspark.ml.feature import Imputer
    df, host = _records_frame(200000, 4)
    ins = ["Destination Port", "Flow Bytes/s", "Fwd IAT"]
    kinds = ["i32", "f64", "f32"]
    for strategy in ("mean", "median", "mode"):
        for mv in (NAN, 0.0, 80.0):
            m = Imputer(inputCols=ins, outputCols=[c + "_i" for c in ins], strategy=strategy, missingValue=mv).fit(df)
            out = m.transform(df)
            for c, k in zip(ins, kinds):
                v = host[c].astype(np.float64)
                want = {"mean": qo.mean, "median": lambda a, missing: qo.quantiles(a, [0.5], missing)[0],
                        "mode": qo.mode}[strategy](v, missing=mv)
                assert _hex([m._surrogates[c]]) == _hex([want]), (strategy, mv, c)
                got = out._column_tensor(c + "_i").cpu().numpy()
                assert got.dtype == host[c].dtype
                exp = qo.fill(host[c], qo.cast(want, k), mv)
                assert got.tobytes() == exp.tobytes(), (strategy, mv, c)
    from pyspark.ml.feature import SparkException
    df2, _ = _records_frame(1000, 5)
    with pytest.raises(SparkException, match="surrogate cannot be computed"):
        Imputer(inputCols=["Destination Port"], outputCols=["o"], missingValue=0.0).fit(df2.where(
            __import__("pyspark.sql.functions", fromlist=["col"]).col("Destination Port") == 0))


def test_imputer_keeps_each_type_next_to_derived_columns():
    """raw i32 and f32 fields imputed together with derived f64 and i32 columns: every output keeps its input's type and
    equals the same column imputed alone"""
    from pyspark.ml.feature import Imputer
    df, host = _records_frame(100000, 6)
    df = Imputer(inputCols=["Flow Bytes/s", "Destination Port"], outputCols=["fb", "port_i"], strategy="mean",
                 missingValue=80.0).fit(df).transform(df)
    fb = df._column_tensor("fb").cpu().numpy()
    port_i = df._column_tensor("port_i").cpu().numpy()
    assert fb.dtype == np.float64 and port_i.dtype == np.int32
    ins = ["Destination Port", "fb", "Fwd IAT", "port_i"]
    vals = {"Destination Port": host["Destination Port"], "fb": fb, "Fwd IAT": host["Fwd IAT"], "port_i": port_i}
    kinds = {"Destination Port": "i32", "fb": "f64", "Fwd IAT": "f32", "port_i": "i32"}
    for mv in (0.0, NAN):
        m = Imputer(inputCols=ins, outputCols=[c + "_o" for c in ins], strategy="mean", missingValue=mv).fit(df)
        out = m.transform(df)
        for c in ins:
            want = qo.mean(vals[c].astype(np.float64), missing=mv)
            assert _hex([m._surrogates[c]]) == _hex([want]), (mv, c)
            got = out._column_tensor(c + "_o").cpu().numpy()
            exp = qo.fill(vals[c], qo.cast(want, kinds[c]), mv)
            assert got.dtype == exp.dtype and got.tobytes() == exp.tobytes(), (mv, c)
            alone = Imputer(inputCol=c, outputCol="a", strategy="mean", missingValue=mv).fit(df).transform(df)
            assert alone._column_tensor("a").cpu().numpy().tobytes() == got.tobytes(), (mv, c)


def test_bucketizer_and_discretizer():
    from pyspark.ml.feature import Bucketizer, QuantileDiscretizer, SparkException
    from pyspark.sql import SparkSession
    spark = SparkSession.builder.getOrCreate()
    df = spark.createDataFrame([(v,) for v in [0.1, 0.4, 1.2, 1.5, NAN, NAN]], ["values"])
    b = QuantileDiscretizer(numBuckets=2, inputCol="values", outputCol="buckets", handleInvalid="keep").fit(df)
    assert b.getSplits() == [-INF, 0.4, INF]
    assert list(b.transform(df)._column_tensor("buckets").cpu().numpy()) == [0, 1, 1, 1, 2, 2]
    assert b.setHandleInvalid("skip").transform(df).count() == 4
    with pytest.raises(SparkException, match="NaN"):
        b.setHandleInvalid("error").transform(df)
    with pytest.raises(SparkException, match="out of Bucketizer bounds"):
        Bucketizer(splits=[0.0, 0.5, 1.0], inputCol="values", outputCol="b", handleInvalid="keep").transform(df)
    # raw record fields, several columns in one launch, against the oracle
    rdf, host = _records_frame(300000, 8)
    ins = ["Destination Port", "Flow Bytes/s", "Fwd IAT"]
    qd = QuantileDiscretizer(inputCols=ins, outputCols=[c + "_b" for c in ins], numBucketsArray=[4, 10, 300],
                             handleInvalid="keep")
    bz = qd.fit(rdf)
    for c, k, s in zip(ins, [4, 10, 300], bz.getSplitsArray()):
        v = host[c].astype(np.float64)
        assert _hex(s) == _hex(qo.discretizer_splits(v, k)), c
    out = bz.transform(rdf)
    for c, s in zip(ins, bz.getSplitsArray()):
        got = out._column_tensor(c + "_b").cpu().numpy()
        want = np.array([qo.bucket(x, s) for x in host[c].astype(np.float64)])
        assert np.array_equal(got, want), c
    kept = bz.setHandleInvalid("skip").transform(rdf)
    assert kept.count() == int((~np.isnan(host["Flow Bytes/s"])).sum())
    from pyspark.ml.feature import IllegalArgumentException
    inf = spark.createDataFrame([(v,) for v in [INF, INF, NAN, INF]], ["v"])
    with pytest.raises(IllegalArgumentException, match="splits of column v"):        # only [-inf, +inf] is left
        QuantileDiscretizer(numBuckets=3, inputCol="v", outputCol="b", handleInvalid="keep").fit(inf)


def test_min_max_and_max_abs_equal_oracle():
    from b200flow import quantile as q
    m = _matrix(100000, 12, np.float64)
    t = torch.from_numpy(m).cuda()
    st = q.column_stats(t)
    for lo, hi in ((0.0, 1.0), (-1.0, 3.0)):
        scale = [(hi - lo) / r if r != 0 else 0.0 for r in st.max - st.min]
        got = q.min_max(t, st.min, scale, lo, 0.5 * (hi - lo) + lo).cpu().numpy()
        want = qo.min_max(m, st.min, st.max, lo, hi)
        assert got.tobytes() == want.tobytes()
    want_abs = [max(abs(qo.sorted_values(m[:, j])[0]), abs(qo.sorted_values(m[:, j])[-1])) for j in range(m.shape[1])]
    assert _hex(st.max_abs) == _hex(want_abs)


def test_scalers_keep_plan_provenance():
    from pyspark.ml.feature import MaxAbsScaler, MinMaxScaler, RobustScaler, VectorAssembler
    from feature_helpers import kdd_frame
    df, feats = kdd_frame(50000, 2, seed=17)
    lazy = VectorAssembler(inputCols=feats, outputCol="features").transform(df)
    assert lazy._cols["features"].lazy
    x = lazy._cols["features"]._maker(lazy._rec).to(torch.float64)
    from pyspark.sql import ColumnData
    cols = dict(lazy._cols); cols["features"] = ColumnData("vector", x, "f64", lazy._cols["features"].meta, None)
    dense = lazy._with(cols=cols)
    for est in (RobustScaler(inputCol="features", outputCol="s", withCentering=True),
                RobustScaler(inputCol="features", outputCol="s", lower=0.1, upper=0.9), MaxAbsScaler(inputCol="features", outputCol="s")):
        m1, m2 = est.fit(lazy), est.fit(dense)
        assert lazy._cols["features"].lazy
        for a in ("_median", "_range", "_max_abs"):
            if hasattr(m1, a):
                assert _hex(getattr(m1, a)) == _hex(getattr(m2, a))
        o1, o2 = m1.transform(lazy), m2.transform(dense)
        assert o1._cols["s"].prov is not None and o1._cols["s"].prov[0] == "plan"
        assert o1._column_tensor("s").cpu().numpy().tobytes() == o2._column_tensor("s").cpu().numpy().tobytes()
    xm = x.cpu().numpy()
    r = RobustScaler(inputCol="features", outputCol="s").fit(lazy)
    for j in range(xm.shape[1]):
        qq = qo.quantiles(xm[:, j], [0.25, 0.5, 0.75])
        assert _hex([r.median[j], r.range[j]]) == _hex([qq[1], qq[2] - qq[0]])
    mm = MinMaxScaler(inputCol="features", outputCol="s").fit(lazy)
    got = mm.transform(lazy)._column_tensor("s").cpu().numpy()
    assert got.tobytes() == qo.min_max(xm, mm.originalMin.toArray(), mm.originalMax.toArray()).tobytes()


def test_pipeline_and_cross_validator():
    from pyspark.ml import Pipeline
    from pyspark.ml.classification import RandomForestClassifier
    from pyspark.ml.evaluation import MulticlassClassificationEvaluator
    from pyspark.ml.feature import Imputer, QuantileDiscretizer, RobustScaler, VectorAssembler
    from pyspark.ml.tuning import CrossValidator, ParamGridBuilder
    df, host = _records_frame(60000, 11)
    from pyspark.ml.feature import StringIndexer
    df = StringIndexer(inputCol="label", outputCol="label_num").fit(df).transform(df)
    pipe = Pipeline(stages=[Imputer(inputCols=["Flow Bytes/s"], outputCols=["fb"], strategy="median"),
                            VectorAssembler(inputCols=["Destination Port", "fb", "Fwd IAT"], outputCol="raw", handleInvalid="keep"),
                            RobustScaler(inputCol="raw", outputCol="features"),
                            RandomForestClassifier(labelCol="label_num", numTrees=4, maxDepth=4, seed=3)])
    out = pipe.fit(df).transform(df)
    assert out.count() == 60000 and "prediction" in out.columns
    qd = QuantileDiscretizer(inputCol="Fwd IAT", outputCol="iat_b")
    est = Pipeline(stages=[qd, VectorAssembler(inputCols=["Destination Port", "iat_b"], outputCol="features"),
                           RandomForestClassifier(labelCol="label_num", numTrees=3, maxDepth=3, seed=3)])
    grid = ParamGridBuilder().addGrid(qd.numBuckets, [2, 5]).build()
    cvm = CrossValidator(estimator=est, estimatorParamMaps=grid, evaluator=MulticlassClassificationEvaluator(
        labelCol="label_num"), numFolds=2, seed=7).fit(df)
    assert len(cvm.avgMetrics) == 2


def test_approx_quantile():
    df, host = _records_frame(50000, 13)
    v = host["Flow Bytes/s"].astype(np.float64)
    got = df.approxQuantile("Flow Bytes/s", [0.1, 0.5, 0.9], 0.01)
    assert _hex(got) == _hex(qo.quantiles(v, [0.1, 0.5, 0.9]))
    both = df.stat.approxQuantile(["Flow Bytes/s", "Fwd IAT"], [0.5], 0.0)
    assert _hex(both[1]) == _hex(qo.quantiles(host["Fwd IAT"].astype(np.float64), [0.5]))
    with pytest.raises(ValueError):
        df.approxQuantile("Flow Bytes/s", [1.5], 0.0)
    with pytest.raises(ValueError):
        df.approxQuantile("Flow Bytes/s", [0.5], -1.0)
