"""The preprocessing stages over TWO RANKS: column statistics, quantiles, Imputer surrogates (mean, median, mode),
RobustScaler, MinMaxScaler, MaxAbsScaler, QuantileDiscretizer splits and approxQuantile equal the single-process run byte
for byte for even and uneven shards and an empty first or last shard, and an all-missing column raises on both ranks.
Two gloo ranks share one GPU; the NCCL case needs two GPUs and is skipped otherwise."""
import numpy as np
import pytest
import torch

from ranks import block, run, two_gpus

pytestmark = pytest.mark.gpu

N = 30000
SPLITS = {"even": 15000, "uneven": 11000, "empty_first": 0, "empty_last": N}


def _data():
    rng = np.random.default_rng(6)
    m = np.stack([rng.normal(0, 10, N), np.where(rng.random(N) < 0.9, 0.0, np.round(rng.exponential(5, N))),
                  rng.normal(0, 1, N)], 1)
    m[rng.random(N) < 0.05, 2] = np.nan
    m[rng.random(N) < 0.01, 0] = np.inf
    return m


def _hex(a):
    return [float(v).hex() for v in np.asarray(a, np.float64).reshape(-1)]


def _run(m, dev):
    from pyspark.ml.feature import (Imputer, MaxAbsScaler, MinMaxScaler, QuantileDiscretizer, RobustScaler,
                                    SparkException, VectorAssembler)
    from pyspark.sql import SparkSession
    import pandas as pd
    spark = SparkSession.builder.getOrCreate()
    df = spark.createDataFrame(pd.DataFrame({"a": m[:, 0], "b": m[:, 1], "c": m[:, 2]}))
    out = {}
    for s in ("mean", "median", "mode"):
        im = Imputer(inputCols=["a", "b", "c"], outputCols=["a2", "b2", "c2"], strategy=s, missingValue=0.0).fit(df)
        out["imputer_" + s] = _hex([im._surrogates[k] for k in "abc"])
    vdf = VectorAssembler(inputCols=["a", "b", "c"], outputCol="f", handleInvalid="keep").transform(df)
    r = RobustScaler(inputCol="f", outputCol="o", lower=0.1, upper=0.8).fit(vdf)
    out["robust"] = _hex(list(r.median) + list(r.range))
    out["maxabs"] = _hex(list(MaxAbsScaler(inputCol="f", outputCol="o").fit(vdf).maxAbs))
    mm = MinMaxScaler(inputCol="f", outputCol="o").fit(vdf)
    out["minmax"] = _hex(list(mm.originalMin) + list(mm.originalMax))
    bz = QuantileDiscretizer(inputCols=["a", "b", "c"], outputCols=["x", "y", "z"], numBucketsArray=[5, 60, 200],
                             handleInvalid="keep").fit(df)
    out["splits"] = [_hex(s) for s in bz.getSplitsArray()]
    out["approx"] = [_hex(v) for v in df.approxQuantile(["a", "b", "c"], [0.0, 0.14, 0.5, 1.0], 0.0)]
    try:
        Imputer(inputCols=["b"], outputCols=["o"], missingValue=0.0).fit(df.where(__import__(
            "pyspark.sql.functions", fromlist=["col"]).col("b") == 0))
        out["raised"] = False
    except SparkException:
        out["raised"] = True
    return out


def _ranks(rank, grp, dev):
    m = _data()
    res = {}
    for name, cut in SPLITS.items():
        lo, hi = block(rank, cut, N)
        res[name] = _run(m[lo:hi], dev)
    return res


def _two_ranks(tmp_path, mode):
    got = run(tmp_path, _ranks, mode=mode)
    want = _run(_data(), torch.device("cuda", 0))
    assert want["raised"] is True
    for rank in (0, 1):
        for name in SPLITS:
            assert got[rank][name] == want, (rank, name)


def test_feature_scaling_two_gloo_ranks_equal_one_process(tmp_path):
    _two_ranks(tmp_path, "gloo")


@two_gpus
def test_feature_scaling_two_nccl_ranks_equal_one_process(tmp_path):
    _two_ranks(tmp_path, "nccl")
