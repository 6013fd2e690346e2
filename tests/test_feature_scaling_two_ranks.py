"""The preprocessing stages over TWO RANKS: column statistics, quantiles, Imputer surrogates (mean, median, mode),
RobustScaler, MinMaxScaler, MaxAbsScaler, QuantileDiscretizer splits and approxQuantile equal the single-process run byte
for byte for even and uneven shards and an empty first or last shard, and an all-missing column raises on both ranks.
Two gloo ranks share one GPU; the NCCL case needs two GPUs and is skipped otherwise."""
import json
import os
import time
import traceback

import numpy as np
import pytest
import torch

from feature_helpers import free_port

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


def _worker(rank, world, port, out_dir, backend):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    gpu = rank if backend == "nccl" else 0
    torch.cuda.set_device(gpu)
    kw = {"device_id": torch.device("cuda", gpu)} if backend == "nccl" else {}
    dist.init_process_group(backend, rank=rank, world_size=world, **kw)
    try:
        m = _data()
        res = {}
        for name, cut in SPLITS.items():
            lo, hi = (0, cut) if rank == 0 else (cut, N)
            res[name] = _run(m[lo:hi], torch.device("cuda", gpu))
        open(os.path.join(out_dir, "res%d.json" % rank), "w").write(json.dumps(res))
    except Exception:
        open(os.path.join(out_dir, "error%d.txt" % rank), "w").write(traceback.format_exc())
        raise
    finally:
        try:
            dist.destroy_process_group()
        except Exception:
            pass


def _two_ranks(tmp_path, backend):
    import torch.multiprocessing as mp
    ctx = mp.start_processes(_worker, args=(2, free_port(), str(tmp_path), backend), nprocs=2, join=False, start_method="spawn")
    deadline = time.time() + 600
    failed = None
    try:
        while not ctx.join(timeout=5):
            if time.time() > deadline:
                failed = "workers hung"
                break
    except Exception as e:
        failed = "worker failed: %s" % e
    if failed:
        for pr in ctx.processes:
            if pr.is_alive():
                pr.kill()
        errs = "\n".join("--- rank %d\n%s" % (r, open(tmp_path / ("error%d.txt" % r)).read()) for r in (0, 1)
                         if (tmp_path / ("error%d.txt" % r)).exists())
        pytest.fail("%s\n%s" % (failed, errs))
    want = json.loads(json.dumps(_run(_data(), torch.device("cuda", 0))))
    assert want["raised"] is True
    for rank in (0, 1):
        got = json.loads(open(tmp_path / ("res%d.json" % rank)).read())
        for name in SPLITS:
            assert got[name] == want, (rank, name)


def test_feature_scaling_two_gloo_ranks_equal_one_process(tmp_path):
    _two_ranks(tmp_path, "gloo")


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_feature_scaling_two_nccl_ranks_equal_one_process(tmp_path):
    _two_ranks(tmp_path, "nccl")
