"""CrossValidator with TWO RANKS ON ONE GPU (gloo group, as in tests/test_two_ranks_one_gpu.py): each rank holds a block of
the rows; fold ids are keyed by the global row index, the fits all-reduce their histograms and grid_confusion all-reduces
its counts, so avgMetrics and the best model equal the single-process result exactly."""
import json
import os
import socket
import time
import traceback

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

N = 30000


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _cv(rec, dicts):
    from b200flow import synth
    from pyspark.ml import Pipeline
    from pyspark.ml.classification import RandomForestClassifier
    from pyspark.ml.evaluation import MulticlassClassificationEvaluator
    from pyspark.ml.feature import StringIndexer, VectorAssembler
    from pyspark.ml.tuning import CrossValidator, ParamGridBuilder
    from pyspark.sql import DataFrame
    df = DataFrame.fromRecords(rec, synth.kdd_schema(), dicts)
    cats = synth.KDD_CATEGORICAL
    df = Pipeline(stages=[StringIndexer(inputCol=c, outputCol=c + "_num") for c in cats + ["label"]]).fit(df).transform(df)
    feats = [c for c in df.columns if c not in cats + ["label", "label_num"]]
    df = VectorAssembler(inputCols=feats, outputCol="features").transform(df).select(["features", "label_num"])
    rf = RandomForestClassifier(labelCol="label_num", maxBins=70, seed=4)
    grid = ParamGridBuilder().addGrid(rf.numTrees, [2, 5]).addGrid(rf.maxDepth, [2, 6]).build()
    ev = MulticlassClassificationEvaluator(labelCol="label_num", metricName="f1")
    m = CrossValidator(estimator=rf, estimatorParamMaps=grid, evaluator=ev, numFolds=3, seed=2019).fit(df)
    return m.avgMetrics, m.bestModel._forest.export()


def _worker(rank, world, port, out_dir):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from b200flow import synth
        rec, dicts = synth.make_kdd(N, 5, seed=17, device="cuda:0")
        lo, hi = (0, 11000) if rank == 0 else (11000, N)                       # uneven blocks
        avg, ex = _cv(rec[lo:hi].contiguous(), dicts)
        if rank == 0:
            open(os.path.join(out_dir, "avg.json"), "w").write(json.dumps([float.hex(v) for v in avg]))
            np.savez(os.path.join(out_dir, "best.npz"), **ex)
        open(os.path.join(out_dir, "ok%d" % rank), "w").write("ok")
    except Exception:
        open(os.path.join(out_dir, "error%d.txt" % rank), "w").write(traceback.format_exc())
        raise
    finally:
        try:
            dist.destroy_process_group()
        except Exception:
            pass


def test_cross_validator_two_ranks_equals_single_process(tmp_path):
    import torch.multiprocessing as mp
    ctx = mp.start_processes(_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=False, start_method="spawn")
    deadline = time.time() + 300
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
    from b200flow import synth
    rec, dicts = synth.make_kdd(N, 5, seed=17, device="cuda:0")
    avg, ex = _cv(rec, dicts)
    assert json.loads(open(tmp_path / "avg.json").read()) == [float.hex(v) for v in avg]
    got = np.load(tmp_path / "best.npz")
    assert all(np.array_equal(got[k], ex[k]) for k in ex)
