"""Binary evaluation with TWO RANKS ON ONE GPU (gloo group, as in tests/test_two_ranks_one_gpu.py): each rank reduces its
shard to distinct (score, pos, neg) triples, the triples are all-gathered and reduced again, so the areas and the curve
points equal the single-process result bit for bit — also when one rank holds no rows.  A CrossValidator scored by
areaUnderROC gives the same avgMetrics as one process."""
import json
import os
import time
import traceback

import numpy as np
import pytest
import torch

from test_tuning_two_ranks import _free_port

pytestmark = pytest.mark.gpu

N = 30000
SPLITS = {"uneven": 11000, "empty_shard": N}


def _data():
    rng = np.random.default_rng(5)
    sc = np.concatenate([rng.integers(0, 700, (3, N // 2)) / 699.0, rng.random((3, N - N // 2))], axis=1)
    sc[:, ::97] = -0.0
    y = (rng.random(N) < 0.4).astype(np.float64)
    return sc, y


def _areas(sc, y):
    from b200flow.metrics import binary_metrics
    out = {}
    ts, ty = torch.from_numpy(np.ascontiguousarray(sc)).cuda(), torch.from_numpy(np.ascontiguousarray(y)).cuda()
    for bins in (0, 1000):
        r1 = binary_metrics(ts[0], ty, num_bins=bins, curves=True)
        r3 = binary_metrics(ts, ty, num_bins=bins, curves=True)
        out["s1_%d" % bins] = [float.hex(r1["areaUnderROC"]), float.hex(r1["areaUnderPR"]), r1["curves"]["tp"].tolist(),
                               r1["curves"]["fp"].tolist(), [float.hex(v) for v in r1["curves"]["score"]]]
        out["s3_%d" % bins] = [[float.hex(v) for v in r3["areaUnderROC"]], [float.hex(v) for v in r3["areaUnderPR"]],
                               [c["tp"].tolist() for c in r3["curves"]]]
    return out


def _cv(rec, dicts):
    from b200flow import synth
    from pyspark.ml import Pipeline
    from pyspark.ml.classification import RandomForestClassifier
    from pyspark.ml.evaluation import BinaryClassificationEvaluator
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
    ev = BinaryClassificationEvaluator(labelCol="label_num", metricName="areaUnderROC")
    return [float.hex(v) for v in CrossValidator(estimator=rf, estimatorParamMaps=grid, evaluator=ev, numFolds=3,
                                                 seed=2019).fit(df).avgMetrics]


def _worker(rank, world, port, out_dir):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        sc, y = _data()
        res = {}
        for name, cut in SPLITS.items():
            lo, hi = (0, cut) if rank == 0 else (cut, N)
            res[name] = _areas(sc[:, lo:hi], y[lo:hi])
        from b200flow import synth
        rec, dicts = synth.make_kdd(N, 2, seed=17, device="cuda:0")
        lo, hi = (0, 13000) if rank == 0 else (13000, N)
        res["cv"] = _cv(rec[lo:hi].contiguous(), dicts)
        open(os.path.join(out_dir, "res%d.json" % rank), "w").write(json.dumps(res))
    except Exception:
        open(os.path.join(out_dir, "error%d.txt" % rank), "w").write(traceback.format_exc())
        raise
    finally:
        try:
            dist.destroy_process_group()
        except Exception:
            pass


def test_binary_evaluation_two_ranks_equals_single_process(tmp_path):
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
    sc, y = _data()
    want = json.loads(json.dumps(_areas(sc, y)))
    from b200flow import synth
    rec, dicts = synth.make_kdd(N, 2, seed=17, device="cuda:0")
    cv = _cv(rec, dicts)
    for rank in (0, 1):
        got = json.loads(open(tmp_path / ("res%d.json" % rank)).read())
        for name in SPLITS:
            assert got[name] == want, (rank, name)
        assert got["cv"] == cv, rank
