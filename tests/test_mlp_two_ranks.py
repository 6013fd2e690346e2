"""MultilayerPerceptronClassifier over TWO RANKS: chunk partials are computed from each 4096-row chunk's rows alone (a
straddling chunk by the rank holding its first row) and chained rank to rank, so the loss and gradient at fixed weights
and a whole fit's weights and objective history equal the single-process run byte for byte — for even and uneven
shards, a shard shorter than one chunk and an empty shard.  Two gloo ranks share one GPU; the NCCL case needs two GPUs
and is skipped otherwise."""
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
LAYERS = [41, 16, 5]
SPLITS = {"even": 15000, "uneven": 11000, "short_first": 2500, "short_last": 28000, "empty_last": N, "empty_first": 0}


def _data():
    rng = np.random.default_rng(8)
    means = rng.normal(0.0, 1.0, (5, 41))
    y = rng.integers(0, 5, N)
    return np.ascontiguousarray(means[y] + rng.normal(0.0, 1.0, (N, 41))), y.astype(np.int32)


def _run(x, y, dev, grp):
    from b200flow import dist as bdist, mlp as bm
    xt, yt = torch.from_numpy(x).to(dev), torch.from_numpy(y).to(dev)
    off, _ = bdist.global_offset(xt.shape[0], dev, grp)
    sh = bdist.Shards(xt.shape[0], off, grp, dev)
    w = torch.from_numpy(bm.init_weights(LAYERS, 3)).to(dev)
    t = bm.loss_grad_sums(xt, yt, LAYERS, w, sh).cpu().numpy()
    fit = bm.mlp_fit(xt, yt, LAYERS, max_iter=6, seed=3, group=grp)
    return {"sums": [v.hex() for v in t], "weights": [v.hex() for v in fit.weights.cpu().numpy()],
            "hist": [v.hex() for v in fit.objective_history], "it": fit.iterations}


def _worker(rank, world, port, out_dir, backend):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    gpu = rank if backend == "nccl" else 0
    torch.cuda.set_device(gpu)
    kw = {"device_id": torch.device("cuda", gpu)} if backend == "nccl" else {}
    dist.init_process_group(backend, rank=rank, world_size=world, **kw)
    try:
        x, y = _data()
        res = {}
        for name, cut in SPLITS.items():
            lo, hi = (0, cut) if rank == 0 else (cut, N)
            res[name] = _run(x[lo:hi], y[lo:hi], torch.device("cuda", gpu), dist.group.WORLD)
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
    ctx = mp.start_processes(_worker, args=(2, _free_port(), str(tmp_path), backend), nprocs=2, join=False, start_method="spawn")
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
    x, y = _data()
    want = json.loads(json.dumps(_run(x, y, torch.device("cuda", 0), None)))
    for rank in (0, 1):
        got = json.loads(open(tmp_path / ("res%d.json" % rank)).read())
        for name in SPLITS:
            assert got[name] == want, (rank, name)


def test_mlp_two_gloo_ranks_equal_one_process(tmp_path):
    _two_ranks(tmp_path, "gloo")


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_mlp_two_nccl_ranks_equal_one_process(tmp_path):
    _two_ranks(tmp_path, "nccl")
