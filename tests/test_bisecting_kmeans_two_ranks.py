"""BisectingKMeans over TWO RANKS: every split decision comes from grouped-sum totals that keep their chunk order across
shards, so the tree, centers, sizes, costs, training cost, predictions and computeCost equal the single-process result
byte for byte — for even and uneven shards, a shard shorter than one 4096-row chunk and an empty first or last shard.
Two gloo ranks share one GPU; the NCCL case needs two GPUs and is skipped otherwise."""
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
SPLITS = {"even": 15000, "uneven": 11000, "short_first": 2500, "short_last": 28000, "empty_last": N, "empty_first": 0}


def _data():
    rng = np.random.default_rng(8)
    means = rng.normal(0.0, 3.0, (9, 41))
    x = means[rng.integers(0, 9, N)] + rng.normal(0.0, 1.0, (N, 41))
    x[::5] = x[0]                                          # a heavy block of repeated rows
    return np.ascontiguousarray(x)


def _run(x, dev, lo=0):
    """the fit of this rank's rows x (global rows lo ..) -> comparable values; predictions are gathered by the caller."""
    from b200flow import bisecting_kmeans as bb
    xt = torch.from_numpy(x).to(dev)
    out = {}
    for k, it, mdcs in ((12, 8, 1.0), (5, 2, 0.02)):
        r = bb.bkm_fit(xt, k, max_iter=it, min_divisible=mdcs, seed=21)
        t = r.tree
        out["%d_%d" % (k, it)] = [t.heap.tolist(), t.left.tolist(), t.right.tolist(), t.leaf.tolist(), t.size.tolist(),
                                  [v.hex() for v in t.center.ravel()], [v.hex() for v in t.cost], float(r.training_cost).hex(),
                                  r.levels, bb.compute_cost(xt, t).hex(), bb.cluster_sizes(r.leaf, k).tolist(),
                                  r.leaf.cpu().numpy().tolist(), [v.hex() for v in r.dist.cpu().numpy()]]
    return out


def _worker(rank, world, port, out_dir, backend):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    gpu = rank if backend == "nccl" else 0
    torch.cuda.set_device(gpu)
    kw = {"device_id": torch.device("cuda", gpu)} if backend == "nccl" else {}
    dist.init_process_group(backend, rank=rank, world_size=world, **kw)
    try:
        x = _data()
        res = {}
        for name, cut in SPLITS.items():
            lo, hi = (0, cut) if rank == 0 else (cut, N)
            res[name] = _run(x[lo:hi], torch.device("cuda", gpu))
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
    want = json.loads(json.dumps(_run(_data(), torch.device("cuda", 0))))
    got = [json.loads(open(tmp_path / ("res%d.json" % r)).read()) for r in (0, 1)]
    for name, cut in SPLITS.items():
        for key, w in want.items():
            a, b = got[0][name][key], got[1][name][key]
            assert a[:-2] == b[:-2] == w[:-2], (name, key)
            assert a[-2] + b[-2] == w[-2] and a[-1] + b[-1] == w[-1], (name, key)   # rank 0 holds rows [0, cut)
            assert len(a[-2]) == cut


def test_bisecting_kmeans_two_gloo_ranks_equal_one_process(tmp_path):
    _two_ranks(tmp_path, "gloo")


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_bisecting_kmeans_two_nccl_ranks_equal_one_process(tmp_path):
    _two_ranks(tmp_path, "nccl")
