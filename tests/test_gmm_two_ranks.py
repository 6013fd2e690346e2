"""GaussianMixture over TWO RANKS: the E-step and moment partials keep their chunk order across shards (a straddling chunk
is computed by the rank holding its first row, running totals pass rank to rank, the eigendecompositions are rank 0's), so
weights, means, covariances, log-likelihood, iteration count, cluster sizes and the transform's probabilities and
predictions equal the single-process result byte for byte — for even and uneven shards, a shard shorter than one 4096-row
chunk and an empty shard.  Two gloo ranks share one GPU; the NCCL case needs two GPUs and is skipped otherwise."""
import json
import os
import time
import traceback

import numpy as np
import pytest
import torch

from test_kmeans_two_ranks import SPLITS, N
from test_tuning_two_ranks import _free_port

pytestmark = pytest.mark.gpu


def _data():
    """four tight clusters, whose densities clear Spark's EPSILON floor, so that EM separates them (at unit scale in 41
    dimensions every responsibility would be 1/k)."""
    rng = np.random.default_rng(18)
    means = rng.normal(0.0, 0.05, (4, 41))
    return np.ascontiguousarray(means[rng.integers(0, 4, N)] + rng.normal(0.0, 0.0025, (N, 41)))


def _run(x, dev):
    from b200flow import gmm as bg
    xt = torch.from_numpy(x).to(dev)
    r = bg.gmm_fit(xt, 4, max_iter=6, tol=0.0, seed=21)
    prob, pred = bg.gmm_predict(xt, r)
    hx = lambda a: [float(v).hex() for v in np.asarray(a).ravel()]       # noqa: E731
    return {"weights": hx(r.weights), "means": hx(r.means), "covs": hx(r.covariances), "ll": float(r.log_likelihood).hex(),
            "it": r.num_iter, "sizes": r.cluster_sizes.tolist(), "prob": hx(prob.cpu().numpy()),
            "pred": pred.cpu().numpy().tolist()}


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
    deadline = time.time() + 900
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
    want = _run(_data(), torch.device("cuda", 0))
    top = np.array([float.fromhex(v) for v in want["prob"]]).reshape(N, 4).max(1)
    assert top.mean() > 0.99 and min(want["sizes"]) > 0.2 * N      # the fit separates the clusters
    for rank in (0, 1):
        got = json.loads(open(tmp_path / ("res%d.json" % rank)).read())
        for name, cut in SPLITS.items():
            g = got[name]
            lo, hi = (0, cut) if rank == 0 else (cut, N)
            for key in ("weights", "means", "covs", "ll", "it", "sizes"):
                assert g[key] == want[key], (rank, name, key)
            k = 4
            assert g["prob"] == want["prob"][lo * k:hi * k], (rank, name, "prob")
            assert g["pred"] == want["pred"][lo:hi], (rank, name, "pred")


def test_gmm_two_gloo_ranks_equal_one_process(tmp_path):
    _two_ranks(tmp_path, "gloo")


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_gmm_two_nccl_ranks_equal_one_process(tmp_path):
    _two_ranks(tmp_path, "nccl")
