"""PCA and Pearson correlation over TWO RANKS: the column sums and the centred-Gram partials keep their chunk order across
shards (a straddling chunk is computed by the rank holding its first row, running totals pass rank to rank, the
eigendecomposition is rank 0's), so pc, explainedVariance, the mean, the covariance, the correlation matrix and the
transformed rows equal the single-process result byte for byte — for even and uneven shards (a cut inside a chunk), fewer
than 4096 rows in total and an empty shard.  Two gloo ranks share one GPU; the NCCL case needs two GPUs and is skipped
otherwise."""
import json
import os
import time
import traceback

import numpy as np
import pytest
import torch

from test_tuning_two_ranks import _free_port

pytestmark = pytest.mark.gpu

N, D, K = 30000, 41, 6
# name -> (rows in total, rows of rank 0)
CASES = {"even": (N, 15000), "uneven": (N, 11000), "chunk_aligned": (N, 8192), "short_first": (N, 2500),
         "short_total": (3000, 1200), "empty_last": (N, N), "empty_first": (N, 0)}


def _data():
    rng = np.random.default_rng(31)
    w = rng.normal(size=(8, D)) * (3.0 * 2.0 ** -np.arange(8))[:, None]
    return np.ascontiguousarray(rng.normal(size=(N, 8)) @ w + rng.normal(0.0, 0.05, (N, D)) + rng.normal(0.0, 2.0, D))


def _run(x, dev):
    from b200flow import pca as bp
    xt = torch.from_numpy(x).to(dev)
    fit = bp.pca_fit(xt, K)
    hx = lambda a: [float(v).hex() for v in np.asarray(a).ravel()]       # noqa: E731
    return {"pc": hx(fit.pc), "ev": hx(fit.explained_variance), "mean": hx(fit.mean), "cov": hx(fit.cov),
            "pearson": hx(bp.pearson(xt)), "rows": hx(bp.pca_transform(xt, fit).cpu().numpy())}


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
        for name, (total, cut) in CASES.items():
            lo, hi = (0, cut) if rank == 0 else (cut, total)
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
    x = _data()
    want = {total: _run(x[:total], torch.device("cuda", 0)) for total in sorted({t for t, _ in CASES.values()})}
    ev = np.array([float.fromhex(v) for v in want[N]["ev"]])
    assert np.all(np.diff(ev) < 0) and ev.sum() > 0.9                  # the planted directions are found, in order
    for rank in (0, 1):
        got = json.loads(open(tmp_path / ("res%d.json" % rank)).read())
        for name, (total, cut) in CASES.items():
            g, w = got[name], want[total]
            lo, hi = (0, cut) if rank == 0 else (cut, total)
            for key in ("pc", "ev", "mean", "cov", "pearson"):
                assert g[key] == w[key], (rank, name, key)
            assert g["rows"] == w["rows"][lo * K:hi * K], (rank, name, "rows")


def test_pca_two_gloo_ranks_equal_one_process(tmp_path):
    _two_ranks(tmp_path, "gloo")


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_pca_two_nccl_ranks_equal_one_process(tmp_path):
    _two_ranks(tmp_path, "nccl")
