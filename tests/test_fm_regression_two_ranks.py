"""FMRegressor over TWO RANKS: the squared-error factorization-machine partials are computed from each 4096-row chunk's
rows alone and chained rank to rank, and the optimiser state is the same on every rank, so adamW, gd and mini-batch fits
equal the single-process run byte for byte, for even and uneven shards, a shard shorter than one chunk and empty first
and last shards.  A non-finite label on one rank makes both raise.  Two gloo ranks share one GPU."""
import json
import os
import time
import traceback

import numpy as np
import pytest
import torch

from test_tuning_two_ranks import _free_port

pytestmark = pytest.mark.gpu

N, D = 30000, 23
SPLITS = {"even": 15000, "uneven": 11000, "short_first": 2500, "short_last": 28000, "empty_last": N, "empty_first": 0}


def _data():
    rng = np.random.default_rng(8)
    x = rng.normal(0.0, 1.0, (N, D)) * (rng.random((N, D)) < 0.6)
    y = x[:, 0] * x[:, 1] + x @ rng.normal(0.0, 0.2, D) + rng.normal(0.0, 0.5, N)
    return np.ascontiguousarray(x), y


def _hex(a):
    return [float(v).hex() for v in np.asarray(a, np.float64).reshape(-1)]


def _run(x, y, dev, grp):
    from b200flow import dist as bdist, fm as bfm
    xt, yt = torch.from_numpy(x).to(dev), torch.from_numpy(y).to(dev)
    out = {}
    cases = {"adamw": bfm.FMParams(factor_size=4, max_iter=8, step_size=0.05, seed=3),
             "gd_batch": bfm.FMParams(factor_size=3, max_iter=8, step_size=0.05, solver="gd", mini_batch_fraction=0.4,
                                      reg_param=0.01, seed=4)}
    for name, p in cases.items():
        f = bfm.fm_regression_fit(xt, yt, p, group=grp)
        out[name] = {"V": _hex(f.factors), "w": _hex(f.linear), "b": float(f.intercept).hex(),
                     "hist": _hex(f.objective_history), "it": f.iterations}
    off, _ = bdist.global_offset(xt.shape[0], dev, grp)
    bad = yt.clone()
    if xt.shape[0] and off + xt.shape[0] == N:             # only the rank holding the last global row sees the NaN
        bad[-1] = float("nan")
    try:
        bfm.fm_regression_fit(xt, bad, cases["adamw"], group=grp)
        out["raised"] = False
    except ValueError:
        out["raised"] = True
    return out


def _worker(rank, world, port, out_dir):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        x, y = _data()
        res = {}
        for name, cut in SPLITS.items():
            lo, hi = (0, cut) if rank == 0 else (cut, N)
            res[name] = _run(x[lo:hi], y[lo:hi], torch.device("cuda", 0), dist.group.WORLD)
        open(os.path.join(out_dir, "res%d.json" % rank), "w").write(json.dumps(res))
    except Exception:
        open(os.path.join(out_dir, "error%d.txt" % rank), "w").write(traceback.format_exc())
        raise
    finally:
        try:
            dist.destroy_process_group()
        except Exception:
            pass


def test_fm_regression_two_gloo_ranks_equal_one_process(tmp_path):
    import torch.multiprocessing as mp
    ctx = mp.start_processes(_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=False, start_method="spawn")
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
    assert want["raised"]
    for rank in (0, 1):
        got = json.loads(open(tmp_path / ("res%d.json" % rank)).read())
        for name in SPLITS:
            assert got[name] == want, (rank, name)
