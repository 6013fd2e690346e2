"""GBTRegressor with rows sharded over TWO RANKS ON ONE GPU (gloo): both processes run the real kernels on cuda:0.  This
exercises the global-row-keyed findSplits sample and Bernoulli subsample weights, the all-reduced label scale, the
all-reduced max |r| behind every iteration's residual grid, the per-level int64 histogram all-reduce, evaluateEachIteration's
all-reduced sums, the rank-wide label check and a rank whose shard is EMPTY walking every collective.  The models and the
per-iteration losses must be byte-identical to the single-process ones."""
import os
import socket
import time
import traceback

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _data(dev):
    g = torch.Generator(device=dev).manual_seed(37)
    n, F = 24000, 20
    x = torch.randint(0, 8, (n, F), device=dev, generator=g).to(torch.float64)
    x[:, :10] += torch.rand((n, 10), device=dev, generator=g, dtype=torch.float64)
    y = 1e4 * x[:, 0] - 300.0 * x[:, 11] + torch.randn(n, device=dev, generator=g, dtype=torch.float64) * 50.0
    arity = [0] * 10 + [8] * 10
    return x, y, arity


def _params(loss):
    from b200flow import gbt_regression as bgr
    return bgr.GBTRegressorParams(max_iter=4, step_size=0.5, max_depth=5, max_bins=16, subsampling_rate=0.8, seed=2019, loss=loss)


def _result(model, xs, ys, grp):
    out = {k: v for k, v in model.export().items()}
    out["E"] = np.array(model.E, np.int64)
    out["each"] = np.array(model.evaluate_each_iteration(xs, ys, "squared", group=grp)
                           + model.evaluate_each_iteration(xs, ys, "absolute", group=grp))
    return out


def _worker(rank, world, port, out_dir):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from b200flow import dist as bdist, gbt_regression as bgr
        dev = torch.device("cuda", 0)
        x, y, arity = _data(dev)
        n = x.shape[0]
        grp = bdist.group()
        lo, hi = bdist.shard_bounds(n, rank, world)
        out = {}
        for name, (a, b) in (("even", (lo, hi)), ("uneven", (0, 9000) if rank == 0 else (9000, n)),
                             ("empty", (0, n) if rank == 0 else (n, n))):
            off, tot = bdist.global_offset(b - a, dev, grp)
            assert tot == n and off == a
            xs, ys = x[a:b].contiguous(), y[a:b].contiguous()
            for loss in ("squared", "absolute"):
                model = bgr.fit_gbt_regressor(xs, ys, arity, _params(loss), row_offset=off, group=grp)
                out[name + "_" + loss] = _result(model, xs, ys, grp)
        # a NaN label on rank 1 only: both ranks refuse, none waits in a collective
        yb = y[lo:hi].clone()
        if rank == 1:
            yb[5] = float("nan")
        try:
            bgr.fit_gbt_regressor(x[lo:hi].contiguous(), yb, arity, _params("squared"), row_offset=lo, group=grp)
            refused = np.zeros(1)
        except ValueError:
            refused = np.ones(1)
        np.save(os.path.join(out_dir, "refused%d.npy" % rank), refused)
        if rank == 0:
            for name, d in out.items():
                np.savez(os.path.join(out_dir, name + ".npz"), **d)
        open(os.path.join(out_dir, "ok%d" % rank), "w").write("ok")
    except Exception:
        open(os.path.join(out_dir, "error%d.txt" % rank), "w").write(traceback.format_exc())
        raise
    finally:
        try:
            dist.destroy_process_group()
        except Exception:
            pass


def test_two_ranks_one_gpu_gbt_regression_equals_single_process(tmp_path):
    import torch.multiprocessing as mp
    ctx = mp.start_processes(_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=False, start_method="spawn")
    deadline = time.time() + 300
    failed = None
    try:
        while not ctx.join(timeout=5):
            if time.time() > deadline:
                failed = "workers hung"
                break
    except Exception as e:                                                    # a worker raised: its traceback is on file
        failed = "worker failed: %s" % e
    if failed:
        for pr in ctx.processes:
            if pr.is_alive():
                pr.kill()
        errs = "\n".join("--- rank %d\n%s" % (r, open(tmp_path / ("error%d.txt" % r)).read()) for r in (0, 1)
                         if (tmp_path / ("error%d.txt" % r)).exists())
        pytest.fail("%s\n%s" % (failed, errs))
    from b200flow import gbt_regression as bgr
    x, y, arity = _data(torch.device("cuda", 0))
    for loss in ("squared", "absolute"):
        single = _result(bgr.fit_gbt_regressor(x, y, arity, _params(loss)), x, y, None)
        for name in ("even", "uneven", "empty"):
            got = np.load(tmp_path / ("%s_%s.npz" % (name, loss)))
            assert sorted(got.files) == sorted(single)
            for k in single:
                assert np.array_equal(got[k].view(np.uint8), np.asarray(single[k]).view(np.uint8)), "%s shards, %s: %s" % (name, loss, k)
        assert (single["is_leaf"] == 0).sum() > 20
    assert [float(np.load(tmp_path / ("refused%d.npy" % r))[0]) for r in (0, 1)] == [1.0, 1.0]
