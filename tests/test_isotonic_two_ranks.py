"""IsotonicRegression over TWO RANKS: every rank gathers all rows in rank order (padded with zero-weight rows) and runs the
same single-device fit, so isotonic and antitonic, weighted and unweighted fits equal the single-process run byte for
byte for even and uneven shards and an empty first or last shard.  A NaN label or a negative weight on one rank makes
both raise.  Two gloo ranks share one GPU; the NCCL case needs two GPUs and is skipped otherwise."""
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
SPLITS = {"even": 15000, "uneven": 11000, "empty_first": 0, "empty_last": N}


def _data():
    rng = np.random.default_rng(4)
    x = np.round(rng.uniform(0.0, 50.0, N), 2)
    y = np.log1p(x) + rng.normal(0, 0.4, N)
    w = rng.uniform(0.0, 2.0, N)
    w[rng.random(N) < 0.1] = 0.0
    return x, y, w


def _hex(a):
    return [float(v).hex() for v in np.asarray(a, np.float64).reshape(-1)]


def _run(x, y, w, dev, grp):
    from b200flow import isotonic as biso
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)      # noqa: E731
    xt, yt, wt = t(x), t(y), t(w)
    out = {}
    for name, (ww, iso, chunk) in {"weighted": (wt, True, 0), "antitonic": (wt, False, 0), "unweighted": (None, True, 3),
                                   "f32": (wt, True, 0)}.items():
        f = biso.isotonic_fit(xt.float() if name == "f32" else xt, yt, ww, isotonic=iso, group=grp, chunk=chunk)
        out[name] = {"b": _hex(f.boundaries), "p": _hex(f.predictions)}
    from b200flow import dist as bdist
    ro, _ = bdist.global_offset(xt.shape[0], dev, grp)
    last = bool(xt.shape[0]) and ro + xt.shape[0] == N         # only the rank holding the last global row sees the bad value
    raised = []
    for col in ("label", "weight"):
        yy, ww = yt.clone(), wt.clone()
        if last:
            (yy if col == "label" else ww)[-1] = float("nan") if col == "label" else -1.0
        try:
            biso.isotonic_fit(xt, yy, ww, group=grp)
            raised.append(False)
        except ValueError:
            raised.append(True)
    out["raised"] = raised
    return out


def _worker(rank, world, port, out_dir, backend):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    gpu = rank if backend == "nccl" else 0
    torch.cuda.set_device(gpu)
    kw = {"device_id": torch.device("cuda", gpu)} if backend == "nccl" else {}
    dist.init_process_group(backend, rank=rank, world_size=world, **kw)
    try:
        x, y, w = _data()
        res = {}
        for name, cut in SPLITS.items():
            lo, hi = (0, cut) if rank == 0 else (cut, N)
            res[name] = _run(x[lo:hi], y[lo:hi], w[lo:hi], torch.device("cuda", gpu), dist.group.WORLD)
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
    x, y, w = _data()
    want = json.loads(json.dumps(_run(x, y, w, torch.device("cuda", 0), None)))
    assert want["raised"] == [True, True]
    assert want["f32"] != want["weighted"]                     # the f32 rounding of x is visible ...
    for rank in (0, 1):
        got = json.loads(open(tmp_path / ("res%d.json" % rank)).read())
        for name in SPLITS:
            assert got[name] == want, (rank, name)             # ... and the same on every layout


def test_isotonic_two_gloo_ranks_equal_one_process(tmp_path):
    _two_ranks(tmp_path, "gloo")


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_isotonic_two_nccl_ranks_equal_one_process(tmp_path):
    _two_ranks(tmp_path, "nccl")
