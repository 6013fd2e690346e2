"""GeneralizedLinearRegression over TWO RANKS: the per-row partials and the weighted Gram partials are computed from each
4096-row chunk's rows alone and chained rank to rank, and the D x D solves run on rank 0 and are broadcast, so poisson/log
with weights and an offset, binomial/probit, gamma/inverse and tweedie 1.5 fits and their summaries equal the
single-process run byte for byte, for even and uneven shards, a shard shorter than one chunk and empty first and last
shards.  A negative poisson label on one rank makes both raise.  Two gloo ranks share one GPU; the NCCL case needs two
GPUs and is skipped otherwise."""
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
    x = np.abs(rng.normal(0.0, 1.0, (N, D))) * rng.uniform(0.05, 0.2, D)
    y = rng.poisson(np.exp(x @ rng.normal(0.0, 0.5, D) + 0.3)).astype(float)
    return np.ascontiguousarray(x), y, rng.uniform(0.5, 2.0, N), rng.normal(0.0, 0.05, N)


def _hex(a):
    return [float(v).hex() for v in np.asarray(a, np.float64).reshape(-1)]


def _run(x, y, w, off, dev, grp):
    from b200flow import glm as bg
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)      # noqa: E731
    xt, yt, wt, ot = t(x), t(y), t(w), t(off)
    out = {}
    cases = {"poisson": (bg.GLMParams(family="poisson"), yt, wt, ot),
             "probit": (bg.GLMParams(family="binomial", link="probit"), (yt > 1).double(), None, None),
             "gamma": (bg.GLMParams(family="gamma", link="inverse"), yt + 1.0, wt, None),
             "tweedie": (bg.GLMParams(family="tweedie", variance_power=1.5, link_power=0.0, max_iter=8), yt, None, ot)}
    for name, (p, yy, ww, oo) in cases.items():
        f = bg.glm_fit(xt, yy, p, weight=ww, offset=oo, group=grp)
        s = bg.summarize(xt, yy, f, p, weight=ww, offset=oo, group=grp)
        out[name] = {"coef": _hex(f.coef), "b": float(f.intercept).hex(), "it": f.iterations,
                     "diag": None if f.diag_inv_atwa is None else _hex(f.diag_inv_atwa),
                     "summary": _hex([s.deviance, s.null_deviance, s.dispersion] + ([] if s.aic is None else [s.aic])
                                     + list(s.std_errors) + list(s.p_values)) + [s.num_instances, s.rank]}
    from b200flow import dist as bdist
    ro, _ = bdist.global_offset(xt.shape[0], dev, grp)
    bad = yt.clone()
    if xt.shape[0] and ro + xt.shape[0] == N:              # only the rank holding the last global row sees the bad label
        bad[-1] = -1.0
    raised = []
    for p in (bg.GLMParams(family="poisson"), bg.GLMParams(family="tweedie", variance_power=1.5)):
        try:
            bg.glm_fit(xt, bad, p, group=grp)
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
        x, y, w, off = _data()
        res = {}
        for name, cut in SPLITS.items():
            lo, hi = (0, cut) if rank == 0 else (cut, N)
            res[name] = _run(x[lo:hi], y[lo:hi], w[lo:hi], off[lo:hi], torch.device("cuda", gpu), dist.group.WORLD)
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
    x, y, w, off = _data()
    want = json.loads(json.dumps(_run(x, y, w, off, torch.device("cuda", 0), None)))
    assert want["raised"] == [True, True]
    for rank in (0, 1):
        got = json.loads(open(tmp_path / ("res%d.json" % rank)).read())
        for name in SPLITS:
            assert got[name] == want, (rank, name)


def test_glm_two_gloo_ranks_equal_one_process(tmp_path):
    _two_ranks(tmp_path, "gloo")


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_glm_two_nccl_ranks_equal_one_process(tmp_path):
    _two_ranks(tmp_path, "nccl")
