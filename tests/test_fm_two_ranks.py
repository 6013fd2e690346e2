"""FMClassifier and OneVsRest(FMClassifier) over TWO RANKS: the factorization-machine partials are computed from each
4096-row chunk's rows alone (a straddling chunk by the rank holding its first row), the mini-batch draw follows the global
row, and the partials are chained rank to rank, so the loss and gradient totals, a binary fit (with the whole set and
with miniBatchFraction = 0.5) and a OneVsRest fit equal the single-process run byte for byte — for even and uneven shards,
a shard shorter than one chunk and an empty shard.  An invalid label on one rank makes both raise.  Through the pyspark
shim, a rank whose shard is empty or holds only label 0 decides numClasses as the other does: the fit equals one process,
and a label set that is not binary overall makes both ranks raise.  Two gloo ranks share one GPU; the NCCL case needs two
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

N = 30000
D, K, KF = 41, 5, 4
SPLITS = {"even": 15000, "uneven": 11000, "short_first": 2500, "short_last": 28000, "empty_last": N, "empty_first": 0}


def _data():
    rng = np.random.default_rng(8)
    means = rng.normal(0.0, 1.0, (K, D))
    y = rng.integers(0, K, N)
    return np.ascontiguousarray(means[y] + rng.normal(0.0, 1.0, (N, D))), y.astype(np.int32)


def _hex(a):
    return [float(v).hex() for v in np.asarray(a).reshape(-1)]


def _fits_hex(fits):
    return [{"v": _hex(f.factors), "w": _hex(f.linear), "b": float(f.intercept).hex(), "hist": _hex(f.objective_history),
             "it": f.iterations} for f in fits]


def _run(x, y, dev, grp):
    from b200flow import dist as bdist, fm as bfm
    xt, yt = torch.from_numpy(x).to(dev), torch.from_numpy(y).to(dev)
    off, _ = bdist.global_offset(xt.shape[0], dev, grp)
    sh = bdist.Shards(xt.shape[0], off, grp, dev)
    rng = np.random.default_rng(2)
    w = torch.from_numpy(rng.normal(0, 0.1, (K, D * (KF + 1) + 1))).to(dev)
    pos = torch.arange(K, dtype=torch.int32, device=dev)
    out = {"sums": _hex(bfm.fm_loss_grad_totals(xt, yt, pos, w, KF, 1.0, 43, sh).cpu().numpy()),
           "sums_batch": _hex(bfm.fm_loss_grad_totals(xt, yt, pos, w, KF, 0.5, 44, sh).cpu().numpy())}
    p = bfm.FMParams(factor_size=KF, max_iter=8, step_size=0.05, reg_param=0.01, seed=7)
    pb = bfm.FMParams(factor_size=KF, max_iter=8, step_size=0.5, mini_batch_fraction=0.5, solver="gd", seed=7)
    out["binary"] = _fits_hex(bfm.fm_fit_classes(xt, (yt == 2).to(torch.int32), [1], p, group=grp))
    out["binary_batch"] = _fits_hex(bfm.fm_fit_classes(xt, (yt == 2).to(torch.int32), [1], pb, group=grp))
    out["ovr"] = _fits_hex(bfm.fm_fit_classes(xt, yt, range(K), p, group=grp))
    bad = yt.clone()
    if xt.shape[0] and off + xt.shape[0] == N:             # only the rank holding the last global row sees the bad label
        bad[-1] = K + 3
    try:
        bfm.fm_fit_classes(xt, bad, range(K), p, group=grp)
        out["raised"] = False
    except ValueError:
        out["raised"] = True
    return out


class _Frame:
    """the two columns FMClassifier.fit reads, without label metadata"""

    def __init__(self, x, y):
        from pyspark.sql import ColumnData
        self._cols = {"features": ColumnData("vector", x, "f64"), "label": ColumnData("numeric", y, "f64")}

    def _column_tensor(self, name):
        return self._cols[name].data


def _shim_data():
    """the rows sorted by a binary label, label 0 first, so that a short first shard holds only label 0"""
    x, y = _data()
    yb = (y == 2).astype(np.float64)
    order = np.argsort(yb, kind="stable")
    return np.ascontiguousarray(x[order]), yb[order], int((yb == 0).sum())


def _shim_cases(n0):
    """name -> (global row cut between the ranks, label transform)"""
    return {"empty_first": (0, None), "only_label_0_first": (n0 // 2, None), "empty_last": (N, None),
            "one_class": (n0 // 2, "zeros"), "three_classes": (n0 // 2, "two_on_last_row")}


def _shim_run(x, y, lo, hi, how, dev):
    from pyspark.ml.classification import FMClassifier
    y = y.copy()
    if how == "zeros":
        y[:] = 0.0
    elif how == "two_on_last_row":
        y[-1] = 2.0
    df = _Frame(torch.from_numpy(x[lo:hi]).to(dev), torch.from_numpy(y[lo:hi]).to(dev))
    try:
        f = FMClassifier(factorSize=KF, maxIter=8, stepSize=0.05, seed=3).fit(df)._fit_result
    except Exception as e:                                 # IllegalArgumentException
        return {"raised": str(e)}
    return _fits_hex([f])[0]


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
        xs, ys, n0 = _shim_data()
        res["shim"] = {}
        for name, (cut, how) in _shim_cases(n0).items():
            lo, hi = (0, cut) if rank == 0 else (cut, N)
            res["shim"][name] = _shim_run(xs, ys, lo, hi, how, torch.device("cuda", gpu))
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
    assert want["raised"] is True
    xs, ys, n0 = _shim_data()
    want_shim = {name: _shim_run(xs, ys, 0, N, how, torch.device("cuda", 0)) for name, (_, how) in _shim_cases(n0).items()}
    assert want_shim["one_class"] == {"raised": "FMClassifier only supports binary classification. 1 classes detected in label"}
    assert want_shim["three_classes"]["raised"].startswith("FMClassifier only supports binary classification. 3 classes")
    for rank in (0, 1):
        got = json.loads(open(tmp_path / ("res%d.json" % rank)).read())
        for name in SPLITS:
            assert got[name] == want, (rank, name)
        for name in want_shim:
            assert got["shim"][name] == want_shim[name], (rank, name)


def test_fm_two_gloo_ranks_equal_one_process(tmp_path):
    _two_ranks(tmp_path, "gloo")


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_fm_two_nccl_ranks_equal_one_process(tmp_path):
    _two_ranks(tmp_path, "nccl")
