"""Feature selection over TWO RANKS: the dictionaries are merged from every rank's keys, the contingency counts are int64
sums, and the class sums and centred sums keep their chunk order across shards, so the p-values, statistics, degrees of
freedom and selected features equal the single-process result byte for byte — for even, uneven, chunk-aligned, short and
empty shards.  A column with more than 10000 distinct values on one rank only raises on both.  Two gloo ranks share one
GPU; the NCCL case needs two GPUs and is skipped otherwise."""
import json
import os
import time
import traceback

import numpy as np
import pytest
import torch

from test_tuning_two_ranks import _free_port

pytestmark = pytest.mark.gpu

N, D = 30000, 12
CASES = {"even": (N, 15000), "uneven": (N, 11000), "chunk_aligned": (N, 8192), "short_first": (N, 2500),
         "short_total": (3000, 1200), "empty_last": (N, N), "empty_first": (N, 0)}


def _data():
    rng = np.random.default_rng(31)
    y = rng.integers(0, 4, N).astype(np.float64)
    x = rng.integers(0, 6, (N, D)).astype(np.float64)
    x[:, ::2] += np.floor(y[:, None] * rng.uniform(0, 1.5, (N, D // 2)))
    x[:, 1::3] = rng.normal(size=(N, len(range(1, D, 3)))) + 0.05 * y[:, None]
    x[:, 1::3] = np.round(x[:, 1::3], 2)                        # continuous-looking, but < 10000 values
    yc = x[:, 0] * 0.3 + rng.normal(size=N)
    return x, y, yc


def _run(x, y, yc, dev):
    from b200flow import selection as bs
    xt, yt, yct = (torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in (x, y, yc))
    hx = lambda a: [float(v).hex() for v in np.asarray(a, np.float64).ravel()]       # noqa: E731
    out = {}
    for name, res in (("chi", bs.chi_square_test(xt, yt)), ("anova", bs.anova_test(xt, yt)), ("fv", bs.f_value_test(xt, yct))):
        out[name] = {"p": hx(res.p_values), "s": hx(res.statistics), "dof": [int(v) for v in res.dof],
                     "sel": [bs.select(res.p_values, m, t) for m, t in (("numTopFeatures", 4), ("fdr", 0.05), ("fpr", 0.01))]}
    out["var"] = hx(bs.variances(xt))
    return out


def _worker(rank, world, port, out_dir, backend):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    gpu = rank if backend == "nccl" else 0
    torch.cuda.set_device(gpu)
    kw = {"device_id": torch.device("cuda", gpu)} if backend == "nccl" else {}
    dist.init_process_group(backend, rank=rank, world_size=world, **kw)
    try:
        from b200flow import selection as bs
        x, y, yc = _data()
        res = {}
        dev = torch.device("cuda", gpu)
        for name, (total, cut) in CASES.items():
            lo, hi = (0, cut) if rank == 0 else (cut, total)
            res[name] = _run(x[lo:hi], y[lo:hi], yc[lo:hi], dev)
        wide = np.zeros((20000, 2))                             # rank 1 alone sees 10001 values in column 1
        if rank == 1:
            wide[:10001, 1] = np.arange(10001)
        try:
            bs.chi_square_test(torch.from_numpy(wide).to(dev), torch.zeros(20000, dtype=torch.float64, device=dev))
            res["overflow"] = "no error"
        except bs.TooManyValuesError as e:
            res["overflow"] = str(e)
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
    x, y, yc = _data()
    want = {total: _run(x[:total], y[:total], yc[:total], torch.device("cuda", 0)) for total in sorted({t for t, _ in CASES.values()})}
    assert want[N]["chi"]["sel"][0] and want[N]["anova"]["sel"][0]
    for rank in (0, 1):
        got = json.loads(open(tmp_path / ("res%d.json" % rank)).read())
        for name, (total, _) in CASES.items():
            assert got[name] == want[total], (rank, name)
        assert "more than 10000 distinct values in column 1" in got["overflow"], rank


def test_selection_two_gloo_ranks_equal_one_process(tmp_path):
    _two_ranks(tmp_path, "gloo")


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_selection_two_nccl_ranks_equal_one_process(tmp_path):
    _two_ranks(tmp_path, "nccl")
