"""MultilayerPerceptronClassifier over TWO RANKS: chunk partials are computed from each 4096-row chunk's rows alone (a
straddling chunk by the rank holding its first row) and chained rank to rank, so the loss and gradient at fixed weights
and a whole fit's weights and objective history equal the single-process run byte for byte — for even and uneven
shards, a shard shorter than one chunk and an empty shard.  Two gloo ranks share one GPU; the NCCL case needs two GPUs
and is skipped otherwise."""
import numpy as np
import pytest
import torch

from ranks import SPLITS, block, run, two_gpus

pytestmark = pytest.mark.gpu

N = 30000
LAYERS = [41, 16, 5]


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


def _ranks(rank, grp, dev):
    x, y = _data()
    res = {}
    for name, cut in SPLITS(N).items():
        lo, hi = block(rank, cut, N)
        res[name] = _run(x[lo:hi], y[lo:hi], dev, grp)
    return res


def _two_ranks(tmp_path, mode):
    got = run(tmp_path, _ranks, mode=mode)
    x, y = _data()
    want = _run(x, y, torch.device("cuda", 0), None)
    for rank in (0, 1):
        for name in SPLITS(N):
            assert got[rank][name] == want, (rank, name)


def test_mlp_two_gloo_ranks_equal_one_process(tmp_path):
    _two_ranks(tmp_path, "gloo")


@two_gpus
def test_mlp_two_nccl_ranks_equal_one_process(tmp_path):
    _two_ranks(tmp_path, "nccl")
