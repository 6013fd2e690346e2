"""BisectingKMeans over TWO RANKS: every split decision comes from grouped-sum totals that keep their chunk order across
shards, so the tree, centers, sizes, costs, training cost, predictions and computeCost equal the single-process result
byte for byte — for even and uneven shards, a shard shorter than one 4096-row chunk and an empty first or last shard.
Two gloo ranks share one GPU; the NCCL case needs two GPUs and is skipped otherwise."""
import numpy as np
import pytest
import torch

from ranks import SPLITS, block, run, two_gpus

pytestmark = pytest.mark.gpu

N = 30000


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


def _ranks(rank, grp, dev):
    x = _data()
    res = {}
    for name, cut in SPLITS(N).items():
        lo, hi = block(rank, cut, N)
        res[name] = _run(x[lo:hi], dev)
    return res


def _two_ranks(tmp_path, mode):
    got = run(tmp_path, _ranks, mode=mode)
    want = _run(_data(), torch.device("cuda", 0))
    for name, cut in SPLITS(N).items():
        for key, w in want.items():
            a, b = got[0][name][key], got[1][name][key]
            assert a[:-2] == b[:-2] == w[:-2], (name, key)
            assert a[-2] + b[-2] == w[-2] and a[-1] + b[-1] == w[-1], (name, key)   # rank 0 holds rows [0, cut)
            assert len(a[-2]) == cut


def test_bisecting_kmeans_two_gloo_ranks_equal_one_process(tmp_path):
    _two_ranks(tmp_path, "gloo")


@two_gpus
def test_bisecting_kmeans_two_nccl_ranks_equal_one_process(tmp_path):
    _two_ranks(tmp_path, "nccl")
