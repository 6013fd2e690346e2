"""KMeans and the silhouette over TWO RANKS: the grouped sums keep their chunk order across shards (a straddling chunk is
summed by the rank holding its first row, running totals pass rank to rank), so centers, cost, sizes, iteration count
and silhouette equal the single-process result byte for byte — for even and uneven shards, a shard shorter than one
4096-row chunk and an empty shard.  Two gloo ranks share one GPU (as in tests/test_two_ranks_one_gpu.py); the NCCL case
needs two GPUs and is skipped otherwise."""
import numpy as np
import pytest
import torch

from ranks import SPLITS, block, run, two_gpus

pytestmark = pytest.mark.gpu

N = 30000


def _data():
    rng = np.random.default_rng(8)
    means = rng.normal(0.0, 3.0, (9, 41))
    return np.ascontiguousarray(means[rng.integers(0, 9, N)] + rng.normal(0.0, 1.0, (N, 41)))


def _run(x, dev):
    from b200flow import kmeans as bk
    xt = torch.from_numpy(x).to(dev)
    out = {}
    for init, k in (("k-means||", 12), ("random", 5)):
        r = bk.kmeans_fit(xt, k, init=init, max_iter=8, seed=21)
        out[init] = [[v.hex() for v in r.centers.cpu().numpy().ravel()], float(r.training_cost).hex(), r.num_iter,
                     r.cluster_sizes.tolist(), bk.silhouette(xt, r.cluster).hex()]
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
    for rank in (0, 1):
        for name in SPLITS(N):
            assert got[rank][name] == want, (rank, name)


def test_kmeans_two_gloo_ranks_equal_one_process(tmp_path):
    _two_ranks(tmp_path, "gloo")


@two_gpus
def test_kmeans_two_nccl_ranks_equal_one_process(tmp_path):
    _two_ranks(tmp_path, "nccl")
