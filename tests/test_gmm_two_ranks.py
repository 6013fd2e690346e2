"""GaussianMixture over TWO RANKS: the E-step and moment partials keep their chunk order across shards (a straddling chunk
is computed by the rank holding its first row, running totals pass rank to rank, the eigendecompositions are rank 0's), so
weights, means, covariances, log-likelihood, iteration count, cluster sizes and the transform's probabilities and
predictions equal the single-process result byte for byte — for even and uneven shards, a shard shorter than one 4096-row
chunk and an empty shard.  Two gloo ranks share one GPU; the NCCL case needs two GPUs and is skipped otherwise."""
import numpy as np
import pytest
import torch

from ranks import SPLITS, block, run, two_gpus

pytestmark = pytest.mark.gpu

N = 30000


def _data():
    """four tight clusters, whose densities clear Spark's EPSILON floor, so that EM separates them (at unit scale in 41
    dimensions every responsibility would be 1/k)."""
    rng = np.random.default_rng(18)
    means = rng.normal(0.0, 0.05, (4, 41))
    return np.ascontiguousarray(means[rng.integers(0, 4, N)] + rng.normal(0.0, 0.0025, (N, 41)))


def _run(x, dev):
    from b200flow import gmm as bg
    xt = torch.from_numpy(x).to(dev)
    r = bg.gmm_fit(xt, 4, max_iter=6, tol=0.0, seed=21)
    prob, pred = bg.gmm_predict(xt, r)
    hx = lambda a: [float(v).hex() for v in np.asarray(a).ravel()]       # noqa: E731
    return {"weights": hx(r.weights), "means": hx(r.means), "covs": hx(r.covariances), "ll": float(r.log_likelihood).hex(),
            "it": r.num_iter, "sizes": r.cluster_sizes.tolist(), "prob": hx(prob.cpu().numpy()),
            "pred": pred.cpu().numpy().tolist()}


def _ranks(rank, grp, dev):
    x = _data()
    res = {}
    for name, cut in SPLITS(N).items():
        lo, hi = block(rank, cut, N)
        res[name] = _run(x[lo:hi], dev)
    return res


def _two_ranks(tmp_path, mode):
    got = run(tmp_path, _ranks, mode=mode, timeout=900)
    want = _run(_data(), torch.device("cuda", 0))
    top = np.array([float.fromhex(v) for v in want["prob"]]).reshape(N, 4).max(1)
    assert top.mean() > 0.99 and min(want["sizes"]) > 0.2 * N      # the fit separates the clusters
    for rank in (0, 1):
        for name, cut in SPLITS(N).items():
            g = got[rank][name]
            lo, hi = block(rank, cut, N)
            for key in ("weights", "means", "covs", "ll", "it", "sizes"):
                assert g[key] == want[key], (rank, name, key)
            k = 4
            assert g["prob"] == want["prob"][lo * k:hi * k], (rank, name, "prob")
            assert g["pred"] == want["pred"][lo:hi], (rank, name, "pred")


def test_gmm_two_gloo_ranks_equal_one_process(tmp_path):
    _two_ranks(tmp_path, "gloo")


@two_gpus
def test_gmm_two_nccl_ranks_equal_one_process(tmp_path):
    _two_ranks(tmp_path, "nccl")
