"""PCA and Pearson correlation over TWO RANKS: the column sums and the centred-Gram partials keep their chunk order across
shards (a straddling chunk is computed by the rank holding its first row, running totals pass rank to rank, the
eigendecomposition is rank 0's), so pc, explainedVariance, the mean, the covariance, the correlation matrix and the
transformed rows equal the single-process result byte for byte — for even and uneven shards (a cut inside a chunk), fewer
than 4096 rows in total and an empty shard.  Two gloo ranks share one GPU; the NCCL case needs two GPUs and is skipped
otherwise."""
import numpy as np
import pytest
import torch

from ranks import block, run, two_gpus

pytestmark = pytest.mark.gpu

N, D, K = 30000, 41, 6
# name -> (rows in total, rows of rank 0)
CASES = {"even": (N, 15000), "uneven": (N, 11000), "chunk_aligned": (N, 8192), "short_first": (N, 2500),
         "short_total": (3000, 1200), "empty_last": (N, N), "empty_first": (N, 0)}


def _data():
    rng = np.random.default_rng(31)
    w = rng.normal(size=(8, D)) * (3.0 * 2.0 ** -np.arange(8))[:, None]
    return np.ascontiguousarray(rng.normal(size=(N, 8)) @ w + rng.normal(0.0, 0.05, (N, D)) + rng.normal(0.0, 2.0, D))


def _run(x, dev):
    from b200flow import pca as bp
    xt = torch.from_numpy(x).to(dev)
    fit = bp.pca_fit(xt, K)
    hx = lambda a: [float(v).hex() for v in np.asarray(a).ravel()]       # noqa: E731
    return {"pc": hx(fit.pc), "ev": hx(fit.explained_variance), "mean": hx(fit.mean), "cov": hx(fit.cov),
            "pearson": hx(bp.pearson(xt)), "rows": hx(bp.pca_transform(xt, fit).cpu().numpy())}


def _ranks(rank, grp, dev):
    x = _data()
    res = {}
    for name, (total, cut) in CASES.items():
        lo, hi = block(rank, cut, total)
        res[name] = _run(x[lo:hi], dev)
    return res


def _two_ranks(tmp_path, mode):
    got = run(tmp_path, _ranks, mode=mode)
    x = _data()
    want = {total: _run(x[:total], torch.device("cuda", 0)) for total in sorted({t for t, _ in CASES.values()})}
    ev = np.array([float.fromhex(v) for v in want[N]["ev"]])
    assert np.all(np.diff(ev) < 0) and ev.sum() > 0.9                  # the planted directions are found, in order
    for rank in (0, 1):
        for name, (total, cut) in CASES.items():
            g, w = got[rank][name], want[total]
            lo, hi = block(rank, cut, total)
            for key in ("pc", "ev", "mean", "cov", "pearson"):
                assert g[key] == w[key], (rank, name, key)
            assert g["rows"] == w["rows"][lo * K:hi * K], (rank, name, "rows")


def test_pca_two_gloo_ranks_equal_one_process(tmp_path):
    _two_ranks(tmp_path, "gloo")


@two_gpus
def test_pca_two_nccl_ranks_equal_one_process(tmp_path):
    _two_ranks(tmp_path, "nccl")
