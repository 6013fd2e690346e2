"""FMRegressor over TWO RANKS: the squared-error factorization-machine partials are computed from each 4096-row chunk's
rows alone and chained rank to rank, and the optimiser state is the same on every rank, so adamW, gd and mini-batch fits
equal the single-process run byte for byte, for even and uneven shards, a shard shorter than one chunk and empty first
and last shards.  A non-finite label on one rank makes both raise.  Two gloo ranks share one GPU."""
import numpy as np
import pytest
import torch

from ranks import SPLITS, block, run

pytestmark = pytest.mark.gpu

N, D = 30000, 23


def _data():
    rng = np.random.default_rng(8)
    x = rng.normal(0.0, 1.0, (N, D)) * (rng.random((N, D)) < 0.6)
    y = x[:, 0] * x[:, 1] + x @ rng.normal(0.0, 0.2, D) + rng.normal(0.0, 0.5, N)
    return np.ascontiguousarray(x), y


def _hex(a):
    return [float(v).hex() for v in np.asarray(a, np.float64).reshape(-1)]


def _run(x, y, dev, grp):
    from b200flow import dist as bdist, fm as bfm
    xt, yt = torch.from_numpy(x).to(dev), torch.from_numpy(y).to(dev)
    out = {}
    cases = {"adamw": bfm.FMParams(factor_size=4, max_iter=8, step_size=0.05, seed=3),
             "gd_batch": bfm.FMParams(factor_size=3, max_iter=8, step_size=0.05, solver="gd", mini_batch_fraction=0.4,
                                      reg_param=0.01, seed=4)}
    for name, p in cases.items():
        f = bfm.fm_regression_fit(xt, yt, p, group=grp)
        out[name] = {"V": _hex(f.factors), "w": _hex(f.linear), "b": float(f.intercept).hex(),
                     "hist": _hex(f.objective_history), "it": f.iterations}
    off, _ = bdist.global_offset(xt.shape[0], dev, grp)
    bad = yt.clone()
    if xt.shape[0] and off + xt.shape[0] == N:             # only the rank holding the last global row sees the NaN
        bad[-1] = float("nan")
    try:
        bfm.fm_regression_fit(xt, bad, cases["adamw"], group=grp)
        out["raised"] = False
    except ValueError:
        out["raised"] = True
    return out


def _ranks(rank, grp, dev):
    x, y = _data()
    res = {}
    for name, cut in SPLITS(N).items():
        lo, hi = block(rank, cut, N)
        res[name] = _run(x[lo:hi], y[lo:hi], dev, grp)
    return res


def test_fm_regression_two_gloo_ranks_equal_one_process(tmp_path):
    got = run(tmp_path, _ranks)
    x, y = _data()
    want = _run(x, y, torch.device("cuda", 0), None)
    assert want["raised"]
    for rank in (0, 1):
        for name in SPLITS(N):
            assert got[rank][name] == want, (rank, name)
