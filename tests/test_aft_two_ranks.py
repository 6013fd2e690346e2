"""AFTSurvivalRegression over TWO RANKS: the AFT partials are computed from each 4096-row chunk's rows alone and chained
rank to rank (the censor travelling with the rows), so fits with and without an intercept equal the single-process run
byte for byte, for even and uneven shards, a shard shorter than one chunk and empty first and last shards.  A bad censor
or a non-positive label on one rank makes both raise.  Two gloo ranks share one GPU."""
import numpy as np
import pytest
import torch

from ranks import SPLITS, block, run

pytestmark = pytest.mark.gpu

N, D = 30000, 41


def _data():
    rng = np.random.default_rng(8)
    x = rng.normal(0.0, 1.0, (N, D)) * rng.uniform(0.2, 5.0, D) + rng.normal(0.0, 2.0, D)
    t = np.exp(x @ (rng.normal(0.0, 0.3, D) / x.std(0)) + 1.0 + 0.5 * np.log(rng.exponential(1.0, N)))
    c = (rng.random(N) < 0.7).astype(np.float64)
    return np.ascontiguousarray(x), t, c


def _hex(a):
    return [float(v).hex() for v in np.asarray(a, np.float64).reshape(-1)]


def _run(x, t, c, dev, grp):
    from b200flow import aft as baft, dist as bdist
    xt, tt, ct = torch.from_numpy(x).to(dev), torch.from_numpy(t).to(dev), torch.from_numpy(c).to(dev)
    out = {}
    for name, p in (("intercept", baft.AFTParams(max_iter=25)), ("origin", baft.AFTParams(max_iter=25, fit_intercept=False))):
        f = baft.aft_fit(xt, tt, ct, p, group=grp)
        out[name] = {"coef": _hex(f.coef), "b": float(f.intercept).hex(), "scale": float(f.scale).hex(),
                     "hist": _hex(f.objective_history), "it": f.iterations}
    off, _ = bdist.global_offset(xt.shape[0], dev, grp)
    raised = []
    for what in ("censor", "label"):
        tb, cb = tt.clone(), ct.clone()
        if xt.shape[0] and off + xt.shape[0] == N:       # only the rank holding the last global row sees the bad value
            (cb if what == "censor" else tb)[-1] = 0.5 if what == "censor" else 0.0
        try:
            baft.aft_fit(xt, tb, cb, baft.AFTParams(max_iter=3), group=grp)
            raised.append(False)
        except ValueError:
            raised.append(True)
    out["raised"] = raised
    return out


def _ranks(rank, grp, dev):
    x, t, c = _data()
    res = {}
    for name, cut in SPLITS(N).items():
        lo, hi = block(rank, cut, N)
        res[name] = _run(x[lo:hi], t[lo:hi], c[lo:hi], dev, grp)
    return res


def test_aft_two_gloo_ranks_equal_one_process(tmp_path):
    got = run(tmp_path, _ranks)
    x, t, c = _data()
    want = _run(x, t, c, torch.device("cuda", 0), None)
    assert want["raised"] == [True, True]
    for rank in (0, 1):
        for name in SPLITS(N):
            assert got[rank][name] == want, (rank, name)
