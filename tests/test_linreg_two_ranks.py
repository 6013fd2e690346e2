"""LinearRegression over TWO RANKS: the least-squares / Huber partials and the labelled Gram partials are computed from
each 4096-row chunk's rows alone and chained rank to rank, and the D x D solves run on rank 0 and are broadcast, so the
normal, L-BFGS + L1 and Huber fits and the summary metrics equal the single-process run byte for byte, for even and
uneven shards, a shard shorter than one chunk and empty first and last shards.  A NaN label on one rank makes both raise.
Two gloo ranks share one GPU; the NCCL case needs two GPUs and is skipped otherwise."""
import numpy as np
import pytest
import torch

from ranks import SPLITS, block, run, two_gpus

pytestmark = pytest.mark.gpu

N, D = 30000, 41


def _data():
    rng = np.random.default_rng(8)
    x = rng.normal(0.0, 1.0, (N, D)) * rng.uniform(0.2, 5.0, D) + rng.normal(0.0, 2.0, D)
    y = x @ rng.normal(0.0, 1.0, D) + 2.0 + rng.standard_t(3, N)
    return np.ascontiguousarray(x), y


def _hex(a):
    return [float(v).hex() for v in np.asarray(a, np.float64).reshape(-1)]


def _fit_json(f):
    return {"coef": _hex(f.coef), "b": float(f.intercept).hex(), "scale": float(f.scale).hex(),
            "hist": _hex(f.objective_history), "it": f.iterations, "solver": f.solver,
            "diag": None if f.diag_inv_atwa is None else _hex(f.diag_inv_atwa)}


def _run(x, y, dev, grp):
    from b200flow import linreg as blr
    xt, yt = torch.from_numpy(x).to(dev), torch.from_numpy(y).to(dev)
    out = {}
    cases = {"normal": blr.LinRegParams(),
             "lbfgs_l1": blr.LinRegParams(solver="l-bfgs", reg_param=0.05, elastic_net_param=1.0, max_iter=15),
             "huber": blr.LinRegParams(loss="huber", reg_param=0.01, max_iter=15)}
    for name, p in cases.items():
        f = blr.linreg_fit(xt, yt, p, group=grp)
        out[name] = _fit_json(f)
        if name == "normal":
            s = blr.summarize(xt, yt, f, True, group=grp)
            out["summary"] = _hex([s.mse, s.rmse, s.mae, s.r2, s.r2adj, s.explained_variance] + s.deviance_residuals
                                  + list(s.std_errors) + list(s.p_values)) + [s.num_instances, s.degrees_of_freedom]
    from b200flow import dist as bdist
    off, _ = bdist.global_offset(xt.shape[0], dev, grp)
    bad = yt.clone()
    if xt.shape[0] and off + xt.shape[0] == N:             # only the rank holding the last global row sees the NaN
        bad[-1] = float("nan")
    raised = []
    for p in cases.values():
        try:
            blr.linreg_fit(xt, bad, p, group=grp)
            raised.append(False)
        except ValueError:
            raised.append(True)
    out["raised"] = raised
    return out


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
    assert want["raised"] == [True, True, True]
    for rank in (0, 1):
        for name in SPLITS(N):
            assert got[rank][name] == want, (rank, name)


def test_linreg_two_gloo_ranks_equal_one_process(tmp_path):
    _two_ranks(tmp_path, "gloo")


@two_gpus
def test_linreg_two_nccl_ranks_equal_one_process(tmp_path):
    _two_ranks(tmp_path, "nccl")
