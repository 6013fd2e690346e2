"""GeneralizedLinearRegression over TWO RANKS: the per-row partials and the weighted Gram partials are computed from each
4096-row chunk's rows alone and chained rank to rank, and the D x D solves run on rank 0 and are broadcast, so poisson/log
with weights and an offset, binomial/probit, gamma/inverse and tweedie 1.5 fits and their summaries equal the
single-process run byte for byte, for even and uneven shards, a shard shorter than one chunk and empty first and last
shards.  A negative poisson label on one rank makes both raise.  Two gloo ranks share one GPU; the NCCL case needs two
GPUs and is skipped otherwise."""
import numpy as np
import pytest
import torch

from ranks import SPLITS, block, run, two_gpus

pytestmark = pytest.mark.gpu

N, D = 30000, 23


def _data():
    rng = np.random.default_rng(8)
    x = np.abs(rng.normal(0.0, 1.0, (N, D))) * rng.uniform(0.05, 0.2, D)
    y = rng.poisson(np.exp(x @ rng.normal(0.0, 0.5, D) + 0.3)).astype(float)
    return np.ascontiguousarray(x), y, rng.uniform(0.5, 2.0, N), rng.normal(0.0, 0.05, N)


def _hex(a):
    return [float(v).hex() for v in np.asarray(a, np.float64).reshape(-1)]


def _run(x, y, w, off, dev, grp):
    from b200flow import glm as bg
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)      # noqa: E731
    xt, yt, wt, ot = t(x), t(y), t(w), t(off)
    out = {}
    cases = {"poisson": (bg.GLMParams(family="poisson"), yt, wt, ot),
             "probit": (bg.GLMParams(family="binomial", link="probit"), (yt > 1).double(), None, None),
             "gamma": (bg.GLMParams(family="gamma", link="inverse"), yt + 1.0, wt, None),
             "tweedie": (bg.GLMParams(family="tweedie", variance_power=1.5, link_power=0.0, max_iter=8), yt, None, ot)}
    for name, (p, yy, ww, oo) in cases.items():
        f = bg.glm_fit(xt, yy, p, weight=ww, offset=oo, group=grp)
        s = bg.summarize(xt, yy, f, p, weight=ww, offset=oo, group=grp)
        out[name] = {"coef": _hex(f.coef), "b": float(f.intercept).hex(), "it": f.iterations,
                     "diag": None if f.diag_inv_atwa is None else _hex(f.diag_inv_atwa),
                     "summary": _hex([s.deviance, s.null_deviance, s.dispersion] + ([] if s.aic is None else [s.aic])
                                     + list(s.std_errors) + list(s.p_values)) + [s.num_instances, s.rank]}
    from b200flow import dist as bdist
    ro, _ = bdist.global_offset(xt.shape[0], dev, grp)
    bad = yt.clone()
    if xt.shape[0] and ro + xt.shape[0] == N:              # only the rank holding the last global row sees the bad label
        bad[-1] = -1.0
    raised = []
    for p in (bg.GLMParams(family="poisson"), bg.GLMParams(family="tweedie", variance_power=1.5)):
        try:
            bg.glm_fit(xt, bad, p, group=grp)
            raised.append(False)
        except ValueError:
            raised.append(True)
    out["raised"] = raised
    return out


def _ranks(rank, grp, dev):
    x, y, w, off = _data()
    res = {}
    for name, cut in SPLITS(N).items():
        lo, hi = block(rank, cut, N)
        res[name] = _run(x[lo:hi], y[lo:hi], w[lo:hi], off[lo:hi], dev, grp)
    return res


def _two_ranks(tmp_path, mode):
    got = run(tmp_path, _ranks, mode=mode)
    x, y, w, off = _data()
    want = _run(x, y, w, off, torch.device("cuda", 0), None)
    assert want["raised"] == [True, True]
    for rank in (0, 1):
        for name in SPLITS(N):
            assert got[rank][name] == want, (rank, name)


def test_glm_two_gloo_ranks_equal_one_process(tmp_path):
    _two_ranks(tmp_path, "gloo")


@two_gpus
def test_glm_two_nccl_ranks_equal_one_process(tmp_path):
    _two_ranks(tmp_path, "nccl")
