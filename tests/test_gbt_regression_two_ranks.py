"""GBTRegressor with rows sharded over TWO RANKS ON ONE GPU (gloo): both processes run the real kernels on cuda:0.  This
exercises the global-row-keyed findSplits sample and Bernoulli subsample weights, the all-reduced label scale, the
all-reduced max |r| behind every iteration's residual grid, the per-level int64 histogram all-reduce, evaluateEachIteration's
all-reduced sums, the rank-wide label check and a rank whose shard is EMPTY walking every collective.  The models and the
per-iteration losses must be byte-identical to the single-process ones."""
import numpy as np
import pytest
import torch

from ranks import block, run

pytestmark = pytest.mark.gpu


def _data(dev):
    g = torch.Generator(device=dev).manual_seed(37)
    n, F = 24000, 20
    x = torch.randint(0, 8, (n, F), device=dev, generator=g).to(torch.float64)
    x[:, :10] += torch.rand((n, 10), device=dev, generator=g, dtype=torch.float64)
    y = 1e4 * x[:, 0] - 300.0 * x[:, 11] + torch.randn(n, device=dev, generator=g, dtype=torch.float64) * 50.0
    arity = [0] * 10 + [8] * 10
    return x, y, arity


def _params(loss):
    from b200flow import gbt_regression as bgr
    return bgr.GBTRegressorParams(max_iter=4, step_size=0.5, max_depth=5, max_bins=16, subsampling_rate=0.8, seed=2019, loss=loss)


def _result(model, xs, ys, grp):
    out = {k: v for k, v in model.export().items()}
    out["E"] = np.array(model.E, np.int64)
    out["each"] = np.array(model.evaluate_each_iteration(xs, ys, "squared", group=grp)
                           + model.evaluate_each_iteration(xs, ys, "absolute", group=grp))
    return out


def _ranks(rank, grp, dev):
    from b200flow import dist as bdist, gbt_regression as bgr
    x, y, arity = _data(dev)
    n = x.shape[0]
    lo, hi = bdist.shard_bounds(n, rank, 2)
    out = {}
    for name, (a, b) in (("even", (lo, hi)), ("uneven", block(rank, 9000, n)), ("empty", block(rank, n, n))):
        off, tot = bdist.global_offset(b - a, dev, grp)
        assert tot == n and off == a
        xs, ys = x[a:b].contiguous(), y[a:b].contiguous()
        for loss in ("squared", "absolute"):
            model = bgr.fit_gbt_regressor(xs, ys, arity, _params(loss), row_offset=off, group=grp)
            out[name + "_" + loss] = _result(model, xs, ys, grp)
    # a NaN label on rank 1 only: both ranks refuse, none waits in a collective
    yb = y[lo:hi].clone()
    if rank == 1:
        yb[5] = float("nan")
    try:
        bgr.fit_gbt_regressor(x[lo:hi].contiguous(), yb, arity, _params("squared"), row_offset=lo, group=grp)
        refused = False
    except ValueError:
        refused = True
    return out, refused


def test_two_ranks_one_gpu_gbt_regression_equals_single_process(tmp_path):
    (out, refused0), (_, refused1) = run(tmp_path, _ranks, timeout=300)
    from b200flow import gbt_regression as bgr
    x, y, arity = _data(torch.device("cuda", 0))
    for loss in ("squared", "absolute"):
        single = _result(bgr.fit_gbt_regressor(x, y, arity, _params(loss)), x, y, None)
        for name in ("even", "uneven", "empty"):
            got = out["%s_%s" % (name, loss)]
            assert sorted(got) == sorted(single)
            for k in single:
                assert np.array_equal(got[k].view(np.uint8), np.asarray(single[k]).view(np.uint8)), "%s shards, %s: %s" % (name, loss, k)
        assert (single["is_leaf"] == 0).sum() > 20
    assert [refused0, refused1] == [True, True]
