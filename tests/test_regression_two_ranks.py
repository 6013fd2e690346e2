"""RandomForestRegressor, DecisionTreeRegressor and RegressionEvaluator with rows sharded over TWO RANKS ON ONE GPU (gloo):
both processes run the real kernels on cuda:0.  This exercises the global-row-keyed findSplits sample and Poisson bag
weights, the all-reduced label scale and tree weights behind the label grid, the per-level int64 histogram all-reduce, the
evaluator's all-reduced limb sums, the rank-wide label check and a rank whose shard is EMPTY walking every collective.  The
models and metrics must be byte-identical to the single-process ones."""
import numpy as np
import pytest
import torch

from ranks import block, run

pytestmark = pytest.mark.gpu


def _data(dev):
    from b200flow import synth
    g = torch.Generator(device=dev).manual_seed(31)
    n, F = 24000, 20
    x = torch.randint(0, 8, (n, F), device=dev, generator=g).to(torch.float64)
    x[:, :10] += torch.rand((n, 10), device=dev, generator=g, dtype=torch.float64)
    y = 1e4 * x[:, 0] - 300.0 * x[:, 11] + torch.randn(n, device=dev, generator=g, dtype=torch.float64) * 50.0
    arity = [0] * 10 + [8] * 10
    return x, y, arity


def _flat(rf, dt, m):
    return dict(metrics=np.array([m[k] for k in sorted(m)]), **{"rf_" + k: v for k, v in rf.export().items()},
                **{"dt_" + k: v for k, v in dt.export().items()})


def _ranks(rank, grp, dev):
    from b200flow import dist as bdist, metrics as bm, regression as br
    x, y, arity = _data(dev)
    n = x.shape[0]
    lo, hi = bdist.shard_bounds(n, rank, 2)
    p = br.RegressorParams(num_trees=4, max_depth=5, max_bins=16, subsampling_rate=0.8, seed=2019)
    out = {}
    for name, (a, b) in (("even", (lo, hi)), ("uneven", block(rank, 9000, n)), ("empty", block(rank, n, n))):
        off, tot = bdist.global_offset(b - a, dev, grp)
        assert tot == n and off == a
        xs, ys = x[a:b].contiguous(), y[a:b].contiguous()
        rf = br.fit_rf_regressor(xs, ys, arity, p, row_offset=off, group=grp)
        dt = br.fit_dt_regressor(xs, ys, arity, p, row_offset=off, group=grp)
        out[name] = _flat(rf, dt, bm.regression_metrics(ys, rf.predict(xs), group=grp))
    # a NaN label on rank 1 only: both ranks refuse, none waits in a collective
    yb = y[lo:hi].clone()
    if rank == 1:
        yb[5] = float("nan")
    try:
        br.fit_rf_regressor(x[lo:hi].contiguous(), yb, arity, p, row_offset=lo, group=grp)
        refused = False
    except ValueError:
        refused = True
    return out, refused


def test_two_ranks_one_gpu_regression_equals_single_process(tmp_path):
    (out, refused0), (_, refused1) = run(tmp_path, _ranks, timeout=300)
    from b200flow import metrics as bm, regression as br
    x, y, arity = _data(torch.device("cuda", 0))
    p = br.RegressorParams(num_trees=4, max_depth=5, max_bins=16, subsampling_rate=0.8, seed=2019)
    rf, dt = br.fit_rf_regressor(x, y, arity, p), br.fit_dt_regressor(x, y, arity, p)
    single = _flat(rf, dt, bm.regression_metrics(y, rf.predict(x)))
    for name in ("even", "uneven", "empty"):
        got = out[name]
        assert sorted(got) == sorted(single)
        for k in single:
            assert np.array_equal(got[k].view(np.uint8), np.asarray(single[k]).view(np.uint8)), "%s shards: %s" % (name, k)
    assert (single["rf_is_leaf"] == 0).sum() > 20
    assert [refused0, refused1] == [True, True]
