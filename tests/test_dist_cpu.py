"""Host-side logic of the row-sharded (multi-GPU) path, exercised with 2 CPU processes over gloo:
block partition, global row offsets, integer all-reduce of per-shard histograms == unsharded histogram,
and shard-independent RNG streams (bagging weights / randomSplit ids are slices of the global stream)."""
import numpy as np
import torch

import oracle
from b200flow import dist as bdist
from ranks import block, run


def _sharding(rank, grp, dev):
    assert bdist.group() is not None
    n, F, C, NB, m = 10007, 12, 3, 16, 4
    rng = np.random.default_rng(0)                      # same global data in every rank
    tp = rng.integers(0, NB, size=(n, 16), dtype=np.uint8); tp[:, F] = rng.integers(0, C, n)
    lo, hi = bdist.shard_bounds(n, rank, 2)
    off, tot = bdist.global_offset(hi - lo, dev)
    assert (off, tot) == (lo, n)
    cdf = oracle.poisson_cdf_table(1.0)
    w_local = oracle.bag_weights(99, 3, hi - lo, cdf, row_offset=off)          # counter RNG keyed by GLOBAL row
    w_full = oracle.bag_weights(99, 3, n, cdf)
    assert np.array_equal(w_local, w_full[:, lo:hi])
    sid = oracle.random_split(2019, hi - lo, [0.75, 1.0], row_offset=off)
    assert np.array_equal(sid, oracle.random_split(2019, n, [0.75, 1.0])[lo:hi])
    subset = oracle.feature_subset(5, 1, 7, F, m)
    rows = np.nonzero(w_local[1])[0].astype(np.int32)
    h = oracle.hist_node(tp[lo:hi], F, rows, w_local[1][rows], subset, NB, C)
    ht = torch.from_numpy(h.astype(np.int32))
    bdist.all_reduce_sum_(ht)                                                    # R7r: the per-level collective
    rows_f = np.nonzero(w_full[1])[0].astype(np.int32)
    want = oracle.hist_node(tp, F, rows_f, w_full[1][rows_f], subset, NB, C)
    assert np.array_equal(ht.numpy().astype(np.int64), want)


def test_two_rank_sharding_gloo(tmp_path):
    run(tmp_path, _sharding, mode="cpu", timeout=300)


def _gather(rank, grp, dev):
    from b200flow import forest as fr
    F = 3
    n_s, cap = (1000, 1024) if rank == 0 else (1050, 2048)      # ADVICE r1: 1050 > the other rank's capacity
    col = torch.arange(n_s, dtype=torch.float64) + 10000.0 * rank
    sample = torch.zeros(F * cap, dtype=torch.float64)
    for f in range(F):
        sample.view(F, cap)[f, :n_s] = col + 0.25 * f
    out, tot, new_cap = fr._gather_sample(sample, n_s, cap, F, grp)
    assert tot == 2050 and new_cap == 4096 and out.numel() == F * new_cap
    got = out.view(F, new_cap)[:, :tot]
    want0 = torch.cat([torch.arange(1000, dtype=torch.float64), torch.arange(1050, dtype=torch.float64) + 10000.0])
    for f in range(F):
        assert torch.equal(got[f], want0 + 0.25 * f)


def test_gather_sample_uneven_shards_gloo(tmp_path):
    # the findSplits sample of every rank is exchanged in blocks of the agreed (widest) width, whatever the local capacity
    run(tmp_path, _gather, mode="cpu", timeout=300)


def test_shard_bounds_cover_everything():
    for n in (0, 1, 7, 1000, 4898431):
        for world in (1, 2, 3, 8):
            b = [bdist.shard_bounds(n, r, world) for r in range(world)]
            assert b[0][0] == 0 and b[-1][1] == n and all(b[i][1] == b[i + 1][0] for i in range(world - 1))
            assert max(h - l for l, h in b) - min(h - l for l, h in b) <= 1
    assert bdist.group() is None and bdist.global_offset(5, torch.device("cpu")) == (0, 5)


def _fits(x, y, C, grp=None):
    from b200flow import linear
    xs, ys = torch.from_numpy(x), torch.from_numpy(y)
    nb = linear.nb_fit(xs, ys, C, 1.0, group=grp)
    lr = linear.lr_fit(xs, ys, C, max_iter=60, reg_param=0.1, elastic_net=0.5, tol=1e-12, family="multinomial", group=grp)
    return dict(pi=nb.pi.numpy(), theta=nb.theta.numpy(), coef=lr.coef.numpy(), b=lr.intercept.numpy(), hist=np.array(lr.objective_history))


def _linear_data():
    rng = np.random.default_rng(4)                       # same global data in every rank
    n, D, C = 3001, 9, 4
    y = rng.integers(0, C, n)
    x = rng.poisson(rng.uniform(0.5, 5.0, size=(C, D))[y]).astype(np.float64)
    x[:, 2] = 3.0
    return x, y, C


def _linear(rank, grp, dev):
    x, y, C = _linear_data()
    lo, hi = block(rank, 700, len(y))                    # uneven shards
    return _fits(x[lo:hi], y[lo:hi], C, grp)


def test_naive_bayes_and_logistic_regression_on_row_shards_gloo(tmp_path):
    """SURVEY 8f-4 under one process per GPU: the sufficient statistics (NB) and the loss / gradient sums (LR) are all-reduced,
    so every rank ends with the same model, equal to the single-process one up to the association of the fp64 partial sums."""
    a, b = run(tmp_path, _linear, mode="cpu", timeout=300)
    one = _fits(*_linear_data())
    for k in a:
        assert np.array_equal(a[k], b[k]), k                                         # the ranks agree bit for bit
    assert np.allclose(a["pi"], one["pi"], atol=1e-12) and np.allclose(a["theta"], one["theta"], atol=1e-12)
    assert abs(a["hist"][-1] - one["hist"][-1]) < 1e-9
    assert np.abs(a["coef"] - one["coef"]).max() < 1e-5 and np.abs(a["b"] - one["b"]).max() < 1e-5
