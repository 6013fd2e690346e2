"""OneVsRest(GBTClassifier)'s class-batched trainer with rows sharded over TWO RANKS ON ONE GPU (gloo): both processes run the
real kernels on cuda:0.  Even shards on the dense path, uneven and empty shards on the fused record path; every class's
model must be byte-identical to the single-process one, and a label beyond the class count on one rank makes both refuse."""
import numpy as np
import pytest
import torch

from ranks import block, run
from util import kdd_luts_gpu, kdd_plan

pytestmark = pytest.mark.gpu

K = 5


def _exports(model):
    return {"%d_%s" % (k, key): v for k, m in enumerate(model.models) for key, v in m.export().items()}


def _ranks(rank, grp, dev):
    from b200flow import dist as bdist, gbt as bg, synth
    n = 24000
    rec, dicts = synth.make_kdd(n, K, seed=31, device=dev)              # identical global data in both ranks
    schema = synth.kdd_schema()
    lo, hi = bdist.shard_bounds(n, rank, 2)
    luts, ordered = kdd_luts_gpu(rec[lo:hi].contiguous(), schema, dicts, grp)
    assert len(ordered["label"]) == K
    plan = kdd_plan(schema, luts, ordered)
    arity = [0] * 38 + [len(ordered[c]) for c in synth.KDD_CATEGORICAL]
    p = bg.GBTParams(max_iter=4, max_depth=5, max_bins=70, subsampling_rate=0.8, feature_subset_strategy="sqrt", seed=2019)
    out = {}
    for name, (a, b) in (("even", (lo, hi)), ("uneven", block(rank, 9000, n)), ("empty", block(rank, n, n))):
        shard = rec[a:b].contiguous()
        off, tot = bdist.global_offset(b - a, dev, grp)
        assert tot == n and off == a
        if name == "even":                                               # dense matrix path
            x, y, _ = plan.run(shard, torch.float64)
            model = bg.fit_gbt_ovr(x, y, K, arity, p, row_offset=off, group=grp)
        else:                                                             # fused record path
            model = bg.fit_gbt_ovr_records(shard, plan, K, arity, p, row_offset=off, group=grp)
        out[name] = _exports(model)
    # a label beyond the class count on rank 1 only: both ranks refuse, none waits in a collective
    x, y, _ = plan.run(rec[lo:hi].contiguous(), torch.float64)
    if rank == 1:
        y = y.clone(); y[5] = K
    try:
        bg.fit_gbt_ovr(x, y, K, arity, p, row_offset=lo, group=grp)
        refused = False
    except ValueError:
        refused = True
    single = _exports(bg.fit_gbt_ovr_records(rec, plan, K, arity, p)) if rank == 0 else None
    return out, single, refused


def test_two_ranks_one_gpu_ovr_equals_single_process(tmp_path):
    (out, single, refused0), (_, _, refused1) = run(tmp_path, _ranks, timeout=300)
    for name in ("even", "uneven", "empty"):
        got = out[name]
        assert sorted(got) == sorted(single)
        for k in single:
            assert np.array_equal(got[k].view(np.uint8), single[k].view(np.uint8)), "%s shards: %s" % (name, k)
    for k in range(K):
        assert (single["%d_is_leaf" % k] == 0).sum() > 4
    assert [refused0, refused1] == [True, True]
