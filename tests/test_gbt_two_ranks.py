"""GBTClassifier with rows sharded over TWO RANKS ON ONE GPU (gloo): both processes run the real kernels on cuda:0.  This
exercises the global row count behind the residual grid, the global-row-keyed findSplits sample and Bernoulli subsample,
the per-level int64 histogram all-reduce, the rank-wide label check and a rank whose shard is EMPTY walking every
collective.  The model must be byte-identical to the single-process model."""
import numpy as np
import pytest
import torch

from ranks import block, run
from util import kdd_luts_gpu, kdd_plan

pytestmark = pytest.mark.gpu


def _ranks(rank, grp, dev):
    from b200flow import dist as bdist, gbt as bg, synth
    n = 30000
    rec, dicts = synth.make_kdd(n, 2, seed=23, device=dev)              # identical global data in both ranks
    schema = synth.kdd_schema()
    lo, hi = bdist.shard_bounds(n, rank, 2)
    luts, ordered = kdd_luts_gpu(rec[lo:hi].contiguous(), schema, dicts, grp)
    plan = kdd_plan(schema, luts, ordered)
    arity = [0] * 38 + [len(ordered[c]) for c in synth.KDD_CATEGORICAL]
    p = bg.GBTParams(max_iter=5, max_depth=5, max_bins=70, subsampling_rate=0.8, feature_subset_strategy="sqrt", seed=2019)
    out = {}
    for name, (a, b) in (("even", (lo, hi)), ("uneven", block(rank, 11000, n)), ("empty", block(rank, n, n))):
        shard = rec[a:b].contiguous()
        off, tot = bdist.global_offset(b - a, dev, grp)
        assert tot == n and off == a
        if name == "even":                                               # dense matrix path
            x, y, _ = plan.run(shard, torch.float64)
            model = bg.fit_gbt(x, y, arity, p, row_offset=off, group=grp)
        else:                                                             # fused record path
            model = bg.fit_gbt_records(shard, plan, arity, p, row_offset=off, group=grp)
        out[name] = model.export()
    # a label outside {0, 1} on rank 1 only: both ranks refuse, none waits in a collective
    x, y, _ = plan.run(rec[lo:hi].contiguous(), torch.float64)
    if rank == 1:
        y = y.clone(); y[5] = 2
    try:
        bg.fit_gbt(x, y, arity, p, row_offset=lo, group=grp)
        refused = False
    except ValueError:
        refused = True
    single = bg.fit_gbt_records(rec, plan, arity, p).export() if rank == 0 else None
    return out, single, refused


def test_two_ranks_one_gpu_gbt_equals_single_process(tmp_path):
    (out, single, refused0), (_, _, refused1) = run(tmp_path, _ranks, timeout=300)
    for name in ("even", "uneven", "empty"):
        got = out[name]
        assert sorted(got) == sorted(single)
        for k in single:
            assert np.array_equal(got[k].view(np.uint8), single[k].view(np.uint8)), "%s shards: %s" % (name, k)
    assert (single["is_leaf"] == 0).sum() > 20
    assert [refused0, refused1] == [True, True]
