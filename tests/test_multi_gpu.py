"""Real multi-GPU check (needs >= 2 GPUs: `gpurun --gpus 2 -- python -m pytest tests/test_multi_gpu.py -m gpu`):
rows sharded over 2 ranks + NCCL all-reduce of the level histograms must reproduce the 1-GPU forest byte for byte."""
import numpy as np
import pytest
import torch

from ranks import block, run, two_gpus
from util import kdd_luts_gpu, kdd_plan

pytestmark = pytest.mark.gpu


def _ranks(rank, grp, dev):
    import torch.distributed as dist
    from b200flow import dist as bdist, forest as fr, synth
    n = 60000
    rec, dicts = synth.make_kdd(n, 5, seed=17, device=dev)              # identical global data in both ranks
    schema = synth.kdd_schema()
    lo, hi = bdist.shard_bounds(n, rank, 2)
    shard = rec[lo:hi].contiguous()
    luts, ordered = kdd_luts_gpu(shard, schema, dicts, grp)
    plan = kdd_plan(schema, luts, ordered)
    x, y, _ = plan.run(shard, torch.float64)
    arity = [0] * 38 + [len(ordered[c]) for c in synth.KDD_CATEGORICAL]
    C = len(ordered["label"])
    p = fr.ForestParams(num_trees=8, max_bins=70, max_depth=10, seed=2019)
    off, _ = bdist.global_offset(hi - lo, dev)
    model = fr.fit_forest(x, y, C, arity, p, row_offset=off, group=bdist.group())
    ex = model.export()
    fr.RS_MIN_BYTES = 0            # every level through reduce-scatter -> sharded scoring -> all-gather of the split records
    fr.RS_CHUNKS = 3               # ... in three pipelined slot ranges
    ex_rs = fr.fit_forest(x, y, C, arity, p, row_offset=off, group=bdist.group()).export()
    fr.RS_MIN_BYTES = 8 << 20
    fr.RS_CHUNKS = 1
    # uneven shards (21,000 / 39,000 rows: different findSplits sample capacities per rank) on the fused record path
    ulo, uhi = block(rank, 21000, n)
    ushard = rec[ulo:uhi].contiguous()
    uoff, _ = bdist.global_offset(uhi - ulo, dev)
    ex_uneven = fr.fit_forest_records(ushard, plan, C, arity, p, row_offset=uoff, group=bdist.group()).export()
    # one rank without any row: it still takes part in every collective
    eshard = rec if rank == 0 else rec[:0].contiguous()
    eoff, _ = bdist.global_offset(eshard.shape[0], dev)
    ex_empty = fr.fit_forest_records(eshard, plan, C, arity, p, row_offset=eoff, group=bdist.group()).export()
    single = None
    if rank == 0:
        xf, yf, _ = plan.run(rec, torch.float64)
        single = fr.fit_forest(xf, yf, C, arity, p).export()
    dist.barrier()
    return ex, ex_rs, ex_uneven, ex_empty, single


@two_gpus
def test_two_gpu_forest_is_byte_identical_to_one_gpu(tmp_path):
    a, c, d, e, b = run(tmp_path, _ranks, mode="nccl", timeout=200)[0]
    assert sorted(a) == sorted(b)
    for k in a:
        assert np.array_equal(a[k], b[k]), k
        assert np.array_equal(c[k], b[k]), "reduce-scatter path: " + k
        assert np.array_equal(d[k], b[k]), "uneven shards, record path: " + k
        assert np.array_equal(e[k], b[k]), "empty shard: " + k
    assert len(a["nid"]) > 500
    print("2-GPU forests (all-reduce, pipelined reduce-scatter, uneven shards on the record path, one empty shard) == 1-GPU forest: "
          "%d nodes, byte-identical" % len(a["nid"]))
