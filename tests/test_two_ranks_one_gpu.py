"""Row-sharded training with TWO RANKS ON ONE GPU: both processes run the real CUDA kernels on cuda:0 and exchange the level
histograms through a gloo group (b200flow.dist stages CUDA tensors through host memory for gloo).  This exercises the
multi-rank control flow — global row offsets, the gathered findSplits sample, the per-level histogram all-reduce, ranks whose
shards are uneven or EMPTY — on the driver's 1-GPU box, where tests/test_multi_gpu.py (NCCL, 2 GPUs) is skipped.
The forest must be byte-identical to the single-process forest (SURVEY.md 8e: integer sums, global-row-keyed RNG)."""
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist

from ranks import block, run
from util import kdd_luts_gpu, kdd_plan

pytestmark = pytest.mark.gpu


def _ranks(rank, grp, dev, out_dir):
    from b200flow import dist as bdist, forest as fr, synth
    n = 40000
    rec, dicts = synth.make_kdd(n, 5, seed=17, device=dev)              # identical global data in both ranks
    schema = synth.kdd_schema()
    lo, hi = bdist.shard_bounds(n, rank, 2)
    luts, ordered = kdd_luts_gpu(rec[lo:hi].contiguous(), schema, dicts, grp)
    plan = kdd_plan(schema, luts, ordered)
    arity = [0] * 38 + [len(ordered[c]) for c in synth.KDD_CATEGORICAL]
    C = len(ordered["label"])
    p = fr.ForestParams(num_trees=6, max_bins=70, max_depth=8, seed=2019)
    out = {}
    for name, (a, b) in (("even", (lo, hi)), ("uneven", block(rank, 13000, n)), ("empty", block(rank, n, n))):
        shard = rec[a:b].contiguous()
        off, tot = bdist.global_offset(b - a, dev, grp)
        assert tot == n and off == a
        if name == "even":                                               # dense matrix path
            x, y, _ = plan.run(shard, torch.float64)
            model = fr.fit_forest(x, y, C, arity, p, row_offset=off, group=grp)
        else:                                                             # fused record path
            model = fr.fit_forest_records(shard, plan, C, arity, p, row_offset=off, group=grp)
        out[name] = model.export()
        # the sharded evaluator: every rank (also the one without rows) joins both collectives
        raw, prob, pred, lab = model.predict_records(shard, plan, want_label=True)
        cm = bdist.all_reduce_sum_(fr.confusion_matrix(pred, lab.to(torch.float64), C), grp)
        out[name]["cm"] = cm.cpu().numpy()
    # spark.read.csv under one process per GPU: same schema and dictionary codes on every rank, a row block each
    from b200flow import csvio
    csv_path = os.path.join(out_dir, "flows.csv")
    if rank == 0:
        rng = np.random.default_rng(3)
        with open(csv_path + ".tmp", "w") as f:
            f.write("a,b,proto,c\n")
            for i in range(5001):
                f.write("%d,%s,%s,%s\n" % (rng.integers(-9, 9), repr(float(rng.standard_normal())), ["tcp", "udp", "icmp", "gre"][int(rng.integers(0, 4)) if i > 2500 else 0],
                                            "" if i % 97 == 0 else str(i)))
        os.replace(csv_path + ".tmp", csv_path)
    dist.barrier()
    part, sch, dcts = csvio.read_csv([csv_path], header=True, infer_schema=True, shard=(rank, 2))
    res = {"forest": out, "csv_part": part.cpu().numpy(), "csv_meta": repr((sch.names, sch.types, dcts))}
    if rank == 0:
        whole, sch_w, dcts_w = csvio.read_csv([csv_path], header=True, infer_schema=True)
        res["csv_whole"], res["csv_meta_whole"] = whole.cpu().numpy(), repr((sch_w.names, sch_w.types, dcts_w))
        single = fr.fit_forest_records(rec, plan, C, arity, p)
        ex = single.export()
        _, _, pred, lab = single.predict_records(rec, plan, want_label=True)
        ex["cm"] = fr.confusion_matrix(pred, lab.to(torch.float64), C).cpu().numpy()
        res["single"] = ex
    return res


def test_two_ranks_one_gpu_forest_equals_single_process(tmp_path):
    got = run(tmp_path, _ranks, args=(str(tmp_path),), timeout=240)
    single = got[0]["single"]
    for name in ("even", "uneven", "empty"):
        forest = got[0]["forest"][name]
        assert sorted(forest) == sorted(single)
        for k in single:
            assert np.array_equal(forest[k], single[k]), "%s shards: %s" % (name, k)
    assert len(single["nid"]) > 300
    # the CSV reader's row blocks: concatenated they are the whole file, with one schema and one dictionary (rank 1's block
    # alone holds "udp" / "icmp" / "gre": the codes still come from the global order of first appearance)
    parts = [got[r]["csv_part"] for r in (0, 1)]
    whole = got[0]["csv_whole"]
    assert parts[0].shape[0] == 2500 and parts[1].shape[0] == 2501 and np.array_equal(np.concatenate(parts), whole)
    metas = {got[0]["csv_meta"], got[1]["csv_meta"], got[0]["csv_meta_whole"]}
    assert len(metas) == 1 and "'code'" in metas.pop()
