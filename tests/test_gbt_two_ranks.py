"""GBTClassifier with rows sharded over TWO RANKS ON ONE GPU (gloo): both processes run the real kernels on cuda:0.  This
exercises the global row count behind the residual grid, the global-row-keyed findSplits sample and Bernoulli subsample,
the per-level int64 histogram all-reduce, the rank-wide label check and a rank whose shard is EMPTY walking every
collective.  The model must be byte-identical to the single-process model."""
import os
import socket
import time
import traceback

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _worker(rank, world, port, out_dir):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from b200flow import dist as bdist, encode as enc, gbt as bg, synth
        dev = torch.device("cuda", 0)
        n = 30000
        rec, dicts = synth.make_kdd(n, 2, seed=23, device=dev)              # identical global data in both ranks
        schema = synth.kdd_schema()
        grp = bdist.group()
        luts, ordered = {}, {}
        lo, hi = bdist.shard_bounds(n, rank, world)
        for c in synth.KDD_CATEGORICAL + ["label"]:
            cnt = bdist.all_reduce_sum_(enc.category_counts(rec[lo:hi].contiguous(), schema, c, len(dicts[c]))).cpu().numpy()
            ordered[c], luts[c] = enc.string_index_order(cnt, dicts[c])
        plan = enc.EncodePlan(schema)
        for c in synth.KDD_COLUMNS:
            if c not in synth.KDD_CATEGORICAL and c != "label":
                plan.add_numeric(c)
        for c in synth.KDD_CATEGORICAL:
            plan.add_index(c, luts[c])
        plan.set_label("label", luts["label"])
        arity = [0] * 38 + [len(ordered[c]) for c in synth.KDD_CATEGORICAL]
        p = bg.GBTParams(max_iter=5, max_depth=5, max_bins=70, subsampling_rate=0.8, feature_subset_strategy="sqrt", seed=2019)
        out = {}
        for name, (a, b) in (("even", (lo, hi)), ("uneven", (0, 11000) if rank == 0 else (11000, n)), ("empty", (0, n) if rank == 0 else (n, n))):
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
            out["refused"] = {"v": np.zeros(1)}
        except ValueError:
            out["refused"] = {"v": np.ones(1)}
        np.save(os.path.join(out_dir, "refused%d.npy" % rank), out.pop("refused")["v"])
        if rank == 0:
            for name, ex in out.items():
                np.savez(os.path.join(out_dir, name + ".npz"), **ex)
            np.savez(os.path.join(out_dir, "single.npz"), **bg.fit_gbt_records(rec, plan, arity, p).export())
        open(os.path.join(out_dir, "ok%d" % rank), "w").write("ok")
    except Exception:
        open(os.path.join(out_dir, "error%d.txt" % rank), "w").write(traceback.format_exc())
        raise
    finally:
        try:
            dist.destroy_process_group()
        except Exception:
            pass


def test_two_ranks_one_gpu_gbt_equals_single_process(tmp_path):
    import torch.multiprocessing as mp
    ctx = mp.start_processes(_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=False, start_method="spawn")
    deadline = time.time() + 300
    failed = None
    try:
        while not ctx.join(timeout=5):
            if time.time() > deadline:
                failed = "workers hung"
                break
    except Exception as e:                                                    # a worker raised: its traceback is on file
        failed = "worker failed: %s" % e
    if failed:
        for pr in ctx.processes:
            if pr.is_alive():
                pr.kill()
        errs = "\n".join("--- rank %d\n%s" % (r, open(tmp_path / ("error%d.txt" % r)).read()) for r in (0, 1)
                         if (tmp_path / ("error%d.txt" % r)).exists())
        pytest.fail("%s\n%s" % (failed, errs))
    single = np.load(tmp_path / "single.npz")
    for name in ("even", "uneven", "empty"):
        got = np.load(tmp_path / (name + ".npz"))
        assert sorted(got.files) == sorted(single.files)
        for k in single.files:
            assert np.array_equal(got[k].view(np.uint8), single[k].view(np.uint8)), "%s shards: %s" % (name, k)
    assert (single["is_leaf"] == 0).sum() > 20
    assert [float(np.load(tmp_path / ("refused%d.npy" % r))[0]) for r in (0, 1)] == [1.0, 1.0]
