"""OneVsRest(GBTClassifier)'s class-batched trainer with rows sharded over TWO RANKS ON ONE GPU (gloo): both processes run the
real kernels on cuda:0.  Even shards on the dense path, uneven and empty shards on the fused record path; every class's
model must be byte-identical to the single-process one, and a label beyond the class count on one rank makes both refuse."""
import os
import socket
import time
import traceback

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

K = 5


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _exports(model):
    return {"%d_%s" % (k, key): v for k, m in enumerate(model.models) for key, v in m.export().items()}


def _worker(rank, world, port, out_dir):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from b200flow import dist as bdist, encode as enc, gbt as bg, synth
        dev = torch.device("cuda", 0)
        n = 24000
        rec, dicts = synth.make_kdd(n, K, seed=31, device=dev)              # identical global data in both ranks
        schema = synth.kdd_schema()
        grp = bdist.group()
        luts, ordered = {}, {}
        lo, hi = bdist.shard_bounds(n, rank, world)
        for c in synth.KDD_CATEGORICAL + ["label"]:
            cnt = bdist.all_reduce_sum_(enc.category_counts(rec[lo:hi].contiguous(), schema, c, len(dicts[c]))).cpu().numpy()
            ordered[c], luts[c] = enc.string_index_order(cnt, dicts[c])
        assert len(ordered["label"]) == K
        plan = enc.EncodePlan(schema)
        for c in synth.KDD_COLUMNS:
            if c not in synth.KDD_CATEGORICAL and c != "label":
                plan.add_numeric(c)
        for c in synth.KDD_CATEGORICAL:
            plan.add_index(c, luts[c])
        plan.set_label("label", luts["label"])
        arity = [0] * 38 + [len(ordered[c]) for c in synth.KDD_CATEGORICAL]
        p = bg.GBTParams(max_iter=4, max_depth=5, max_bins=70, subsampling_rate=0.8, feature_subset_strategy="sqrt", seed=2019)
        out = {}
        for name, (a, b) in (("even", (lo, hi)), ("uneven", (0, 9000) if rank == 0 else (9000, n)), ("empty", (0, n) if rank == 0 else (n, n))):
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
            refused = np.zeros(1)
        except ValueError:
            refused = np.ones(1)
        np.save(os.path.join(out_dir, "refused%d.npy" % rank), refused)
        if rank == 0:
            for name, ex in out.items():
                np.savez(os.path.join(out_dir, name + ".npz"), **ex)
            np.savez(os.path.join(out_dir, "single.npz"), **_exports(bg.fit_gbt_ovr_records(rec, plan, K, arity, p)))
        open(os.path.join(out_dir, "ok%d" % rank), "w").write("ok")
    except Exception:
        open(os.path.join(out_dir, "error%d.txt" % rank), "w").write(traceback.format_exc())
        raise
    finally:
        try:
            dist.destroy_process_group()
        except Exception:
            pass


def test_two_ranks_one_gpu_ovr_equals_single_process(tmp_path):
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
    for k in range(K):
        assert (single["%d_is_leaf" % k] == 0).sum() > 4
    assert [float(np.load(tmp_path / ("refused%d.npy" % r))[0]) for r in (0, 1)] == [1.0, 1.0]
