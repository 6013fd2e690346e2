"""Two-rank runs for the tests that prove a result is identical for any world size: `run` starts two ranks under one
process group, runs a test's body in each and returns both results.  A failing rank's traceback, or where each rank sits
when the deadline passes, ends up in the test's failure message, and no rank outlives the call."""
import faulthandler
import multiprocessing
import multiprocessing.connection
import os
import pickle
import socket
import time
import traceback

import pytest
import torch
import torch.distributed as dist

two_gpus = pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")


def free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def block(rank, cut, n):
    """rank 0 holds the global rows [0, cut), rank 1 the rows [cut, n)"""
    return (0, cut) if rank == 0 else (cut, n)


def SPLITS(n):
    """name -> rank 0's row count: even and uneven shards, a shard shorter than one 4096-row chunk first or last, and an
    empty last or first shard"""
    return {"even": n // 2, "uneven": 11000, "short_first": 2500, "short_last": n - 2000, "empty_last": n, "empty_first": 0}


def _rank(rank, port, out, deadline, mode, body, args):
    # dumped shortly before the parent gives up, so that a hang says where each rank is stuck
    left = deadline - time.time()
    faulthandler.dump_traceback_later(max(left - 5, left / 2, 0.1), file=open(os.path.join(out, "stack%d.txt" % rank), "w"))
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE="2")
    dev = torch.device("cpu") if mode == "cpu" else torch.device("cuda", rank if mode == "nccl" else 0)
    try:
        try:
            if mode != "cpu":
                torch.cuda.set_device(dev)
            kw = {"device_id": dev} if mode == "nccl" else {}
            dist.init_process_group("nccl" if mode == "nccl" else "gloo", rank=rank, world_size=2, **kw)
            result = body(rank, dist.group.WORLD, dev, *args)
            with open(os.path.join(out, "result%d.pkl" % rank), "wb") as f:
                pickle.dump(result, f)
        finally:
            if dist.is_initialized():
                dist.destroy_process_group()
    except BaseException:
        with open(os.path.join(out, "error%d.txt" % rank), "w") as f:
            f.write(traceback.format_exc())
        raise


def run(tmp_path, body, args=(), mode="gloo", timeout=600):
    """body(rank, group, device, *args) on two spawned ranks -> [rank 0's result, rank 1's result].  body is a
    module-level function and its result is pickled.  mode "cpu": gloo without CUDA; "gloo": both ranks on cuda:0;
    "nccl": rank r on cuda:r.  A rank that fails, or ranks still running after timeout seconds, fail the test."""
    port, deadline = free_port(), time.time() + timeout
    ctx = multiprocessing.get_context("spawn")
    procs = [ctx.Process(target=_rank, args=(r, port, str(tmp_path), deadline, mode, body, args)) for r in (0, 1)]
    try:
        for p in procs:
            p.start()
        while True:
            codes = [p.exitcode for p in procs]
            if codes == [0, 0]:
                return [pickle.loads((tmp_path / ("result%d.pkl" % r)).read_bytes()) for r in (0, 1)]
            failed = any(c not in (None, 0) for c in codes)
            if failed or time.time() > deadline:
                break
            multiprocessing.connection.wait([p.sentinel for p in procs if p.exitcode is None], timeout=1)
        msg = ["%s (exit codes %s)" % ("worker failed" if failed else "workers hung", codes)]
        for r in (0, 1):
            err, stack = tmp_path / ("error%d.txt" % r), tmp_path / ("stack%d.txt" % r)
            if err.exists():
                msg.append("--- rank %d\n%s" % (r, err.read_text()))
            if not failed and codes[r] is None and stack.exists():
                msg.append("--- rank %d stack\n%s" % (r, stack.read_text()[-3000:]))
        pytest.fail("\n".join(msg))
    finally:
        for p in procs:
            if p.pid is not None:
                p.kill()
                p.join()
