"""The two-rank harness itself, on the CPU (gloo, no device): both ranks' results come back, a rank that raises fails the
test with its traceback, and ranks still running at the deadline fail it with their stacks.  No rank outlives the call."""
import multiprocessing
import time

import pytest
import torch

from ranks import run


def _sum(rank, grp, dev):
    import torch.distributed as dist
    t = torch.tensor([rank + 1.0], device=dev)
    dist.all_reduce(t, group=grp)
    return rank, float(t)


def test_both_ranks_return(tmp_path):
    assert run(tmp_path, _sum, mode="cpu", timeout=120) == [(0, 3.0), (1, 3.0)]


def _raise_on_rank_1(rank, grp, dev):
    if rank == 1:
        raise ValueError("rank 1 refuses")
    return rank


def test_a_rank_that_raises_fails_the_run(tmp_path):
    with pytest.raises(pytest.fail.Exception) as e:
        run(tmp_path, _raise_on_rank_1, mode="cpu", timeout=120)
    msg = str(e.value)
    assert msg.startswith("worker failed") and "--- rank 1\nTraceback" in msg and "ValueError: rank 1 refuses" in msg
    assert multiprocessing.active_children() == []


def _sleep_on_rank_1(rank, grp, dev):
    if rank == 1:
        time.sleep(120)
    return rank


def test_ranks_past_the_deadline_fail_the_run(tmp_path):
    start = time.time()
    with pytest.raises(pytest.fail.Exception) as e:
        run(tmp_path, _sleep_on_rank_1, mode="cpu", timeout=10)
    msg = str(e.value)
    assert msg.startswith("workers hung") and "--- rank 1 stack" in msg and "in _sleep_on_rank_1" in msg
    assert multiprocessing.active_children() == [] and time.time() - start < 60
