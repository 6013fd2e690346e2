"""Row sharding over ranks (one process per GPU, torch.distributed): SURVEY.md §8(e).

Rows are independent units; rank r holds a contiguous block of the global row range.  The only
data-path collective of the trainer is the per-level histogram all-reduce (forest.fit_forest); the fit-time
one-offs (category counts, moments, the findSplits sample, confusion counts) are tiny all-reduces/all-gathers.
Works with the NCCL backend on GPUs and with gloo on CPU tensors (used by the CPU tests)."""
import torch
import torch.distributed as dist


def group():
    """the default process group when running under torchrun with world_size > 1, else None."""
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        return dist.group.WORLD
    return None


def shard_bounds(n_total, rank, world):
    """contiguous block partition: rank r owns rows [r*n/G, (r+1)*n/G)."""
    return (n_total * rank) // world, (n_total * (rank + 1)) // world


def global_offset(n_local, device, grp=None):
    """(first global row index of this rank's block, global row count) from the local counts."""
    grp = grp if grp is not None else group()
    if grp is None:
        return 0, int(n_local)
    world, rank = dist.get_world_size(grp), dist.get_rank(grp)
    counts = [int(c.item()) for c in all_gather_list(torch.tensor([int(n_local)], dtype=torch.int64, device=device), grp)]
    return sum(counts[:rank]), sum(counts)


def _staged(t, grp):
    """gloo moves CUDA tensors only for broadcast / all_reduce: everything else (and, for uniformity, those two) is staged
    through host memory when the group is gloo — the 2-ranks-on-one-GPU tests run the real kernels over a gloo group."""
    return t.is_cuda and dist.get_backend(grp) == "gloo"


def is_nccl(grp):
    return grp is not None and dist.get_backend(grp) == "nccl"


def all_reduce_(t, grp, op=None):
    """in-place all-reduce (sum by default) on whatever backend the group has."""
    op = dist.ReduceOp.SUM if op is None else op
    if _staged(t, grp):
        c = t.cpu()
        dist.all_reduce(c, op=op, group=grp)
        t.copy_(c)
    else:
        dist.all_reduce(t, op=op, group=grp)
    return t


def all_gather_list(t, grp):
    """equal-shape all-gather -> list of tensors (one per rank) on t's device."""
    world = dist.get_world_size(grp)
    if _staged(t, grp):
        c = t.cpu()
        parts = [torch.empty_like(c) for _ in range(world)]
        dist.all_gather(parts, c, group=grp)
        return [p.to(t.device) for p in parts]
    parts = [torch.empty_like(t) for _ in range(world)]
    dist.all_gather(parts, t, group=grp)
    return parts


def send(t, dst, grp):
    """point-to-point send to group rank dst (staged through host memory under gloo)."""
    d = dist.get_global_rank(grp, dst)
    dist.send(t.cpu() if _staged(t, grp) else t, dst=d, group=grp)


def recv_(t, src, grp):
    """point-to-point receive from group rank src into t, in place."""
    s = dist.get_global_rank(grp, src)
    if _staged(t, grp):
        c = t.cpu()
        dist.recv(c, src=s, group=grp)
        t.copy_(c)
    else:
        dist.recv(t, src=s, group=grp)
    return t


def broadcast_(t, src, grp):
    """in-place broadcast from group rank src."""
    s = dist.get_global_rank(grp, src)
    if _staged(t, grp):
        c = t.cpu()
        dist.broadcast(c, src=s, group=grp)
        t.copy_(c)
    else:
        dist.broadcast(t, src=s, group=grp)
    return t


def all_reduce_sum_(t, grp=None):
    """in-place sum over ranks (integer tensors stay exact -> bit-identical models for any world size)."""
    grp = grp if grp is not None else group()
    if grp is not None:
        all_reduce_(t, grp)
    return t
