"""Row sharding over ranks (one process per GPU, torch.distributed): SURVEY.md §8(e).

Rows are independent units; rank r holds a contiguous block of the global row range.  The only
data-path collective of the trainer is the per-level histogram all-reduce (forest.fit_forest); the fit-time
one-offs (category counts, moments, the findSplits sample, confusion counts) are tiny all-reduces/all-gathers.
Works with the NCCL backend on GPUs and with gloo on CPU tensors (used by the CPU tests).

The chunk-order sums (KMeans' grouped sums, the MLP's loss and gradient) share one layout, Shards: global rows are cut
into 4096-row chunks, a chunk's partial is computed from that chunk's rows alone, and the total is the sequential sum of
the partials in chunk order.  A chunk that straddles shards is computed by the rank holding its first row (chunk_tail
collects the later ranks' leading rows), and the running totals pass rank to rank (chunk_chain), so the totals are the
same bits for any world size."""
import torch
import torch.distributed as dist

from ._lib import call, ptr

CHUNK = 4096


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


class Shards:
    """the global row layout: every rank's (first global row, row count), gathered once per fit."""

    def __init__(self, n, row_offset, grp, device):
        self.grp = grp
        if grp is None:
            self.rank, self.offs, self.ns = 0, [int(row_offset)], [int(n)]
        else:
            self.rank = dist.get_rank(grp)
            parts = all_gather_list(torch.tensor([int(row_offset), int(n)], dtype=torch.int64, device=device), grp)
            self.offs = [int(p[0]) for p in parts]
            self.ns = [int(p[1]) for p in parts]
        self.total = sum(self.ns)
        # rows at the head of a shard that belong to a chunk starting on an earlier rank
        self.lead = [min(m, (-o) % CHUNK) for o, m in zip(self.offs, self.ns)]
        self.owner = [self._holder(CHUNK * (o // CHUNK)) if ld else -1 for o, ld in zip(self.offs, self.lead)]

    def _holder(self, row):
        return next(r for r, (o, m) in enumerate(zip(self.offs, self.ns)) if o <= row < o + m)


def chunk_tail(values, ids, sh):
    """(t0, tail values, tail ids) of this rank's rows values [n, W] / ids [n] (ids may be None): t0 is the first local
    row of its trailing, possibly straddling chunk, and the tail is rows [t0, n) followed by the leading rows of the later
    ranks whose chunk starts here (sent as f64; the ids as f64 too, back to int32).  Collective when any shard has leading
    rows.  Rows [lead, t0) are whole chunks."""
    n, W = values.shape
    rank, grp = sh.rank, sh.grp
    lead = sh.lead[rank]
    t0 = lead + max(n - lead, 0) // CHUNK * CHUNK
    tail_v, tail_i = values[t0:], (ids[t0:] if ids is not None else None)
    if grp is not None and any(sh.lead):                   # the owner of a straddling chunk collects the rows of later ranks
        buf = torch.zeros((CHUNK - 1, W + 1), dtype=torch.float64, device=values.device)
        buf[:lead, :W] = values[:lead]
        if ids is not None:
            buf[:lead, W] = ids[:lead].to(torch.float64)
        parts = all_gather_list(buf, grp)
        extra = [parts[s][:sh.lead[s]] for s in range(len(parts)) if sh.owner[s] == rank]
        if extra:
            ex = torch.cat(extra)
            tail_v = torch.cat([tail_v.to(torch.float64), ex[:, :W]]).contiguous()
            tail_i = torch.cat([tail_i, ex[:, W].to(torch.int32)]).contiguous() if ids is not None else None
    return t0, tail_v, tail_i


def chunk_chain(partials, n_chunks, G, W, sh, more=()):
    """totals [G, W] f64: the running totals received from the previous rank (+0.0 on rank 0), plus this rank's
    partials [n_chunks, G, W] added in chunk order (b200flow_group_sums_chain), sent on to the next rank; the last rank's
    totals are broadcast, so every rank returns the same bits.  `more` yields further (partials, n_chunks) batches, the
    chunks that follow in order; each is added before the next is drawn, so a rank need not hold all its partials at once."""
    totals = torch.zeros((G, W), dtype=torch.float64, device=partials.device)
    rank, grp = sh.rank, sh.grp
    world = len(sh.ns)
    if grp is not None and rank > 0:
        recv_(totals, rank - 1, grp)
    call("b200flow_group_sums_chain", ptr(partials), n_chunks, G, W, ptr(totals))
    for p, n in more:
        call("b200flow_group_sums_chain", ptr(p), n, G, W, ptr(totals))
    if grp is not None:
        if rank < world - 1:
            send(totals, rank + 1, grp)
        broadcast_(totals, world - 1, grp)
    return totals
