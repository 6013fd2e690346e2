"""KMeans (k-means|| or random init, then Lloyd) and the silhouette on the device (DESIGN.md §5c).

Distances come from csrc/kmeans.cu's assign kernel (exact squared distances summed in feature order, no FMA).  Every sum
that decides the model (center sums, costs, silhouette statistics and mean) is one grouped sum with a fixed rounding order:
global rows are cut into 4096-row chunks, a chunk's partial is the sequential sum of its member rows, and the total is the
sequential sum of the partials in chunk order.  Under torch.distributed the rows are contiguous shards; a chunk that
straddles shards is summed by the rank holding its first row, and the running totals pass rank to rank.  So the centers,
the costs and the silhouette are the same bits for any world size, and the same bits as a numpy restatement.
"""
import numpy as np
import torch

from . import _lib
from . import dist as bdist
from ._lib import call, ptr

CHUNK = bdist.CHUNK
_Shards = bdist.Shards
MAX_D = 256            # kmeans_assign stages a row tile and a center tile of every feature in shared memory
MAX_GROUPS = 4096      # group_sums counting-sorts a chunk by group in shared memory
PURPOSE_KMNS = 0x4B4D4E53
PURPOSE_KMPP = 0x4B4D5050
_M32 = 0xFFFFFFFF


# ------------------------------------------------------------------------------------------------ host Philox
def philox(seed, purpose, c0, c1=0, c2=0, c3=0):
    """Philox4x32-10 of the device (csrc/common.cuh): key (lo32(seed) ^ purpose, hi32(seed)) -> 4 words."""
    k0, k1 = (int(seed) & _M32) ^ purpose, (int(seed) >> 32) & _M32
    c = [c0 & _M32, c1 & _M32, c2 & _M32, c3 & _M32]
    for _ in range(10):
        p0, p1 = 0xD2511F53 * c[0], 0xCD9E8D57 * c[2]
        c = [(p1 >> 32) ^ c[1] ^ k0, p1 & _M32, (p0 >> 32) ^ c[3] ^ k1, p0 & _M32]
        k0, k1 = (k0 + 0x9E3779B9) & _M32, (k1 + 0xBB67AE85) & _M32
    return c


def uniform(w0, w1):
    """the 53-bit uniform in [0, 1) of two Philox words."""
    return float((w0 << 21) | (w1 >> 11)) * 2.0 ** -53


def row_key(seed, row):
    """the step-0 key of a global row, as kmeans_row_keys writes it (int64, top bit flipped: signed order = key order)."""
    w = philox(seed, PURPOSE_KMNS, row, row >> 32)
    v = ((w[0] << 32) | w[1]) ^ (1 << 63)
    return v - (1 << 64) if v >> 63 else v


class _Draws:
    """the host-side stream of local k-means++: draw i = uniform of Philox(seed, 'KMPP', (i_lo, i_hi, 0, 0))."""

    def __init__(self, seed):
        self.seed, self.i = int(seed), 0

    def next(self):
        w = philox(self.seed, PURPOSE_KMPP, self.i, self.i >> 32)
        self.i += 1
        return uniform(w[0], w[1])


# ------------------------------------------------------------------------------------------------ kernels
def assign(x, centers):
    """(cluster int32 [n], squared distance f64 [n]) of every row of x [n, D] to its first nearest center."""
    n, D = x.shape
    cl = torch.empty(max(n, 1), dtype=torch.int32, device=x.device)
    d = torch.empty(max(n, 1), dtype=torch.float64, device=x.device)
    call("b200flow_kmeans_assign", ptr(x), n, D, D, ptr(centers), centers.shape[0], ptr(cl), ptr(d))
    return cl[:n], d[:n]


def grouped_sum(values, ids, G, sh):
    """(totals f64 [G, W], counts int64 [G]) of values [n, W] f64 grouped by ids int32 [n] (None: one group), summed in the
    fixed chunk order of the module docstring; the same bits on every rank."""
    n, W = values.shape
    dev = values.device
    values = values.contiguous()
    off, lead = sh.offs[sh.rank], sh.lead[sh.rank]
    t0, tail_v, tail_i = bdist.chunk_tail(values, ids, sh)
    nfull = (t0 - lead) // CHUNK
    n_tail = tail_v.shape[0]
    n_chunks = nfull + (1 if n_tail else 0)
    partials = torch.empty((max(n_chunks, 1), G, W), dtype=torch.float64, device=dev)
    counts = torch.zeros(G, dtype=torch.int64, device=dev)
    if nfull:
        call("b200flow_group_sums", ptr(values[lead:t0]), W, ptr(ids[lead:t0]) if ids is not None else None, t0 - lead, W, G,
             off + lead, ptr(partials), ptr(counts))
    if n_tail:
        call("b200flow_group_sums", ptr(tail_v), W, ptr(tail_i) if ids is not None else None, n_tail, W, G, off + t0,
             ptr(partials[nfull:]), ptr(counts))
    totals = bdist.chunk_chain(partials, n_chunks, G, W, sh)
    if sh.grp is not None:
        bdist.all_reduce_(counts, sh.grp)
    return totals, counts


def _sum1(v, sh):
    """the grouped sum of one column with one group, as a float."""
    return float(grouped_sum(v.reshape(-1, 1), None, 1, sh)[0].item())


def _sqdist(a, b):
    """host squared distances with the kernel's rounding: rows of a [m, D] against b [D] or [m, D]."""
    acc = np.zeros(a.shape[0])
    for j in range(a.shape[1]):
        t = a[:, j] - b[..., j]
        acc = acc + t * t
    return acc


def _distinct_rows(rows):
    """rows de-duplicated by their exact bytes, first occurrence kept, in order."""
    seen, keep = set(), []
    for i, r in enumerate(rows):
        b = r.tobytes()
        if b not in seen:
            seen.add(b)
            keep.append(i)
    return rows[keep]


def _gather_rows(rows, sh):
    """every rank's rows [m_r, D] concatenated in rank order (= global row order), as a host array."""
    if sh.grp is None:
        return rows.cpu().numpy()
    D = rows.shape[1]
    m = torch.tensor([rows.shape[0]], dtype=torch.int64, device=rows.device)
    import torch.distributed as dist
    mx = m.clone()
    bdist.all_reduce_(mx, sh.grp, op=dist.ReduceOp.MAX)
    cap = max(int(mx.item()), 1)
    buf = torch.zeros((cap, D), dtype=torch.float64, device=rows.device)
    buf[:rows.shape[0]] = rows
    counts = [int(c.item()) for c in bdist.all_gather_list(m, sh.grp)]
    parts = bdist.all_gather_list(buf, sh.grp)
    return torch.cat([p[:c] for p, c in zip(parts, counts)]).cpu().numpy()


def _smallest_keys(x, seed, sh, k):
    """the rows of the k smallest step-0 keys (ties: lower global row), in key order, as a host array."""
    n = x.shape[0]
    keys = torch.empty(max(n, 1), dtype=torch.int64, device=x.device)
    call("b200flow_kmeans_row_keys", int(seed) & 0xFFFFFFFFFFFFFFFF, sh.offs[sh.rank], n, ptr(keys))
    keys = keys[:n]
    m = min(k, n)
    kk, order = torch.sort(keys, stable=True)              # equal keys keep row order
    kk, order = kk[:m], order[:m]
    rows = x[order]
    grow = order.to(torch.int64) + sh.offs[sh.rank]
    if sh.grp is None:
        return rows.cpu().numpy()
    D = x.shape[1]
    pk = torch.full((k,), 2 ** 63 - 1, dtype=torch.int64, device=x.device); pk[:m] = kk
    pr = torch.full((k,), 2 ** 63 - 1, dtype=torch.int64, device=x.device); pr[:m] = grow
    pv = torch.zeros((k, D), dtype=torch.float64, device=x.device); pv[:m] = rows
    ks = torch.cat(bdist.all_gather_list(pk, sh.grp)).cpu().numpy()
    rs = torch.cat(bdist.all_gather_list(pr, sh.grp)).cpu().numpy()
    vs = torch.cat(bdist.all_gather_list(pv, sh.grp)).cpu().numpy()
    sel = np.lexsort((rs, ks))[:min(k, sh.total)]
    return vs[sel]


def _local_kmeans_pp(points, weights, k, seed, max_iter=30):
    """Spark's LocalKMeans.kMeansPlusPlus over weighted candidates, with the KMPP draws and exact distances (DESIGN §5c)."""
    rnd = _Draws(seed)
    m = points.shape[0]

    def pick(cum, r):
        if not 0.0 < r:
            return 0
        return min(int(np.searchsorted(cum, r, side="left")), m - 1)

    cw = np.add.accumulate(np.concatenate([[0.0], weights]))[1:]
    centers = [points[pick(cw, rnd.next() * cw[-1])]]
    cost = _sqdist(points, centers[0])
    for _ in range(1, k):
        cc = np.add.accumulate(np.concatenate([[0.0], cost * weights]))[1:]
        c = points[pick(cc, rnd.next() * cc[-1])]
        centers.append(c)
        cost = np.minimum(_sqdist(points, c), cost)
    centers = np.array(centers)
    old = np.full(m, -1)
    for _ in range(max_iter):
        dist = np.stack([_sqdist(points, c) for c in centers], axis=1)
        idx = np.argmin(dist, axis=1)
        moved = bool((idx != old).any())
        old = idx
        new = centers.copy()
        for j in range(k):
            mem = np.nonzero(idx == j)[0]
            if mem.size == 0:
                new[j] = points[min(int(rnd.next() * m), m - 1)]
                continue
            s = np.add.accumulate(np.vstack([np.zeros(points.shape[1]), weights[mem, None] * points[mem]]))[-1]
            cnt = np.add.accumulate(np.concatenate([[0.0], weights[mem]]))[-1]
            new[j] = s * (1.0 / cnt)
        centers = new
        if not moved:
            break
    return centers


def _init_parallel(x, k, steps, seed, sh):
    """k-means|| (Spark's initKMeansParallel with the KMNS draws): -> host centers [k' <= k, D]."""
    dev = x.device
    first = _smallest_keys(x, seed, sh, 1)
    cands = [first]
    new = torch.from_numpy(first).to(dev)
    cost = torch.full((x.shape[0],), float("inf"), dtype=torch.float64, device=dev)
    from .rows import compact_many
    for step in range(1, steps + 1):
        if new.shape[0]:
            _, d = assign(x, new)
            cost = torch.minimum(cost, d)
        sum_cost = _sum1(cost, sh)
        flag = torch.empty(max(x.shape[0], 1), dtype=torch.uint8, device=dev)
        call("b200flow_kmeans_select", int(seed) & 0xFFFFFFFFFFFFFFFF, sh.offs[sh.rank], x.shape[0], step, ptr(cost), k,
             sum_cost, ptr(flag))
        (rows,), _ = compact_many([x], flag[:x.shape[0]])
        chosen = _gather_rows(rows, sh)
        cands.append(chosen)
        new = torch.from_numpy(chosen).to(dev)
    cands = _distinct_rows(np.concatenate(cands))
    if cands.shape[0] <= k:
        return cands
    cl, _ = assign(x, torch.from_numpy(cands).to(dev))
    w = torch.bincount(cl.to(torch.int64), minlength=cands.shape[0])
    if sh.grp is not None:
        bdist.all_reduce_(w, sh.grp)
    return _local_kmeans_pp(cands, w.cpu().numpy().astype(np.float64), k, seed)


class KMeansResult:
    def __init__(self, centers, num_iter, training_cost, cluster_sizes, cluster=None, dist=None):
        self.centers, self.num_iter, self.training_cost, self.cluster_sizes = centers, num_iter, training_cost, cluster_sizes
        self.cluster, self.dist = cluster, dist          # the final model's assignment of the local rows


def lloyd(x, centers, max_iter, tol, sh):
    """Lloyd passes from host centers [k, D] (Spark's runAlgorithm with exact distances and the grouped sums)."""
    dev = x.device
    centers = np.array(centers, dtype=np.float64)
    k = centers.shape[0]
    it, converged, cost = 0, False, 0.0
    while it < max_iter and not converged:
        cl, d = assign(x, torch.from_numpy(centers).to(dev))
        cost = _sum1(d, sh)
        sums, counts = grouped_sum(x, cl, k, sh)
        sums, counts = sums.cpu().numpy(), counts.cpu().numpy()
        converged = True
        new = centers.copy()
        for j in np.nonzero(counts)[0]:
            c = sums[j] * (1.0 / float(counts[j]))
            if converged and _sqdist(c[None, :], centers[j])[0] > tol * tol:
                converged = False
            new[j] = c
        centers = new
        it += 1
    ct = torch.from_numpy(centers).to(dev)
    cl, d = assign(x, ct)
    sizes = torch.bincount(cl.to(torch.int64), minlength=k)
    if sh.grp is not None:
        bdist.all_reduce_(sizes, sh.grp)
    return KMeansResult(ct, it, cost, sizes.cpu().numpy(), cl, d)


def _check_x(x):
    if not (torch.is_tensor(x) and x.is_cuda and x.dim() == 2 and x.dtype == torch.float64):
        raise _lib.B200FlowError("kmeans needs a CUDA float64 [n, D] matrix")
    if not 1 <= x.shape[1] <= MAX_D:
        raise _lib.UnsupportedParamError("kmeans supports 1 to %d features, got %d" % (MAX_D, x.shape[1]))
    return x.contiguous()


def kmeans_fit(x, k, init="k-means||", init_steps=2, max_iter=20, tol=1e-4, seed=0, row_offset=None, group=None):
    """KMeans.fit on the rows x [n, D] (this rank's contiguous shard; row_offset = its first global row, default from
    dist.global_offset).  -> KMeansResult(centers [k' <= k, D] f64 device, num_iter, training_cost, cluster_sizes int64)."""
    x = _check_x(x)
    k, init_steps, max_iter = int(k), int(init_steps), int(max_iter)
    if k < 2:
        raise ValueError("k must be > 1, got %d" % k)
    if k > MAX_GROUPS:
        raise _lib.UnsupportedParamError("k must be at most %d on this path, got %d" % (MAX_GROUPS, k))
    if init not in ("k-means||", "random"):
        raise ValueError("initMode must be k-means|| or random, got %r" % (init,))
    if init_steps <= 0 or max_iter < 0 or not tol >= 0:
        raise ValueError("initSteps must be > 0, maxIter >= 0 and tol >= 0")
    grp = group if group is not None else bdist.group()
    if row_offset is None:
        row_offset, _ = bdist.global_offset(x.shape[0], x.device, grp)
    sh = _Shards(x.shape[0], row_offset, grp, x.device)
    bad = (~torch.isfinite(x)).any().to(torch.int64).reshape(1)
    if grp is not None:
        bdist.all_reduce_(bad, grp)
    if sh.total == 0 or int(bad.item()):
        raise ValueError("KMeans needs at least one row and finite features")
    if init == "random":
        centers = _distinct_rows(_smallest_keys(x, seed, sh, k))
    else:
        centers = _init_parallel(x, k, init_steps, seed, sh)
    return lloyd(x, centers, max_iter, float(tol), sh)


def kmeans_predict(x, centers):
    """(cluster int32 [n], squared distance f64 [n]) to the nearest of centers [k, D]; the distance is the anomaly score."""
    x = _check_x(x)
    return assign(x, centers.to(torch.float64).contiguous())


def silhouette(x, cluster, row_offset=None, group=None):
    """mean silhouette coefficient (squared Euclidean) of x [n, D] under the int cluster ids [n], identical for any world
    size.  Raises ValueError when fewer than two clusters are present."""
    x = _check_x(x)
    n, D = x.shape
    grp = group if group is not None else bdist.group()
    if row_offset is None:
        row_offset, _ = bdist.global_offset(n, x.device, grp)
    sh = _Shards(n, row_offset, grp, x.device)
    cl = cluster.to(torch.int32).contiguous()
    mx = torch.stack([cl.max() if n else cl.new_zeros(()), cl.min() if n else cl.new_zeros(())]).to(torch.int64)
    mx[1] = -mx[1]
    if grp is not None:
        import torch.distributed as dist
        bdist.all_reduce_(mx, grp, op=dist.ReduceOp.MAX)
    G, lo = int(mx[0].item()) + 1, -int(mx[1].item())
    if lo < 0 or G > MAX_GROUPS:
        raise ValueError("cluster ids must be integers in [0, %d)" % MAX_GROUPS)
    _, norms = assign(x, torch.zeros((1, D), dtype=torch.float64, device=x.device))     # ||x||^2 summed in feature order
    totals, counts = grouped_sum(torch.cat([x, norms.reshape(-1, 1)], 1), cl, G, sh)
    if int((counts > 0).sum().item()) < 2:
        raise ValueError("Number of clusters must be greater than one.")
    Y, psi = totals[:, :D].contiguous(), totals[:, D].contiguous()
    s = torch.empty(max(n, 1), dtype=torch.float64, device=x.device)
    call("b200flow_silhouette_rows", ptr(x), n, D, D, ptr(norms), ptr(cl), ptr(Y), ptr(psi), ptr(counts), G, ptr(s))
    return _sum1(s[:n], sh) / sh.total
