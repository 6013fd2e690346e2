"""BisectingKMeans (Spark 3's top-down divisive k-means) on the device (DESIGN.md §5t).

Each level divides the largest divisible leaf clusters in two.  Rows of a dividing cluster re-pick between its two
children on csrc/bisecting_kmeans.cu's assign kernel (exact squared distances summed in feature order, no FMA, ties to the
left child); the children's sizes, sums and costs are kmeans.grouped_sum totals, so every decision (divisibility, the
top-m choice, children that receive no row, the end of the loop) is taken from totals that are the same bits on every
rank.  The split noise is a host Philox keyed by the cluster's heap index.  transform / computeCost walk the cluster tree
on the predict kernel.  The model is the same bits for any world size and the same bits as tests/bisecting_kmeans_oracle.py.

Deviations from Spark: a cluster's cost is the exact two-pass sum of squared distances to its center (not
Σ‖x‖² − n‖c‖²); children are compared on squared distances (not their square roots); among equally large divisible clusters
the smaller heap index is kept (not hash-map order); the split noise comes from Philox, not one java.util.Random.
"""
import math

import numpy as np
import torch

from . import _lib
from . import dist as bdist
from ._lib import call, ptr
from .kmeans import MAX_GROUPS, _check_x, _Shards, _sum1, assign, grouped_sum, philox, uniform

PURPOSE_BKMS = 0x424B4D53     # split noise: ctr = (heap_lo, heap_hi, feature, 0)
MAX_K = MAX_GROUPS // 2       # one level's 2·m children are the groups of one grouped sum
LEVEL_LIMIT = 63              # Spark's LEVEL_LIMIT: heap indices stay below 2^63
EPSILON = 2.0 ** -52          # MLUtils.EPSILON
_M32 = 0xFFFFFFFF


def split_centers(center, heap, seed):
    """(left, right) = center ∓ ℓ·z, ℓ = 1e-4·‖center‖₂ (summed in feature order), z_j a standard normal by Box–Muller
    from Philox(seed, 'BKMS', (heap_lo, heap_hi, j, 0)): u1 = 1 − uniform(w0, w1), u2 = uniform(w2, w3)."""
    D = center.shape[0]
    acc = 0.0
    for v in center:
        acc = acc + float(v) * float(v)
    level = 1e-4 * math.sqrt(acc)
    left, right = np.empty(D), np.empty(D)
    for j in range(D):
        w = philox(seed, PURPOSE_BKMS, heap & _M32, (heap >> 32) & _M32, j, 0)
        u1, u2 = 1.0 - uniform(w[0], w[1]), uniform(w[2], w[3])
        z = math.sqrt(-2.0 * math.log(u1)) * math.cos(2.0 * math.pi * u2)
        left[j] = float(center[j]) + (-level) * z
        right[j] = float(center[j]) + level * z
    return left, right


# ------------------------------------------------------------------------------------------------ kernels
def bkm_assign(x, node, slot_of_node, centers, present, prev=None):
    """(child int32 [n], dist_prev f64 [n] or None): each row of a dividing node picks between its slot's present children
    (b200flow_bkm_assign)."""
    n, D = x.shape
    child = torch.empty(max(n, 1), dtype=torch.int32, device=x.device)
    dp = torch.empty(max(n, 1), dtype=torch.float64, device=x.device) if prev is not None else None
    call("b200flow_bkm_assign", ptr(x), n, D, D, ptr(node), slot_of_node.shape[0], ptr(slot_of_node), ptr(centers),
         centers.shape[0] // 2, ptr(present), ptr(prev), ptr(child), ptr(dp))
    return child[:n], (dp[:n] if dp is not None else None)


class Tree:
    """the cluster tree in depth-first order (node 0 = root, left before right), as Spark's buildTree numbers it: heap
    [N] (Spark's cluster index), left / right [N] (-1 = absent), leaf [N] (the leaf ordinal, -1 for an internal node),
    size int64 [N], center f64 [N, D], cost f64 [N]; the same arrays on the device for the predict kernel."""

    def __init__(self, heap, left, right, leaf, size, center, cost, device):
        self.heap, self.left, self.right, self.leaf = heap, left, right, leaf
        self.size, self.center, self.cost = size, center, cost
        self.d_left = torch.from_numpy(left).to(device)
        self.d_right = torch.from_numpy(right).to(device)
        self.d_leaf = torch.from_numpy(leaf).to(device)
        self.d_center = torch.from_numpy(np.ascontiguousarray(center)).to(device)

    @property
    def num_leaves(self):
        return int((self.leaf >= 0).sum())

    def leaf_nodes(self):
        """node numbers of the leaves in leaf order."""
        return np.nonzero(self.leaf >= 0)[0][np.argsort(self.leaf[self.leaf >= 0])]


def build_tree(clusters, device):
    """Spark's buildTree over {heap index: (size, center, cost)}: a cluster is internal iff its left child exists; it keeps
    the children that exist; leaves are numbered 0.. depth-first, left before right."""
    heap, left, right, leaf = [], [], [], []
    n_leaf = [0]

    def visit(h):
        u = len(heap)
        heap.append(h); left.append(-1); right.append(-1); leaf.append(-1)
        if 2 * h in clusters:
            for c, arr in ((2 * h, left), (2 * h + 1, right)):
                if c in clusters:
                    arr[u] = visit(c)
        else:
            leaf[u] = n_leaf[0]
            n_leaf[0] += 1
        return u

    visit(1)                                               # recursion depth <= LEVEL_LIMIT
    size = np.array([clusters[h][0] for h in heap], np.int64)
    center = np.array([clusters[h][1] for h in heap], np.float64)
    cost = np.array([clusters[h][2] for h in heap], np.float64)
    return Tree(np.array(heap, np.int64), np.array(left, np.int32), np.array(right, np.int32), np.array(leaf, np.int32),
                size, center, cost, device)


def bkm_predict(x, tree):
    """(leaf int32 [n], squared distance f64 [n] to that leaf's center): the walk of Spark's ClusteringTreeNode.predict."""
    x = _check_x(x)
    n, D = x.shape
    out = torch.empty(max(n, 1), dtype=torch.int32, device=x.device)
    d = torch.empty(max(n, 1), dtype=torch.float64, device=x.device)
    call("b200flow_bkm_predict", ptr(x), n, D, D, ptr(tree.d_left), ptr(tree.d_right), ptr(tree.d_leaf), ptr(tree.d_center),
         tree.heap.shape[0], 0, ptr(out), ptr(d))
    return out[:n], d[:n]


class BisectingKMeansResult:
    def __init__(self, tree, training_cost, levels, leaf, dist):
        self.tree, self.training_cost = tree, training_cost
        self.levels = levels                               # levels that divided at least one cluster
        self.leaf, self.dist = leaf, dist                  # the fitted tree's walk of the local rows

    @property
    def centers(self):
        """leaf centers in leaf order, host f64 [num_leaves, D]."""
        return self.tree.center[self.tree.leaf_nodes()]


def bkm_fit(x, k, max_iter=20, min_divisible=1.0, seed=0, row_offset=None, group=None):
    """BisectingKMeans.fit on the rows x [n, D] (this rank's contiguous shard; row_offset = its first global row, default
    from dist.global_offset) -> BisectingKMeansResult."""
    x = _check_x(x)
    k, max_iter, min_divisible = int(k), int(max_iter), float(min_divisible)
    if k < 2:
        raise ValueError("k must be > 1, got %d" % k)
    if k > MAX_K:
        raise _lib.UnsupportedParamError("k must be at most %d on this path, got %d" % (MAX_K, k))
    if max_iter < 1:
        raise ValueError("maxIter must be >= 1, got %d" % max_iter)
    if not min_divisible > 0.0:
        raise ValueError("minDivisibleClusterSize must be > 0, got %r" % min_divisible)
    grp = group if group is not None else bdist.group()
    if row_offset is None:
        row_offset, _ = bdist.global_offset(x.shape[0], x.device, grp)
    sh = _Shards(x.shape[0], row_offset, grp, x.device)
    bad = (~torch.isfinite(x)).any().to(torch.int64).reshape(1)
    if grp is not None:
        bdist.all_reduce_(bad, grp)
    if sh.total == 0 or int(bad.item()):
        raise ValueError("BisectingKMeans needs at least one row and finite features")
    dev, n, D = x.device, sh.total, x.shape[1]

    sums, _ = grouped_sum(x, None, 1, sh)
    root_center = sums[0].cpu().numpy() * (1.0 / float(n))
    _, d = assign(x, torch.from_numpy(root_center.reshape(1, D)).to(dev))
    clusters = {1: (n, root_center, _sum1(d, sh))}        # heap index -> (size, center, cost)
    dense = [1]                                            # dense node number -> heap index
    node = torch.zeros(x.shape[0], dtype=torch.int32, device=dev)
    min_size = math.ceil(min_divisible) if min_divisible >= 1.0 else math.ceil(min_divisible * n)
    active, need, level = [1], k - 1, 1
    while active and need > 0 and level < LEVEL_LIMIT:
        div = [h for h in active if clusters[h][0] >= min_size and clusters[h][2] > EPSILON * clusters[h][0]]
        if len(div) > need:
            div = sorted(div, key=lambda h: (-clusters[h][0], h))[:need]
        if not div:
            break
        div.sort()
        m = len(div)
        index = {h: u for u, h in enumerate(dense)}
        slot = np.full(len(dense), -1, np.int32)
        centers = np.empty((2 * m, D))
        for s, h in enumerate(div):
            slot[index[h]] = s
            centers[2 * s], centers[2 * s + 1] = split_centers(clusters[h][1], h, seed)
        d_slot = torch.from_numpy(slot).to(dev)
        present = np.ones(2 * m, np.uint8)
        counts = None
        for _ in range(max_iter):
            child, _ = bkm_assign(x, node, d_slot, torch.from_numpy(centers).to(dev), torch.from_numpy(present).to(dev))
            sums, cnt = grouped_sum(x, child, 2 * m, sh)
            sums, counts = sums.cpu().numpy(), cnt.cpu().numpy()
            present = (counts > 0).astype(np.uint8)
            for c in np.nonzero(counts)[0]:
                centers[c] = sums[c] * (1.0 / float(counts[c]))
        # the final pass: the rows' new leaves, and the cost of the last refined assignment against its own centers
        new, dist_prev = bkm_assign(x, node, d_slot, torch.from_numpy(centers).to(dev), torch.from_numpy(present).to(dev),
                                    prev=child)
        cost, _ = grouped_sum(dist_prev.reshape(-1, 1), child, 2 * m, sh)
        cost = cost.cpu().numpy()[:, 0]
        lut = np.full(2 * m, -1, np.int32)
        children = []
        for s, h in enumerate(div):
            for c in (2 * s, 2 * s + 1):
                if counts[c]:
                    hc = 2 * h + (c & 1)
                    clusters[hc] = (int(counts[c]), centers[c].copy(), float(cost[c]))
                    lut[c] = len(dense)
                    dense.append(hc)
                    children.append(hc)
        d_lut = torch.from_numpy(lut).to(dev)
        node = torch.where(new >= 0, d_lut[new.clamp(min=0).to(torch.int64)], node)
        active, need, level = children, need - m, level + 1
    tree = build_tree(clusters, dev)
    training_cost = 0.0
    for u in tree.leaf_nodes():
        training_cost = training_cost + float(tree.cost[u])
    leaf, dist = bkm_predict(x, tree)
    return BisectingKMeansResult(tree, training_cost, level - 1, leaf, dist)


def compute_cost(x, tree, row_offset=None, group=None):
    """Σ over the rows of the squared distance to the leaf the walk reaches, a grouped sum (the same bits for any world
    size)."""
    x = _check_x(x)
    grp = group if group is not None else bdist.group()
    if row_offset is None:
        row_offset, _ = bdist.global_offset(x.shape[0], x.device, grp)
    sh = _Shards(x.shape[0], row_offset, grp, x.device)
    _, d = bkm_predict(x, tree)
    return _sum1(d, sh)


def cluster_sizes(leaf, k, group=None):
    """int64 [k]: the rows per leaf ordinal, zeros for ordinals the tree lacks (all-reduced over ranks)."""
    grp = group if group is not None else bdist.group()
    sizes = torch.bincount(leaf.to(torch.int64), minlength=k)[:k]
    if grp is not None:
        bdist.all_reduce_(sizes, grp)
    return sizes.cpu().numpy()
