"""numpy restatement of BisectingKMeans (b200flow/bisecting_kmeans.py, DESIGN.md §5t).

Written from the contract, not from the product: Spark 3's BisectingKMeans.run loop (divisible clusters, the top-m choice,
maxIter refinement passes, the final assignment), splitCenter with Philox Box–Muller noise, buildTree and
ClusteringTreeNode.predict, as plain loops.  Distances, grouped sums and Philox come from tests/kmeans_oracle.py; nothing
is imported from b200flow."""
import math

import numpy as np

import kmeans_oracle as ko

BKMS = 0x424B4D53
LEVEL_LIMIT = 63
EPS = 2.0 ** -52


def split(center, heap, seed):
    """(left, right) = center + (∓ℓ)·z, ℓ = 1e-4·sqrt(Σ c_j² in feature order), z_j by Box–Muller from Philox(seed, BKMS,
    (heap_lo, heap_hi, j, 0)) with u1 = 1 − u(w0, w1), u2 = u(w2, w3)."""
    D = center.shape[0]
    s = 0.0
    for v in center:
        s = s + float(v) * float(v)
    ell = 1e-4 * math.sqrt(s)
    j = np.arange(D, dtype=np.uint64)
    w = ko.philox(seed, BKMS, heap & 0xFFFFFFFF, heap >> 32, j, 0)
    ua, ub = ko.uniforms(w[0], w[1]), ko.uniforms(w[2], w[3])
    z = np.array([math.sqrt(-2.0 * math.log(1.0 - float(a))) * math.cos(2.0 * math.pi * float(b)) for a, b in zip(ua, ub)])
    return center + (-ell) * z, center + ell * z


def pair_assign(x, node, slot, centers, present, prev=None):
    """the assign kernel: child [n] (2s / 2s+1 / -1) and, with prev, dist_prev [n]."""
    n = x.shape[0]
    child = np.full(n, -1, np.int32)
    dprev = np.zeros(n)
    keys = np.array(sorted(slot), np.int64)
    pos = np.minimum(np.searchsorted(keys, node), keys.shape[0] - 1)
    s_row = np.where(keys[pos] == node, np.array([slot[h] for h in keys], np.int64)[pos], -1)
    for s in np.unique(s_row[s_row >= 0]):
        rows = np.nonzero(s_row == s)[0]
        dd = ko.sqdist(x[rows], centers[2 * s:2 * s + 2])
        pl, pr = bool(present[2 * s]), bool(present[2 * s + 1])
        go_right = pr & ((not pl) | (dd[:, 1] < dd[:, 0]))
        ch = np.where(go_right, 2 * s + 1, 2 * s)
        if not pl and not pr:
            ch[:] = -1
        child[rows] = ch
        if prev is not None:
            p = prev[rows]
            dprev[rows] = np.where(p == 2 * s, dd[:, 0], np.where(p == 2 * s + 1, dd[:, 1], 0.0))
    return child, dprev


def fit(x, k, max_iter=20, min_divisible=1.0, seed=0):
    """-> dict(clusters {heap: (size, center, cost)}, tree, training_cost, levels)."""
    n, D = x.shape
    root = ko.group_sums(x, None, 1)[0][0] * (1.0 / n)
    cost = ko.group_sums(ko.assign(x, root[None, :])[1][:, None], None, 1)[0][0, 0]
    clusters = {1: (n, root, float(cost))}
    node = np.ones(n, np.int64)                            # the row's cluster, by heap index
    min_size = math.ceil(min_divisible) if min_divisible >= 1.0 else math.ceil(min_divisible * n)
    active, need, level, levels = [1], k - 1, 1, 0
    while active and need > 0 and level < LEVEL_LIMIT:
        div = [h for h in active if clusters[h][0] >= min_size and clusters[h][2] > EPS * clusters[h][0]]
        if len(div) > need:
            div = sorted(div, key=lambda h: (-clusters[h][0], h))[:need]
        if not div:
            break
        div = sorted(div)
        m = len(div)
        slot = {h: s for s, h in enumerate(div)}
        centers = np.vstack([np.vstack(split(clusters[h][1], h, seed)) for h in div])
        present = np.ones(2 * m, bool)
        for _ in range(max_iter):
            child, _ = pair_assign(x, node, slot, centers, present)
            sums, counts = ko.group_sums(x, np.where(child >= 0, child, 2 * m), 2 * m + 1)
            present = counts[:2 * m] > 0
            for c in np.nonzero(present)[0]:
                centers[c] = sums[c] * (1.0 / float(counts[c]))
        new, dprev = pair_assign(x, node, slot, centers, present, prev=child)
        csum = ko.group_sums(dprev[:, None], np.where(child >= 0, child, 2 * m), 2 * m + 1)[0][:, 0]
        children = []
        for s, h in enumerate(div):
            for c in (2 * s, 2 * s + 1):
                if present[c]:
                    clusters[2 * h + (c & 1)] = (int(counts[c]), centers[c].copy(), float(csum[c]))
                    children.append(2 * h + (c & 1))
        heap_of_child = np.array([2 * div[c // 2] + (c & 1) for c in range(2 * m)], np.int64)
        node = np.where(new >= 0, heap_of_child[np.maximum(new, 0)], node)
        active, need, level, levels = children, need - m, level + 1, levels + 1
    tree = build_tree(clusters)
    tc = 0.0
    for u in tree["leaf_order"]:
        tc = tc + tree["cost"][u]
    return {"clusters": clusters, "tree": tree, "training_cost": tc, "levels": levels}


def build_tree(clusters):
    """Spark's buildTree: internal iff the left child exists; existing children only; DFS leaf numbering."""
    t = {"heap": [], "left": [], "right": [], "leaf": []}
    count = [0]

    def visit(h):
        u = len(t["heap"])
        t["heap"].append(h); t["left"].append(-1); t["right"].append(-1); t["leaf"].append(-1)
        if 2 * h in clusters:
            t["left"][u] = visit(2 * h)
            if 2 * h + 1 in clusters:
                t["right"][u] = visit(2 * h + 1)
        else:
            t["leaf"][u] = count[0]
            count[0] += 1
        return u

    visit(1)
    out = {key: np.array(v, np.int64 if key == "heap" else np.int32) for key, v in t.items()}
    out["size"] = np.array([clusters[h][0] for h in t["heap"]], np.int64)
    out["center"] = np.array([clusters[h][1] for h in t["heap"]])
    out["cost"] = np.array([clusters[h][2] for h in t["heap"]])
    leaves = [u for u in range(len(t["heap"])) if t["leaf"][u] >= 0]
    out["leaf_order"] = sorted(leaves, key=lambda u: t["leaf"][u])
    return out


def _paired(a, c):
    """squared distance of row i of a to row i of c, summed in feature order from 0.0."""
    acc = np.zeros(a.shape[0])
    for j in range(a.shape[1]):
        t = a[:, j] - c[:, j]
        acc = acc + t * t
    return acc


def predict(x, left, right, leaf, center, root=0):
    """ClusteringTreeNode.predict for every row: (leaf ordinal [n], squared distance to that leaf's center [n]).  At an
    internal node the row goes to the existing child with the smaller distance, a tie to the first (left) one."""
    n = x.shape[0]
    left, right, leaf = np.asarray(left), np.asarray(right), np.asarray(leaf)
    u = np.full(n, root, np.int64)
    d = ko.sqdist(x, center[root:root + 1])[:, 0] if leaf[root] >= 0 else np.zeros(n)
    for _ in range(LEVEL_LIMIT):
        idx = np.nonzero(leaf[u] < 0)[0]
        if idx.size == 0:
            break
        a, b = left[u[idx]], right[u[idx]]
        da = np.where(a >= 0, _paired(x[idx], center[np.maximum(a, 0)]), np.inf)
        db = np.where(b >= 0, _paired(x[idx], center[np.maximum(b, 0)]), np.inf)
        take_a = (a >= 0) & ((b < 0) | (da <= db))
        u[idx] = np.where(take_a, a, b)
        d[idx] = np.where(take_a, da, db)
    return leaf[u].astype(np.int32), d


def predict_tree(x, tree):
    return predict(x, tree["left"], tree["right"], tree["leaf"], tree["center"])


def compute_cost(x, tree):
    return float(ko.group_sums(predict_tree(x, tree)[1][:, None], None, 1)[0][0, 0])
