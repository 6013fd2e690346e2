"""Plain restatement of one level of the forest's level loop (csrc/forest.cu), one function per kernel:

  route_ref  route_hist_level (and partition_level): route every entry of a parent by its split, keep it on the side whose
             child is not a leaf, and add it to that child's histogram over the child's feature subset;
  score_ref  score_level: MLlib's binsToBestSplit over one node's histogram (Gini, first maximum over features in subset
             order, then over splits), with the arithmetic of calculateImpurityStats;
  grow_ref   grow_level: the node pool, masks, counts and the next level's slots of one scored level.

numpy and Python floats only: integer histograms are exact int64, every fp64 sum runs sequentially from 0.0 and nothing is
fused (Python's float ops round once each), so gains equal the kernel's to the bit."""
import numpy as np

from b200flow._lib import NODE_DTYPE, SPLIT_DTYPE

DBL_MAX = float(np.finfo(np.float64).max)


# ------------------------------------------------------------------------------------------------ route_hist_level
def split_goes_left(sp, bins):
    """left-or-right of records whose split feature has the given bins (continuous: bin <= bin_thr; categorical: mask bit)."""
    bins = np.asarray(bins, np.int64)
    if int(sp["kind"]) == 0:
        return bins <= int(sp["bin_thr"])
    mask = np.asarray(sp["mask"], np.uint64)
    words = mask[bins >> 6]
    return ((words >> (bins & 63).astype(np.uint64)) & np.uint64(1)).astype(bool)


def route_ref(bins, labels, ent, seg_begin, seg_end, n_chunks, chunk_rows, split, child_slot, subset_next, n_bins, C,
              n_next):
    """b200flow_route_hist_level on records given as a bin matrix bins [n_rec][F] and labels [n_rec].

    ent [E][2] = {record, weight}; parent s owns ent[seg_begin[s]:seg_end[s]] and its first n_chunks[s] * chunk_rows entries
    are routed (the chunk table of plan_route).  An entry goes left or right by split[s] (feature max(feat, 0)) and is kept
    when child_slot[2 s + side] >= 0.  subset_next [n_next][m] = the children's feature subsets (None: no histograms).
    Returns (hist int64 [n_next][m][n_bins][C] or None, left [n_slots] and right [n_slots] lists of kept {record, weight}
    arrays, cursors int64 [n_slots][2] = their sizes)."""
    bins = np.asarray(bins); labels = np.asarray(labels, np.int64); ent = np.asarray(ent, np.int64)
    n_slots = len(seg_begin)
    hist = None
    if subset_next is not None:
        subset_next = np.asarray(subset_next, np.int64)
        hist = np.zeros((n_next, subset_next.shape[1], n_bins, C), np.int64)
    left, right = [], []
    cursors = np.zeros((n_slots, 2), np.int64)
    for s in range(n_slots):
        b = int(seg_begin[s]); e = min(int(seg_end[s]), b + int(n_chunks[s]) * chunk_rows)
        part = ent[b:max(b, e)]
        sp = split[s]
        go_left = split_goes_left(sp, bins[part[:, 0], max(int(sp["feat"]), 0)])
        kept = []
        for side, sel in ((0, go_left), (1, ~go_left)):
            cs = int(child_slot[2 * s + side])
            if cs < 0:
                kept.append(part[:0]); continue
            mine = part[sel]
            kept.append(mine)
            if hist is not None:
                rec, w, lab = mine[:, 0], mine[:, 1], labels[mine[:, 0]]
                for j in range(subset_next.shape[1]):
                    np.add.at(hist[cs, j], (bins[rec, subset_next[cs, j]].astype(np.int64), lab), w)
        left.append(kept[0]); right.append(kept[1])
        cursors[s] = (len(kept[0]), len(kept[1]))
    return hist, left, right, cursors


# ------------------------------------------------------------------------------------------------ score_level
def gini(counts, tot):
    """Gini.calculate: 1 - sum (c_k / tot)^2 in class order, 0 for an empty node."""
    if tot == 0.0:
        return 0.0
    imp = 1.0
    for c in counts:
        f = float(c) / tot
        imp = imp - f * f
    return imp


def _fsum(values):
    acc = 0.0
    for v in values:
        acc = acc + float(v)
    return acc


def split_gain(L, tot, parent_imp, min_inst, min_gain):
    """calculateImpurityStats for left counts L of a node with class counts tot (ints): the gain, or -DBL_MAX when a child
    has fewer than min_inst instances or the gain is below min_gain."""
    R = [t - l for t, l in zip(tot, L)]
    lc, rc = _fsum(L), _fsum(R)
    if lc < float(min_inst) or rc < float(min_inst):
        return -DBL_MAX
    t = lc + rc
    gl, gr = gini(L, lc), gini(R, rc)
    gain = parent_imp - (lc / t) * gl - (rc / t) * gr
    return -DBL_MAX if gain < min_gain else gain


def score_ref(hist_slot, subset, feat_bins, feat_kind, level, max_depth, min_instances, min_info_gain):
    """b200flow_score_level for one slot: hist_slot [m][n_bins][C] integer counts over subset[j].  The node's class counts
    are the first subset feature's counts summed over its bins.  Candidates, in MLlib's scan order (subset position, split):
      continuous (kind 0)            split s < nb - 1: left = bins 0..s;
      ordered categorical (kind 1)   categories ranked by centroid (multiclass: the category's Gini, binary: its class-1
                                     count; empty categories last; stable), split s < nb - 1: left = the first s + 1 ranked;
      unordered categorical (kind 2) split s < 2^(nb-1) - 1: left = the categories whose bit is set in s + 1.
    Returns (split record SPLIT_DTYPE, node counts, left counts, right counts) — children's counts are those of the best
    valid candidate even when the node stays a leaf, zero when there is none."""
    h = np.asarray(hist_slot, np.int64)
    m, _, C = h.shape
    nb0 = int(feat_bins[int(subset[0])])
    tot = [int(v) for v in h[0, :nb0].sum(0)]
    parent_imp = gini(tot, _fsum(tot))
    best = None                                     # (gain, j, s, kind, L, mask)
    for j in range(m):
        f = int(subset[j]); nb, kind = int(feat_bins[f]), int(feat_kind[f])
        hj = [[int(v) for v in h[j, b]] for b in range(nb)]
        if kind == 2:
            cands = []
            for s in range((1 << (nb - 1)) - 1):
                bits = s + 1
                L = [sum(hj[c][k] for c in range(nb) if (bits >> c) & 1) for k in range(C)]
                cands.append((s, L, [bits, 0, 0, 0]))
        else:
            order = list(range(nb))
            if kind == 1:
                def centroid(c):
                    cnt = _fsum(hj[c])
                    if cnt == 0.0:
                        return DBL_MAX
                    return gini(hj[c], cnt) if C > 2 else float(hj[c][1])
                cen = [centroid(c) for c in range(nb)]
                order = sorted(range(nb), key=lambda c: cen[c])      # sorted() is stable
            cands, L, mask = [], [0] * C, [0, 0, 0, 0]
            for s in range(nb - 1):
                c = order[s]
                L = [L[k] + hj[c][k] for k in range(C)]
                if kind == 1:
                    mask = list(mask); mask[c >> 6] |= 1 << (c & 63)
                cands.append((s, L, mask if kind == 1 else [0, 0, 0, 0]))
        for s, L, mask in cands:
            g = split_gain(L, tot, parent_imp, min_instances, min_info_gain)
            if g == -DBL_MAX:
                continue
            if best is None or g > best[0]:
                best = (g, j, s, kind, L, mask)
    out = np.zeros(1, SPLIT_DTYPE)[0]
    has = best is not None
    leaf = not (has and best[0] > 0.0) or level >= max_depth
    out["gain"] = best[0] if has else -DBL_MAX
    out["impurity"] = parent_imp
    out["feat"], out["kind"], out["bin_thr"] = -1, 0, 0
    flags = 1 if leaf else 0
    L = best[4] if has else [0] * C
    R = [t - l for t, l in zip(tot, L)] if has else [0] * C
    if not leaf:
        g, j, s, kind, _, mask = best
        out["feat"], out["kind"], out["bin_thr"] = int(subset[j]), 0 if kind == 0 else 1, s
        out["mask"] = np.array(mask, np.uint64)
        if level + 1 == max_depth or gini(L, _fsum(L)) == 0.0:
            flags |= 2
        if level + 1 == max_depth or gini(R, _fsum(R)) == 0.0:
            flags |= 4
    out["flags"] = flags
    return out, np.array(tot, np.int64), np.array(L, np.int64), np.array(R, np.int64)


# ------------------------------------------------------------------------------------------------ grow_level
def grow_ref(slot_tree, slot_nid, slot_node, split, node_counts, left_counts, right_counts, nodes, node_mask, pool_counts,
             node_tree, pool_size, pool_capacity):
    """b200flow_grow_level on host copies (nodes NODE_DTYPE [cap], node_mask uint64 [cap][4] or None, pool_counts [cap][C],
    node_tree [cap]; they are updated in place).  Slots are taken in order: a split slot s gets children at
    pool_size + 2 * (splits before s), and each non-leaf child the next slot index after those of the earlier slots.
    Returns (counters {pool, n_next, overflow, pool before}, next_tree, next_nid, next_node, next_parent, child_slot);
    when the grown pool would exceed pool_capacity the overflow flag is set and nothing is written."""
    n_slots = len(split)
    is_split = (split["flags"] & 1) == 0
    grown = pool_size + 2 * int(is_split.sum())
    child_slot = np.full(2 * n_slots, -1, np.int64)
    nxt = dict(tree=[], nid=[], node=[], parent=[])
    if grown > pool_capacity:
        return (pool_size, 0, 1, pool_size), *[np.zeros(0, np.int64)] * 4, None
    child = pool_size
    for s in range(n_slots):
        sp, node, nid, tree = split[s], int(slot_node[s]), int(slot_nid[s]), int(slot_tree[s])
        pool_counts[node] = node_counts[s]
        nd = np.zeros(1, NODE_DTYPE)[0]
        nd["nid"], nd["feat"], nd["kind_bin"], nd["left"] = nid, -1, 0, -1
        if is_split[s]:
            nd["feat"], nd["kind_bin"], nd["left"] = sp["feat"], (int(sp["kind"]) << 16) | (int(sp["bin_thr"]) & 0xFFFF), child
            if node_mask is not None:
                node_mask[node] = sp["mask"]
            for side in (0, 1):
                ch = np.zeros(1, NODE_DTYPE)[0]
                ch["feat"], ch["kind_bin"], ch["left"], ch["nid"] = -1, 0, -1, (nid * 2 + side) & 0xFFFFFFFF
                nodes[child + side] = ch
                node_tree[child + side] = tree
                pool_counts[child + side] = (left_counts if side == 0 else right_counts)[s]
                if not (int(sp["flags"]) & (2 << side)):
                    child_slot[2 * s + side] = len(nxt["tree"])
                    nxt["tree"].append(tree); nxt["nid"].append((nid * 2 + side) & 0xFFFFFFFF)
                    nxt["node"].append(child + side); nxt["parent"].append(2 * s + side)
            child += 2
        nodes[node] = nd
    n_next = len(nxt["tree"])
    return ((grown, n_next, 0, pool_size), *[np.array(nxt[k], np.int64) for k in ("tree", "nid", "node", "parent")],
            child_slot)
