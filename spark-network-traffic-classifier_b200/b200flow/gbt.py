"""GBTClassifier (binary, LogLoss) on libb200flow.so: GradientBoostedTrees.boost with one regression tree per iteration
(DESIGN.md §5e).

Host logic only.  findSplits, binning and the de-duplication of the binned rows are the forest's (forest._TrainingRows,
once per fit); every tree runs the forest's level loop with the variance kernels of csrc/gbt.cu.  Residuals sit on a
fixed-point grid, so the level histograms are exact int64 sums: with rows sharded over ranks the one all-reduce per level
is exact and the model is the same bits for any number of ranks.

fit_gbt_ovr trains OneVsRest(GBTClassifier)'s K binary problems (label == k) in one level loop, K trees side by side per
iteration (DESIGN.md §5f); every class's model is the same bits as fit_gbt on the relabelled rows.
"""
import math
from dataclasses import dataclass

import numpy as np
import torch

from . import _lib
from . import forest as fr
from ._lib import NODE_DTYPE, call, ptr
from .forest import _timed


@dataclass
class GBTParams:
    """Spark 3 GBTClassifier Param defaults."""
    max_iter: int = 20
    step_size: float = 0.1
    max_depth: int = 5
    max_bins: int = 32
    min_instances_per_node: int = 1
    min_info_gain: float = 0.0
    subsampling_rate: float = 1.0
    feature_subset_strategy: str = "all"
    seed: int = 0


def grid_shift(n_global):
    """(S, S2) of the residual grid: q = rint(r 2^S), q2 = rint(r̂^2 2^S2); |r| <= 4 keeps every sum over n rows below 2^62."""
    lg = int(math.ceil(math.log2(max(int(n_global), 2))))
    return 60 - lg, 58 - lg


def subsample_cdf(rate):
    """the one-threshold inverse CDF that makes b200flow_bag_weights draw Bernoulli(rate) weights in {0, 1}"""
    cdf = np.full(32, 0xFFFFFFFF, np.uint32)
    cdf[0] = int(math.floor((1.0 - rate) * 4294967296.0))
    return cdf


def export_pool(fo, stats):
    """canonical host copy of a variance-tree pool (ForestModel fo whose leaf_prob[:, 0] is the payload, stats int64 [pool][3])
    ordered by (tree, node id)"""
    n = fo.n_nodes
    nodes = fo.nodes[:n].cpu().numpy().view(NODE_DTYPE).reshape(-1)
    tree = fo.node_tree[:n].cpu().numpy()
    order = np.lexsort((nodes["nid"], tree))
    mask = (fo.node_mask[:n].cpu().numpy().view(np.uint64) if fo.node_mask is not None else np.zeros((n, 4), np.uint64))
    is_leaf = (nodes["feat"] < 0).astype(np.int32)
    kind = np.where(is_leaf == 1, 0, nodes["kind_bin"] >> 16).astype(np.int32)
    bin_thr = np.where(is_leaf == 1, 0, nodes["kind_bin"] & 0xffff).astype(np.int32)
    mask = np.where(is_leaf[:, None] == 1, 0, mask).astype(np.uint64)
    return dict(tree=tree[order], nid=nodes["nid"][order], feat=np.where(is_leaf == 1, -1, nodes["feat"])[order],
                kind=kind[order], bin_thr=bin_thr[order], is_leaf=is_leaf[order], mask=mask[order],
                gain=fo.node_gain[:n].cpu().numpy()[order], payload=fo.leaf_prob[:n, 0].cpu().numpy()[order],
                stats=stats[:n].cpu().numpy()[order])


class GBTModel:
    """Device-resident boosted trees: one node pool (roots = nodes 0..T-1), payload[node] = tree weight x leaf value."""

    def __init__(self, forest, tree_weights, stats, S):
        self.forest = forest                            # ForestModel with C = 1 over the payloads: binning and the tree walk
        self.T, self.F = forest.T, forest.F
        self.tree_weights = list(tree_weights)
        self.stats, self.S = stats, S                   # int64 [pool][3] {Σw, Σw·q, Σw·q2}

    @property
    def n_nodes(self):
        return self.forest.n_nodes

    def margin(self, x):
        """Σ_t payload of the leaf each row reaches, in tree order from +0.0 (GBTClassificationModel.margin)."""
        raw, _, _ = self.forest.predict(x, want_raw=True, want_prob=False)
        return raw.view(-1)

    def _output(self, margin):
        n = margin.shape[0]
        dev = margin.device
        raw = torch.empty((n, 2), dtype=torch.float64, device=dev)
        prob = torch.empty((n, 2), dtype=torch.float64, device=dev)
        pred = torch.empty(n, dtype=torch.float64, device=dev)
        call("b200flow_gbt_output", ptr(margin.contiguous()), n, ptr(raw), ptr(prob), ptr(pred))
        return raw, prob, pred

    def predict(self, x):
        """-> (rawPrediction [n, 2], probability [n, 2], prediction [n]) on a dense feature matrix."""
        return self._output(self.margin(x))

    def predict_records(self, rec, plan, round_f32=False, on_invalid="ignore"):
        """the same from raw flow records + the encode plan of the feature vector (fused encode -> bins)"""
        raw, _, _, _ = self.forest.predict_records(rec, plan, want_raw=True, want_prob=False, round_f32=round_f32,
                                                   on_invalid=on_invalid)
        return self._output(raw.view(-1))

    def export(self):
        """canonical host copy ordered by (tree, node id): the forest export's structure + payload, gain and int64 stats"""
        return export_pool(self.forest, self.stats)

    def feature_importances(self):
        """featureImportances with perTreeNormalization = false (SPARK-26721): Σ gain · count over the internal nodes of all
        trees, normalised once."""
        ex = self.export()
        v = np.zeros(self.F)
        sel = ex["is_leaf"] == 0
        np.add.at(v, ex["feat"][sel], ex["gain"][sel] * ex["stats"][sel, 0].astype(np.float64))
        return v / v.sum() if v.sum() > 0 else v


def fit_gbt(x, labels, arity, params, row_offset=0, group=None):
    """GradientBoostedTrees.boost on a dense CUDA feature matrix x [n, F] (f32/f64) and labels [n] in {0, 1}.  arity as
    for fit_forest; with `group`, x / labels are this rank's row shard starting at global row `row_offset`."""
    return _fit(fr._DenseSource(x, labels), arity, params, row_offset, group)


def fit_gbt_records(rec, plan, arity, params, row_offset=0, group=None, round_f32=False):
    """the same on raw flow records [n, row_bytes] + the encode plan of their feature vector (plan.label = a label column
    with at most two values)"""
    if plan.label is None:
        raise ValueError("fit_gbt_records: the encode plan has no label column (EncodePlan.set_label)")
    return _fit(fr._RecordSource(rec, plan, round_f32), arity, params, row_offset, group)


def fit_gbt_ovr(x, labels, K, arity, params, row_offset=0, group=None):
    """OneVsRest(GBTClassifier) on a dense CUDA feature matrix: the K problems (labels == k) for k < K, with labels [n] in
    [0, K), K <= 256, trained together.  -> OvRGBTModel whose models[k] equals fit_gbt(x, labels == k, ...) bit for bit."""
    return _fit(fr._DenseSource(x, labels), arity, params, row_offset, group, n_classes=K)


def fit_gbt_ovr_records(rec, plan, K, arity, params, row_offset=0, group=None, round_f32=False):
    """the same on raw flow records [n, row_bytes] + the encode plan of their feature vector (plan.label = the label column)"""
    if plan.label is None:
        raise ValueError("fit_gbt_ovr_records: the encode plan has no label column (EncodePlan.set_label)")
    return _fit(fr._RecordSource(rec, plan, round_f32), arity, params, row_offset, group, n_classes=K)


class OvRGBTModel:
    """OneVsRest over K binary GBT models trained together.  models[k] is class k's GBTModel on its own node pool; `forest`
    is the combined pool (K·T trees, tree k·T + t = class k's tree t) with C = K, whose leaf_prob[node] is one-hot on the class
    of the node's tree and carries the node's payload.  One b200flow_predict_forest over it gives every class's margin — class k's
    column adds its own payloads and +0.0 for the other classes' trees, in tree order from +0.0, so it has the bits of
    models[k].margin — and the first argmax under Spark's `>` rule."""

    def __init__(self, models, forest):
        self.models, self.forest = list(models), forest
        self.K, self.T, self.F = len(self.models), self.models[0].T, forest.F

    def predict(self, x):
        """-> (rawPrediction [n, K] = each class's margin, prediction [n]) on a dense feature matrix."""
        raw, _, pred = self.forest.predict(x, want_raw=True, want_prob=False)
        return raw, pred

    def predict_records(self, rec, plan, round_f32=False, on_invalid="ignore"):
        """the same from raw flow records + the encode plan of the feature vector (fused encode -> bins)"""
        raw, _, pred, _ = self.forest.predict_records(rec, plan, want_raw=True, want_prob=False, round_f32=round_f32,
                                                      on_invalid=on_invalid)
        return raw, pred


class LevelLoop:
    """the level loop of the variance trees, shared by GBTClassifier, OneVsRest(GBTClassifier) and the regressors
    (b200flow/regression.py): every level builds the slots' {Σw, Σw·q, Σw·q2} histograms (gbt_hist_level, in slot groups
    that keep one level within forest.HIST_BUDGET_BYTES), all-reduces them (exact int64 sums), scores them (gbt_score_level
    with the grid scales S, S2), grows the pool and partitions the entries to the children.  rq [.][2] holds {q, q2} per
    unique record; n_iter = T makes it OneVsRest's class-major pool (tree k·T + t reads class k's rq block, and draws the
    feature subsets of tree t)."""

    def __init__(self, tp, stride, rq, U, F, m, n_bins, feat_bins, feat_kind, S, S2, seed, params, group, stats, n_iter=None):
        self.tp, self.stride, self.rq, self.U, self.F, self.m, self.n_bins = tp, stride, rq, U, F, m, n_bins
        self.feat_bins, self.feat_kind, self.S, self.S2, self.seed, self.p = feat_bins, feat_kind, S, S2, seed, params
        self.group, self.stats, self.n_iter = group, stats, n_iter
        self.per_slot = m * n_bins * 3
        self.group_slots = max(1, fr.HIST_BUDGET_BYTES // (self.per_slot * 8))

    def grow(self, pool, ent, ent2, seg_begin, seg_end, slot_tree):
        """grow the trees rooted at pool nodes slot_tree (one level-0 slot each, whose entries are ent[seg_begin:seg_end])
        to the end; -> (ent, ent2), swapped as the partitions left them"""
        from . import dist as bdist
        p, dev, m, n_bins, tp, stride, rq = self.p, pool.dev, self.m, self.n_bins, self.tp, self.stride, self.rq
        per_slot, group_slots, group, ovr, T, CH = self.per_slot, self.group_slots, self.group, self.n_iter is not None, self.n_iter, fr.CHUNK_ROWS
        n_slots, level = int(slot_tree.numel()), 0
        slot_nid = torch.ones(n_slots, dtype=torch.int32, device=dev)
        slot_node = slot_tree.clone()
        while n_slots > 0:
            subset = torch.empty((n_slots, m), dtype=torch.int16, device=dev)
            # the feature subsets are keyed by the iteration, as in the K separate fits: class k's tree t draws tree t's
            slot_iter = torch.remainder(slot_tree, T) if ovr else slot_tree
            call("b200flow_feature_subsets", self.seed, n_slots, ptr(slot_iter), ptr(slot_nid), self.F, m, ptr(subset))
            slot_class = torch.div(slot_tree, T, rounding_mode="floor") if ovr else None
            chunk_off, off_h = fr.chunk_table(seg_end - seg_begin)
            n_chunks = int(off_h[-1])
            split = torch.empty((n_slots, 64), dtype=torch.uint8, device=dev)
            st = torch.empty((3, n_slots, 3), dtype=torch.int64, device=dev)   # node, left, right
            for g0 in range(0, n_slots, group_slots):      # slot groups keep one level's histograms within HIST_BUDGET_BYTES
                g1 = min(n_slots, g0 + group_slots)
                hist = torch.zeros((g1 - g0) * per_slot, dtype=torch.int64, device=dev)
                gch = int(off_h[g1] - off_h[g0])
                if gch > 0:
                    coff = (chunk_off[g0:g1 + 1] - chunk_off[g0]).contiguous()
                    if ovr:
                        _timed("gbt_hist_level", "b200flow_gbt_hist_level_classes", ptr(tp), stride, ptr(ent), ptr(rq), self.U,
                               ptr(slot_class[g0:g1]), g1 - g0, ptr(seg_begin[g0:g1]), ptr(seg_end[g0:g1]), ptr(coff), gch, CH,
                               ptr(subset[g0:g1]), m, n_bins, ptr(hist))
                    else:
                        _timed("gbt_hist_level", "b200flow_gbt_hist_level", ptr(tp), stride, ptr(ent), ptr(rq), g1 - g0,
                               ptr(seg_begin[g0:g1]), ptr(seg_end[g0:g1]), ptr(coff), gch, CH, ptr(subset[g0:g1]), m, n_bins,
                               ptr(hist))
                if group is not None:                   # the one data-path collective: exact int64 sums
                    bdist.all_reduce_(hist, group)
                _timed("gbt_score_level", "b200flow_gbt_score_level", ptr(hist), g1 - g0, ptr(subset[g0:g1]), m, n_bins,
                       ptr(self.feat_bins), ptr(self.feat_kind), self.S, self.S2, level, p.max_depth, int(p.min_instances_per_node),
                       float(p.min_info_gain), ptr(split[g0:g1]), ptr(st[0, g0:g1]), ptr(st[1, g0:g1]), ptr(st[2, g0:g1]))
                del hist
            next_tree = torch.empty(2 * n_slots, dtype=torch.int32, device=dev)
            next_nid = torch.empty(2 * n_slots, dtype=torch.int32, device=dev)
            next_node = torch.empty(2 * n_slots, dtype=torch.int32, device=dev)
            next_parent = torch.empty(2 * n_slots, dtype=torch.int32, device=dev)
            pool.grow_level(n_slots, slot_tree, slot_nid, slot_node, split, st[0], st[1], st[2], next_tree, next_nid, next_node,
                            next_parent)
            pool.node_gain[slot_node.long()] = split.view(torch.float64)[:, 2]
            n_next = pool.commit(pool.counters[:3].cpu())
            self.stats["levels"] += 1; self.stats["slots"] += n_slots
            if n_next == 0:
                break
            cursors = torch.zeros(2 * n_slots, dtype=torch.int32, device=dev)
            if n_chunks > 0:
                _timed("partition_level", "b200flow_partition_level", ptr(tp), stride, ptr(ent), ptr(ent2), n_slots, ptr(seg_begin),
                       ptr(seg_end), ptr(chunk_off), n_chunks, CH, ptr(split), ptr(cursors))
            next_begin = torch.empty(n_next, dtype=torch.int64, device=dev)
            next_end = torch.empty(n_next, dtype=torch.int64, device=dev)
            call("b200flow_next_segments", n_next, None, ptr(next_parent), ptr(seg_begin), ptr(seg_end), ptr(cursors), ptr(next_begin),
                 ptr(next_end))
            ent, ent2 = ent2, ent
            slot_tree, slot_nid, slot_node = next_tree[:n_next], next_nid[:n_next], next_node[:n_next]
            seg_begin, seg_end = next_begin, next_end
            n_slots = n_next
            level += 1
        return ent, ent2


def check_boosting_params(p):
    """the parameter checks GBTClassifier and GBTRegressor share"""
    if not (0 <= p.max_depth <= 30):
        raise ValueError("maxDepth must be in [0, 30], got %d" % p.max_depth)
    if int(p.max_iter) < 1:
        raise ValueError("maxIter must be >= 1, got %d" % p.max_iter)
    if not (0.0 < p.step_size <= 1.0):
        raise ValueError("stepSize must be in (0, 1], got %r" % p.step_size)
    if not (0.0 < p.subsampling_rate <= 1.0):
        raise ValueError("subsamplingRate must be in (0, 1], got %r" % p.subsampling_rate)


def _fit(src, arity, params, row_offset=0, group=None, n_classes=None):
    """the boosting loop.  n_classes None: the binary problem of the label byte.  n_classes = K: the K problems (label == k)
    side by side — the pool holds K·T trees, class-major (tree k·T + t), margin and rq are [K][U], every iteration's entries
    are repeated in K segments (one per class root) and one level loop grows all K trees."""
    from . import dist as bdist
    _lib.require_cuda()
    p = params
    check_boosting_params(p)
    ovr = n_classes is not None
    K = int(n_classes) if ovr else 1
    if not (1 <= K <= 256):
        raise ValueError("OneVsRest on the GBT trainer needs 1 <= numClasses <= 256 (labels are stored as one byte), got %d" % K)
    dev = src.device
    n, F = src.n, src.F
    T = int(p.max_iter)
    seed = int(p.seed) & 0xFFFFFFFFFFFFFFFF
    strategy = "all" if str(p.feature_subset_strategy) == "auto" else p.feature_subset_strategy
    # num_classes = 2 only shapes the metadata, so the bins are the binary fit's; de-duplication keys on (bins, label byte), and
    # with K classes those records refine each relabelled problem's records: the trees see the same integer histogram sums
    rows = fr._TrainingRows(src, 2, arity, p.max_bins, 1, strategy, seed, row_offset, group).read()
    tp, U, m, n_bins = rows.tp, rows.U, rows.m, rows.n_bins
    feat_bins, feat_kind, stride = rows.feat_bins, rows.feat_kind, fr.tp_stride(F)
    S, S2 = grid_shift(rows.n_global)
    # labels must be 0 or 1 (OneVsRest: below K) on EVERY rank: the flag is summed over the ranks first, so that all of them
    # raise together
    top = K - 1 if ovr else 1
    bad = (tp[:U, F] > top).any().reshape(1).to(torch.int64) if U > 0 else torch.zeros(1, dtype=torch.int64, device=dev)
    if group is not None:
        bdist.all_reduce_(bad, group)
    if int(bad.item()):
        if ovr:
            raise ValueError("OneVsRest: a label is not in [0, %d)" % K)
        raise ValueError("GBTClassifier currently only supports binary classification: a label is not 0 or 1")

    # subsampling weights W[iteration][unique record] (Bernoulli, tree index = iteration); without subsampling every
    # iteration sees each unique record with its multiplicity
    sub = p.subsampling_rate < 1.0
    TW = T if sub else 1
    cdf_host = subsample_cdf(p.subsampling_rate) if sub else None
    W = fr.bag_weights(rows, TW, cdf_host, _lib.h2d(cdf_host.view(np.int32), dev) if sub else None, False, seed, row_offset)

    # node pool: roots 0..K·T-1
    TK = K * T
    pool = fr.NodePool(TK, max(1024, TK * min(1 << (p.max_depth + 1), 64)), bool((rows.kind > 0).any()), 3, torch.int64, dev)

    weights = [1.0] + [float(p.step_size)] * (T - 1)
    tree_weight = _lib.h2d(np.asarray(weights * K, np.float64), dev)
    payload = torch.zeros(pool.cap, dtype=torch.float64, device=dev)
    margin = torch.zeros(max(K * U, 1), dtype=torch.float64, device=dev)          # [K][U]
    rq = torch.zeros((max(K * U, 1), 2), dtype=torch.int64, device=dev)           # [K][U][2]: class blocks stay 16-byte aligned
    if ovr:
        call("b200flow_gbt_update_classes", ptr(tp), stride, F, U, K, None, None, None, -1, T, S, S2, ptr(margin), ptr(rq))
    else:
        call("b200flow_gbt_update", ptr(tp), stride, F, U, None, None, None, -1, S, S2, ptr(margin), ptr(rq))

    bag = fr.Bag(1, U, dev)
    ent = torch.empty((max(K * U, 1), 2), dtype=torch.int32, device=dev)        # class k's segment starts at k·U
    ent2 = torch.empty_like(ent)
    stats_t = dict(levels=0, slots=0, rows=n, unique_rows=U, S=S)
    loop = LevelLoop(tp, stride, rq, U, F, m, n_bins, feat_bins, feat_kind, S, S2, seed, p, group, stats_t,
                     n_iter=T if ovr else None)
    if ovr:
        cls_base = torch.arange(K, dtype=torch.int64, device=dev) * U
        cls_root = torch.arange(K, dtype=torch.int32, device=dev) * T

    for t in range(T):
        # ---- this iteration's entries {unique record, weight}: the non-zero weights, in unique-id order
        Wt = W[(t if sub else 0) * U:(t if sub else 0) * U + max(U, 1)]
        bag.count(Wt)
        bag.fill(Wt, ent)
        if ovr:             # the same entries for every class: one segment per class root k·T + t
            if K > 1 and U > 0:
                ent[:K * U].view(K, U, 2)[1:] = ent[:U]
            seg_begin = cls_base.clone()
            seg_end = cls_base + bag.total
            slot_tree = cls_root + t
        else:
            seg_begin = torch.zeros(1, dtype=torch.int64, device=dev)
            seg_end = bag.total.clone()
            slot_tree = torch.full((1,), t, dtype=torch.int32, device=dev)
        ent, ent2 = loop.grow(pool, ent, ent2, seg_begin, seg_end, slot_tree)
        # ---- leaf values of the pool so far, then F and the next residuals of every unique record
        if payload.shape[0] < pool.cap:
            payload = torch.zeros(pool.cap, dtype=torch.float64, device=dev)
        call("b200flow_gbt_leaf_values", pool.size, ptr(pool.stats), ptr(pool.node_tree), ptr(tree_weight), S, ptr(payload))
        if ovr:
            _timed("gbt_update", "b200flow_gbt_update_classes", ptr(tp), stride, F, U, K, ptr(pool.nodes), ptr(pool.node_mask),
                   ptr(payload), t, T, S, S2, ptr(margin), ptr(rq))
        else:
            _timed("gbt_update", "b200flow_gbt_update", ptr(tp), stride, F, U, ptr(pool.nodes), ptr(pool.node_mask), ptr(payload), t,
                   S, S2, ptr(margin), ptr(rq))

    if ovr:
        return _ovr_model(rows, K, T, weights, S, stats_t, pool, payload, margin, U)
    model = GBTModel(pool.model(rows, T, payload[:pool.size].reshape(pool.size, 1).contiguous()), weights, pool.stats, S)
    model.train_stats = stats_t
    model.train_margin = margin[:U]                      # F of every unique training record (rows: train_margin[train_uid])
    model.train_uid = rows.uid
    model.feat_kind, model.feat_bins, model.n_bins, model.m = rows.kind, feat_bins, n_bins, m
    return model


def _ovr_model(rows, K, T, weights, S, stats_t, pool, payload, margin, U):
    """the K·T-tree pool -> OvRGBTModel: each class's nodes compacted into their own pool (pool order kept, so its roots
    k·T..k·T+T-1 become 0..T-1 and sibling pairs stay adjacent; left indices remapped), and the combined C = K forest."""
    nodes, node_mask, stats, node_tree, node_gain = pool.nodes, pool.node_mask, pool.stats, pool.node_tree, pool.node_gain
    n = pool.size
    dev = nodes.device
    F = rows.F
    tree = node_tree[:n]
    cls = torch.div(tree, T, rounding_mode="floor").long()
    sels = [torch.nonzero(cls == k).view(-1) for k in range(K)]
    rank = torch.empty(n, dtype=torch.int64, device=dev)         # every node's index within its class, in pool order
    for sel in sels:
        rank[sel] = torch.arange(sel.numel(), dtype=torch.int64, device=dev)
    nd32 = nodes[:n].view(torch.int32).view(n, 4)
    left = nd32[:, 2].long()
    new_left = torch.where(left >= 0, rank[left.clamp(min=0)], left).to(torch.int32)
    models = []
    for k, sel in enumerate(sels):
        nk = sel.numel()
        nk32 = nd32[sel].clone()
        nk32[:, 2] = new_left[sel]
        nodes_k = nk32.contiguous().view(torch.uint8).view(nk, 16)
        mask_k = node_mask[sel].contiguous() if node_mask is not None else None
        tree_k = (tree[sel] - k * T).contiguous()
        forest_k = fr.ForestModel(T, 1, F, rows.arity, rows.mpb, rows.thresholds, rows.n_thr, nodes_k, mask_k, None, tree_k,
                                  payload[sel].reshape(nk, 1).contiguous(), node_gain[sel].contiguous(), nk, dt_mode=False)
        mk = GBTModel(forest_k, weights, stats[sel].contiguous(), S)
        mk.train_margin = margin[k * U:(k + 1) * U]
        mk.train_uid = rows.uid
        mk.feat_kind, mk.feat_bins, mk.n_bins, mk.m = rows.kind, rows.feat_bins, rows.n_bins, rows.m
        models.append(mk)
    leaf = torch.zeros((max(n, 1), K), dtype=torch.float64, device=dev)
    if n > 0:
        leaf[torch.arange(n, device=dev), cls] = payload[:n]
    model = OvRGBTModel(models, pool.model(rows, K * T, leaf))
    model.train_stats = stats_t
    return model
