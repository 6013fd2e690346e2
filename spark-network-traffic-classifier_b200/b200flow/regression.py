"""DecisionTreeRegressor / RandomForestRegressor on libb200flow.so (DESIGN.md §5l): RandomForest.run with the Variance
impurity, T bagged regression trees grown side by side.

Host logic only.  findSplits, binning and de-duplication are the forest's (forest._TrainingRows), the bag weights are the
forest classifier's Poisson draws, and the trees grow in the variance-tree level loop of gbt.LevelLoop (the kernels of
csrc/gbt.cu); csrc/regression.cu adds the label check, the label grid and the leaf table.  Labels sit on a fixed-point grid
whose scale comes from the data (label_grid), so the level histograms are exact int64 sums and the model is the same bits
for any number of ranks and any shard layout.
"""
import math
from dataclasses import dataclass

import numpy as np
import torch

from . import _lib
from . import forest as fr
from . import gbt as bg
from ._lib import call, ptr

E_MIN, E_MAX = -300, 300           # label scale exponents; max |y| above 2^E_MAX is refused, below 2^E_MIN the grid stays 2^E_MIN


@dataclass
class RegressorParams:
    """Spark 3 RandomForestRegressor Param defaults (DecisionTreeRegressor: num_trees = 1, no bootstrap)."""
    num_trees: int = 20
    max_depth: int = 5
    max_bins: int = 32
    min_instances_per_node: int = 1
    min_info_gain: float = 0.0
    feature_subset_strategy: str = "auto"
    subsampling_rate: float = 1.0
    seed: int = 0
    bootstrap: bool = True


def resolve_strategy(strategy, num_trees):
    """featureSubsetStrategy 'auto' for regression: 'all' for one tree, 'onethird' for a forest (build_metadata's own 'auto'
    is the classification rule, sqrt)"""
    s = str(strategy)
    if s == "auto":
        return "all" if int(num_trees) == 1 else "onethird"
    return s


def label_grid(max_abs, w_max):
    """(E, S, S2) of the label grid.  y' = y 2^-E with max |y| <= 2^E, so |y'| <= 1 and the scaling is exact; q = rint(y' 2^S),
    q2 = rint((q 2^-S)^2 2^S2).  Bound: a tree's entries carry at most w_max = the largest total bag weight of any tree, so
    every histogram cell (and every node) has Σw·|q| <= w_max 2^S and Σw·q2 <= w_max 2^S2; with S = S2 = 61 - ceil(log2 w_max)
    both stay <= 2^61 < 2^62, and so do the left / right differences the scorer takes.  The scorer and the leaf table get
    S - E and S2 - 2E: then sums, variances, gains and leaf values come out in label units.  max |y| = 0 takes E = 0."""
    lg = int(math.ceil(math.log2(max(int(w_max), 2))))
    S = 61 - lg
    if not max_abs > 0.0:
        E = 0
    else:
        mnt, e = math.frexp(float(max_abs))       # max_abs = mnt 2^e, 0.5 <= mnt < 1
        E = e - 1 if mnt == 0.5 else e
    if E > E_MAX:
        raise ValueError("a label of magnitude %r is beyond the regression trainer's range (|label| <= 2^%d)" % (max_abs, E_MAX))
    return max(E, E_MIN), S, S


class _LabelledSource(fr._DenseSource):
    """a dense feature matrix with f64 labels: binning also checks the labels, finds max |y| and, when the record has eight
    spare bytes, stores each row's label bits right after the label byte, so that de-duplication keys on (bins, label)"""

    def __init__(self, x, y, in_record):
        super().__init__(x, None)
        self.y, self.in_record = y, in_record
        self.flags = torch.zeros(2, dtype=torch.int64, device=x.device)     # [non-finite labels, max |y| bits]

    def bin(self, thresholds, n_thr, arity_dev, mpb, bad, want_label_out=False):
        tp, _ = super().bin(thresholds, n_thr, arity_dev, mpb, bad)
        call("b200flow_reg_labels", ptr(self.y), self.n, ptr(tp) if self.in_record else None, tp.shape[1], self.F + 1,
             ptr(self.flags))
        return tp, None


def _labelled_rows(x, y, arity, max_bins, num_trees, strategy, seed, row_offset, group):
    """the front half of a regression fit on a dense feature matrix x [n, F] and labels y [n]: -> (the _LabelledSource, whose y
    holds the labels as f64 on x's device, the read forest._TrainingRows).  The label bits ride in the record's padding when
    there is room, so records merge only when bins AND label are equal — such rows also share every boosting residual; without
    room every row stays its own record.  num_classes = 2: every categorical feature is ordered by centroid, as for GBT's
    regression trees."""
    n, F = x.shape
    if y.shape[0] != n:
        raise ValueError("%d labels for %d rows" % (y.shape[0], n))
    src = _LabelledSource(x, y.to(device=x.device, dtype=torch.float64).contiguous(), fr.tp_stride(F) - (F + 1) >= 8)
    rows = fr._TrainingRows(src, 2, arity, max_bins, num_trees, strategy, seed, row_offset, group, key_bytes=F + 9,
                            dedup=None if src.in_record else False).read()
    return src, rows


class RegressionModel:
    """Device-resident regression trees: one node pool (roots = nodes 0..T-1), payload[node] = the node's mean label.
    prediction = (Σ over the trees, in tree order from +0.0, of the reached leaf's payload) / T."""

    def __init__(self, forest, stats, E, S, S2, var_forest=None):
        self.forest = forest                    # ForestModel with C = 1 over the payloads: binning and the tree walk
        self.var_forest = var_forest            # one tree, C = 2 over (payload, leaf variance), or None
        self.T, self.F = forest.T, forest.F
        self.stats, self.E, self.S, self.S2 = stats, E, S, S2      # int64 [pool][3] {Σw, Σw·q, Σw·q2} on the label grid

    @property
    def n_nodes(self):
        return self.forest.n_nodes

    def _pred(self, raw):
        s = raw.reshape(-1).contiguous()                  # C = 1: [n] (de-duplicated predict) or [n, 1]
        if self.T > 1:
            call("b200flow_reg_divide", ptr(s), s.shape[0], float(self.T), ptr(s))
        return s

    def predict(self, x):
        """-> prediction [n] f64 on a dense feature matrix"""
        raw, _, _ = self.forest.predict(x, want_raw=True, want_prob=False)
        return self._pred(raw)

    def predict_records(self, rec, plan, round_f32=False, on_invalid="ignore"):
        """the same from raw flow records + the encode plan of the feature vector (fused encode -> bins)"""
        raw, _, _, _ = self.forest.predict_records(rec, plan, want_raw=True, want_prob=False, round_f32=round_f32,
                                                   on_invalid=on_invalid)
        return self._pred(raw)

    def predict_with_variance(self, x=None, rec=None, plan=None, round_f32=False, on_invalid="ignore"):
        """decision tree only: -> (prediction [n], variance of the reached leaf [n]) from a dense matrix or from records"""
        if self.var_forest is None:
            raise ValueError("the leaf variance is only kept for a single decision tree")
        if x is not None:
            raw, _, _ = self.var_forest.predict(x, want_raw=True, want_prob=False)
        else:
            raw, _, _, _ = self.var_forest.predict_records(rec, plan, want_raw=True, want_prob=False, round_f32=round_f32,
                                                           on_invalid=on_invalid)
        return raw[:, 0].contiguous(), raw[:, 1].contiguous()

    def export(self):
        """canonical host copy ordered by (tree, node id): structure, payload, gain and the int64 stats"""
        return bg.export_pool(self.forest, self.stats)

    def feature_importances(self):
        """TreeEnsembleModel.featureImportances: per tree Σ gain · count over the internal nodes, normalised per tree, summed
        over the trees and normalised once"""
        ex = self.export()
        imp = np.zeros(self.F)
        for t in range(self.T):
            sel = (ex["tree"] == t) & (ex["is_leaf"] == 0)
            v = np.zeros(self.F)
            np.add.at(v, ex["feat"][sel], ex["gain"][sel] * ex["stats"][sel, 0].astype(np.float64))
            if v.sum() > 0:
                imp += v / v.sum()
        return imp / imp.sum() if imp.sum() > 0 else imp


def fit_dt_regressor(x, y, arity, params, row_offset=0, group=None):
    """DecisionTreeRegressor (RandomForest.run, one tree, strategy 'all', no bagging) on a dense CUDA feature matrix x [n, F]
    (f32/f64) and f64 labels y [n].  With `group`, x / y are this rank's row shard starting at global row `row_offset`."""
    p = RegressorParams(**{**params.__dict__, "num_trees": 1, "feature_subset_strategy": "all", "bootstrap": False})
    return _fit(x, y, arity, p, row_offset, group, want_variance=True)


def fit_rf_regressor(x, y, arity, params, row_offset=0, group=None):
    """RandomForestRegressor on a dense CUDA feature matrix x [n, F] and f64 labels y [n]: params.num_trees trees with the
    forest classifier's Poisson(subsamplingRate) bag weights per (tree, global row)."""
    return _fit(x, y, arity, params, row_offset, group)


def _fit(x, y, arity, p, row_offset=0, group=None, want_variance=False):
    from . import dist as bdist
    import torch.distributed as dist
    _lib.require_cuda()
    if not (0 <= p.max_depth <= 30):
        raise ValueError("maxDepth must be in [0, 30], got %d" % p.max_depth)
    T = int(p.num_trees)
    if T < 1:
        raise ValueError("numTrees must be >= 1, got %d" % T)
    if not (0.0 < p.subsampling_rate <= 1.0):
        raise ValueError("subsamplingRate must be in (0, 1], got %r" % p.subsampling_rate)
    seed = int(p.seed) & 0xFFFFFFFFFFFFFFFF
    src, rows = _labelled_rows(x, y, arity, p.max_bins, T, resolve_strategy(p.feature_subset_strategy, T), seed, row_offset,
                               group)
    dev = x.device
    n, F = x.shape
    stride = fr.tp_stride(F)
    tp, U, m, n_bins = rows.tp, rows.U, rows.m, rows.n_bins
    # ---- bag weights W[tree][unique record] (the forest classifier's draws); a decision tree weighs each record by its
    # multiplicity
    bagging = p.bootstrap and T > 1
    cdf_host = np.ascontiguousarray(fr.poisson_cdf_table(p.subsampling_rate)) if bagging else None
    W = fr.bag_weights(rows, T, cdf_host, _lib.h2d(cdf_host.view(np.int32), dev) if bagging else None, True, seed, row_offset)
    # ---- the label check, max |y| and the largest tree weight: one all-reduce (MAX) of [bad flag, max |y| bits, totals]
    totals = torch.zeros(T, dtype=torch.int64, device=dev)
    call("b200flow_reg_tree_weights", ptr(W), T, U, ptr(totals))
    if group is not None:
        bdist.all_reduce_(totals, group)
    head = torch.cat([(src.flags[0:1] > 0).to(torch.int64), src.flags[1:2], totals.max().reshape(1)])
    if group is not None:
        bdist.all_reduce_(head, group, op=dist.ReduceOp.MAX)
    bad, max_bits, w_max = (int(v) for v in head.cpu())
    if bad:
        raise ValueError("a label is NaN or infinite: regression labels must be finite")
    max_abs = float(np.array([max_bits], np.int64).view(np.float64)[0])
    E, S, S2 = label_grid(max_abs, w_max)
    rq = torch.zeros((max(U, 1), 2), dtype=torch.int64, device=dev)
    if U > 0:
        call("b200flow_reg_grid", ptr(tp) if src.in_record else None, stride, F + 1, None if src.in_record else ptr(src.y), U, E,
             S, S2, ptr(rq))

    # ---- entries {unique record, weight} of every tree, tree-major: one level-0 segment per tree root
    bag = fr.Bag(T, U, dev)
    bag.count(W)
    n_ent = int(bag.total.item())
    ent = torch.empty((max(n_ent, 1), 2), dtype=torch.int32, device=dev)
    ent2 = torch.empty_like(ent)
    bag.fill(W, ent)
    del W
    seg_begin, seg_end = bag.segments()

    pool = fr.NodePool(T, max(1024, T * min(1 << (p.max_depth + 1), 64)), bool((rows.kind > 0).any()), 3, torch.int64, dev)
    stats_t = dict(levels=0, slots=0, rows=n, unique_rows=U, entries=n_ent, E=E, S=S, S2=S2)
    loop = bg.LevelLoop(tp, stride, rq, U, F, m, n_bins, rows.feat_bins, rows.feat_kind, S - E, S2 - 2 * E, seed, p, group,
                        stats_t)
    loop.grow(pool, ent, ent2, seg_begin, seg_end, torch.arange(T, dtype=torch.int32, device=dev))

    width = 2 if want_variance else 1
    table = torch.zeros((max(pool.size, 1), width), dtype=torch.float64, device=dev)
    call("b200flow_reg_leaf_table", pool.size, ptr(pool.stats), S - E, S2 - 2 * E, ptr(table), width)
    model = RegressionModel(pool.model(rows, T, table[:, 0:1].contiguous()), pool.stats, E, S, S2,
                            pool.model(rows, T, table.contiguous()) if want_variance else None)
    model.train_stats = stats_t
    model.feat_kind, model.feat_bins, model.n_bins, model.m = rows.kind, rows.feat_bins, n_bins, m
    return model
