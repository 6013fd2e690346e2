"""GBTRegressor on libb200flow.so (DESIGN.md §5m): GradientBoostedTrees.boost with SquaredError or AbsoluteError, one
regression tree per iteration.

Host logic only.  findSplits, binning and de-duplication are the regressors' (regression._LabelledSource through
forest._TrainingRows: records key on bins and label), the subsample weights are GBTClassifier's Bernoulli draws, and every
tree grows in gbt.LevelLoop.  What is new is the residual grid: r = -loss.gradient(F, y) has no a-priori bound, so each
iteration m puts r on a grid whose exponent E_m comes from the all-reduced max |r| (exact, so it is the same for any
world size and shard layout), and tree m is scored and valued with its own scale S - E_m.  csrc/regression.cu adds the
margin / residual update and the per-tree leaf values.
"""
from dataclasses import dataclass

import numpy as np
import torch

from . import _lib
from . import forest as fr
from . import gbt as bg
from . import regression as rg
from ._lib import call, ptr

LOSSES = {"squared": 0, "absolute": 1}


@dataclass
class GBTRegressorParams:
    """Spark 3 GBTRegressor Param defaults."""
    max_iter: int = 20
    step_size: float = 0.1
    max_depth: int = 5
    max_bins: int = 32
    min_instances_per_node: int = 1
    min_info_gain: float = 0.0
    subsampling_rate: float = 1.0
    feature_subset_strategy: str = "all"
    seed: int = 0
    loss: str = "squared"


def residual_exponent(max_abs):
    """E_m of iteration m's grid from M_m = the all-reduced max |r|: label_grid's rule (M <= 2^E, M = 0 gives 0, clamped below
    at 2^-300); beyond 2^300 the residuals cannot be put on a grid and the fit is refused"""
    if max_abs > 2.0 ** rg.E_MAX:
        raise ValueError("a boosting residual of magnitude %r is beyond the regression trainer's range (|r| <= 2^%d)"
                         % (max_abs, rg.E_MAX))
    return rg.label_grid(max_abs, 2)[0]


class GBTRegressionModel:
    """Device-resident boosted regression trees: one node pool (roots = nodes 0..T-1), payload[node] = tree weight x leaf
    value.  prediction = Σ_t payload of the leaf each row reaches, in tree order from +0.0 (the training margin's order)."""

    def __init__(self, forest, tree_weights, stats, E, S, S2):
        self.forest = forest                            # ForestModel with C = 1 over the payloads: binning and the tree walk
        self.T, self.F = forest.T, forest.F
        self.tree_weights = list(tree_weights)
        self.stats, self.E, self.S, self.S2 = stats, list(E), S, S2      # int64 [pool][3]; tree t's grid is 2^-(S - E[t])

    @property
    def n_nodes(self):
        return self.forest.n_nodes

    def predict(self, x):
        """-> prediction [n] f64 on a dense feature matrix"""
        raw, _, _ = self.forest.predict(x, want_raw=True, want_prob=False)
        return raw.reshape(-1)

    def predict_records(self, rec, plan, round_f32=False, on_invalid="ignore"):
        """the same from raw flow records + the encode plan of the feature vector (fused encode -> bins)"""
        raw, _, _, _ = self.forest.predict_records(rec, plan, want_raw=True, want_prob=False, round_f32=round_f32,
                                                   on_invalid=on_invalid)
        return raw.reshape(-1)

    def _prefix(self, k):
        """the model of the first k trees: the same pool and payloads, walked from roots 0..k-1 only"""
        fo = self.forest
        pre = fr.ForestModel(k, 1, fo.F, fo.arity, fo.max_bins, fo.thresholds, fo.n_thr, fo.nodes, fo.node_mask, None,
                             fo.node_tree, fo.leaf_prob, fo.node_gain, fo.n_nodes, dt_mode=False)
        pre._layout = fo._forest_layout()                # per-tree blocks in tree order: the first k are the prefix's
        return pre

    def prefix_predictions(self, x):
        """-> generator of the predictions [n] of the first k = 1..T trees on a dense feature matrix: the rows are binned
        and de-duplicated once, and each prefix sums its trees in tree order from +0.0, as a model of k trees does"""
        tp, _ = self.forest.bin(x)
        n = tp.shape[0]
        uid = None
        if fr.DEDUP and n > 0:
            tp, uid, _ = fr.dedup_rows(tp, self.F)
        for k in range(1, self.T + 1):
            raw, _, _ = self._prefix(k).predict_binned(tp, want_raw=True, want_prob=False)
            if uid is None:
                yield raw.reshape(-1)
                continue
            out = torch.empty(n, dtype=torch.float64, device=tp.device)
            call("b200flow_gather_rows", ptr(raw.contiguous()), 8, ptr(uid), n, ptr(out))
            yield out

    def evaluate_each_iteration(self, x, y, loss, group=None):
        """GBTRegressionModel.evaluateEachIteration: [mean loss of the first m + 1 trees for m < T]; squared is
        RegressionEvaluator's mse and absolute its mae on each prefix model's predictions, bit for bit"""
        from .metrics import regression_metrics
        if loss not in LOSSES:
            raise ValueError("loss must be one of %s, got %r" % (sorted(LOSSES), loss))
        key = "mse" if loss == "squared" else "mae"
        y = y.to(torch.float64).reshape(-1).contiguous()
        return [regression_metrics(y, p, group=group)[key] for p in self.prefix_predictions(x)]

    def export(self):
        """canonical host copy ordered by (tree, node id): structure, payload, gain and the int64 stats"""
        return bg.export_pool(self.forest, self.stats)

    def leaf_values(self, ex=None):
        """every node's unweighted value in label units, (Σw·q 2^-(S - E_t)) / Σw with its tree's own scale, in export order"""
        ex = self.export() if ex is None else ex
        sh = self.S - np.asarray(self.E, np.int64)[ex["tree"]]
        with np.errstate(all="ignore"):
            return (ex["stats"][:, 1].astype(np.float64) * np.ldexp(1.0, -sh)) / ex["stats"][:, 0].astype(np.float64)

    def feature_importances(self):
        """featureImportances with perTreeNormalization = false: Σ gain · count over the internal nodes of all trees,
        normalised once"""
        ex = self.export()
        v = np.zeros(self.F)
        sel = ex["is_leaf"] == 0
        np.add.at(v, ex["feat"][sel], ex["gain"][sel] * ex["stats"][sel, 0].astype(np.float64))
        return v / v.sum() if v.sum() > 0 else v


def fit_gbt_regressor(x, y, arity, params, row_offset=0, group=None):
    """GradientBoostedTrees.boost for regression on a dense CUDA feature matrix x [n, F] (f32/f64) and f64 labels y [n].
    With `group`, x / y are this rank's row shard starting at global row `row_offset`."""
    from . import dist as bdist
    import torch.distributed as dist
    _lib.require_cuda()
    p = params
    bg.check_boosting_params(p)
    if p.loss not in LOSSES:
        raise ValueError("lossType must be one of %s, got %r" % (sorted(LOSSES), p.loss))
    loss = LOSSES[p.loss]
    T = int(p.max_iter)
    seed = int(p.seed) & 0xFFFFFFFFFFFFFFFF
    strategy = "all" if str(p.feature_subset_strategy) == "auto" else p.feature_subset_strategy
    src, rows = rg._labelled_rows(x, y, arity, p.max_bins, 1, strategy, seed, row_offset, group)
    dev = x.device
    n, F = x.shape
    stride = fr.tp_stride(F)
    tp, U, m, n_bins = rows.tp, rows.U, rows.m, rows.n_bins

    # subsampling weights W[iteration][unique record] (GBTClassifier's Bernoulli draws per (iteration, global row))
    sub = p.subsampling_rate < 1.0
    TW = T if sub else 1
    cdf_host = bg.subsample_cdf(p.subsampling_rate) if sub else None
    W = fr.bag_weights(rows, TW, cdf_host, _lib.h2d(cdf_host.view(np.int32), dev) if sub else None, False, seed, row_offset)

    # ---- the label check and max |y| on every rank; S = S2 = 61 - ceil(log2 n): a tree's weights never exceed n
    head = torch.cat([(src.flags[0:1] > 0).to(torch.int64), src.flags[1:2]])
    if group is not None:
        bdist.all_reduce_(head, group, op=dist.ReduceOp.MAX)
    bad, max_bits = (int(v) for v in head.cpu())
    if bad:
        raise ValueError("a label is NaN or infinite: regression labels must be finite")
    E, S, S2 = rg.label_grid(float(np.array([max_bits], np.int64).view(np.float64)[0]), rows.n_global)

    pool = fr.NodePool(T, max(1024, T * min(1 << (p.max_depth + 1), 64)), bool((rows.kind > 0).any()), 3, torch.int64, dev)
    weights = [1.0] + [float(p.step_size)] * (T - 1)
    payload = torch.zeros(pool.cap, dtype=torch.float64, device=dev)
    margin = torch.zeros(max(U, 1), dtype=torch.float64, device=dev)
    resid = torch.zeros(max(U, 1), dtype=torch.float64, device=dev)
    rq = torch.zeros((max(U, 1), 2), dtype=torch.int64, device=dev)
    mx = torch.zeros(1, dtype=torch.int64, device=dev)
    y_vec = None if src.in_record else src.y                    # else the label is read from the record's bytes [F + 1, F + 9)

    def update(tree):
        mx.zero_()
        fr._timed("gbr_update", "b200flow_gbr_update", ptr(tp), stride, F + 1, ptr(y_vec), U, ptr(pool.nodes),
                  ptr(pool.node_mask), ptr(payload), tree, loss, ptr(margin), ptr(resid), ptr(mx))
    update(-1)                                          # F = +0.0, r = y

    bag = fr.Bag(1, U, dev)
    ent = torch.empty((max(U, 1), 2), dtype=torch.int32, device=dev)
    ent2 = torch.empty_like(ent)
    Es = []
    stats_t = dict(levels=0, slots=0, rows=n, unique_rows=U, S=S, S2=S2, E=Es)
    loop = bg.LevelLoop(tp, stride, rq, U, F, m, n_bins, rows.feat_bins, rows.feat_kind, S - E, S2 - 2 * E, seed, p, group,
                        stats_t)
    for t in range(T):
        if t > 0:                                       # the one host read of the iteration: E_m from the reduced max |r|
            if group is not None:
                bdist.all_reduce_(mx, group, op=dist.ReduceOp.MAX)
            E = residual_exponent(float(np.array([_read(mx)], np.int64).view(np.float64)[0]))
        Es.append(E)
        if U > 0:
            fr._timed("gbr_grid", "b200flow_reg_grid", None, stride, F + 1, ptr(resid), U, E, S, S2, ptr(rq))
        loop.S, loop.S2 = S - E, S2 - 2 * E
        # ---- this iteration's entries {unique record, weight}: the non-zero weights, in unique-id order
        Wt = W[(t if sub else 0) * U:(t if sub else 0) * U + max(U, 1)]
        bag.count(Wt)
        bag.fill(Wt, ent)
        ent, ent2 = loop.grow(pool, ent, ent2, torch.zeros(1, dtype=torch.int64, device=dev), bag.total.clone(),
                              torch.full((1,), t, dtype=torch.int32, device=dev))
        if payload.shape[0] < pool.cap:                 # earlier trees' payloads are kept: they are not recomputed
            grown = torch.zeros(pool.cap, dtype=torch.float64, device=dev)
            grown[:payload.shape[0]] = payload
            payload = grown
        call("b200flow_gbr_leaf_values", pool.size, ptr(pool.stats), ptr(pool.node_tree), t, weights[t], S - E, ptr(payload))
        update(t)

    forest = pool.model(rows, T, payload[:pool.size].reshape(pool.size, 1).contiguous())
    model = GBTRegressionModel(forest, weights, pool.stats, Es, S, S2)
    model.train_stats = stats_t
    model.train_margin = margin[:U]                      # F of every unique training record (rows: train_margin[train_uid])
    model.train_uid = rows.uid
    model.feat_kind, model.feat_bins, model.n_bins, model.m = rows.kind, rows.feat_bins, n_bins, m
    return model


def _read(mx):
    """host copy of the device scalar mx.  With forest.PROFILE set, the device time from the read's start until the stream
    resumes after it (the copy and the host round trip the GPU waits through) is recorded as 'gbr_sync'."""
    if fr.PROFILE is None:
        return int(mx.item())
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    v = int(mx.item())
    e1.record()
    fr.PROFILE.setdefault("gbr_sync", []).append((e0, e1))
    return v
