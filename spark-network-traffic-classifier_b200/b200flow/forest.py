"""RandomForest / DecisionTree trainer and batch predictor on libb200flow.so.

Host logic only (the level loop MLlib runs on the Spark driver: RandomForest.run, SURVEY.md §3.3);
every per-row / per-node computation is a kernel in csrc/forest.cu, csrc/treeprep.cu, csrc/predict.cu.
Reference call sites: kdd99.py:61,64,79,82; cicids17.py:65,68,83,86.

Rows may be sharded over ranks (one process per GPU): each rank holds a contiguous block of rows
starting at global index `row_offset`; the only data-path collective is one all-reduce (sum, int32)
of the per-node histograms per tree level (R7r).  Integer sums + counter-based RNG make the model
bit-identical for any number of ranks.
"""
import math
from dataclasses import dataclass

import numpy as np
import torch

from . import _lib
from ._lib import NODE_DTYPE, SPLIT_DTYPE, B200FlowError, UnsupportedParamError, call, ptr

import os as _os
CHUNK_ROWS = 2048                  # entries per CTA in hist_level / partition_level (<= 2048)
FUSED = True                       # use route_hist_level (partition + next-level histogram in one pass) when it fits
TOP_LEVELS = int(_os.environ.get("B200FLOW_TOP_LEVELS", "8"))   # tree levels the grid predict kernel walks in shared memory (0 = none)
DEDUP = True                       # run the level loop on unique binned records (flow records repeat massively)
_PIN = True                        # read the per-level counts into pinned host memory
PROFILE = None                     # set to a dict to collect per-kernel CUDA-event timings (bench.py)


def _timed(name, fn, *args):
    """run one C-ABI call; when PROFILE is a dict, bracket it with CUDA events on the launching stream."""
    if PROFILE is None:
        return call(fn, *args)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    call(fn, *args)
    e1.record()
    PROFILE.setdefault(name, []).append((e0, e1))


def profile_totals():
    """-> {kernel: (launches, total_ms)} from the recorded events (synchronises)."""
    torch.cuda.synchronize()
    return {k: (len(v), sum(a.elapsed_time(b) for a, b in v)) for k, v in (PROFILE or {}).items()
            if not k.startswith("_")}


ENTRY_BOUND_BYTES = 8 << 30        # the two entry buffers are sized by the bound T * U (no host read of the exact count) up to this many bytes
HIST_BUDGET_BYTES = int(_os.environ.get("B200FLOW_HIST_BUDGET_GB", "10")) << 30   # cap of one level's histogram buffer (MLlib: maxMemoryInMB; 10 GB of an 80 GB H100); beyond it the level is processed in node groups by the unfused kernels
# Multi-GPU: level histograms of at least this many bytes are REDUCE-SCATTERED by node (each rank then scores only its own
# nodes and the 64-byte split records are all-gathered) instead of all-reduced: half the NVLink bytes, 1/world of the scoring.
# Smaller levels are latency-bound and keep the single all-reduce.
RS_MIN_BYTES = int(_os.environ.get("B200FLOW_RS_MIN_BYTES", str(8 << 20)))
RS_CHUNKS = int(_os.environ.get("B200FLOW_RS_CHUNKS", "1"))   # slot ranges per level whose reduce-scatter overlaps the scoring of the previous range


@dataclass
class ForestParams:
    """MLlib Param defaults (SURVEY.md §8a R0)."""
    num_trees: int = 20
    max_depth: int = 5
    max_bins: int = 32
    min_instances_per_node: int = 1
    min_info_gain: float = 0.0
    feature_subset_strategy: str = "auto"
    subsampling_rate: float = 1.0
    impurity: str = "gini"
    seed: int = 0
    bootstrap: bool = True         # False for DecisionTreeClassifier (numTrees == 1)


def tp_stride(F):
    """TreePoint record stride: F bins + label, padded to whole 64-byte HBM bursts so that one random
    record gather costs exactly ceil((F+1)/64) bursts (both level kernels gather records at random)."""
    return (F + 1 + 63) // 64 * 64


def poisson_cdf_table(rate=1.0):
    """32 uint32 thresholds floor(CDF(k)*2^32), saturating (DESIGN.md §RNG, A.4)."""
    out = np.empty(32, np.uint32)
    term = math.exp(-rate); cdf = 0.0
    for k in range(32):
        cdf += term
        out[k] = min(int(math.floor(cdf * 4294967296.0)), 0xFFFFFFFF)
        term = term * rate / (k + 1)
    if out[30] != 0xFFFFFFFF:
        raise UnsupportedParamError("subsamplingRate %.3f too large: bag weights must stay below 31" % rate)
    return out


def bag_weights(rows, T, cdf_host, cdf_dev, by_record, seed, row_offset):
    """W int32 [T][U]: the summed weights of every (weight row, unique record) of read _TrainingRows, drawn per (row t, global
    row) from the 32-threshold inverse CDF cdf_host (cdf_dev: its device copy, staged by the caller).  cdf_host None: every
    record weighs its multiplicity.  by_record: draw over the rows grouped by unique record (one RED per warp run and weight
    row instead of one per row), when there are draws and records repeat."""
    n, U, uid, dev = rows.n, rows.U, rows.uid, rows.src.device
    W = torch.zeros(max(T * U, 1), dtype=torch.int32, device=dev)
    if n > 0:
        perm = uperm = None
        if by_record and cdf_host is not None and uid is not None and U < n:
            gsize = torch.empty(U, dtype=torch.int32, device=dev); cursor = torch.empty(U, dtype=torch.int32, device=dev)
            goff = torch.empty(U + 1, dtype=torch.int64, device=dev)
            perm = torch.empty(n, dtype=torch.int32, device=dev); uperm = torch.empty(n, dtype=torch.int32, device=dev)
            _timed("group_rows", "b200flow_group_rows", ptr(uid), n, U, ptr(gsize), ptr(goff), ptr(cursor), ptr(perm), ptr(uperm))
        _timed("bag_weights", "b200flow_bag_weights", seed, T, int(row_offset), n, ptr(cdf_dev),
               cdf_host.ctypes.data if cdf_host is not None else None, ptr(uperm if perm is not None else uid), ptr(perm), U, ptr(W))
    return W


def build_metadata(n_rows, F, num_classes, arity, max_bins, num_trees, strategy="auto"):
    """DecisionTreeMetadata.buildMetadata (A.1): (maxPossibleBins, feat_kind[F], numFeaturesPerNode)."""
    arity = np.asarray(arity, np.int32)
    mpb = int(min(max_bins, n_rows))
    if mpb > 256:
        raise UnsupportedParamError("maxBins > 256 is not supported (bins are stored as uint8)")
    if arity.size and int(arity.max()) > mpb:
        raise ValueError("DecisionTree requires maxBins (= %d) to be at least as large as the number of values in each "
                         "categorical feature, but a categorical feature has %d values. Consider removing this and other "
                         "categorical features with a large number of values, or add more training examples."
                         % (mpb, int(arity.max())))
    if arity.size and int(arity.max()) > 255:
        raise UnsupportedParamError("a categorical feature with %d categories is not supported: bins are stored as uint8, and "
                                    "with 256 categories no bin is left for a value unseen at fit time (at most 255)"
                                    % int(arity.max()))
    kind = np.zeros(F, np.int32)
    U = int(math.floor(math.log(mpb // 2 + 1) / math.log(2.0) + 1)) if num_classes > 2 else 0
    for f in range(F):
        if arity[f] > 1:
            kind[f] = 2 if (num_classes > 2 and arity[f] <= U) else 1
        elif arity[f] == 1:
            kind[f] = 1
    s = str(strategy)
    if s == "auto":
        s = "all" if num_trees == 1 else "sqrt"
    if s == "all": m = F
    elif s == "sqrt": m = int(math.ceil(math.sqrt(F)))
    elif s == "log2": m = max(1, int(math.ceil(math.log(F) / math.log(2))))
    elif s == "onethird": m = int(math.ceil(F / 3.0))
    else:
        try:
            v = float(s)
        except ValueError:
            raise ValueError("Supported featureSubsetStrategy values: auto, all, onethird, sqrt, log2, (0.0-1.0], [1-n]; got %r" % strategy)
        m = int(v) if ("." not in s and v >= 1) else int(math.ceil(v * F))
    return mpb, kind, max(1, min(m, F))


def pack_records(tp, F, field_desc, rec_bytes):
    """byte TreePoint records tp[U][stride] -> bit-packed records [U][rec_bytes] (uint8) of the layout whose device
    descriptors are field_desc (_lib.packed_layout)"""
    packed = torch.empty((max(tp.shape[0], 1), rec_bytes), dtype=torch.uint8, device=tp.device)
    call("b200flow_pack_records", ptr(tp), tp.shape[1], tp.shape[0], F, ptr(field_desc), rec_bytes, ptr(packed))
    return packed


def dedup_rows(tp, key_bytes, sync=True):
    """unique TreePoint records of a binned batch: -> (tp_unique [U, stride], uid int32 [n], U).  Flow records repeat
    massively (KDD99: 4.9 M rows, ~1.07 M distinct), so both the level loop and the batch predictor run per unique record."""
    n, stride = tp.shape
    dev = tp.device
    cap_tab = 1
    while cap_tab < 2 * n:
        cap_tab <<= 1
    table = torch.empty(cap_tab, dtype=torch.int32, device=dev); minrow = torch.empty(cap_tab, dtype=torch.int32, device=dev)
    slot_of = torch.empty(n, dtype=torch.int32, device=dev); rep = torch.empty(n, dtype=torch.int32, device=dev)
    flag = torch.empty(n, dtype=torch.int32, device=dev); pos = torch.empty(n + 1, dtype=torch.int64, device=dev)
    uid = torch.empty(n, dtype=torch.int32, device=dev); total = torch.zeros(1, dtype=torch.int64, device=dev)
    tpu = torch.empty_like(tp)
    _timed("dedup_rows", "b200flow_dedup_rows", ptr(tp), n, stride, key_bytes, ptr(table), ptr(minrow), cap_tab, ptr(slot_of), ptr(rep),
           ptr(flag), ptr(pos), ptr(total), ptr(uid), ptr(tpu))
    if not sync:                       # caller reads the count together with its other device scalars
        return tpu, uid, total
    U = int(total.item())
    return tpu[:U], uid, U


def _i32(a, dev):
    return _lib.h2d(np.ascontiguousarray(a, np.int32), dev)


class InvalidRowsError(ValueError):
    """NaN / null numeric cells or unseen dictionary codes met while assembling rows (VectorAssembler / StringIndexerModel
    handleInvalid="error"); raised when the fused record path meets them — Spark raises at the same point: the action."""


class _DenseSource:
    """training / test rows as a dense CUDA feature matrix x [n, F] (f32/f64) + int32 labels: the materialised
    VectorAssembler output (kdd99.py:46)."""

    def __init__(self, x, labels=None):
        self.x, self.labels = x, (labels.to(torch.int32).contiguous() if labels is not None else None)
        self.n, self.F = x.shape
        self.device = x.device

    def sample(self, seed, keep, row_offset, sample, cap, n_s_dev):
        call("b200flow_sample_rows", ptr(self.x), _lib.dtype_code(self.x), self.n, self.F, self.x.stride(0), seed, keep, int(row_offset),
             ptr(sample), cap, ptr(n_s_dev))

    def bin(self, thresholds, n_thr, arity_dev, mpb, bad, want_label_out=False):
        stride = tp_stride(self.F)
        tp = torch.empty((self.n, stride), dtype=torch.uint8, device=self.device)
        _timed("bin_rows", "b200flow_bin_rows", ptr(self.x), _lib.dtype_code(self.x), self.n, self.F, self.x.stride(0), ptr(thresholds), ptr(n_thr),
               ptr(arity_dev), mpb, ptr(self.labels), ptr(tp), stride, ptr(bad[0:1]))
        return tp, self.labels


class _RecordSource:
    """rows as raw AoS flow records + the encode plan that would assemble their feature vector: sampled and binned
    straight from the records by the fused kernels (SURVEY.md 8d "Encode -> bins"), the dense matrix never exists.
    round_f32: the plan's vector would have been an f32 matrix (only matters for scaled slots, whose f32 rounding the
    bins must see)."""

    def __init__(self, rec, plan, round_f32=False, with_label=True):
        if rec.dtype != torch.uint8 or rec.dim() != 2 or rec.shape[1] != plan.schema.row_bytes:
            raise ValueError("records must be uint8 [n, %d]" % plan.schema.row_bytes)
        self.rec, self.plan, self.round_f32 = rec, plan, 1 if round_f32 else 0
        self.n, self.F = rec.shape[0], plan.n_out
        self.device = rec.device
        self.with_label = with_label and plan.label is not None

    def _thr_f32(self, arity_dev):
        """1 when every slot's value is exactly a float (f32 fields / ranks / one-hot flags unscaled, or an f32 matrix being
        emulated): the fused kernel may then search float thresholds (rounded down) — the same bins, half the bytes."""
        if self.round_f32:
            return 1
        return 1 if all(s[0] in (_lib.SRC_F32, _lib.SRC_INDEX, _lib.SRC_ONEHOT) and s[5] == 0.0 and s[6] == 1.0 for s in self.plan.slots) else 0

    def sample(self, seed, keep, row_offset, sample, cap, n_s_dev):
        _, slots, lut_t, _ = self.plan._device_tables(self.device)
        call("b200flow_sample_records", ptr(self.rec), self.n, self.plan.schema.row_bytes, ptr(slots), self.F, ptr(lut_t), self.round_f32,
             seed, keep, int(row_offset), ptr(sample), cap, ptr(n_s_dev))

    def bin(self, thresholds, n_thr, arity_dev, mpb, bad, want_label_out=False):
        _, slots, lut_t, lut_total = self.plan._device_tables(self.device)
        stride = tp_stride(self.F)
        tp = torch.empty((self.n, stride), dtype=torch.uint8, device=self.device)
        loff, llo, lln = self.plan.label if self.with_label else (-1, 0, 0)
        lab = torch.empty(self.n, dtype=torch.int32, device=self.device) if (want_label_out and self.with_label) else None
        _timed("encode_bins", "b200flow_encode_bins", ptr(self.rec), self.n, self.plan.schema.row_bytes, ptr(slots), self.F, ptr(lut_t), lut_total,
               loff, llo, lln, int(self.plan.check_nan), self.round_f32, self._thr_f32(arity_dev), ptr(thresholds), ptr(n_thr), ptr(arity_dev), mpb, ptr(tp), stride,
               ptr(lab), ptr(bad))
        return tp, lab


class ForestModel:
    """Device-resident forest: one node pool for all trees (roots = nodes 0..T-1)."""

    def __init__(self, T, C, F, arity, max_bins, thresholds, n_thr, nodes, node_mask, pool_counts, node_tree,
                 leaf_prob, node_gain, n_nodes, dt_mode):
        self.T, self.C, self.F, self.max_bins, self.dt_mode = T, C, F, max_bins, dt_mode
        self.arity = np.asarray(arity, np.int32)
        self.thresholds, self.n_thr = thresholds, n_thr          # device [F, max_bins-1] f64, [F] i32
        self.nodes, self.node_mask, self.pool_counts = nodes, node_mask, pool_counts
        self.node_tree, self.leaf_prob, self.node_gain, self.n_nodes = node_tree, leaf_prob, node_gain, n_nodes
        self._arity_dev = _i32(self.arity, thresholds.device)

    def bin(self, x, labels=None):
        """TreePoint.findBin (R5) with this model's thresholds: dense [n, F] -> uint8 [n, stride]."""
        n, F = x.shape
        if F != self.F:
            raise ValueError("expected %d features, got %d" % (self.F, F))
        bad = torch.zeros(2, dtype=torch.int32, device=x.device)
        tp, _ = _DenseSource(x, labels).bin(self.thresholds, self.n_thr, self._arity_dev, self.max_bins, bad)
        return tp, bad[0:1]

    def _top_table(self):
        """the first TOP_LEVELS levels of every tree, heap-indexed by node id, for the grid predict kernel's shared-memory
        stage (built once per model)."""
        if TOP_LEVELS <= 0:
            return None, 0
        if getattr(self, "_top", None) is None:
            self._top = torch.zeros((self.T << TOP_LEVELS, 4), dtype=torch.int32, device=self.nodes.device)
            call("b200flow_build_top_nodes", ptr(self.nodes), ptr(self.node_tree), self.n_nodes, self.T, TOP_LEVELS, ptr(self._top))
        return self._top, TOP_LEVELS

    def _forest_layout(self):
        """(layout uint64 [words], tree_off int64 [T+1]): every tree's nodes, left-set masks and leaf votes in one contiguous
        block, which the predict kernel stages whole in shared memory (built once per model; one host read of the size)."""
        if getattr(self, "_layout", None) is None:
            dev = self.nodes.device
            scratch = torch.empty(2 * self.n_nodes + 4 * self.T, dtype=torch.int32, device=dev)
            tree_off = torch.empty(self.T + 1, dtype=torch.int64, device=dev)
            call("b200flow_forest_layout_size", ptr(self.nodes), ptr(self.node_tree), self.n_nodes, self.T, self.C, ptr(scratch),
                 ptr(tree_off))
            layout = torch.empty(max(int(tree_off[self.T].item()), 2), dtype=torch.int64, device=dev)
            call("b200flow_build_forest_layout", ptr(self.nodes), ptr(self.node_mask), ptr(self.leaf_prob), ptr(self.pool_counts),
                 ptr(self.node_tree), self.n_nodes, self.T, self.C, 1 if self.dt_mode else 0, ptr(scratch), ptr(tree_off),
                 ptr(layout))
            self._layout = (layout, tree_off)
        return self._layout

    def predict_binned(self, tp, want_raw=True, want_prob=True):
        n = tp.shape[0]
        dev = tp.device
        raw = torch.empty((n, self.C), dtype=torch.float64, device=dev) if want_raw else None
        prob = torch.empty((n, self.C), dtype=torch.float64, device=dev) if want_prob else None
        pred = torch.empty(n, dtype=torch.float64, device=dev)
        if n == 0:
            return raw, prob, pred
        layout, tree_off = self._forest_layout()
        _timed("predict", "b200flow_predict_forest", ptr(tp), tp.shape[1], self.F, n, ptr(layout), ptr(tree_off), self.T, self.C,
               ptr(raw), ptr(prob), ptr(pred))
        return raw, prob, pred

    def predict(self, x, want_raw=True, want_prob=True):
        """RandomForestClassificationModel.transform (R9): rawPrediction, probability, prediction.  The trees are walked
        once per UNIQUE binned record; the results are then spread back to the rows.  A categorical value outside
        [0, arity) is binned to `arity` (at most 255, see build_metadata), which no left set contains, so it goes right at
        every split on that feature — what MLlib's CategoricalSplit.shouldGoLeft does with an unseen category when the
        split's left set holds at most half of the categories."""
        tp, _ = self.bin(x)
        return self._predict_tp(tp, want_raw, want_prob)

    def predict_records(self, rec, plan, want_raw=True, want_prob=True, round_f32=False, want_label=False, on_invalid="ignore"):
        """the same from raw flow records + the encode plan of the feature vector (fused encode -> bins, no dense matrix).
        -> (raw, prob, pred, label int32 | None).  on_invalid="error": NaN cells (plan.check_nan) / unseen codes raise."""
        src = _RecordSource(rec, plan, round_f32, with_label=want_label)
        if src.F != self.F:
            raise ValueError("expected %d features, got %d" % (self.F, src.F))
        bad = torch.zeros(2, dtype=torch.int32, device=rec.device)
        tp, lab = src.bin(self.thresholds, self.n_thr, self._arity_dev, self.max_bins, bad, want_label_out=want_label)
        out = self._predict_tp(tp, want_raw, want_prob, bad if on_invalid == "error" else None)
        return out + (lab,)

    def _predict_tp(self, tp, want_raw=True, want_prob=True, bad=None):
        n = tp.shape[0]
        if not DEDUP or n == 0:
            if bad is not None and int(bad[1].item()):
                raise InvalidRowsError("%d NaN/null cells or unseen labels in the rows to transform" % int(bad[1].item()))
            return self.predict_binned(tp, want_raw, want_prob)
        tpu, uid, u_dev = dedup_rows(tp, self.F, sync=False)  # the label byte is not part of a test record's identity
        head = (torch.cat([u_dev, bad.to(torch.int64)]) if bad is not None else u_dev).cpu()    # ONE host read
        if bad is not None and int(head[2]):
            raise InvalidRowsError("%d NaN/null cells or unseen labels in the rows to transform" % int(head[2]))
        U = int(head[0])
        raw_u, prob_u, pred_u = self.predict_binned(tpu[:U], want_raw, want_prob)

        def spread(src, width):
            if src is None:
                return None
            out = torch.empty((n, width) if width > 1 else (n,), dtype=torch.float64, device=tp.device)
            call("b200flow_gather_rows", ptr(src), 8 * width, ptr(uid), n, ptr(out))
            return out
        return spread(raw_u, self.C), spread(prob_u, self.C), spread(pred_u, 1)

    def grid_confusion(self, x_or_records, tree_cuts, depth_cuts, labels=None, plan=None, round_f32=False, cm_side=None,
                       group=None, max_depth_cuts_per_launch=0):
        """confusion matrices of every truncated forest on labelled validation rows: -> int64 [I, J, S, S] (host), where
        [i, j] counts (label, prediction) of the first tree_cuts[i] trees cut at depth depth_cuts[j] — exactly what
        confusion_matrix(predict(...)) gives for the (tree_cuts[i], depth_cuts[j]) forest fitted on its own (DESIGN.md §5a).
        Dense path: x [n, F] and int labels [n]; record path: raw records + an encode plan with its label column set.
        S = max(C, cm_side); labels >= S are not counted.  Under torch.distributed the counts are summed over the ranks."""
        from . import dist as bdist
        tree_cuts = np.ascontiguousarray(sorted(set(int(t) for t in tree_cuts)), np.int32)
        depth_cuts = np.ascontiguousarray(sorted(set(int(d) for d in depth_cuts)), np.int32)
        if plan is None:
            if labels is None:
                raise ValueError("grid_confusion: the dense path needs the labels")
            src = _DenseSource(x_or_records, labels)
        else:
            if plan.label is None:
                raise ValueError("grid_confusion: the encode plan has no label column (EncodePlan.set_label)")
            src = _RecordSource(x_or_records, plan, round_f32)
        if src.F != self.F:
            raise ValueError("expected %d features, got %d" % (self.F, src.F))
        S = max(self.C, int(cm_side or 0))
        dev = src.device
        cm = torch.zeros((len(tree_cuts), len(depth_cuts), S, S), dtype=torch.int64, device=dev)
        n = src.n
        if n > 0:
            bad = torch.zeros(2, dtype=torch.int32, device=dev)
            tp, _ = src.bin(self.thresholds, self.n_thr, self._arity_dev, self.max_bins, bad)
            tpu, uid, U = dedup_rows(tp, self.F + 1)        # a validation record's identity includes its label
            gsize = torch.empty(U, dtype=torch.int32, device=dev); cursor = torch.empty(U, dtype=torch.int32, device=dev)
            goff = torch.empty(U + 1, dtype=torch.int64, device=dev)
            perm = torch.empty(n, dtype=torch.int32, device=dev); uperm = torch.empty(n, dtype=torch.int32, device=dev)
            _timed("group_rows", "b200flow_group_rows", ptr(uid), n, U, ptr(gsize), ptr(goff), ptr(cursor), ptr(perm), ptr(uperm))
            top, K = self._top_table()
            _timed("predict_grid", "b200flow_predict_grid_confusion", ptr(tpu), tpu.shape[1], self.F, U, ptr(gsize), ptr(self.nodes),
                   ptr(self.node_mask), ptr(self.leaf_prob), ptr(self.pool_counts), self.T, self.C, 1 if self.dt_mode else 0,
                   ptr(top), K, tree_cuts.ctypes.data, len(tree_cuts), depth_cuts.ctypes.data, len(depth_cuts), S,
                   int(max_depth_cuts_per_launch), ptr(cm))
        return bdist.all_reduce_sum_(cm, group).cpu()

    GRID_SCORE_BUDGET = 2 << 30            # bytes of [tree cuts, J, U] fp64 scores per grid_binary_metrics block

    def grid_binary_metrics(self, x_or_records, tree_cuts, depth_cuts, labels=None, plan=None, num_bins=1000, group=None,
                            round_f32=False, max_depth_cuts_per_launch=0):
        """areaUnderROC / areaUnderPR of every truncated forest on labelled validation rows: -> float64 [I, J, 2] (host), where
        [i, j] is what BinaryClassificationEvaluator(numBins=num_bins) gives on rawPrediction[1] of the (tree_cuts[i],
        depth_cuts[j]) forest fitted on its own (DESIGN.md §5a, §5b).  A row is positive iff its label >= 1.  The rows are
        de-duplicated on (bins, label) with their multiplicities as integer counts, predict_grid_scores writes every grid
        point's score per distinct record, and binary_metrics runs over the I·J segments (in blocks of tree cuts when the
        scores would exceed GRID_SCORE_BUDGET bytes).  Under torch.distributed every rank returns the same bits."""
        from . import dist as bdist
        from .metrics import binary_metrics
        if self.C < 2:
            raise ValueError("grid_binary_metrics: the score is rawPrediction[1], the forest has %d class(es)" % self.C)
        tree_cuts = np.ascontiguousarray(sorted(set(int(t) for t in tree_cuts)), np.int32)
        depth_cuts = np.ascontiguousarray(sorted(set(int(d) for d in depth_cuts)), np.int32)
        if plan is None:
            if labels is None:
                raise ValueError("grid_binary_metrics: the dense path needs the labels")
            src = _DenseSource(x_or_records, labels)
        else:
            if plan.label is None:
                raise ValueError("grid_binary_metrics: the encode plan has no label column (EncodePlan.set_label)")
            src = _RecordSource(x_or_records, plan, round_f32)
        if src.F != self.F:
            raise ValueError("expected %d features, got %d" % (self.F, src.F))
        dev = src.device
        I, J = len(tree_cuts), len(depth_cuts)
        U = 0
        if src.n > 0:
            bad = torch.zeros(2, dtype=torch.int32, device=dev)
            tp, _ = src.bin(self.thresholds, self.n_thr, self._arity_dev, self.max_bins, bad)
            tpu, uid, U = dedup_rows(tp, self.F + 1)        # a validation record's identity includes its label
            tpu = tpu.contiguous()
            gsize = torch.empty(U, dtype=torch.int32, device=dev); cursor = torch.empty(U, dtype=torch.int32, device=dev)
            goff = torch.empty(U + 1, dtype=torch.int64, device=dev)
            perm = torch.empty(src.n, dtype=torch.int32, device=dev); uperm = torch.empty(src.n, dtype=torch.int32, device=dev)
            _timed("group_rows", "b200flow_group_rows", ptr(uid), src.n, U, ptr(gsize), ptr(goff), ptr(cursor), ptr(perm), ptr(uperm))
            positive = tpu[:, self.F] >= 1
            pos = torch.where(positive, gsize, 0).contiguous()
            neg = torch.where(positive, 0, gsize).contiguous()
        else:
            pos = neg = torch.zeros(0, dtype=torch.int32, device=dev)
        mx = torch.tensor([U], dtype=torch.int64, device=dev)   # every rank takes the same blocks: size them by the widest shard
        grp = group if group is not None else bdist.group()
        if grp is not None:
            import torch.distributed as dist
            bdist.all_reduce_(mx, grp, op=dist.ReduceOp.MAX)
        per_cut = J * max(int(mx.item()), 1) * 8
        step = max(1, min(I, self.GRID_SCORE_BUDGET // per_cut))
        out = np.empty((I, J, 2), np.float64)
        top, K = self._top_table()
        for i0 in range(0, I, step):
            cuts = np.ascontiguousarray(tree_cuts[i0:i0 + step])
            scores = torch.empty((len(cuts), J, U), dtype=torch.float64, device=dev)
            if U > 0:
                _timed("predict_grid", "b200flow_predict_grid_scores", ptr(tpu), tpu.shape[1], self.F, U, ptr(self.nodes),
                       ptr(self.node_mask), ptr(self.leaf_prob), ptr(self.pool_counts), self.T, self.C, 1 if self.dt_mode else 0,
                       ptr(top), K, cuts.ctypes.data, len(cuts), depth_cuts.ctypes.data, J, int(max_depth_cuts_per_launch),
                       ptr(scores))
            r = binary_metrics(scores.reshape(len(cuts) * J, U), pos=pos, neg=neg, num_bins=num_bins, group=grp)
            out[i0:i0 + len(cuts), :, 0] = np.asarray(r["areaUnderROC"]).reshape(len(cuts), J)
            out[i0:i0 + len(cuts), :, 1] = np.asarray(r["areaUnderPR"]).reshape(len(cuts), J)
        return out

    def export(self):
        """Canonical host copy, nodes ordered by (tree, MLlib node id) — what parity tests compare."""
        n = self.n_nodes
        nodes = self.nodes[:n].cpu().numpy().view(NODE_DTYPE).reshape(-1)
        tree = self.node_tree[:n].cpu().numpy()
        counts = self.pool_counts[:n].cpu().numpy().view(np.uint32).astype(np.int64)
        mask = (self.node_mask[:n].cpu().numpy().view(np.uint64) if self.node_mask is not None
                else np.zeros((n, 4), np.uint64))
        gain = self.node_gain[:n].cpu().numpy()
        order = np.lexsort((nodes["nid"], tree))
        is_leaf = (nodes["feat"] < 0).astype(np.int32)
        kind = np.where(is_leaf == 1, 0, nodes["kind_bin"] >> 16).astype(np.int32)
        bin_thr = np.where(is_leaf == 1, 0, nodes["kind_bin"] & 0xffff).astype(np.int32)
        mask = np.where(is_leaf[:, None] == 1, 0, mask).astype(np.uint64)
        return dict(tree=tree[order], nid=nodes["nid"][order], feat=nodes["feat"][order], kind=kind[order],
                    bin_thr=bin_thr[order], is_leaf=is_leaf[order], gain=gain[order], mask=mask[order],
                    counts=counts[order])

    def feature_importances(self):
        """TreeEnsembleModel.featureImportances: per tree Σ gain·count over internal nodes, normalised per tree,
        averaged over trees and normalised (host-side, from the canonical export)."""
        ex = self.export()
        imp = np.zeros(self.F)
        for t in range(self.T):
            sel = (ex["tree"] == t) & (ex["is_leaf"] == 0)
            v = np.zeros(self.F)
            np.add.at(v, ex["feat"][sel], ex["gain"][sel] * ex["counts"][sel].sum(1))
            if v.sum() > 0:
                imp += v / v.sum()
        return imp / imp.sum() if imp.sum() > 0 else imp


def _gather_sample(sample, n_s, cap, F, group):
    """all-gather the per-rank findSplits samples (column-major [F, cap]) into one buffer.  The ranks agree on the widest
    sample first and exchange (F, mx) blocks padded to that width — local capacities differ when the shards are uneven."""
    import torch.distributed as dist
    world = dist.get_world_size(group)
    from . import dist as bdist
    counts = [int(c.item()) for c in bdist.all_gather_list(torch.tensor([n_s], dtype=torch.int64, device=sample.device), group)]
    mx = max(max(counts), 1)
    mine = torch.zeros((F, mx), dtype=torch.float64, device=sample.device)
    if n_s > 0:
        mine[:, :n_s] = sample.view(F, cap)[:, :n_s]
    parts = bdist.all_gather_list(mine, group)
    tot = sum(counts)
    new_cap = 1
    while new_cap < max(tot, 2):
        new_cap <<= 1
    out = torch.empty((F, new_cap), dtype=torch.float64, device=sample.device)
    pos = 0
    for p, c in zip(parts, counts):
        out[:, pos:pos + c] = p[:, :c]; pos += c
    return out.view(-1), tot, new_cap


class _TrainingRows:
    """The front half of RandomForest.run, shared by the forest and the GBT trainers: the global row count, the metadata,
    findSplits (R4), binning (R5) and the de-duplication of the binned rows.  The constructor only enqueues device work;
    read() then fetches the bad-cell counts, the bin count, the sample count and the unique-record count in ONE host read, so
    the caller can prepare what does not depend on them in between, while the GPU works through the queue."""

    def __init__(self, src, num_classes, arity, max_bins, num_trees, strategy, seed, row_offset, group, key_bytes=None,
                 dedup=None):
        """key_bytes: the record bytes de-duplication compares (default F + 1: bins and label byte); dedup=False keeps the
        binned rows as they are (default: DEDUP)"""
        from . import dist as bdist
        dev = src.device
        n, F, C, T = src.n, src.F, num_classes, num_trees
        n_global = n
        if group is not None:
            t = torch.tensor([n], dtype=torch.int64, device=dev)
            bdist.all_reduce_(t, group)
            n_global = int(t.item())
        mpb, kind, m = build_metadata(n_global, F, C, arity, max_bins, T, strategy)
        arity = np.asarray(arity, np.int32)
        arity_dev = _i32(arity, dev)

        # ---- R4 findSplits: Bernoulli row sample keyed by global row, sort + stride walk on device
        has_cont = bool((arity == 0).any())
        frac = min(1.0, max(mpb * mpb, 10000) / float(max(n_global, 1))) if has_cont else 1.0
        keep = int(frac * 4294967296.0)
        expect = n if frac >= 1.0 else int(n * frac + 6.0 * math.sqrt(max(n * frac, 1.0)) + 64)
        cap = 1
        while cap < max(min(expect, n), 2):
            cap <<= 1
        sample = torch.empty(F * cap, dtype=torch.float64, device=dev)
        n_s_dev = torch.zeros(1, dtype=torch.int32, device=dev)
        thresholds = torch.zeros((F, mpb - 1), dtype=torch.float64, device=dev)
        n_thr = torch.zeros(F, dtype=torch.int32, device=dev)
        if has_cont:
            src.sample(seed, keep, row_offset, sample, cap, n_s_dev)
            if group is not None:
                n_s = int(n_s_dev.item())
                if n_s > cap:
                    raise B200FlowError("findSplits sample overflow (%d > %d)" % (n_s, cap))
                sample, n_s, cap = _gather_sample(sample, n_s, cap, F, group)
                call("b200flow_find_splits", ptr(sample), cap, n_s, F, ptr(arity_dev), mpb, ptr(thresholds), ptr(n_thr), None)
            else:       # single GPU: the sample count stays on the device (checked with the other counts below: one host sync)
                call("b200flow_find_splits", ptr(sample), cap, cap, F, ptr(arity_dev), mpb, ptr(thresholds), ptr(n_thr), ptr(n_s_dev))
        del sample

        # ---- R5 binning (dense matrix: bin_rows; raw records: the fused encode -> bins kernel)
        bad = torch.zeros(2, dtype=torch.int32, device=dev)
        tp, _ = src.bin(thresholds, n_thr, arity_dev, mpb, bad)
        feat_bins = torch.where(arity_dev > 0, arity_dev, n_thr + 1).to(torch.int32).contiguous()
        feat_kind = _i32(kind, dev)
        # ---- de-duplicate the binned rows: the level loop runs on UNIQUE TreePoint records carrying summed bag weights.
        # Everything is enqueued first; ONE host read then fetches the bad-cell counts, the bin count, the sample count and U.
        dedup = n > 0 and (DEDUP if dedup is None else bool(dedup))
        if dedup:
            tp, uid, u_dev = dedup_rows(tp, F + 1 if key_bytes is None else key_bytes, sync=False)
        else:
            uid, u_dev = None, torch.full((1,), n, dtype=torch.int64, device=dev)
        self.src, self.group, self.n, self.F, self.n_global = src, group, n, F, n_global
        self.mpb, self.kind, self.m, self.arity, self.arity_dev = mpb, kind, m, arity, arity_dev
        self.has_cont, self.cap, self.n_s_dev, self.thresholds, self.n_thr = has_cont, cap, n_s_dev, thresholds, n_thr
        self.bad, self.tp, self.feat_bins, self.feat_kind = bad, tp, feat_bins, feat_kind
        self.dedup, self.uid, self.u_dev = dedup, uid, u_dev

    def read(self):
        """-> self with n_bins (the widest feature's bin count), U (unique records) and tp trimmed to them; head = the host copy
        of [bad cells, NaN cells, n_bins, sample count, U, feat_bins...]."""
        bad, feat_bins, n_s_dev, u_dev, tp, F = self.bad, self.feat_bins, self.n_s_dev, self.u_dev, self.tp, self.F
        has_cont, group, cap, dedup, dev = self.has_cont, self.group, self.cap, self.dedup, self.src.device
        stride = tp_stride(F)
        head = torch.cat([bad.to(torch.int64), feat_bins.max().reshape(1).to(torch.int64), n_s_dev.to(torch.int64), u_dev,
                          feat_bins.to(torch.int64)]).cpu()
        if int(head[1]) != 0:
            raise InvalidRowsError("%d NaN/null cells or unseen labels in the training rows" % int(head[1]))
        if int(head[0]) != 0:
            raise ValueError("categorical feature value outside [0, arity) or non-integral in %d cells" % int(head[0]))
        if has_cont and group is None and int(head[3]) > cap:
            raise B200FlowError("findSplits sample overflow (%d > %d)" % (int(head[3]), cap))
        n_bins, U = int(head[2]), int(head[4])
        if dedup:
            tp = tp[:U]
        if tp.shape[0] == 0:                                  # a rank without rows still walks the level loop (its collectives): give the
            tp = torch.zeros((1, stride), dtype=torch.uint8, device=dev)   # kernels a real pointer (data_ptr() of an empty tensor is NULL)
        self.head, self.n_bins, self.U, self.tp = head, n_bins, U, tp
        return self


class Bag:
    """the entries {unique record, weight} of T weight rows W [T][U]: the non-zero weights, tree-major and in unique-id order.
    count() enqueues bag_count (the non-zeros of every 1024-record block) and its scan into the block offsets, whose total
    (the entry count) stays on the device; fill() writes the entries.  Tree t's entries are [blk_off[t·nb], blk_off[(t+1)·nb])."""

    def __init__(self, T, U, dev):
        self.T, self.U, self.nb = T, U, (U + 1023) // 1024
        self.blk_cnt = torch.zeros(max(T * self.nb, 1), dtype=torch.int32, device=dev)
        self.blk_off = torch.zeros(T * self.nb + 1, dtype=torch.int64, device=dev)
        self.total = torch.zeros(1, dtype=torch.int64, device=dev)

    def count(self, W):
        if self.U > 0:
            call("b200flow_bag_count", ptr(W), self.T, self.U, ptr(self.blk_cnt))
        call("b200flow_exclusive_scan_i32_to_i64", ptr(self.blk_cnt), self.T * self.nb, ptr(self.blk_off), ptr(self.total))

    def fill(self, W, ent):
        if self.U > 0:
            call("b200flow_bag_fill", ptr(W), self.T, self.U, ptr(self.blk_off), ptr(ent))

    def segments(self):
        """-> (seg_begin, seg_end) int64 [T]: every tree's entry range, one level-0 slot per tree"""
        idx = torch.arange(self.T, dtype=torch.int64, device=self.blk_off.device) * self.nb
        return self.blk_off[idx].contiguous(), self.blk_off[idx + self.nb].contiguous()


def chunk_table(lens):
    """(device offsets int64 [ns + 1], their host copy) of the CHUNK_ROWS-entry chunks of slots holding lens [ns] entries: the
    chunk table of hist_level, partition_level and their variance-tree forms (one host read)"""
    nch = ((lens + (CHUNK_ROWS - 1)) // CHUNK_ROWS).to(torch.int32).contiguous()
    off = torch.empty(nch.shape[0] + 1, dtype=torch.int64, device=lens.device)
    call("b200flow_exclusive_scan_i32_to_i64", ptr(nch), nch.shape[0], ptr(off), None)
    return off, off.cpu()


class NodePool:
    """the growing node pool of a fit: roots 0..n_roots-1, and per node the statistics grow_level copies from the scored
    slots — int32 [cap, C] class counts for the forest, int64 [cap, 3] {Σw, Σw·q, Σw·q2} for the variance trees.  grow_level
    sees them as opaque 32-bit words."""

    def __init__(self, n_roots, cap, with_mask, stat_width, stat_dtype, dev):
        self.dev, self.cap, self.size = dev, cap, n_roots
        self.nodes = torch.zeros((cap, 16), dtype=torch.uint8, device=dev)
        self.node_mask = torch.zeros((cap, 4), dtype=torch.int64, device=dev) if with_mask else None
        self.stats = torch.zeros((cap, stat_width), dtype=stat_dtype, device=dev)
        self.node_tree = torch.zeros(cap, dtype=torch.int32, device=dev)
        self.node_gain = torch.zeros(cap, dtype=torch.float64, device=dev)
        root = np.zeros(n_roots, NODE_DTYPE); root["feat"] = -1; root["left"] = -1; root["nid"] = 1
        self.nodes[:n_roots] = _lib.h2d(root.view(np.uint8).reshape(n_roots, 16), dev)
        self.node_tree[:n_roots] = torch.arange(n_roots, dtype=torch.int32, device=dev)
        self.counters = None

    def grow(self, need):
        if need <= self.cap:
            return
        new_cap = self.cap
        while new_cap < need:
            new_cap *= 2

        def ext(t):
            nt = torch.zeros((new_cap,) + tuple(t.shape[1:]), dtype=t.dtype, device=self.dev)
            nt[:self.cap] = t
            return nt
        self.nodes, self.stats, self.node_tree, self.node_gain = ext(self.nodes), ext(self.stats), ext(self.node_tree), ext(self.node_gain)
        if self.node_mask is not None:
            self.node_mask = ext(self.node_mask)
        self.cap = new_cap

    def grow_level(self, n_slots, slot_tree, slot_nid, slot_node, split, node_st, left_st, right_st, next_tree, next_nid,
                   next_node, next_parent, child_slot=None):
        """enqueue grow_level: the slots' nodes are written and their children appended (the pool first grows to hold them).
        The counters [pool size, n_next, overflow, pool size before, route chunks, ...] + per-block scratch live across levels:
        the pool size carries over on the device, everything else is rewritten by grow_level / the scans, so they are only
        re-allocated when a level needs more scratch (no per-level fill launches).  commit() takes their host copy."""
        self.grow(self.size + 2 * n_slots)
        nblk = (n_slots + 255) // 256
        if self.counters is None or self.counters.numel() < 8 + nblk + 1:
            fresh = torch.zeros(8 + 2 * nblk + 1024, dtype=torch.int64, device=self.dev)
            if self.counters is None:
                fresh[0:1].fill_(self.size)
            else:
                fresh[:8] = self.counters[:8]
            self.counters = fresh
        words = self.stats.shape[1] * self.stats.element_size() // 4
        _timed("grow_level", "b200flow_grow_level", n_slots, ptr(slot_tree), ptr(slot_nid), ptr(slot_node), ptr(split), ptr(node_st),
               ptr(left_st), ptr(right_st), words, ptr(self.nodes), ptr(self.node_mask), ptr(self.stats), ptr(self.node_tree),
               self.cap, ptr(next_tree), ptr(next_nid), ptr(next_node), ptr(next_parent), ptr(child_slot), ptr(self.counters))

    def commit(self, cnt):
        """cnt: the host copy of counters[:3] after grow_level -> the number of next-level slots (the pool size moves on)"""
        if int(cnt[2]) != 0:
            raise B200FlowError("node pool overflow (capacity %d)" % self.cap)
        self.size = int(cnt[0])
        return int(cnt[1])

    def model(self, rows, T, leaf, class_counts=False, dt_mode=False):
        """the ForestModel of trees 0..T-1 of this pool, binned as rows, with leaf table leaf [size, C]; class_counts: the
        stats are the class counts the forest's grid predictors and export read"""
        return ForestModel(T, leaf.shape[1], rows.F, rows.arity, rows.mpb, rows.thresholds, rows.n_thr, self.nodes,
                           self.node_mask, self.stats if class_counts else None, self.node_tree, leaf, self.node_gain,
                           self.size, dt_mode)


def fit_forest(x, labels, num_classes, arity, params, row_offset=0, group=None):
    """RandomForest.run (R4-R8) on a dense CUDA feature matrix x [n, F] (f32/f64) and int32 labels [n].

    arity[f] = 0 for a continuous feature, else the number of categories (from the StringIndexer's
    nominal metadata, SURVEY.md F7).  With `group`, x/labels are this rank's row shard starting at
    global row `row_offset`.  Returns a ForestModel."""
    return _fit(_DenseSource(x, labels), num_classes, arity, params, row_offset, group)


def fit_forest_records(rec, plan, num_classes, arity, params, row_offset=0, group=None, round_f32=False):
    """the same on raw flow records [n, row_bytes] + the encode plan of their feature vector (plan.label = the label
    column): findSplits samples and TreePoint bins come straight from the records (fused encode -> bins)."""
    if plan.label is None:
        raise ValueError("fit_forest_records: the encode plan has no label column (EncodePlan.set_label)")
    return _fit(_RecordSource(rec, plan, round_f32), num_classes, arity, params, row_offset, group)


def _fit(src, num_classes, arity, params, row_offset=0, group=None):
    import torch.distributed as dist
    from . import dist as bdist
    _lib.require_cuda()
    p = params
    if p.impurity != "gini":
        raise UnsupportedParamError("impurity=%r: only 'gini' is implemented on the CUDA path" % p.impurity)
    if not (0 <= p.max_depth <= 30):
        raise ValueError("maxDepth must be in [0, 30], got %d" % p.max_depth)
    dev = src.device
    n, F = src.n, src.F
    C = int(num_classes)
    if not (1 <= C <= 256):
        raise ValueError("numClasses must be in [1, 256] (labels are stored as one byte), got %d" % C)
    T = int(p.num_trees)
    seed = int(p.seed) & 0xFFFFFFFFFFFFFFFF
    rows = _TrainingRows(src, C, arity, p.max_bins, T, p.feature_subset_strategy, seed, row_offset, group)
    kind, m, feat_bins, feat_kind = rows.kind, rows.m, rows.feat_bins, rows.feat_kind
    stride = tp_stride(F)
    # host-side preparation that does not depend on the counts runs BEFORE the read, while the GPU works through the queue
    bagging = p.bootstrap and T > 1
    cdf_host = np.ascontiguousarray(poisson_cdf_table(p.subsampling_rate)) if bagging else None
    cdf = _lib.h2d(cdf_host.view(np.int32), dev) if bagging else None
    # node pool, sized so that typical forests never re-allocate
    pool = NodePool(T, max(4096, 4 * T, min(T << (min(p.max_depth, 18) + 1), 1 << 20)), bool((kind > 0).any()), C, torch.int32,
                    dev)
    rows.read()
    n_bins, U, tp, head = rows.n_bins, rows.U, rows.tp, rows.head
    # launch shape of the fused kernel: entries per routing chunk and subset features per pass (wide nodes — many classes,
    # or a DecisionTree's all-feature histograms — are accumulated in several feature passes, the first of which routes)
    desc_host, rec_bytes = _lib.packed_layout(head[5:5 + F].numpy(), C) if FUSED else (None, 0)
    cfg = _lib.route_hist_config(F, m, n_bins, C, rec_bytes) if FUSED else None
    fused = cfg is not None
    route_ch, m_pass = cfg if fused else (CHUNK_ROWS, m)
    route_passes = -(-m // m_pass)
    hsz = m * n_bins * C
    # the fused kernel gathers bit-packed records when they save a 16-byte granule (KDD: 32 instead of 48 bytes staged);
    # everything else (the unfused kernels, predict) keeps reading the byte records
    rec_tp, rec_stride, field_desc = tp, stride, None
    if fused and rec_bytes:
        field_desc = _lib.h2d(desc_host, dev)
        rec_tp, rec_stride = pack_records(tp, F, field_desc, rec_bytes), rec_bytes
    # ---- R6 bagging: W[tree][unique] = summed Poisson weights; entries = non-zero (unique, weight) pairs per tree
    W = bag_weights(rows, T, cdf_host, cdf, True, seed, row_offset)
    bag = Bag(T, U, dev)
    bag.count(W)
    # the entry count E stays on the device when its upper bound T * U (every record drawn by every tree) is affordable:
    # one host round trip less; the exact count is read with the last level's counters
    E = T * U if T * U * 16 <= ENTRY_BOUND_BYTES else int(bag.total.item())
    ent = torch.empty((max(E, 1), 2), dtype=torch.int32, device=dev)     # {unique record index, weight}
    ent2 = torch.empty_like(ent)
    bag.fill(W, ent)
    del W
    rows.uid = None                    # the row -> record map is not needed past the bag weights
    # ---- level 0 slots: one per tree
    slot_tree = torch.arange(T, dtype=torch.int32, device=dev)
    slot_nid = torch.ones(T, dtype=torch.int32, device=dev)
    slot_node = torch.arange(T, dtype=torch.int32, device=dev)
    seg_begin, seg_end = bag.segments()
    n_slots = T
    level = 0
    per_slot_hist = m * n_bins * C * 4
    group_slots = max(1, HIST_BUDGET_BYTES // per_slot_hist)
    stats = dict(levels=0, slots=0, entries=0, hist_launches=0, rows=n, unique_rows=U)

    stats["route_chunk"], stats["route_passes"] = route_ch if fused else 0, route_passes if fused else 0
    stats["record_format"], stats["record_bytes"] = ("packed", rec_bytes) if field_desc is not None else ("bytes", stride)

    def level_subsets(ns, s_tree, s_nid):
        sub = torch.empty((ns, m), dtype=torch.int16, device=dev)
        call("b200flow_feature_subsets", seed, ns, ptr(s_tree), ptr(s_nid), F, m, ptr(sub))
        return sub

    def plan_route(ns, split_, begin_, end_, total_out, s_node=None, gain_out=None, cursors_=None):
        """enqueue the chunk table of a fused routing pass (+ the gains of the scored nodes, + zeroed partition cursors); the
        chunk count lands in the device scalar `total_out`."""
        nch = torch.empty(ns, dtype=torch.int32, device=dev)
        call("b200flow_plan_route", ns, ptr(split_), ptr(begin_), ptr(end_), route_ch, ptr(s_node), ptr(gain_out), ptr(nch), ptr(cursors_))
        roff = torch.empty(ns + 1, dtype=torch.int64, device=dev)
        call("b200flow_exclusive_scan_i32_to_i64", ptr(nch), ns, ptr(roff), ptr(total_out))
        if PROFILE is not None:
            PROFILE.setdefault("_route_entries", []).append(torch.where(nch > 0, end_ - begin_, torch.zeros_like(end_)).sum())
        return roff

    route_chunks_max = E // route_ch + 1                 # + one ragged chunk per parent slot, added per call

    world = dist.get_world_size(group) if group is not None else 1
    rank = dist.get_rank(group) if group is not None else 0
    REC = 64 + 12 * C                                    # bytes per slot of the scored result: split record + 3 count vectors
    use_rs = world > 1 and bdist.is_nccl(group)          # reduce-scatter + sharded scoring needs NCCL (gloo test groups all-reduce)

    def score_sharded(h_full, gs, sub, lvl, split_, nc_, lc_, rc_):
        """R7r + R8 over `world` ranks: reduce-scatter the level histograms by node block, score this rank's block, all-gather
        the results.  The level is cut into RS_CHUNKS slot ranges whose reduce-scatters are all enqueued first (NCCL's own
        stream), so chunk k is scored while chunk k+1 is still on the wire; the 64 + 12 C byte results travel back in one
        asynchronous all-gather per chunk.  h_full holds the level's slots + world - 1 slots of zero padding."""
        K = int(max(1, min(RS_CHUNKS, gs, (gs * hsz * 4) // max(RS_MIN_BYTES, 1))))
        bounds = [gs * i // K for i in range(K + 1)]
        ev0 = None
        if PROFILE is not None:
            ev0 = torch.cuda.Event(enable_timing=True); ev0.record()
        jobs = []
        for k in range(K):
            s0, g = bounds[k], bounds[k + 1] - bounds[k]
            per = -(-g // world)
            mine = torch.empty(per * hsz, dtype=torch.int32, device=dev)
            # rank r reduces slots [s0 + r * per, s0 + (r + 1) * per); whatever lies beyond the chunk's g slots is ignored
            w = dist.reduce_scatter_tensor(mine, h_full[s0 * hsz:(s0 + world * per) * hsz], group=group, async_op=True)
            jobs.append((s0, g, per, mine, w))
        gathers = []
        for s0, g, per, mine, w in jobs:
            w.wait()
            lo = rank * per
            cnt = max(0, min(per, g - lo))
            local = torch.empty(per * REC, dtype=torch.uint8, device=dev)
            sec = [local[:per * 64], local[per * 64:per * (64 + 4 * C)], local[per * (64 + 4 * C):per * (64 + 8 * C)], local[per * (64 + 8 * C):]]
            if cnt > 0:
                _timed("score_level", "b200flow_score_level", ptr(mine), cnt, ptr(sub[s0 + lo:s0 + lo + cnt]), m, n_bins, C, ptr(feat_bins),
                       ptr(feat_kind), lvl, p.max_depth, int(p.min_instances_per_node), float(p.min_info_gain), ptr(sec[0]), ptr(sec[1]),
                       ptr(sec[2]), ptr(sec[3]))
            gathered = torch.empty((world, per * REC), dtype=torch.uint8, device=dev)
            gw = dist.all_gather_into_tensor(gathered, local, group=group, async_op=True)
            gathers.append((s0, per, gathered, gw))
        for s0, per, gathered, gw in gathers:               # in chunk order: a chunk's padded tail is overwritten by its successor
            gw.wait()
            o = 0
            for dst, width in ((split_, 64), (nc_.view(torch.uint8), 4 * C), (lc_.view(torch.uint8), 4 * C), (rc_.view(torch.uint8), 4 * C)):
                dst.view(-1)[s0 * width:(s0 + world * per) * width].view(world, per * width).copy_(gathered[:, o:o + per * width])
                o += per * width
        if ev0 is not None:
            ev1 = torch.cuda.Event(enable_timing=True); ev1.record()
            PROFILE.setdefault("level_exchange", []).append((ev0, ev1))

    def run_route(roff, rch_dev, n_parents, split_, child_slot_, cursors_, next_subset_, n_next_cap, route=True):
        """fused pass: route the entries of the planned parent slots to their children and build the children's histograms
        (returns the zero-initialised, now filled, histogram buffer of the next level).  The chunk count stays on the device
        (rch_dev), so the pass can be enqueued before the host knows how many children were created.  route=False builds
        the histograms only (level 0, whose segments do not change; the deepest scored level, whose entries nobody reads)."""
        hist_next = torch.zeros((n_next_cap + world - 1) * hsz, dtype=torch.int32, device=dev)   # + padding for the node-block scatter
        cmax = route_chunks_max + n_parents
        scratch = torch.empty(cmax * 4, dtype=torch.int32, device=dev)
        _timed("route_hist_level", "b200flow_route_hist_level", ptr(rec_tp), rec_stride, F, ptr(field_desc), ptr(ent), ptr(ent2), n_parents,
               ptr(seg_begin), ptr(seg_end), ptr(roff), ptr(rch_dev), cmax, route_ch, ptr(split_), ptr(child_slot_), ptr(cursors_),
               ptr(scratch), ptr(next_subset_), m, n_bins, C, ptr(hist_next), 1 if route else 0)
        _lib.launches += route_passes - 1
        stats["hist_launches"] += route_passes
        return hist_next

    side_stream = torch.cuda.Stream(device=dev)
    host_cnt = torch.empty(5, dtype=torch.int64).pin_memory() if _PIN else None
    subset = level_subsets(n_slots, slot_tree, slot_nid)
    hist_ready = None                  # histogram of the CURRENT level when the fused kernel already built it
    if fused and n_slots * hsz * 4 <= HIST_BUDGET_BYTES:        # (not on E: every rank must take the same collective path)
        # level 0 through the same kernel: T pseudo-parents whose split sends every entry "left" into the tree's root
        pseudo = np.zeros(T, SPLIT_DTYPE); pseudo["bin_thr"] = 255; pseudo["flags"] = 4
        pseudo_t = _lib.h2d(pseudo.view(np.uint8).reshape(T, 64), dev)
        child0 = torch.stack([torch.arange(T, dtype=torch.int32, device=dev),
                              torch.full((T,), -1, dtype=torch.int32, device=dev)], 1).contiguous().view(-1)
        cursors0 = torch.zeros(2 * T, dtype=torch.int32, device=dev)
        rch0 = torch.zeros(1, dtype=torch.int64, device=dev)
        roff0 = plan_route(T, pseudo_t, seg_begin, seg_end, rch0)
        hist_full = run_route(roff0, rch0, T, pseudo_t, child0, cursors0, subset, T, route=False)
        hist_ready = hist_full[:T * hsz]
    while n_slots > 0:
        lens = (seg_end - seg_begin) if hist_ready is None else None   # only the unfused kernels need the lengths on the host side
        n_alloc = n_slots + world - 1                        # room for the padded node blocks of the sharded scoring
        split = torch.empty((n_alloc, 64), dtype=torch.uint8, device=dev)
        node_counts = torch.empty((n_alloc, C), dtype=torch.int32, device=dev)
        left_counts = torch.empty((n_alloc, C), dtype=torch.int32, device=dev)
        right_counts = torch.empty((n_alloc, C), dtype=torch.int32, device=dev)
        chunk_off = None
        if hist_ready is None:
            chunk_off, chunk_h = chunk_table(lens)
        groups = [(0, n_slots)] if hist_ready is not None else \
            [(g0, min(n_slots, g0 + group_slots)) for g0 in range(0, n_slots, group_slots)]
        for g0, g1 in groups:
            gs = g1 - g0
            if hist_ready is not None:
                h = hist_ready
            else:
                h = torch.zeros(gs * hsz, dtype=torch.int32, device=dev)
                gch = int(chunk_h[g1] - chunk_h[g0])
                coff = chunk_off if g0 == 0 and g1 == n_slots else (chunk_off[g0:g1 + 1] - chunk_off[g0]).contiguous()
                # R7 HOT LOOP A (unfused form: level 0, and levels whose histograms exceed the fused budget)
                _timed("hist_level", "b200flow_hist_level", ptr(tp), stride, F, ptr(ent), gs,
                       ptr(seg_begin[g0:g1]), ptr(seg_end[g0:g1]), ptr(coff), gch, CHUNK_ROWS, ptr(subset[g0:g1]), m, n_bins, C, ptr(h))
                stats["hist_launches"] += 1
                if PROFILE is not None:
                    PROFILE.setdefault("_hist_entries", []).append(lens[g0:g1].sum())
            if use_rs and hist_ready is not None and gs * hsz * 4 >= RS_MIN_BYTES:
                score_sharded(hist_full, gs, subset, level, split, node_counts, left_counts, right_counts)
                del h
                continue
            if group is not None:                       # R7r: the one data-path collective
                if PROFILE is not None:
                    ev0 = torch.cuda.Event(enable_timing=True); ev0.record()
                bdist.all_reduce_(h, group)
                if PROFILE is not None:
                    ev1 = torch.cuda.Event(enable_timing=True); ev1.record()
                    PROFILE.setdefault("level_exchange", []).append((ev0, ev1))
            # R8 HOT LOOP B
            _timed("score_level", "b200flow_score_level", ptr(h), gs, ptr(subset[g0:g1]), m, n_bins, C, ptr(feat_bins), ptr(feat_kind),
                   level, p.max_depth, int(p.min_instances_per_node), float(p.min_info_gain), ptr(split[g0:g1]),
                   ptr(node_counts[g0:g1]), ptr(left_counts[g0:g1]), ptr(right_counts[g0:g1]))
            del h
        split, node_counts, left_counts, right_counts = split[:n_slots], node_counts[:n_slots], left_counts[:n_slots], right_counts[:n_slots]
        hist_ready = None
        # grow the pool by this level's children and emit the next level's slots
        next_tree = torch.empty(2 * n_slots, dtype=torch.int32, device=dev)
        next_nid = torch.empty(2 * n_slots, dtype=torch.int32, device=dev)
        next_node = torch.empty(2 * n_slots, dtype=torch.int32, device=dev)
        next_parent = torch.empty(2 * n_slots, dtype=torch.int32, device=dev)
        child_slot = torch.empty(2 * n_slots, dtype=torch.int32, device=dev)
        pool.grow_level(n_slots, slot_tree, slot_nid, slot_node, split, node_counts, left_counts, right_counts, next_tree, next_nid,
                        next_node, next_parent, child_slot)
        counters = pool.counters
        n_cap = 2 * n_slots                              # upper bound on the number of next-level slots
        # (the deepest level has only leaf children: nothing to route, nothing to enqueue ahead)
        speculative = fused and n_cap * hsz * 4 <= HIST_BUDGET_BYTES and level + 1 < p.max_depth
        if not speculative:
            pool.node_gain[slot_node.long()] = split.view(torch.float64)[:, 2]
        if speculative:
            # Everything the next level needs is enqueued NOW with device-side counts (children created, routing chunks);
            # the host reads the counts on a side stream while the routing pass runs, so the GPU never waits for Python.
            cursors = torch.empty(2 * n_slots, dtype=torch.int32, device=dev)       # zeroed by plan_route
            roff = plan_route(n_slots, split, seg_begin, seg_end, counters[4:5], slot_node, pool.node_gain, cursors)
            ev_planned = torch.cuda.Event(); ev_planned.record()
            with torch.cuda.stream(side_stream):
                side_stream.wait_event(ev_planned)
                cnt = counters[:5].to("cpu", non_blocking=True) if host_cnt is None else host_cnt.copy_(counters[:5], non_blocking=True)
                ev_read = torch.cuda.Event(); ev_read.record(side_stream)
            next_subset = level_subsets(n_cap, next_tree, next_nid)
            # children at level + 1 == maxDepth - 1 are scored but never split further into routed nodes: their entries are not written
            hist_next = run_route(roff, counters[4:5], n_slots, split, child_slot, cursors, next_subset, n_cap,
                                  route=level + 2 < p.max_depth)
            next_begin = torch.empty(n_cap, dtype=torch.int64, device=dev)
            next_end = torch.empty(n_cap, dtype=torch.int64, device=dev)
            call("b200flow_next_segments", n_cap, ptr(counters[1:2]), ptr(next_parent), ptr(seg_begin), ptr(seg_end), ptr(cursors),
                 ptr(next_begin), ptr(next_end))
            ev_read.synchronize()
        else:
            cnt = counters[:5].cpu()
        n_next = pool.commit(cnt)
        stats["levels"] += 1; stats["slots"] += n_slots
        if n_next == 0:
            break
        next_tree, next_nid, next_node = next_tree[:n_next], next_nid[:n_next], next_node[:n_next]
        if speculative:
            hist_ready = hist_next[:n_next * hsz]             # only the slots that exist travel through the all-reduce
            hist_full = hist_next                             # (+ zero padding: the reduce-scatter path needs equal node blocks)
            next_subset, next_begin, next_end = next_subset[:n_next], next_begin[:n_next], next_end[:n_next]
        else:
            next_subset = level_subsets(n_next, next_tree, next_nid)
            cursors = torch.zeros(2 * n_slots, dtype=torch.int32, device=dev)
            if chunk_off is None:
                chunk_off, chunk_h = chunk_table(seg_end - seg_begin)
            _timed("partition_level", "b200flow_partition_level", ptr(tp), stride, ptr(ent), ptr(ent2),
                   n_slots, ptr(seg_begin), ptr(seg_end), ptr(chunk_off), int(chunk_h[-1]), CHUNK_ROWS, ptr(split), ptr(cursors))
            next_begin = torch.empty(n_next, dtype=torch.int64, device=dev)
            next_end = torch.empty(n_next, dtype=torch.int64, device=dev)
            call("b200flow_next_segments", n_next, None, ptr(next_parent), ptr(seg_begin), ptr(seg_end), ptr(cursors),
                 ptr(next_begin), ptr(next_end))
        ent, ent2 = ent2, ent
        slot_tree, slot_nid, slot_node, subset = next_tree, next_nid, next_node, next_subset
        seg_begin, seg_end = next_begin, next_end
        n_slots = n_next
        level += 1

    leaf_prob = torch.empty((pool.size, C), dtype=torch.float64, device=dev)
    call("b200flow_finalize_forest", pool.size, ptr(pool.stats), C, ptr(leaf_prob))
    stats["entries"] = int(bag.total.item())
    model = pool.model(rows, T, leaf_prob, class_counts=True, dt_mode=(T == 1 and not p.bootstrap))
    model.train_stats = stats
    model.feat_kind, model.feat_bins, model.n_bins, model.m = kind, feat_bins, n_bins, m
    return model


def confusion_matrix(pred, label, C):
    """MulticlassMetrics counting (R10): int64 [C, C], cm[label, pred]."""
    cm = torch.zeros((C, C), dtype=torch.int64, device=pred.device)
    call("b200flow_confusion", ptr(pred.contiguous()), ptr(label.contiguous()), pred.shape[0], C, ptr(cm))
    return cm


def metrics_from_confusion(cm, metric_label=0.0, beta=1.0):
    """MulticlassMetrics (A.8) + macro-F1 from the C x C counts (host, C^2 numbers).  L = the true labels with support > 0.
    The by-label metrics (…ByLabel) are for metric_label and are left out when it is not in L (Spark's tpByClass(label)
    raises); fMeasure uses beta.  fpr(l) = fp(l) / (N - support(l)) is an IEEE division (0/0 is NaN, as on the JVM)."""
    cm = np.asarray(cm, np.float64)
    N = cm.sum()
    sup = cm.sum(1); predl = cm.sum(0); tp = np.diag(cm)
    labs = sup > 0
    with np.errstate(divide="ignore", invalid="ignore"):
        p = np.where(predl > 0, tp / predl, 0.0)
        r = np.where(sup > 0, tp / sup, 0.0)
        f1 = np.where(p + r > 0, 2 * p * r / (p + r), 0.0)
        b2 = beta * beta
        fb = np.where(p + r > 0, (1 + b2) * p * r / (b2 * p + r), 0.0)
        fpr = (predl - tp) / (N - sup)
    w = sup / N if N else sup
    out = dict(accuracy=float(tp[labs].sum() / N) if N else 0.0,
               weightedPrecision=float((p * w)[labs].sum()), weightedRecall=float((r * w)[labs].sum()),
               f1=float((f1 * w)[labs].sum()), macroF1=float(f1[labs].mean()) if labs.any() else 0.0)
    out.update(weightedTruePositiveRate=out["weightedRecall"], weightedFalsePositiveRate=float((fpr * w)[labs].sum()),
               weightedFMeasure=float((fb * w)[labs].sum()),
               hammingLoss=float((N - tp.sum()) / N) if N else 0.0)
    ml = float(metric_label)
    li = int(ml) if np.isfinite(ml) and ml == int(ml) else -1
    if 0 <= li < cm.shape[0] and labs[li]:
        out.update(truePositiveRateByLabel=float(r[li]), falsePositiveRateByLabel=float(fpr[li]), precisionByLabel=float(p[li]),
                   recallByLabel=float(r[li]), fMeasureByLabel=float(fb[li]))
    return out
