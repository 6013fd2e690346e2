"""BinaryClassificationMetrics on the device (BinaryClassificationEvaluator, DESIGN.md §5b).

binary_metrics() sorts the scores of each segment by the CUDA radix sort of csrc/metrics.cu, groups them by distinct value
with integer positive / negative counts, down-samples to numBins points as Spark does and sums the trapezoids of the ROC
and PR curves sequentially in curve order.  Under torch.distributed each rank reduces its shard to distinct triples, the
triples are all-gathered and reduced once more, so every rank returns the same bits for any world size.

regression_metrics() (RegressionEvaluator, DESIGN.md §5l) sums its per-row terms exactly in 128-bit fixed point on the
device (csrc/regression.cu) and rounds each sum once on the host, so it too is the same bits for any world size.
"""
import math

import numpy as np
import torch

from . import _lib
from . import dist as bdist
from ._lib import call, ptr


class InvalidScoresError(ValueError):
    """a NaN score or an empty dataset: Spark orders NaN arbitrarily and has no area for no rows, so both raise here."""


def _as_segments(t, dtype, name):
    t = t if t.dim() == 2 else t.reshape(1, -1)
    if t.dim() != 2:
        raise ValueError("%s must be [n] or [S, n]" % name)
    return t.to(dtype).contiguous()


def binary_counts(scores, pos, neg):
    """scores [S, n] f64, pos / neg int32 [S, n] or [1, n] (shared) -> distinct (score, pos, neg) per segment in descending
    score order: (d_score [S, n], d_pos [S, n], d_neg [S, n], n_distinct int64 [S], n_nan int64 [1]), all on the device."""
    S, n = scores.shape
    dev = scores.device
    cstride = 0 if pos.shape[0] == 1 else n
    if pos.shape[-1] != n or neg.shape != pos.shape or pos.shape[0] not in (1, S):
        raise ValueError("binary_counts: counts must be [n] or [S, n] like the scores")
    scratch = torch.empty(max(_lib.binary_counts_scratch(S, n), 1), dtype=torch.uint8, device=dev)
    d_score = torch.empty((S, n), dtype=torch.float64, device=dev)
    d_pos = torch.empty((S, n), dtype=torch.int64, device=dev)
    d_neg = torch.empty((S, n), dtype=torch.int64, device=dev)
    nd = torch.empty(S, dtype=torch.int64, device=dev)
    nan = torch.empty(1, dtype=torch.int64, device=dev)
    call("b200flow_binary_counts", ptr(scores), n, ptr(pos), ptr(neg), cstride, S, n, ptr(scratch), scratch.numel(),
         ptr(d_score), ptr(d_pos), ptr(d_neg), n, ptr(nd), ptr(nan))
    return d_score, d_pos, d_neg, nd, nan


def _merge_ranks(d_score, d_pos, d_neg, nd, grp):
    """all-gather every rank's distinct triples (padded to the widest count with zero-count items, which binary_counts
    ignores) and reduce their concatenation: the same triples on every rank, whatever the world size."""
    S = d_score.shape[0]
    import torch.distributed as dist
    dev = d_score.device
    w = d_score.shape[1]
    live = torch.arange(w, device=dev)[None, :] < nd[:, None]
    big = torch.maximum(torch.where(live, d_pos, 0).max(), torch.where(live, d_neg, 0).max()) if w else nd.new_zeros(())
    mx = torch.stack([nd.max(), big])                                     # widest triple count, largest count
    bdist.all_reduce_(mx, grp, op=dist.ReduceOp.MAX)
    cap, largest = (int(v) for v in mx.cpu())
    if largest > 2 ** 31 - 1:                                             # the second pass takes int32 counts
        raise ValueError("binary_metrics: %d rows of one rank share one score; at most 2^31 - 1 are supported" % largest)
    if w >= cap:
        sc, ps, ng = d_score[:, :cap], d_pos[:, :cap], d_neg[:, :cap]
    else:
        sc = torch.zeros((S, cap), dtype=torch.float64, device=dev); sc[:, :w] = d_score
        ps = torch.zeros((S, cap), dtype=torch.int64, device=dev); ps[:, :w] = d_pos
        ng = torch.zeros((S, cap), dtype=torch.int64, device=dev); ng[:, :w] = d_neg
    live = torch.arange(cap, device=dev)[None, :] < nd[:, None]           # entries past n_distinct are not triples
    ps = torch.where(live, ps, 0).to(torch.int32)
    ng = torch.where(live, ng, 0).to(torch.int32)
    sc = torch.where(live, sc, 0.0)
    parts = [bdist.all_gather_list(t.contiguous(), grp) for t in (sc, ps, ng)]
    sc, ps, ng = (torch.cat(p, dim=1).contiguous() for p in parts)         # [S, world * cap], rank-major per segment
    d_score, d_pos, d_neg, nd, _ = binary_counts(sc, ps, ng)
    return d_score, d_pos, d_neg, nd


def binary_metrics(scores, labels=None, pos=None, neg=None, num_bins=1000, group=None, curves=False):
    """areaUnderROC / areaUnderPR of BinaryClassificationMetrics(scoreAndLabels, numBins) per segment.

    scores: CUDA f64 [n] or [S, n].  Either labels ([n] shared by the segments, or [S, n]; a row is positive iff
    label > 0.5) or integer counts pos / neg of the same shapes (a row with pos + neg == 0 is ignored).  num_bins >= 0
    (0: no down-sampling).  group: the process group (default: the torch.distributed world when there is one).
    -> {"areaUnderROC", "areaUnderPR"}: floats for 1-D scores, float64 [S] arrays for 2-D; with curves=True also
    "curves": per segment {"score", "tp", "fp"} int64 / f64 arrays of the curve points, and "P", "N" the totals.
    Raises InvalidScoresError on a NaN score or when no rank has a row with a non-zero count (after a global reduction, so
    every rank raises)."""
    if int(num_bins) < 0:
        raise ValueError("numBins must be >= 0, got %r" % (num_bins,))
    one = scores.dim() == 1
    sc = _as_segments(scores, torch.float64, "scores")
    S, n = sc.shape
    if labels is not None:
        lab = _as_segments(labels, torch.float64, "labels")
        ps = (lab > 0.5).to(torch.int32)
        ng = (1 - ps).to(torch.int32)
    else:
        if pos is None or neg is None:
            raise ValueError("binary_metrics needs labels or pos / neg counts")
        ps, ng = _as_segments(pos, torch.int32, "pos"), _as_segments(neg, torch.int32, "neg")
    if ps.shape[-1] != n:
        raise ValueError("labels / counts must have one entry per score")
    grp = group if group is not None else bdist.group()
    d_score, d_pos, d_neg, nd, nan = binary_counts(sc, ps, ng)
    head = torch.cat([nan, nd.sum().reshape(1)])                         # rows with a non-zero count make distinct scores
    if grp is not None:
        bdist.all_reduce_(head, grp)
    n_nan, n_distinct = (int(v) for v in head.cpu())
    if n_nan:
        raise InvalidScoresError("%d NaN scores: BinaryClassificationEvaluator needs ordered scores" % n_nan)
    if n_distinct == 0:
        raise InvalidScoresError("BinaryClassificationEvaluator: the dataset is empty (no row with a non-zero count)")
    if grp is not None:
        d_score, d_pos, d_neg, nd = _merge_ranks(d_score, d_pos, d_neg, nd, grp)
    cap = max(d_score.shape[1], 1)
    dev = sc.device
    auc = torch.empty((S, 2), dtype=torch.float64, device=dev)
    c_score = torch.empty((S, cap), dtype=torch.float64, device=dev)
    c_tp = torch.empty((S, cap), dtype=torch.int64, device=dev)
    c_fp = torch.empty((S, cap), dtype=torch.int64, device=dev)
    c_n = torch.empty(S, dtype=torch.int64, device=dev)
    work = torch.empty(2 * S * cap, dtype=torch.float64, device=dev)
    call("b200flow_binary_curve", ptr(d_score), ptr(d_pos), ptr(d_neg), d_score.shape[1], ptr(nd), S, int(num_bins), ptr(auc),
         ptr(c_score), ptr(c_tp), ptr(c_fp), ptr(c_n), ptr(work))
    a = auc.cpu().numpy()
    out = {"areaUnderROC": float(a[0, 0]) if one else a[:, 0].copy(), "areaUnderPR": float(a[0, 1]) if one else a[:, 1].copy()}
    if curves:
        k = c_n.cpu().numpy()
        cs, ct, cf = c_score.cpu().numpy(), c_tp.cpu().numpy(), c_fp.cpu().numpy()
        pts = [{"score": cs[s, :k[s]], "tp": ct[s, :k[s]], "fp": cf[s, :k[s]]} for s in range(S)]
        out["curves"] = pts[0] if one else pts
        P = np.array([ct[s, k[s] - 1] if k[s] else 0 for s in range(S)], np.int64)     # the last point counts every row
        N = np.array([cf[s, k[s] - 1] if k[s] else 0 for s in range(S)], np.int64)
        out["P"], out["N"] = (int(P[0]), int(N[0])) if one else (P, N)
    return out


# ------------------------------------------------------------------ RegressionEvaluator (DESIGN.md §5l)
_REG_LIMBS = 4                     # 32-bit limbs of one 128-bit fixed-point sum


def _fixed_shift(max_abs, n_global):
    """grid exponent sh of a term whose all-reduced max |t| is max_abs: rint(t 2^sh) keeps |.| <= 2^(126 - ceil(log2 n)), so
    the sum of n such integers stays below 2^126; 0 for a term that is zero everywhere"""
    if not max_abs > 0.0:
        return 0
    mnt, e = math.frexp(max_abs)
    E = e - 1 if mnt == 0.5 else e                       # max_abs <= 2^E
    return 126 - int(math.ceil(math.log2(max(n_global, 2)))) - E


def _fixed_value(limbs, sh):
    """the double nearest to Σ / 2^sh, from the int64 limb sums [4] of one term (one rounding: int -> float)"""
    total = sum(int(v) << (32 * j) for j, v in enumerate(limbs))
    if total == 0:
        return 0.0
    try:                                                 # Python's int / int is correctly rounded
        return total / (1 << sh) if sh >= 0 else float(total * (1 << -sh))
    except OverflowError:
        return math.copysign(math.inf, total)


def _reg_pass(y, p, mode, mean, n_global, grp):
    """-> (bad row count, [sum of each term]) over every rank's rows, each sum the double nearest to the exact sum of the
    terms on their fixed-point grid"""
    import torch.distributed as dist
    dev = y.device
    n = y.shape[0]
    head = torch.zeros(5, dtype=torch.int64, device=dev)
    call("b200flow_reg_eval_max", ptr(y), ptr(p), n, mode, float(mean), ptr(head))
    if grp is not None:
        bdist.all_reduce_(head, grp, op=dist.ReduceOp.MAX)   # [0] only matters as "any"
    h = head.cpu().numpy()
    if h[0]:
        return 1, None
    K = 4 if mode == 0 else 2
    sh = [_fixed_shift(float(h[1 + k:2 + k].view(np.float64)[0]), n_global) for k in range(K)] + [0] * (4 - K)
    limbs = torch.zeros((4, _REG_LIMBS), dtype=torch.int64, device=dev)
    call("b200flow_reg_eval_sums", ptr(y), ptr(p), n, mode, float(mean), sh[0], sh[1], sh[2], sh[3], ptr(limbs))
    if grp is not None:
        bdist.all_reduce_(limbs, grp)                    # exact: integer sums of the limbs
    L = limbs.cpu().numpy()
    return 0, [_fixed_value(L[k], sh[k]) for k in range(K)]


def regression_metrics(label, pred, group=None, through_origin=False):
    """RegressionMetrics of (prediction, label) rows: {'mse', 'rmse', 'mae', 'var', 'r2'}.  Each sum is exact in 128-bit
    fixed point and rounded once, the label mean comes from one such sum, and (y - ȳ)² / (ŷ - ȳ)² are computed per row in fp64
    without FMA: the result is the same bits for any world size or shard layout.  A non-finite label or prediction (or a
    term that overflows) makes every metric NaN; no rows give NaN."""
    _lib.require_cuda()
    y = label.to(torch.float64).reshape(-1).contiguous()
    p = pred.to(torch.float64).reshape(-1).contiguous()
    if y.shape[0] != p.shape[0]:
        raise ValueError("%d labels for %d predictions" % (y.shape[0], p.shape[0]))
    grp = group if group is not None else bdist.group()
    cnt = torch.tensor([y.shape[0]], dtype=torch.int64, device=y.device)
    if grp is not None:
        bdist.all_reduce_(cnt, grp)
    n = int(cnt.item())
    nan = float("nan")
    if n == 0:
        return dict(mse=nan, rmse=nan, mae=nan, var=nan, r2=nan)
    if n >= (1 << 31):
        raise ValueError("RegressionEvaluator: more than 2^31 - 1 rows")
    bad, s0 = _reg_pass(y, p, 0, 0.0, n, grp)
    if bad:
        return dict(mse=nan, rmse=nan, mae=nan, var=nan, r2=nan)
    sy, syy, sserr, sabs = s0
    mean = sy / n
    bad, s1 = _reg_pass(y, p, 1, mean, n, grp)
    if bad:
        return dict(mse=nan, rmse=nan, mae=nan, var=nan, r2=nan)
    sstot, ssreg = s1
    mse = sserr / n
    den = syy if through_origin else sstot
    if den != 0.0:
        r2 = 1.0 - sserr / den
    else:                                                # Java double division: 0/0 = NaN, x/0 = inf
        r2 = nan if sserr == 0.0 else -math.inf
    return dict(mse=mse, rmse=math.sqrt(mse), mae=sabs / n, var=ssreg / n, r2=r2)
