"""Per-column statistics, exact quantiles and the column transforms of the preprocessing stages on the device (Imputer,
RobustScaler, MinMaxScaler, MaxAbsScaler, QuantileDiscretizer, Bucketizer and DataFrame.approxQuantile; DESIGN.md §5s,
csrc/quantile.cu).  Columns are read in place: a contiguous or strided [n] / [n, D] tensor (f32, f64 or i32) or fields of
the raw AoS records.  Every result is a function of integer all-reduces (counts, ordered keys, fixed-point limbs, digit
histograms), so it is the same bits for any world size and shard layout.

Spark [recalled; Spark 3 `ml/feature/Imputer.scala`, `RobustScaler.scala`, `MinMaxScaler.scala`, `MaxAbsScaler.scala`,
`QuantileDiscretizer.scala`, `Bucketizer.scala`, `sql/DataFrameStatFunctions.scala`, `catalyst/util/QuantileSummaries.scala`]:

    Quantiles: approxQuantile ignores NaN and null.  For an exact sample QuantileSummaries.query(q) returns the element of
    rank r = ceil(q n) (1-based, in Double.compare order), the minimum when q <= 0 or r == 0.  The product is fp64:
    0.14 * 50 = 7.000000000000001, so q = 0.14 of 50 values is the 8th (while 0.7 * 10 is exactly 7.0, the 7th).
    A column without a value gives no quantiles ([]).  Probabilities must lie in [0, 1].  The sketch may return any
    element within relativeError * n ranks of the target; the exact element always satisfies that, so relativeError is
    validated to [0, 1] and then has no effect here.
    Imputer: the surrogate of a column is computed from its values that are neither NaN nor missingValue: mean = sum /
    count, median = the q = 0.5 element, mode = the most frequent value, the smallest on ties (-0.0 counts as 0.0).  No
    such value raises "surrogate cannot be computed".  The surrogate is cast to the input type (an integer column
    truncates toward zero) and replaces missingValue and null in transform.
    Bucketizer.binarySearchForBuckets: NaN -> splits.length - 1 when keepInvalid (else an error, or the row is dropped
    under skip, when any input column is NaN); x == splits.last -> splits.length - 2; else
    java.util.Arrays.binarySearch: a hit gives its index, a miss insertion point - 1, and insertion point 0 or
    splits.length (a value outside the splits) raises under every handleInvalid.
    MinMaxScalerModel: (x - originalMin) * (max - min) / (originalMax - originalMin) + min, the constant
    0.5 * (max - min) + min for a column whose range is 0; NaN stays NaN and is skipped by the fit.

Here the sums are exact: mean is the 128-bit fixed-point sum of the finite values (regression.cu's grid) divided by the
count, rounded once; a column with +inf and -inf has mean NaN, with one of them +-inf.  Mode gathers every rank's
non-missing keys of the column (8 bytes x the global rows on each rank) and sorts them once.
"""
import math

import numpy as np
import torch
import torch.distributed as dist

from . import _lib
from . import dist as bdist
from ._lib import F32, F64, I32, call, ptr
from .metrics import _fixed_shift

SMEM_GROUPS = 48            # kQselSmemGroups of csrc/quantile.cu: larger group bounds count in global memory
_NONE_KEY = -1              # 0xFFFFFFFFFFFFFFFF as int64: the padding key of b200flow_mode
_CODE = {torch.float32: F32, torch.float64: F64, torch.int32: I32}
_RECORD_CODE = {"f32": F32, "f64": F64, "i32": I32}


class Columns:
    """D columns of n rows read in place: value (r, c) at base + r row_bytes + desc[2c], dtype desc[2c + 1]."""

    def __init__(self, base, n, row_bytes, desc, device, keep):
        self.base, self.n, self.row_bytes = base, int(n), int(row_bytes)
        self.desc = np.ascontiguousarray(desc, np.int32).reshape(-1)
        self.D = self.desc.shape[0] // 2
        self.device = device
        self._keep = keep                                      # the tensor that owns base
        self._dev = None

    @property
    def dtypes(self):
        return [int(c) for c in self.desc[1::2]]

    def cols(self):
        if self._dev is None:
            self._dev = _lib.h2d(self.desc, self.device)
        return self._dev

    def one(self, c):
        """column c alone"""
        return Columns(self.base, self.n, self.row_bytes, self.desc[2 * c:2 * c + 2], self.device, self._keep)

    def args(self):
        return (self.base, self.row_bytes, self.n, self.D, ptr(self.cols()))


def columns(x):
    """Columns of a CUDA tensor [n] or [n, D] (f32, f64 or i32, any strides)"""
    if x.dtype not in _CODE:
        raise ValueError("columns must be float32, float64 or int32, got %s" % x.dtype)
    if not x.is_cuda:
        raise _lib.B200FlowError("b200flow kernels need CUDA tensors (got %s); there is no CPU fallback" % x.device)
    x2 = x.unsqueeze(1) if x.dim() == 1 else x
    if x2.dim() != 2 or x2.shape[1] < 1:
        raise ValueError("columns must be [n] or [n, D] with D >= 1")
    es = x2.element_size()
    n, D = x2.shape
    row_bytes = x2.stride(0) * es if n > 1 else max(x2.stride(0) * es, D * x2.stride(1) * es, 4)
    desc = np.zeros(2 * D, np.int32)
    desc[0::2] = np.arange(D) * x2.stride(1) * es
    desc[1::2] = _CODE[x2.dtype]
    return Columns(x2.data_ptr() if n else 0, n, max(row_bytes, 4), desc, x2.device, x2)


def record_columns(rec, schema, fields):
    """Columns of numeric fields of raw records (uint8 [n, row_bytes] CUDA tensor)"""
    desc = []
    for f in fields:
        t = schema.type_of[f]
        if t not in _RECORD_CODE:
            raise ValueError("field %s of type %s has no numeric value" % (f, t))
        desc += [schema.offsets[f], _RECORD_CODE[t]]
    n = rec.shape[0]
    return Columns(rec.data_ptr() if n else 0, n, schema.row_bytes, desc, rec.device, rec)


def _as_columns(x):
    return x if isinstance(x, Columns) else columns(x)


def _missing(missing):
    """(has_missing, missing) of a missingValue (None or NaN: only NaN is missing)"""
    if missing is None or missing != missing:
        return 0, 0.0
    return 1, float(missing)


def _key_value(k):
    """the double of an ordered key stored as key ^ 2^63 (int64)"""
    u = (int(k) ^ (1 << 63)) & 0xFFFFFFFFFFFFFFFF
    b = u & ~(1 << 63) if u >> 63 else ~u & 0xFFFFFFFFFFFFFFFF
    return float(np.array([b], np.uint64).view(np.float64)[0])


class ColumnStats:
    """per column (numpy [D]): count of non-missing values, min and max (Double.compare order; NaN without a value),
    max_abs (max(|min|, |max|)), mean (NaN without a value; None unless asked for)"""

    def __init__(self, count, vmin, vmax, mean):
        self.count, self.min, self.max, self.mean = count, vmin, vmax, mean
        self.max_abs = np.maximum(np.abs(vmin), np.abs(vmax))


def column_stats(x, missing=None, group=None, with_mean=False):
    """ColumnStats of the columns x (a tensor or Columns); with a group every rank passes its shard"""
    cs = _as_columns(x)
    D = cs.D
    hm, mv = _missing(missing)
    stats = torch.empty((6, D), dtype=torch.int64, device=cs.device)
    call("b200flow_column_stats", *cs.args(), hm, mv, ptr(stats))
    if group is not None:
        bdist.all_reduce_(stats[:3], group)
        bdist.all_reduce_(stats[3:4], group, op=dist.ReduceOp.MIN)
        bdist.all_reduce_(stats[4:], group, op=dist.ReduceOp.MAX)
    s = stats.cpu().numpy()
    count = s[0].copy()
    nan = float("nan")
    vmin = np.array([_key_value(k) if c else nan for k, c in zip(s[3], count)])
    vmax = np.array([_key_value(k) if c else nan for k, c in zip(s[4], count)])
    mean = None
    if with_mean:
        finite = count - s[1] - s[2]
        if D and int(finite.max()) >= (1 << 31):
            raise ValueError("column statistics support fewer than 2^31 values per column")
        shifts = np.array([_fixed_shift(float(np.array(s[5, j]).view(np.float64)), int(finite[j])) for j in range(D)], np.int32)
        limbs = torch.zeros((D, 4), dtype=torch.int64, device=cs.device)
        shifts_d = _lib.h2d(shifts, cs.device)
        call("b200flow_column_sums", *cs.args(), hm, mv, ptr(shifts_d), ptr(limbs))
        if group is not None:
            bdist.all_reduce_(limbs, group)
        L = limbs.cpu().numpy()
        mean = np.empty(D)
        for j in range(D):
            if count[j] == 0 or (s[1, j] and s[2, j]):
                mean[j] = nan
            elif s[1, j] or s[2, j]:
                mean[j] = math.inf if s[1, j] else -math.inf
            else:
                total = sum(int(v) << (32 * k) for k, v in enumerate(L[j]))
                sh = int(shifts[j])
                mean[j] = total / (int(count[j]) << sh) if sh >= 0 else total * (1 << -sh) / int(count[j])
    return ColumnStats(count, vmin, vmax, mean)


def target_rank(q, n):
    """QuantileSummaries.query's rank of probability q among n values (1-based): ceil(q n) in fp64, 1 for q <= 0"""
    r = int(math.ceil(float(q) * float(n)))
    return min(max(r, 1), int(n))


def check_probabilities(probs):
    probs = [float(p) for p in probs]
    for p in probs:
        if not 0.0 <= p <= 1.0:
            raise ValueError("percentile should be in the range [0.0, 1.0], got %r" % (p,))
    return probs


def select_ranks(x, ranks, missing=None, group=None):
    """the element of each rank (1-based, within its column's non-missing values in Double.compare order): ranks is one
    list per column, every rank within the column's global count -> list of numpy f64 arrays in the given order.  With a
    group every rank passes its shard and the same ranks."""
    cs = _as_columns(x)
    D = cs.D
    if len(ranks) != D:
        raise ValueError("select_ranks needs one rank list per column")
    tcol, trank, where = [], [], []
    for c in range(D):
        order = sorted(range(len(ranks[c])), key=lambda i: ranks[c][i])
        for i in order:
            tcol.append(c); trank.append(int(ranks[c][i])); where.append((c, i))
    out = [np.empty(len(r)) for r in ranks]
    T = len(tcol)
    if T == 0:
        return out
    hm, mv = _missing(missing)
    state = torch.zeros(6 * T + 2 * D + 1, dtype=torch.int64, device=cs.device)
    state[:T] = _lib.h2d(np.asarray(trank, np.int64), cs.device)
    state[4 * T:5 * T] = _lib.h2d(np.asarray(tcol, np.int64), cs.device)
    call("b200flow_quantile_step", T, D, ptr(state), None, 0)
    active = len(set(tcol))
    hist = torch.empty(T * 256, dtype=torch.int64, device=cs.device)
    for p in range(8):
        bound = min(T, active * 256 ** p)
        call("b200flow_quantile_hist", *cs.args(), hm, mv, T, ptr(state), p, bound, ptr(hist))
        if group is not None:
            bdist.all_reduce_(hist[:bound * 256], group)
        call("b200flow_quantile_step", T, D, ptr(state), ptr(hist), 1)
    vals = state[3 * T:4 * T].view(torch.float64).cpu().numpy()
    for (c, i), v in zip(where, vals):
        out[c][i] = v
    return out


def quantiles(x, probs, missing=None, group=None):
    """DataFrame.approxQuantile of each column at probs (one list for every column, or one list per column): list of
    numpy f64 arrays, empty for a column without a value"""
    cs = _as_columns(x)
    per = probs if probs and isinstance(probs[0], (list, tuple, np.ndarray)) else [probs] * cs.D
    per = [check_probabilities(p) for p in per]
    count = column_stats(cs, missing, group).count
    ranks = [[target_rank(q, count[c]) for q in per[c]] if count[c] else [] for c in range(cs.D)]
    return select_ranks(cs, ranks, missing, group)


def mode(x, missing=None, group=None):
    """per column, the most frequent non-missing value (the smallest on ties; NaN without a value): numpy f64 [D]"""
    cs = _as_columns(x)
    hm, mv = _missing(missing)
    out = np.empty(cs.D)
    for c in range(cs.D):
        one = cs.one(c)
        keys = torch.empty(max(cs.n, 1), dtype=torch.int64, device=cs.device)
        cnt = torch.zeros(1, dtype=torch.int64, device=cs.device)
        call("b200flow_mode_keys", one.base, one.row_bytes, one.n, one.desc.ctypes.data, hm, mv, ptr(keys), ptr(cnt))
        keys = keys[:int(cnt.item())]
        if group is not None:
            widest = cnt.clone()
            bdist.all_reduce_(widest, group, op=dist.ReduceOp.MAX)
            pad = torch.full((int(widest.item()),), _NONE_KEY, dtype=torch.int64, device=cs.device)
            pad[:keys.shape[0]] = keys
            keys = torch.cat(bdist.all_gather_list(pad, group))
        M = keys.shape[0]
        if M == 0:
            out[c] = float("nan")
            continue
        keys = keys.contiguous()
        scratch = torch.empty(max(_lib.mode_scratch(M), 1), dtype=torch.uint8, device=cs.device)
        res = torch.empty(2, dtype=torch.float64, device=cs.device)
        call("b200flow_mode", ptr(keys), M, ptr(scratch), scratch.numel(), ptr(res))
        out[c] = float(res[0].item())
    return out


def bucketize(x, splits):
    """Bucketizer over the columns x with splits[c] (strictly increasing, >= 3 each): (out f64 [n, D], row flags uint8 [n]
    (0: a NaN in the row), NaN values, values outside the splits).  NaN gets index len(splits) - 1."""
    cs = _as_columns(x)
    if len(splits) != cs.D:
        raise ValueError("bucketize needs one split list per column")
    flat = np.concatenate([np.asarray(s, np.float64) for s in splits])
    off = np.concatenate([[0], np.cumsum([len(s) for s in splits])]).astype(np.int32)
    dev = cs.device
    out = torch.empty((cs.n, cs.D), dtype=torch.float64, device=dev)
    flags = torch.empty(cs.n, dtype=torch.uint8, device=dev)
    checks = torch.empty(2, dtype=torch.int64, device=dev)
    flat_d, off_d = _lib.h2d(flat, dev), _lib.h2d(off, dev)          # held until the launch: temporaries would share a block
    call("b200flow_bucketize", *cs.args(), ptr(flat_d), ptr(off_d), ptr(out), ptr(flags), ptr(checks))
    nan, oob = (int(v) for v in checks.cpu())
    return out, flags, nan, oob


def cast_surrogate(v, code):
    """the surrogate cast to a column type, as Spark's cast: f32 rounds, i32 truncates toward zero (NaN -> 0, saturating)"""
    if code == F64:
        return float(v)
    if code == F32:
        return float(np.float32(v))
    if v != v:
        return 0
    return int(max(min(math.trunc(v) if math.isfinite(v) else v, 2 ** 31 - 1), -2 ** 31))


def _bits(v, code):
    if code == F64:
        return int(np.array([v], np.float64).view(np.uint64)[0])
    if code == F32:
        return int(np.array([v], np.float32).view(np.uint32)[0])
    return int(np.array([v], np.int32).view(np.uint32)[0])


def fill(x, surrogates, missing=None):
    """Imputer.transform: per column a contiguous tensor of its own dtype, the missing values (NaN, or == missing)
    replaced by the column's surrogate cast to that dtype"""
    cs = _as_columns(x)
    hm, mv = _missing(missing)
    dt = {F32: torch.float32, F64: torch.float64, I32: torch.int32}
    outs = [torch.empty(cs.n, dtype=dt[c], device=cs.device) for c in cs.dtypes]
    bits = np.array([_bits(cast_surrogate(s, c), c) for s, c in zip(surrogates, cs.dtypes)], np.uint64)
    ptrs = np.array([o.data_ptr() for o in outs], np.uint64)
    bits_d, ptrs_d = _lib.h2d(bits, cs.device), _lib.h2d(ptrs, cs.device)
    call("b200flow_impute_fill", *cs.args(), hm, mv, ptr(bits_d), ptr(ptrs_d))
    return outs


def min_max(x, emin, scale, lo, constant):
    """MinMaxScalerModel.transform: f64 [n, D] = (x - emin) * scale + lo, constant where scale == 0, NaN kept"""
    cs = _as_columns(x)
    out = torch.empty((cs.n, cs.D), dtype=torch.float64, device=cs.device)
    emin_d = _lib.h2d(np.asarray(emin, np.float64), cs.device)
    scale_d = _lib.h2d(np.asarray(scale, np.float64), cs.device)
    call("b200flow_min_max", *cs.args(), ptr(emin_d), ptr(scale_d), float(lo), float(constant), ptr(out))
    return out
