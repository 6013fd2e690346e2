"""numpy restatement of the preprocessing stages' rules (b200flow/quantile.py, DESIGN.md §5s): exact quantiles by
QuantileSummaries.query's rank, Imputer surrogates, Bucketizer's binarySearchForBuckets, QuantileDiscretizer's distinct
splits and MinMaxScaler's transform."""
import math
from fractions import Fraction

import numpy as np


def _bits(v):
    return 0x7ff8000000000000 if v != v else int(np.array(v, np.float64).view(np.int64))


def java_binary_search(a, key):
    """java.util.Arrays.binarySearch(double[] a, double key): ties by doubleToLongBits, so -0.0 < 0.0"""
    low, high = 0, len(a) - 1
    while low <= high:
        mid = (low + high) >> 1
        m = float(a[mid])
        if m < key:
            low = mid + 1
        elif m > key:
            high = mid - 1
        elif _bits(m) == _bits(key):
            return mid
        elif _bits(m) < _bits(key):
            low = mid + 1
        else:
            high = mid - 1
    return -(low + 1)


def order_keys(v):
    """Double.compare order of f64 values as uint64 keys (-0.0 < 0.0)"""
    b = np.asarray(v, np.float64).view(np.uint64)
    return np.where(b >> np.uint64(63), ~b, b | np.uint64(1 << 63))


def valid(v, missing=None):
    """the values that are neither NaN nor == missing, as f64"""
    v = np.asarray(v, np.float64)
    keep = ~np.isnan(v)
    if missing is not None and missing == missing:
        keep &= v != missing
    return v[keep]


def sorted_values(v, missing=None):
    x = valid(v, missing)
    return x[np.argsort(order_keys(x), kind="stable")]


def target_rank(q, n):
    return min(max(int(math.ceil(float(q) * float(n))), 1), int(n))


def quantiles(v, probs, missing=None):
    s = sorted_values(v, missing)
    if s.shape[0] == 0:
        return np.zeros(0)
    return np.array([s[target_rank(q, s.shape[0]) - 1] for q in probs])


def mean(v, missing=None):
    """the exact sum of the values rounded once after the division by the count (NaN without a value)"""
    x = valid(v, missing)
    if x.shape[0] == 0:
        return float("nan")
    pinf, ninf = bool(np.any(x == np.inf)), bool(np.any(x == -np.inf))
    if pinf and ninf:
        return float("nan")
    if pinf or ninf:
        return math.inf if pinf else -math.inf
    f = sum((Fraction(float(a)) for a in x), Fraction(0)) / x.shape[0]
    return f.numerator / f.denominator


def mode(v, missing=None):
    """the most frequent value (-0.0 counted as 0.0), the smallest on ties; NaN without a value"""
    x = valid(v, missing)
    if x.shape[0] == 0:
        return float("nan")
    x = np.where(x == 0.0, 0.0, x)
    u, c = np.unique(x, return_counts=True)
    return float(u[np.argmax(c)])


def cast(v, kind):
    """the surrogate in the column type: 'f64', 'f32' (rounded) or 'i32' (toward zero, NaN -> 0, saturating)"""
    if kind == "f64":
        return float(v)
    if kind == "f32":
        return float(np.float32(v))
    if v != v:
        return 0
    return int(max(min(math.trunc(v) if math.isfinite(v) else v, 2 ** 31 - 1), -2 ** 31))


def fill(v, surrogate, missing=None):
    v = np.asarray(v).copy()
    miss = np.isnan(v.astype(np.float64))
    if missing is not None and missing == missing:
        miss |= v.astype(np.float64) == missing
    v[miss] = surrogate
    return v


class OutOfBounds(Exception):
    pass


def bucket(x, splits, keep=True):
    """Spark's Bucketizer.binarySearchForBuckets of one value; NaN -> len(splits) - 1 (keep)"""
    x = float(x)
    K = len(splits)
    if x != x:
        if not keep:
            raise ValueError("NaN")
        return float(K - 1)
    if x == splits[-1]:
        return float(K - 2)
    f = java_binary_search(splits, x)
    if f >= 0:
        return float(f)
    ins = -f - 1
    if ins == 0 or ins == K:
        raise OutOfBounds(x)
    return float(ins - 1)


def distinct_splits(splits):
    s = [float(v) for v in splits]
    s[0], s[-1] = -math.inf, math.inf
    return list(dict.fromkeys(0.0 if v == 0.0 else v for v in s))


def discretizer_splits(v, num_buckets):
    q = quantiles(v, [i / num_buckets for i in range(1, num_buckets)])
    return distinct_splits([-math.inf] + list(q) + [math.inf])


def min_max(x, omin, omax, lo=0.0, hi=1.0):
    """MinMaxScalerModel.transform of [n, D] f64"""
    x = np.asarray(x, np.float64)
    out = np.empty_like(x)
    for j in range(x.shape[1]):
        r = omax[j] - omin[j]
        s = (hi - lo) / r if r != 0.0 else 0.0
        col = x[:, j]
        out[:, j] = np.where(np.isnan(col), col, (col - omin[j]) * s + lo if s != 0.0 else 0.5 * (hi - lo) + lo)
    return out
