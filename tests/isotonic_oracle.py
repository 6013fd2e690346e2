"""Host restatement of IsotonicRegression (DESIGN.md §5p), in plain Python floats (IEEE fp64, no FMA):

  - fit(..., chunk=None): Spark's one-partition algorithm [recalled]: drop zero weights, stable sort by feature in
    java.lang.Double.compare order, makeUnique, the sequential blockBounds PAV, compress, then makeUnique + PAV + compress
    again over those points;
  - fit(..., chunk=C): the same with the device's chunked PAV: Spark's loop on each chunk of C points, then, level by
    level, the loop resumed at the junction of two adjacent ranges of R = C, 2C, 4C, ... points;
  - predict: java.util.Arrays.binarySearch and Spark's interpolation.
"""
import struct

import numpy as np


def _bits(v):
    """java.lang.Double.doubleToLongBits"""
    if v != v:
        return 0x7ff8000000000000
    return struct.unpack("<q", struct.pack("<d", v))[0]


def _order(x):
    """a stable sort of x in java.lang.Double.compare order (-0.0 before 0.0)"""
    b = np.ascontiguousarray(x, dtype=np.float64).view(np.uint64)
    key = np.where(b >> np.uint64(63), ~b, b | np.uint64(1 << 63))
    return np.argsort(key, kind="stable")


def make_unique(y, x, w):
    """Spark's makeUnique on sorted points: each run of == features -> (sumWY / sumW, first feature, sumW), summed in
    order; at most one point is returned as it is"""
    if len(x) <= 1:
        return list(y), list(x), list(w)
    uy, ux, uw = [], [], []
    swy, cx, sw = y[0] * w[0], x[0], w[0]
    for k in range(1, len(x)):
        if x[k] == cx:
            swy += y[k] * w[k]
            sw += w[k]
        else:
            uy.append(swy / sw); ux.append(cx); uw.append(sw)
            swy, cx, sw = y[k] * w[k], x[k], w[k]
    uy.append(swy / sw); ux.append(cx); uw.append(sw)
    return uy, ux, uw


class _Blocks:
    """Spark's in-place PAV state: blockBounds and weights (w, w y)"""

    def __init__(self, uy, uw):
        self.bb = list(range(len(uy)))
        self.W = list(uw)
        self.WY = [w * y for y, w in zip(uy, uw)]

    def avg(self, s):
        return self.WY[s] / self.W[s]

    def merge(self, b1, b2):
        e2 = self.bb[b2]
        self.bb[b1] = e2
        self.bb[e2] = b1
        self.W[b1] = self.W[b1] + self.W[b2]
        self.WY[b1] = self.WY[b1] + self.WY[b2]
        return b1

    def pool_back(self, lo, i):
        while i > lo and self.avg(self.bb[i - 1]) >= self.avg(i):
            i = self.merge(self.bb[i - 1], i)
        return i

    def run(self, lo, hi):
        """Spark's loop over [lo, hi)"""
        i = lo
        while self.bb[i] + 1 < hi:
            nx = self.bb[i] + 1
            if self.avg(i) >= self.avg(nx):
                self.merge(i, nx)
                i = self.pool_back(lo, i)
            else:
                i = nx

    def join(self, lo, mid, hi):
        """the loop resumed at the block ending at mid - 1, over [lo, hi) whose halves are each monotone"""
        i = self.bb[mid - 1]
        while self.bb[i] + 1 < hi and self.avg(i) >= self.avg(self.bb[i] + 1):
            self.merge(i, self.bb[i] + 1)
            i = self.pool_back(lo, i)


def pav(uy, ux, uw, chunk=None):
    """poolAdjacentViolators on unique sorted points -> the output points (y, x, w)"""
    U = len(ux)
    oy, ox, ow = [], [], []
    if U == 0:
        return oy, ox, ow
    B = _Blocks(uy, uw)
    if chunk is None:
        B.run(0, U)
    else:
        for lo in range(0, U, chunk):
            B.run(lo, min(lo + chunk, U))
        R = chunk
        while R < U:
            for lo in range(0, U, 2 * R):
                if lo + R < U:
                    B.join(lo, lo + R, min(lo + 2 * R, U))
            R *= 2
    i = 0
    while i < U:
        e, a = B.bb[i], B.avg(i)
        if ux[e] > ux[i]:
            oy += [a, a]; ox += [ux[i], ux[e]]; ow += [B.W[i] / 2, B.W[i] / 2]
        else:
            oy.append(a); ox.append(ux[i]); ow.append(B.W[i])
        i = e + 1
    return oy, ox, ow


def fit(label, feature, weight=None, isotonic=True, chunk=None):
    """(boundaries, predictions) as numpy f64 of the rows in order; chunk None: Spark's sequential PAV"""
    y = np.asarray(label, np.float64)
    x = np.asarray(feature, np.float64)
    w = np.ones_like(y) if weight is None else np.asarray(weight, np.float64)
    if (w < 0).any():
        raise ValueError("Negative weight")
    keep = w > 0
    y, x, w = y[keep], x[keep], w[keep]
    if not isotonic:
        y = -y
    o = _order(x)
    pts = (y[o].tolist(), x[o].tolist(), w[o].tolist())
    for _ in range(2):
        pts = pav(*make_unique(*pts), chunk=chunk)
    py, px, _ = pts
    p = np.asarray(py, np.float64)
    return np.asarray(px, np.float64), (p if isotonic else -p)


def binary_search(a, key):
    """java.util.Arrays.binarySearch(double[], double)"""
    low, high = 0, len(a) - 1
    while low <= high:
        mid = (low + high) >> 1
        m = float(a[mid])
        if m < key:
            low = mid + 1
        elif m > key:
            high = mid - 1
        else:
            mb, kb = _bits(m), _bits(key)
            if mb == kb:
                return mid
            low, high = (mid + 1, high) if mb < kb else (low, mid - 1)
    return -(low + 1)


def predict(x, boundaries, predictions):
    """Spark's IsotonicRegressionModel.predict at one value"""
    x = float(x)
    f = binary_search(boundaries, x)
    ins = -f - 1
    if ins == 0:
        return float(predictions[0])
    if ins == len(boundaries):
        return float(predictions[-1])
    if f < 0:
        x1, y1 = float(boundaries[ins - 1]), float(predictions[ins - 1])
        x2, y2 = float(boundaries[ins]), float(predictions[ins])
        return y1 + (y2 - y1) * (x - x1) / (x2 - x1)
    return float(predictions[f])
