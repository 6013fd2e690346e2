"""IsotonicRegression on the device (DESIGN.md §5p): a stable radix sort of the features, Spark's makeUnique tie pooling,
a chunked pool-adjacent-violators merge and a binary-search predict (csrc/isotonic.cu).  Under torch.distributed every rank
gathers all rows in rank order and runs the same single-device fit, so the model is the same bits for any world size.

Spark [recalled; Spark 3 `mllib/regression/IsotonicRegression.scala`, `ml/regression/IsotonicRegression.scala`]:

    Rows are (label, feature, weight): the label cast to double, featuresCol itself when numeric or its element
    featureIndex (default 0) when a vector, weightCol or 1.0.  A negative weight fails ("Negative weight at point ...");
    rows of weight 0 are dropped.  isotonic=False negates the labels, fits, and negates the predictions.
    The points are sorted by feature (stable; java.lang.Double.compare, so -0.0 before 0.0).  makeUnique pools each run of
    equal features (primitive ==, so -0.0 == 0.0) into (sumWY / sumW, the run's first feature, sumW) with
    sumWY = y0 w0 + y1 w1 + ... and sumW = w0 + w1 + ... summed in sorted order; an input of at most one point is kept
    as it is.  poolAdjacentViolators keeps blockBounds and weights (w, w y) in place and, from i = 0, merges block i with
    its successor while average(i) >= average(next), then pools backwards while average(prev) >= average(i); each block
    gives (avg, first feature, W / 2) and (avg, last feature, W / 2) when the two features differ, else (avg, feature, W).
    With one partition Spark runs makeUnique + PAV twice: over the rows, then over the first pass's points.  boundaries
    are the final features, predictions the averages.  predict(x): java.util.Arrays.binarySearch(boundaries, x); insertion
    point 0 -> predictions.head, insertion point length -> predictions.last, a hit -> its prediction, else
    y1 + (y2 - y1) * (x - x1) / (x2 - x1).

Here PAV runs as a merge tree (level 0 on chunks of C points, each level joining two adjacent ranges), so the sums
depend on C: the model is bit-reproducible for (rows, C) and equals Spark's sequential PAV to rounding.
Deviations: a NaN or infinite label, feature or weight raises ValueError on every rank; predicting with the empty model of
an all-zero-weight fit raises ValueError; the global row count must be below 2^32.
"""
import numpy as np
import torch
import torch.distributed as dist

from . import _lib
from . import dist as bdist
from ._lib import call

MAX_ROWS = 1 << 32


class IsotonicFit:
    """boundaries (increasing) and predictions, numpy f64 of equal length; empty when every weight was 0"""

    def __init__(self, boundaries, predictions):
        self.boundaries, self.predictions = boundaries, predictions
        self._device = {}

    def on(self, device):
        """(boundaries, predictions) as device tensors"""
        key = str(device)
        if key not in self._device:
            self._device[key] = tuple(torch.from_numpy(a).to(device) for a in (self.boundaries, self.predictions))
        return self._device[key]


def _vector(t, name):
    if t.dim() != 1:
        raise ValueError("IsotonicRegression: %s must be one value per row" % name)
    return t


def _code(t):
    if t.dtype == torch.float32:
        return _lib.F32
    if t.dtype == torch.float64:
        return _lib.F64
    raise ValueError("IsotonicRegression: features must be float32 or float64, got %s" % t.dtype)


def _gather(feature, label, weight, grp):
    """every rank's (label, feature, weight) rows in rank order, [N, 3] f64; the shards are padded to the widest with
    zero-weight rows, which the fit drops"""
    n = feature.shape[0]
    widest = torch.tensor([n], dtype=torch.int64, device=feature.device)
    bdist.all_reduce_(widest, grp, op=dist.ReduceOp.MAX)
    trip = torch.zeros((int(widest.item()), 3), dtype=torch.float64, device=feature.device)
    trip[:n, 0] = label
    trip[:n, 1] = feature
    trip[:n, 2] = 1.0 if weight is None else weight
    return torch.cat(bdist.all_gather_list(trip, grp))


def isotonic_fit(feature, label, weight=None, isotonic=True, group=None, chunk=0):
    """IsotonicFit of the rows (label[i], feature[i], weight[i]): device tensors of one value per row (strided views
    allowed), feature f32 or f64, label and weight f64 (weight None: 1.0).  With a group every rank passes its shard and gets
    the model of all rows in rank order.  chunk forces the PAV chunk size (0: the library's)."""
    _vector(feature, "featuresCol"); _vector(label, "labelCol")
    if weight is not None:
        _vector(weight, "weightCol")
    if label.shape[0] != feature.shape[0] or (weight is not None and weight.shape[0] != feature.shape[0]):
        raise ValueError("IsotonicRegression needs one label and weight per row")
    code = _code(feature)
    label = label.to(torch.float64)
    weight = None if weight is None else weight.to(torch.float64)
    if group is not None:
        rows = _gather(feature, label, weight, group)
        feature, label, weight, code = rows[:, 1], rows[:, 0], rows[:, 2], _lib.F64
    n = int(feature.shape[0])
    if n >= MAX_ROWS:
        raise ValueError("IsotonicRegression supports fewer than 2^32 rows, got %d" % n)
    dev = feature.device
    for t in (feature, label, weight):
        if t is not None and not t.is_cuda:
            raise _lib.B200FlowError("b200flow kernels need CUDA tensors (got %s); there is no CPU fallback" % t.device)
    scratch = torch.empty(max(_lib.isotonic_scratch(n), 1), dtype=torch.uint8, device=dev)
    model = torch.empty((2, max(n, 1)), dtype=torch.float64, device=dev)
    counts = torch.zeros(3, dtype=torch.int64, device=dev)           # bad rows, negative weights, model size
    call("b200flow_isotonic_fit", feature.data_ptr(), code, feature.stride(0), label.data_ptr(), label.stride(0),
         None if weight is None else weight.data_ptr(), 0 if weight is None else weight.stride(0), n, int(bool(isotonic)),
         int(chunk), scratch.data_ptr(), scratch.numel(), model[0].data_ptr(), model[1].data_ptr(),
         counts[2:].data_ptr(), counts[:2].data_ptr())
    bad, neg, K = (int(v) for v in counts.cpu())
    if bad:
        raise ValueError("IsotonicRegression needs finite labels, features and weights (%d rows are not)" % bad)
    if neg:
        i = int(torch.nonzero(weight < 0)[0, 0])
        raise ValueError("Negative weight at point (%r, %r, %r). Weights must be non-negative"
                         % (float(label[i]), float(feature[i]), float(weight[i])))
    host = model[:, :K].cpu().numpy()
    return IsotonicFit(host[0].copy(), host[1].copy())


def _check_model(fit):
    if fit.boundaries.shape[0] == 0:
        raise ValueError("IsotonicRegressionModel is empty: every training weight was 0")


def isotonic_predict(x, fit):
    """device f64 [n]: the model's prediction at each x (device, one value per row, f32 or f64, strided views allowed)"""
    _vector(x, "featuresCol")
    _check_model(fit)
    code = _code(x)
    bx, by = fit.on(x.device)
    out = torch.empty(x.shape[0], dtype=torch.float64, device=x.device)
    call("b200flow_isotonic_predict", x.data_ptr(), code, max(x.stride(0), 1), int(x.shape[0]), bx.data_ptr(),
         by.data_ptr(), int(bx.shape[0]), out.data_ptr())
    return out


def _java_bits(v):
    """java.lang.Double.doubleToLongBits: the IEEE bits as a signed long, every NaN canonical"""
    if v != v:
        return 0x7ff8000000000000
    return int(np.array(v, dtype=np.float64).view(np.int64))


def java_binary_search(a, key):
    """java.util.Arrays.binarySearch(double[] a, double key)"""
    key = float(key)
    low, high = 0, len(a) - 1
    while low <= high:
        mid = (low + high) >> 1
        m = float(a[mid])
        if m < key:
            low = mid + 1
        elif m > key:
            high = mid - 1
        else:
            mb, kb = _java_bits(m), _java_bits(key)
            if mb == kb:
                return mid
            if mb < kb:
                low = mid + 1
            else:
                high = mid - 1
    return -(low + 1)


def predict_value(x, fit):
    """the model's prediction at one value on the host: the same arithmetic as the kernel, so the same bits"""
    _check_model(fit)
    b, p = fit.boundaries, fit.predictions
    f = java_binary_search(b, x)
    ins = -f - 1
    if ins == 0:
        return float(p[0])
    if ins == len(b):
        return float(p[-1])
    if f < 0:
        x1, y1, x2, y2 = float(b[ins - 1]), float(p[ins - 1]), float(b[ins]), float(p[ins])
        return y1 + (y2 - y1) * (float(x) - x1) / (x2 - x1)
    return float(p[f])
