"""MultilayerPerceptronClassifier on the device (DESIGN.md §5d): loss and gradient from csrc/mlp.cu's fused fp64
tensor-core kernel, summed in the chunk order of dist.Shards, and the L-BFGS of linear.lbfgs (or mllib's gradient descent).

Spark [recalled; Spark 3 `ml/classification/MultilayerPerceptronClassifier.scala`, `ml/ann/Layer.scala`,
`mllib/optimization/GradientDescent.scala`]:

    layers = [D, h_1, ..., h_k, K]; hidden layers are affine + sigmoid 1/(1 + exp(-z)), the top layer affine + softmax.
    The flat weight vector holds, layer after layer, W (out x in, column-major: (o, i) at o + i*out) and then b (out).
    AffineLayerModel.randomWeights: every element of layer l's block is (u*4.8 - 2.4) / sqrt(in_l); here u is the
    Philox draw of purpose MLPW, counter (i_lo, i_hi, 0, 0) for flat index i (DESIGN §5), not XORShiftRandom.
    Objective (1/n) sum_r [logsumexp(z_r) - z_r[y_r]] with z the top affine output, no regularisation (ANNUpdater).
    solver "l-bfgs": Breeze LBFGS, 10 corrections; "gd": full-batch GradientDescent, step stepSize / sqrt(t), stop when
    |w_t - w_{t-1}| < tol * max(|w_t|, 1).  rawPrediction is the top affine output (Spark 3's predictRaw).

Deviations: Spark averages over blockSize stacks, which equals this mean only when every partition's row count is a
multiple of blockSize, so blockSize does not change the result here; the loss is log-softmax, never log(softmax), and
cannot overflow to inf; K >= 2 is required.

Every row's loss and gradient is summed into its 4096-row chunk's partial on the device; the partials are added in
chunk order and passed rank to rank (dist.chunk_tail / chunk_chain), and one division by n gives loss and gradient.
So the model is the same bits for any world size, any shard layout and either feature dtype.
"""
import math

import numpy as np
import torch

from . import _lib
from . import dist as bdist
from .kmeans import philox, uniform
from .linear import lbfgs
from ._lib import call, ptr

PURPOSE_MLPW = 0x4D4C5057


def n_params(layers):
    return sum((a + 1) * b for a, b in zip(layers[:-1], layers[1:]))


def init_weights(layers, seed):
    """Spark's randomWeights layout with the MLPW draws: host f64 [P]."""
    out = np.empty(n_params(layers))
    i = 0
    for a, b in zip(layers[:-1], layers[1:]):
        scale = math.sqrt(a)
        for _ in range((a + 1) * b):
            w = philox(seed, PURPOSE_MLPW, i, i >> 32)
            out[i] = (uniform(w[0], w[1]) * 4.8 - 2.4) / scale
            i += 1
    return out


def check_layers(layers):
    """layers as a list of ints; ValueError unless >= 2 positive sizes with K >= 2, UnsupportedParamError beyond the
    kernels' limits (b200flow_mlp_config)."""
    layers = [int(v) for v in layers]
    if len(layers) < 2 or min(layers) <= 0:
        raise ValueError("layers must have at least 2 entries, all > 0, got %s" % layers)
    if layers[-1] < 2:
        raise ValueError("the output layer needs at least 2 classes, got %d" % layers[-1])
    _lib.mlp_config(layers)
    return layers


def _check_x(x, layers):
    if not (torch.is_tensor(x) and x.is_cuda and x.dim() == 2 and x.dtype in (torch.float32, torch.float64)):
        raise _lib.B200FlowError("the MLP needs a CUDA float32 or float64 [n, D] matrix")
    if x.shape[1] != layers[0]:
        raise ValueError("layers[0] = %d does not match the feature size %d" % (layers[0], x.shape[1]))
    return x.contiguous()


def loss_grad_sums(x, y, layers, w, sh):
    """[P + 1] f64 device: the sum over every rank's rows of the loss (slot 0) and its gradient, in chunk order; the same
    bits on every rank.  x [n, D] f32/f64, y int32 [n] (this rank's shard), w f64 [P] device."""
    la = np.ascontiguousarray(layers, dtype=np.int32)
    P = int(w.shape[0])
    dt = _lib.dtype_code(x)
    lead, off = sh.lead[sh.rank], sh.offs[sh.rank]
    t0, tail_x, tail_y = bdist.chunk_tail(x, y, sh)
    nfull = (t0 - lead) // bdist.CHUNK
    n_tail = tail_x.shape[0]
    n_chunks = nfull + (1 if n_tail else 0)
    parts = torch.empty((max(n_chunks, 1), P + 1), dtype=torch.float64, device=w.device)
    if nfull:
        call("b200flow_mlp_loss_grad", ptr(x[lead:t0]), dt, t0 - lead, layers[0], ptr(y[lead:t0]), la.ctypes.data, len(la),
             ptr(w), off + lead, ptr(parts))
    if n_tail:
        call("b200flow_mlp_loss_grad", ptr(tail_x), _lib.dtype_code(tail_x), n_tail, layers[0], ptr(tail_y), la.ctypes.data,
             len(la), ptr(w), off + t0, ptr(parts[nfull:]))
    return bdist.chunk_chain(parts, n_chunks, 1, P + 1, sh).reshape(-1)


class MLPFit:
    __slots__ = ("weights", "objective_history", "iterations")

    def __init__(self, weights, hist, it):
        self.weights, self.objective_history, self.iterations = weights, hist, it


def mlp_fit(x, y, layers, solver="l-bfgs", max_iter=100, tol=1e-6, step_size=0.03, seed=0, initial_weights=None,
            row_offset=None, group=None):
    """MultilayerPerceptronClassifier.fit on this rank's rows x [n, D] (f32 or f64), y [n] integer labels in [0, K).
    An empty shard still joins every collective.  -> MLPFit(weights f64 [P] device, objective history, iterations)."""
    layers = check_layers(layers)
    x = _check_x(x, layers)
    K, P = layers[-1], n_params(layers)
    if solver not in ("l-bfgs", "gd"):
        raise ValueError("solver must be l-bfgs or gd, got %r" % (solver,))
    if int(max_iter) < 0 or not tol > 0 or not step_size > 0:
        raise ValueError("maxIter must be >= 0, tol > 0 and stepSize > 0")
    grp = group if group is not None else bdist.group()
    dev = x.device
    if row_offset is None:
        row_offset, _ = bdist.global_offset(x.shape[0], dev, grp)
    sh = bdist.Shards(x.shape[0], row_offset, grp, dev)
    yf = y.to(device=dev, dtype=torch.float64)
    yi = yf.to(torch.int32).contiguous()
    bad = torch.stack([((yf < 0) | (yf >= K) | (yf != torch.floor(yf))).any(), (~torch.isfinite(x)).any()]).to(torch.int64)
    if grp is not None:
        bdist.all_reduce_(bad, grp)
    if sh.total == 0:
        raise ValueError("MultilayerPerceptronClassifier needs at least one row")
    if int(bad[0].item()):
        raise ValueError("labels must be integers in [0, %d)" % K)
    if int(bad[1].item()):
        raise ValueError("features must be finite")
    if initial_weights is not None:
        w0 = torch.as_tensor(np.asarray(initial_weights, dtype=np.float64)).reshape(-1)
        if w0.numel() != P:
            raise ValueError("initialWeights has %d elements; layers %s need %d" % (w0.numel(), layers, P))
    else:
        w0 = torch.from_numpy(init_weights(layers, seed))
    w0 = w0.to(dev)
    inv_n = 1.0 / sh.total

    def fun(w):
        t = loss_grad_sums(x, yi, layers, w.contiguous(), sh) * inv_n
        return t[0], t[1:]

    if solver == "l-bfgs":
        w, hist, it = lbfgs(fun, w0, int(max_iter), float(tol))
        return MLPFit(w, hist, it)
    w, hist, it = w0, [], 0
    for t in range(1, int(max_iter) + 1):                    # mllib GradientDescent, miniBatchFraction 1, ANNUpdater
        f, g = fun(w)
        hist.append(float(f.item()))
        wn = w - (float(step_size) / math.sqrt(t)) * g
        it = t
        done = float((wn - w).norm().item()) < float(tol) * max(float(wn.norm().item()), 1.0)
        w = wn
        if done:
            break
    return MLPFit(w, hist, it)


def mlp_raw(weights, layers, x):
    """rawPrediction [n, K] f64: the top affine output of every row of x [n, D] (f32 or f64)."""
    layers = check_layers(layers)
    x = _check_x(x, layers)
    n = x.shape[0]
    la = np.ascontiguousarray(layers, dtype=np.int32)
    w = weights.to(device=x.device, dtype=torch.float64).contiguous()
    raw = torch.empty((max(n, 1), layers[-1]), dtype=torch.float64, device=x.device)
    call("b200flow_mlp_forward", ptr(x), _lib.dtype_code(x), n, layers[0], la.ctypes.data, len(la), ptr(w), ptr(raw))
    return raw[:n]
