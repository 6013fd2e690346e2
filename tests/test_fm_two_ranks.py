"""FMClassifier and OneVsRest(FMClassifier) over TWO RANKS: the factorization-machine partials are computed from each
4096-row chunk's rows alone (a straddling chunk by the rank holding its first row), the mini-batch draw follows the global
row, and the partials are chained rank to rank, so the loss and gradient totals, a binary fit (with the whole set and
with miniBatchFraction = 0.5) and a OneVsRest fit equal the single-process run byte for byte — for even and uneven shards,
a shard shorter than one chunk and an empty shard.  An invalid label on one rank makes both raise.  Through the pyspark
shim, a rank whose shard is empty or holds only label 0 decides numClasses as the other does: the fit equals one process,
and a label set that is not binary overall makes both ranks raise.  Two gloo ranks share one GPU; the NCCL case needs two
GPUs and is skipped otherwise."""
import numpy as np
import pytest
import torch

from ranks import SPLITS, block, run, two_gpus

pytestmark = pytest.mark.gpu

N = 30000
D, K, KF = 41, 5, 4


def _data():
    rng = np.random.default_rng(8)
    means = rng.normal(0.0, 1.0, (K, D))
    y = rng.integers(0, K, N)
    return np.ascontiguousarray(means[y] + rng.normal(0.0, 1.0, (N, D))), y.astype(np.int32)


def _hex(a):
    return [float(v).hex() for v in np.asarray(a).reshape(-1)]


def _fits_hex(fits):
    return [{"v": _hex(f.factors), "w": _hex(f.linear), "b": float(f.intercept).hex(), "hist": _hex(f.objective_history),
             "it": f.iterations} for f in fits]


def _run(x, y, dev, grp):
    from b200flow import dist as bdist, fm as bfm
    xt, yt = torch.from_numpy(x).to(dev), torch.from_numpy(y).to(dev)
    off, _ = bdist.global_offset(xt.shape[0], dev, grp)
    sh = bdist.Shards(xt.shape[0], off, grp, dev)
    rng = np.random.default_rng(2)
    w = torch.from_numpy(rng.normal(0, 0.1, (K, D * (KF + 1) + 1))).to(dev)
    pos = torch.arange(K, dtype=torch.int32, device=dev)
    out = {"sums": _hex(bfm.fm_loss_grad_totals(xt, yt, pos, w, KF, 1.0, 43, sh).cpu().numpy()),
           "sums_batch": _hex(bfm.fm_loss_grad_totals(xt, yt, pos, w, KF, 0.5, 44, sh).cpu().numpy())}
    p = bfm.FMParams(factor_size=KF, max_iter=8, step_size=0.05, reg_param=0.01, seed=7)
    pb = bfm.FMParams(factor_size=KF, max_iter=8, step_size=0.5, mini_batch_fraction=0.5, solver="gd", seed=7)
    out["binary"] = _fits_hex(bfm.fm_fit_classes(xt, (yt == 2).to(torch.int32), [1], p, group=grp))
    out["binary_batch"] = _fits_hex(bfm.fm_fit_classes(xt, (yt == 2).to(torch.int32), [1], pb, group=grp))
    out["ovr"] = _fits_hex(bfm.fm_fit_classes(xt, yt, range(K), p, group=grp))
    bad = yt.clone()
    if xt.shape[0] and off + xt.shape[0] == N:             # only the rank holding the last global row sees the bad label
        bad[-1] = K + 3
    try:
        bfm.fm_fit_classes(xt, bad, range(K), p, group=grp)
        out["raised"] = False
    except ValueError:
        out["raised"] = True
    return out


class _Frame:
    """the two columns FMClassifier.fit reads, without label metadata"""

    def __init__(self, x, y):
        from pyspark.sql import ColumnData
        self._cols = {"features": ColumnData("vector", x, "f64"), "label": ColumnData("numeric", y, "f64")}

    def _column_tensor(self, name):
        return self._cols[name].data


def _shim_data():
    """the rows sorted by a binary label, label 0 first, so that a short first shard holds only label 0"""
    x, y = _data()
    yb = (y == 2).astype(np.float64)
    order = np.argsort(yb, kind="stable")
    return np.ascontiguousarray(x[order]), yb[order], int((yb == 0).sum())


def _shim_cases(n0):
    """name -> (global row cut between the ranks, label transform)"""
    return {"empty_first": (0, None), "only_label_0_first": (n0 // 2, None), "empty_last": (N, None),
            "one_class": (n0 // 2, "zeros"), "three_classes": (n0 // 2, "two_on_last_row")}


def _shim_run(x, y, lo, hi, how, dev):
    from pyspark.ml.classification import FMClassifier
    y = y.copy()
    if how == "zeros":
        y[:] = 0.0
    elif how == "two_on_last_row":
        y[-1] = 2.0
    df = _Frame(torch.from_numpy(x[lo:hi]).to(dev), torch.from_numpy(y[lo:hi]).to(dev))
    try:
        f = FMClassifier(factorSize=KF, maxIter=8, stepSize=0.05, seed=3).fit(df)._fit_result
    except Exception as e:                                 # IllegalArgumentException
        return {"raised": str(e)}
    return _fits_hex([f])[0]


def _ranks(rank, grp, dev):
    x, y = _data()
    res = {}
    for name, cut in SPLITS(N).items():
        lo, hi = block(rank, cut, N)
        res[name] = _run(x[lo:hi], y[lo:hi], dev, grp)
    xs, ys, n0 = _shim_data()
    res["shim"] = {}
    for name, (cut, how) in _shim_cases(n0).items():
        lo, hi = block(rank, cut, N)
        res["shim"][name] = _shim_run(xs, ys, lo, hi, how, dev)
    return res


def _two_ranks(tmp_path, mode):
    got = run(tmp_path, _ranks, mode=mode)
    x, y = _data()
    want = _run(x, y, torch.device("cuda", 0), None)
    assert want["raised"] is True
    xs, ys, n0 = _shim_data()
    want_shim = {name: _shim_run(xs, ys, 0, N, how, torch.device("cuda", 0)) for name, (_, how) in _shim_cases(n0).items()}
    assert want_shim["one_class"] == {"raised": "FMClassifier only supports binary classification. 1 classes detected in label"}
    assert want_shim["three_classes"]["raised"].startswith("FMClassifier only supports binary classification. 3 classes")
    for rank in (0, 1):
        for name in SPLITS(N):
            assert got[rank][name] == want, (rank, name)
        for name in want_shim:
            assert got[rank]["shim"][name] == want_shim[name], (rank, name)


def test_fm_two_gloo_ranks_equal_one_process(tmp_path):
    _two_ranks(tmp_path, "gloo")


@two_gpus
def test_fm_two_nccl_ranks_equal_one_process(tmp_path):
    _two_ranks(tmp_path, "nccl")
