"""NaiveBayes over TWO RANKS: the class sums keep their chunk order across shards and the bad-input counts are all-reduced, so
every rank's pi, theta and sigma, and its transform of its own rows, equal the single-process fit and transform bit for bit,
for all four model types, weighted and unweighted, and for even, uneven, short and empty shards.  Two gloo ranks share one
GPU; the NCCL case needs two GPUs and is skipped otherwise."""
import numpy as np
import pytest
import torch

from ranks import SPLITS, block, run, two_gpus

pytestmark = pytest.mark.gpu

N, D, C = 20000, 9, 4
TYPES = ("multinomial", "complement", "bernoulli", "gaussian")


def _data():
    rng = np.random.default_rng(17)
    y = rng.integers(0, C, N).astype(np.float64)
    counts = rng.poisson(1.0 + y[:, None] * np.arange(1, D + 1) / D, (N, D)).astype(np.float64)
    binary = (rng.random((N, D)) < 0.2 + 0.15 * y[:, None]).astype(np.float64)
    w = rng.uniform(0.0, 3.0, N)
    return counts, binary, y, w


def _one(x, xb, y, w, dev, offset):
    from b200flow import linear, naive_bayes as nb
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)          # noqa: E731
    hx = lambda a: [float(v).hex() for v in a.cpu().numpy().ravel()]          # noqa: E731
    out = {}
    for mt in TYPES:
        xs = xb if mt == "bernoulli" else x
        for weighted in (False, True):
            xt = t(xs).to(torch.float32) if mt == "gaussian" else t(xs)       # the gaussian case reads f32 features
            f = nb.nb_fit(xt, t(y), C, mt, 0.5, weights=t(w) if weighted else None, row_offset=offset)
            raw = linear.nb_raw(f, xt) if mt == "multinomial" else nb.nb_raw(f, xt)
            out[mt, weighted] = {"pi": hx(f.pi), "theta": hx(f.theta), "sigma": hx(f.sigma), "raw": hx(raw),
                                 "prob": hx(torch.softmax(raw, 1))}
    return out


def _ranks(rank, grp, dev):
    x, xb, y, w = _data()
    res = {}
    for name, cut in SPLITS(N).items():
        lo, hi = block(rank, cut, N)
        res[name] = _one(x[lo:hi], xb[lo:hi], y[lo:hi], w[lo:hi], dev, lo)
    return res


def _two_ranks(tmp_path, mode):
    got = run(tmp_path, _ranks, mode=mode, timeout=900)
    x, xb, y, w = _data()
    whole = _one(x, xb, y, w, torch.device("cuda", 0), 0)
    for rank in (0, 1):
        for name, cut in SPLITS(N).items():
            lo, hi = block(rank, cut, N)
            for key, want in whole.items():
                have = got[rank][name][key]
                for part in ("pi", "theta", "sigma"):
                    assert have[part] == want[part], (rank, name, key, part)
                for part in ("raw", "prob"):
                    mine, ref = have[part], want[part][lo * C:hi * C]
                    if key[0] == "multinomial":                   # a cuBLAS product (linear.nb_raw): its order depends on n
                        np.testing.assert_allclose([float.fromhex(v) for v in mine], [float.fromhex(v) for v in ref], rtol=1e-12)
                    else:
                        assert mine == ref, (rank, name, key, part)


def test_naive_bayes_two_gloo_ranks_equal_one_process(tmp_path):
    _two_ranks(tmp_path, "gloo")


@two_gpus
def test_naive_bayes_two_nccl_ranks_equal_one_process(tmp_path):
    _two_ranks(tmp_path, "nccl")
