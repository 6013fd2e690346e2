"""Feature selection over TWO RANKS: the dictionaries are merged from every rank's keys, the contingency counts are int64
sums, and the class sums and centred sums keep their chunk order across shards, so the p-values, statistics, degrees of
freedom and selected features equal the single-process result byte for byte — for even, uneven, chunk-aligned, short and
empty shards.  A column with more than 10000 distinct values on one rank only raises on both.  Two gloo ranks share one
GPU; the NCCL case needs two GPUs and is skipped otherwise."""
import numpy as np
import pytest
import torch

from ranks import block, run, two_gpus

pytestmark = pytest.mark.gpu

N, D = 30000, 12
CASES = {"even": (N, 15000), "uneven": (N, 11000), "chunk_aligned": (N, 8192), "short_first": (N, 2500),
         "short_total": (3000, 1200), "empty_last": (N, N), "empty_first": (N, 0)}


def _data():
    rng = np.random.default_rng(31)
    y = rng.integers(0, 4, N).astype(np.float64)
    x = rng.integers(0, 6, (N, D)).astype(np.float64)
    x[:, ::2] += np.floor(y[:, None] * rng.uniform(0, 1.5, (N, D // 2)))
    x[:, 1::3] = rng.normal(size=(N, len(range(1, D, 3)))) + 0.05 * y[:, None]
    x[:, 1::3] = np.round(x[:, 1::3], 2)                        # continuous-looking, but < 10000 values
    yc = x[:, 0] * 0.3 + rng.normal(size=N)
    return x, y, yc


def _run(x, y, yc, dev):
    from b200flow import selection as bs
    xt, yt, yct = (torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in (x, y, yc))
    hx = lambda a: [float(v).hex() for v in np.asarray(a, np.float64).ravel()]       # noqa: E731
    out = {}
    for name, res in (("chi", bs.chi_square_test(xt, yt)), ("anova", bs.anova_test(xt, yt)), ("fv", bs.f_value_test(xt, yct))):
        out[name] = {"p": hx(res.p_values), "s": hx(res.statistics), "dof": [int(v) for v in res.dof],
                     "sel": [bs.select(res.p_values, m, t) for m, t in (("numTopFeatures", 4), ("fdr", 0.05), ("fpr", 0.01))]}
    out["var"] = hx(bs.variances(xt))
    return out


def _ranks(rank, grp, dev):
    from b200flow import selection as bs
    x, y, yc = _data()
    res = {}
    for name, (total, cut) in CASES.items():
        lo, hi = block(rank, cut, total)
        res[name] = _run(x[lo:hi], y[lo:hi], yc[lo:hi], dev)
    wide = np.zeros((20000, 2))                             # rank 1 alone sees 10001 values in column 1
    if rank == 1:
        wide[:10001, 1] = np.arange(10001)
    try:
        bs.chi_square_test(torch.from_numpy(wide).to(dev), torch.zeros(20000, dtype=torch.float64, device=dev))
        res["overflow"] = "no error"
    except bs.TooManyValuesError as e:
        res["overflow"] = str(e)
    return res


def _two_ranks(tmp_path, mode):
    got = run(tmp_path, _ranks, mode=mode, timeout=900)
    x, y, yc = _data()
    want = {total: _run(x[:total], y[:total], yc[:total], torch.device("cuda", 0)) for total in sorted({t for t, _ in CASES.values()})}
    assert want[N]["chi"]["sel"][0] and want[N]["anova"]["sel"][0]
    for rank in (0, 1):
        for name, (total, _) in CASES.items():
            assert got[rank][name] == want[total], (rank, name)
        assert "more than 10000 distinct values in column 1" in got[rank]["overflow"], rank


def test_selection_two_gloo_ranks_equal_one_process(tmp_path):
    _two_ranks(tmp_path, "gloo")


@two_gpus
def test_selection_two_nccl_ranks_equal_one_process(tmp_path):
    _two_ranks(tmp_path, "nccl")
