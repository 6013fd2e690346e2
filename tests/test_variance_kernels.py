"""The variance-tree kernels (csrc/gbt.cu, csrc/regression.cu, csrc/tree_walk.cuh) called one by one through the C ABI, on
synthetic records, entries, residual grids, histograms and node pools whose edges are placed on purpose:

  gbt_hist_level_classes     2, 3 and 23 classes over one entry array, feature passes, segments around the chunk size,
                             negative q and cells near 2^62;
  gbt_score_level            m = 1, 4, 5, 41, ties across warps, within a warp and across lanes, odd and 256-bin features,
                             categoricals with equal centroids, empty categories and arity 256, one-bin features, large and
                             small grid exponents, and every leaf rule including a child impurity at MLUtils.EPSILON;
  gbt_leaf_values, gbr_leaf_values, reg_leaf_table, reg_divide;
  gbt_update, gbt_update_classes, gbt_output, gbr_update: tree walks through continuous and categorical splits (mask words
                             0-3), NaN payloads, exp overflow, zero differences and half-way grid points;
  reg_labels, reg_grid, reg_tree_weights, reg_eval_max, reg_eval_sums.

Integers (histogram cells, node stats, weight totals, limb sums, counts, max bits) are compared exactly with Python int
sums; fp64 values the kernels define to round like Spark's JVM are compared bit for bit with the oracles' restatements.  The
split choice is also checked against an independent exact reference: every candidate's Variance gain as a Fraction.  The
first test needs no GPU: it checks gbt_oracle.best_split against that reference, so that a GPU failure points at a kernel."""
import itertools
from fractions import Fraction

import numpy as np
import pytest
import torch

import gbt_oracle as go
import gbt_regression_oracle as gro
import regression_oracle as ro
from b200flow import _lib, forest as fr
from b200flow._lib import NODE_DTYPE, SPLIT_DTYPE

DEV = "cuda"
SENTINEL = -7
DBL_MAX = go.DBL_MAX


# ------------------------------------------------------------------------------------------------ exact split reference
def exact_split(hist, subset, feat_bins, feat_kind, S, S2, min_inst=1):
    """Spark's Variance split choice on the integer cells, in exact rational arithmetic: impurity Σq2/c - (Σq/c)² on the
    grid, children weighted by their counts; categorical bins ordered by exact centroid (empty categories last, ties by
    index).  -> (candidates [(gain, j, split, L, mask int or None)], index of the first maximum or None, scale) where scale
    is the parent's mean Σw·q2 / Σw."""
    tot = [int(v) for v in hist[0].sum(0)]
    s1, s2 = Fraction(2) ** -S, Fraction(2) ** -S2

    def imp(c, a, b):
        return Fraction(0) if c == 0 else Fraction(b) * s2 / c - (Fraction(a) * s1 / c) ** 2

    parent = imp(*tot)
    cands = []
    for j, f in enumerate(subset):
        nb = int(feat_bins[f])
        raw = [[int(v) for v in hist[j][b]] for b in range(nb)]
        if feat_kind[f]:
            order = sorted(range(nb), key=lambda c: (raw[c][0] == 0, Fraction(raw[c][1], raw[c][0]) if raw[c][0] else 0))
        else:
            order = list(range(nb))
        L = [0, 0, 0]
        for sp in range(nb - 1):
            L = [L[k] + raw[order[sp]][k] for k in range(3)]
            R = [tot[k] - L[k] for k in range(3)]
            if L[0] < min_inst or R[0] < min_inst:
                continue
            g = parent - Fraction(L[0], tot[0]) * imp(*L) - Fraction(R[0], tot[0]) * imp(*R)
            mask = sum(1 << c for c in order[:sp + 1]) if feat_kind[f] else None
            cands.append((g, j, sp, tuple(L), mask))
    best = None
    for i, c in enumerate(cands):
        if best is None or c[0] > cands[best][0]:
            best = i
    scale = Fraction(tot[2]) * s2 / tot[0] if tot[0] else Fraction(0)
    return cands, best, scale


def _mask_int(words):
    return sum(int(w) << (64 * q) for q, w in enumerate(words))


def check_exact(cands, best, scale, j, sp, L, mask, gain, separated):
    """the kernel's (or the oracle's) choice against the exact reference.  separated: the exact best beats every other
    candidate by 1e-6 scale (checked: a construction error otherwise), and the fp64 gain lies within 1e-10 scale of it."""
    assert best is not None
    g, bj, bsp, bL, bmask = cands[best]
    if separated:
        runner = max((c[0] for i, c in enumerate(cands) if i != best), default=None)
        assert runner is None or g - runner >= scale / 10 ** 6, "construction: the case is not separated"
        assert abs(Fraction(gain) - g) <= scale / 10 ** 10, (float(g), gain)
    assert (j, sp) == (bj, bsp), ((j, sp), (bj, bsp))
    assert tuple(int(v) for v in L) == bL
    assert (mask if mask is None else _mask_int(mask)) == bmask


# ------------------------------------------------------------------------------------------------ score cases
def _node(rng, n, fb, fk, subset, n_bins, S, S2, sig, cut=None, noise=0.05, amp=1.0, w_max=3):
    """cells [m][n_bins][3] of n records with random bins (every feature sums to the node's totals); the residual follows
    subset position sig: a step at bin `cut` (continuous) or a random mean per category, plus noise, times amp"""
    m = len(subset)
    bins = np.stack([rng.integers(0, fb[f], n) for f in subset], 1)
    f = subset[sig]
    if fk[f]:
        mu = rng.uniform(-1.5, 1.5, fb[f])[bins[:, sig]]
    else:
        c = (fb[f] - 1) // 2 if cut is None else cut
        mu = np.where(bins[:, sig] > c, 1.0, -0.5)
    r = np.clip(mu + noise * rng.standard_normal(n), -4.0, 4.0) * amp
    q, q2 = go.to_grid(r, S, S2)
    w = rng.integers(1, w_max + 1, n)
    assert m == bins.shape[1]
    return go.node_hist(bins, w, q, q2, n_bins)


def _grid(n, E=0):
    """(S, S2) of a node of n records with weights <= 3 and |r| <= 4 2^E: every cell stays below 2^62"""
    S, S2 = go.grid_shift(12 * n)
    return S - E, S2 - 2 * E


class ScoreGroup:
    """one gbt_score_level launch: slots sharing m, n_bins, feature metadata, grid and leaf parameters.  kind per slot:
    'sep' (exact best separated from the rest), 'tie' (an exact tie the kernel must break), or 'restate' (bytes only)."""

    def __init__(self, fb, fk, n_bins, S, S2, level=0, max_depth=5, min_inst=1, min_gain=0.0):
        self.fb, self.fk = np.asarray(fb, np.int32), np.asarray(fk, np.int32)
        self.n_bins, self.S, self.S2 = n_bins, S, S2
        self.level, self.max_depth, self.min_inst, self.min_gain = level, max_depth, min_inst, min_gain
        self.hists, self.subsets, self.kinds = [], [], []

    def add(self, h, subset, kind):
        self.hists.append(np.asarray(h, np.int64)); self.subsets.append(np.asarray(subset)); self.kinds.append(kind)
        return self


def _sep_group(m, F, fb, fk, n_bins, E, seed, n=4000, sigs=None):
    rng = np.random.default_rng(seed)
    S, S2 = _grid(n, E)
    g = ScoreGroup(fb, fk, n_bins, S, S2)
    for k, sig in enumerate(sigs if sigs is not None else range(m)):
        sub = np.sort(rng.choice(F, m, replace=False)) if F > m else np.arange(m)
        while fb[sub[sig]] < 2:
            sub = np.sort(rng.choice(F, m, replace=False))
        g.add(_node(rng, n, fb, fk, sub, n_bins, S, S2, sig, amp=2.0 ** E), sub, "sep")
    return g


def _wide_features(F, seed):
    """F features up to 256 bins: 256-bin continuous and arity-256 categoricals, odd widths, one-bin features"""
    rng = np.random.default_rng(seed)
    fb = rng.integers(2, 257, F).astype(np.int32)
    fb[:6] = [256, 256, 1, 37, 255, 2]
    fk = (rng.random(F) < 0.35).astype(np.int32)
    fk[:6] = [0, 1, 0, 1, 1, 1]
    fk[fb == 1] = 0
    return fb, fk


def tie_group():
    """exact ties: identical features at positions in different warps (the lower position in the higher warp too) and in
    one warp; splits with the same partition on different lanes, on one lane, and across a round of 32; a categorical whose
    mirrored ranks give bit-equal gains"""
    rng = np.random.default_rng(77)
    m, nb, n = 8, 256, 6000
    fb = np.array([70] * 6 + [256, 256], np.int32)
    fk = np.zeros(8, np.int32)
    S, S2 = _grid(n)
    g = ScoreGroup(fb, fk, nb, S, S2)
    sub = np.arange(m)
    for a, b in ((3, 4), (2, 6), (1, 5), (0, 4)):        # warps 3/0, 2/2, 1/1, 0/0: position a must win
        h = _node(rng, n, fb, fk, sub, nb, S, S2, a, cut=20)
        h[b] = h[a]
        g.add(h, sub, "tie")
    for sig, cut, empty in ((1, 31, range(32, 33)), (2, 40, range(41, 42)), (6, 100, range(101, 134)), (7, 5, range(6, 70))):
        h = _node(rng, n, fb, fk, sub, nb, S, S2, sig, cut=cut)
        for b in empty:                                    # splits cut .. cut + len(empty) now share one partition
            h[sig, empty[-1] + 1] += h[sig, b]; h[sig, b] = 0
        g.add(h, sub, "tie")
    return g


def mirror_group():
    """a categorical and a continuous feature of residuals -3/4, -1/4, 0, 1/4 with counts 1, 4, 4, 1: the first two splits
    (for the categorical: ranks) have exactly equal gains, and bit-equal fp64 gains, so the lowest must win; the other
    features carry nothing"""
    S, S2 = 40, 38
    fb = np.array([4, 4, 3, 2], np.int32)
    fk = np.array([1, 0, 0, 0], np.int32)
    g = ScoreGroup(fb, fk, 4, S, S2)
    for j, cells in ((0, ((1, 1), (0, 4), (-3, 1), (-1, 4))), (1, ((-3, 1), (-1, 4), (0, 4), (1, 1)))):
        h = np.zeros((4, 4, 3), np.int64)
        for b, (v, c) in enumerate(cells):                 # c records of residual v / 4
            h[j, b] = (c, c * v * 2 ** (S - 2), c * v * v * 2 ** (S2 - 4))
        tot = h[j].sum(0)
        for k in range(4):
            if k != j:
                h[k, 0] = tot
        g.add(h, np.arange(4), "tie")
    return g


def categorical_group(E):
    """arity-256 categoricals with runs of equal centroids (identical cells) and forty empty categories, next to
    continuous features; the signal sits on a different position in each slot"""
    rng = np.random.default_rng(256 + E)
    fb = np.array([256, 256, 255, 40, 256, 7], np.int32)
    fk = np.array([1, 1, 1, 0, 1, 1], np.int32)
    n = 20000
    S, S2 = _grid(n, E)
    g = ScoreGroup(fb, fk, 256, S, S2)
    sub = np.arange(6)
    for s in range(6):
        h = _node(rng, n, fb, fk, sub, 256, S, S2, s % 6, noise=0.3, amp=2.0 ** E)
        for j in np.nonzero(fb >= 255)[0]:
            pool = h[j, 10:30].sum(0)
            h[j, 10:30] = pool // 20                         # categories 10-29: one centroid
            h[j, 29] += pool - 20 * (pool // 20)
            h[j, 60] += h[j, 100:140].sum(0)
            h[j, 100:140] = 0                                # empty: ranked last, in index order
        g.add(h, sub, "choice")
    return g


def equal_centroid_min_inst_group():
    """category 0 (one record, centroid -1) and categories 1, 2 of one centroid (100 records and 1): minInstancesPerNode = 2
    admits only the split that ranks category 2 before category 1.  Ranked by index (stable), no split is valid."""
    S, S2 = 40, 38
    g = ScoreGroup([3], [1], 3, S, S2, min_inst=2)
    h = np.zeros((1, 3, 3), np.int64)
    h[0, 0] = (1, -2 ** S, 2 ** S2)
    h[0, 1] = (100, 100 * 2 ** (S - 1), 100 * 2 ** (S2 - 2))
    h[0, 2] = (1, 2 ** (S - 1), 2 ** (S2 - 2))
    g.add(h, [0], "restate")
    h2 = h.copy()
    h2[0, 2] = (2, 2 * 2 ** (S - 1), 2 * 2 ** (S2 - 2))   # now category 2 may stand alone on the right
    g.add(h2, [0], "choice")
    return g


def score_groups():
    """every launch of the scoring tests, by name (the host-only test checks the oracle on the same inputs)"""
    fb41, fk41 = _wide_features(50, 41)
    groups = {
        "m1_odd": _sep_group(1, 1, [37], [0], 37, 0, 1, sigs=[0, 0, 0]),
        "m4": _sep_group(4, 4, [37, 37, 20, 37], [0, 1, 0, 1], 37, 0, 4),
        "m5": _sep_group(5, 5, [9, 33, 2, 17, 33], [1, 0, 0, 1, 0], 33, 0, 5),
        "m41": _sep_group(41, 50, fb41, fk41, 256, 0, 41, n=20000, sigs=[40, 37, 0, 4, 12, 1]),
        "m41_large_S": _sep_group(41, 50, fb41, fk41, 256, -100, 42, n=20000, sigs=[39, 3]),
        "m41_small_S": _sep_group(41, 50, fb41, fk41, 256, 150, 43, n=20000, sigs=[38, 5]),
        "ties": tie_group(),
        "mirror": mirror_group(),
        "categorical": categorical_group(0),
        "categorical_small_S": categorical_group(150),
        "equal_centroids_min_inst": equal_centroid_min_inst_group(),
    }
    return groups


# ------------------------------------------------------------------------------------------------ host-only self-check
_GROUPS = None


def _groups():
    global _GROUPS
    if _GROUPS is None:
        _GROUPS = score_groups()
    return _GROUPS


def _slot_exact(g, s):
    return exact_split(g.hists[s], g.subsets[s], g.fb, g.fk, g.S, g.S2, g.min_inst)


@pytest.mark.parametrize("name", ["m1_odd", "m4", "m5", "m41", "m41_large_S", "m41_small_S", "ties", "mirror", "categorical",
                                  "categorical_small_S", "equal_centroids_min_inst"])
def test_oracle_best_split_equals_exact_reference(name):
    g = _groups()[name]
    for s, kind in enumerate(g.kinds):
        tot = g.hists[s][0].sum(0)
        _, best = go.best_split(g.hists[s], g.subsets[s], g.fb, g.fk, tot, g.S, g.S2, g.min_inst, g.min_gain)
        cands, bi, scale = _slot_exact(g, s)
        if bi is None:
            assert best is None
            continue
        gain, j, sp, L, mask = best
        check_exact(cands, bi, scale, j, sp, L, mask, gain, kind == "sep")
        if kind == "tie":                                  # the case really is a tie
            assert sum(1 for c in cands if c[0] == cands[bi][0]) >= 2


# ------------------------------------------------------------------------------------------------ device helpers
_alive = []


@pytest.fixture(autouse=True)
def _keep_arguments_alive():
    # the kernels run asynchronously on device pointers: every tensor _dev makes lives until the test has synchronised
    yield
    if _alive:
        torch.cuda.synchronize()
        _alive.clear()


def _dev(a):
    a = np.ascontiguousarray(a)
    if a.dtype in (np.uint16, np.uint32, np.uint64):      # same bits as the signed type torch handles everywhere
        a = a.view({2: np.int16, 4: np.int32, 8: np.int64}[a.dtype.itemsize])
    t = torch.from_numpy(a).to(DEV)
    _alive.append(t)
    return t


def _host(t, dtype=None):
    torch.cuda.synchronize()
    a = t.cpu().numpy()
    return a if dtype is None else a.view(dtype)


def _bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.uint64)


def assert_same_f64(got, want, what=""):
    """bit-for-bit, except that any NaN equals any NaN (the device's and numpy's NaN payloads differ)"""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    assert got.shape == want.shape
    both_nan = np.isnan(got) & np.isnan(want)
    bad = (_bits(got) != _bits(want)) & ~both_nan
    assert not bad.any(), "%s: %d differ, first at %s: got %r want %r" % (
        what, bad.sum(), np.argwhere(bad)[0], got[bad][0], want[bad][0])


def _call(name, *args):
    _lib.call(name, *[_lib.ptr(a) if isinstance(a, torch.Tensor) else a for a in args])


# ------------------------------------------------------------------------------------------------ gbt_hist_level_classes
def _hist_ref(tp, ent, rq, seg_begin, seg_end, slot_class, subset, n_bins):
    """{Σw, Σw·q, Σw·q2} [slot][m][n_bins][3] as Python ints"""
    S, m = len(seg_begin), subset.shape[1]
    out = np.zeros((S, m, n_bins, 3), object)
    for s in range(S):
        e = ent[seg_begin[s]:seg_end[s]]
        if not len(e):
            continue
        rec, w = e[:, 0].astype(np.int64), e[:, 1].astype(object)
        q = rq[slot_class[s], rec, 0].astype(object); q2 = rq[slot_class[s], rec, 1].astype(object)
        vals = np.stack([w, w * q, w * q2], 1)
        for j in range(m):
            np.add.at(out[s, j], tp[rec, subset[s, j]].astype(np.int64), vals)
    return out


CH = fr.CHUNK_ROWS


@pytest.mark.gpu
@pytest.mark.parametrize("K,m,n_bins", [(2, 5, 70), (3, 9, 37), (23, 41, 256), (3, 13, 255)])
def test_hist_level_classes(K, m, n_bins):
    # slots of interleaved classes over one entry array; segments of 0, 1, CH - 1, CH, CH + 1 and more entries; with
    # n_bins = 256 and m = 41 the slot histogram (246 KB) goes in three feature passes.  Class 1 (when K = 3: one slot) has
    # q = q2 = B and class 2 q = -B: every cell of the constant feature F - 1 sums to just below ±2^62.
    rng = np.random.default_rng(K * 1000 + m)
    F, U = max(m, 20) + 3, 3000
    stride = fr.tp_stride(F)
    tp = np.zeros((U, stride), np.uint8)
    tp[:, :F] = rng.integers(0, n_bins, (U, F))
    tp[:, F - 1] = n_bins - 1                               # a constant feature: its cell is the slot's total
    lens = [0, 1, CH - 1, CH, CH + 1, 5, 2 * CH + 3, 0, 700, 64][:max(K, 4) + 4] + [int(v) for v in rng.integers(0, 300, 2 * K)]
    n_slots = len(lens)
    slot_class = np.array([(s * 7 + 3) % K for s in range(n_slots)], np.int32)
    seg_begin, seg_end, pos = [], [], int(rng.integers(0, 5))
    for n in lens:
        seg_begin.append(pos); seg_end.append(pos + n); pos += n + int(rng.integers(0, 3))
    E = pos
    ent = np.stack([rng.integers(0, U, E), rng.integers(1, 6, E)], 1).astype(np.int32)
    ent[rng.random(E) < 0.02, 1] = 0                        # zero weights count for nothing
    rq = np.stack([rng.integers(-(1 << 40), 1 << 40, (K, U)), rng.integers(0, 1 << 40, (K, U))], 2).astype(np.int64)
    big = [s for s in range(n_slots) if lens[s] > 0 and slot_class[s] in (1, 2) and K == 3]
    if big:
        for cls, sign in ((1, 1), (2, -1)):
            wsum = max((int(ent[seg_begin[s]:seg_end[s], 1].sum()) for s in big if slot_class[s] == cls), default=1)
            B = ((1 << 62) - 1) // max(wsum, 1)
            rq[cls, :, 0] = sign * B
            rq[cls, :, 1] = B
    subset = np.stack([np.concatenate([np.sort(rng.choice(F - 1, m - 1, replace=False)), [F - 1]]) for _ in range(n_slots)])
    subset = subset.astype(np.uint16)
    nch = [(n + CH - 1) // CH for n in lens]
    chunk_off = np.zeros(n_slots + 1, np.int64); chunk_off[1:] = np.cumsum(nch)
    hist = torch.zeros(n_slots * m * n_bins * 3, dtype=torch.int64, device=DEV)
    _call("b200flow_gbt_hist_level_classes", _dev(tp), stride, _dev(ent), _dev(rq), U, _dev(slot_class), n_slots,
          _dev(np.array(seg_begin, np.int64)), _dev(np.array(seg_end, np.int64)), _dev(chunk_off), int(chunk_off[-1]), CH,
          _dev(subset), m, n_bins, hist)
    got = _host(hist).reshape(n_slots, m, n_bins, 3)
    want = _hist_ref(tp, ent, rq, seg_begin, seg_end, slot_class, subset, n_bins)
    assert max(abs(int(v)) for v in want.ravel()) < 1 << 62
    assert np.array_equal(got.astype(object), want)
    if big:
        top = max(abs(int(v)) for v in want[big, m - 1, n_bins - 1, 1])
        assert top > (1 << 62) - (1 << 46)
        assert min(int(v) for v in want[big, m - 1, n_bins - 1, 1]) < 0


# ------------------------------------------------------------------------------------------------ gbt_score_level
def score_restated(h, subset, g):
    """the split record, node stats and child stats of one slot, from gbt_oracle.best_split and the leaf rules of
    gbt_oracle.grow_tree"""
    tot = h[0].sum(0)
    parent, best = go.best_split(h, subset, g.fb, g.fk, tot, g.S, g.S2, g.min_inst, g.min_gain)
    o = np.zeros(1, SPLIT_DTYPE)
    o["gain"] = best[0] if best is not None else -DBL_MAX
    o["impurity"] = parent
    o["feat"] = -1
    leaf = best is None or not best[0] > 0.0 or g.level >= g.max_depth
    flags = 1 if leaf else 0
    L = best[3] if best is not None else np.zeros(3, np.int64)
    R = tot - L if best is not None else np.zeros(3, np.int64)
    if not leaf:
        _, j, sp, _, mask = best
        o["feat"] = subset[j]; o["kind"] = 0 if mask is None else 1; o["bin_thr"] = sp
        if mask is not None:
            o["mask"] = mask
        il, ir = float(go.variance(L[0], L[1], L[2], g.S, g.S2)), float(go.variance(R[0], R[1], R[2], g.S, g.S2))
        if g.level + 1 == g.max_depth or abs(il) < go.EPSILON:
            flags |= 2
        if g.level + 1 == g.max_depth or abs(ir) < go.EPSILON:
            flags |= 4
    o["flags"] = flags
    return o, tot, L, R


def run_score(g):
    hists = np.stack(g.hists)
    n_slots, m, n_bins, _ = hists.shape
    assert n_bins == g.n_bins and np.abs(hists).max() < 1 << 62
    split = torch.zeros((n_slots, 64), dtype=torch.uint8, device=DEV)
    st = torch.full((3, n_slots, 3), SENTINEL, dtype=torch.int64, device=DEV)
    _call("b200flow_gbt_score_level", _dev(hists), n_slots, _dev(np.stack(g.subsets).astype(np.uint16)), m, n_bins, _dev(g.fb),
          _dev(g.fk), g.S, g.S2, g.level, g.max_depth, g.min_inst, float(g.min_gain), split, st[0], st[1], st[2])
    got, stats = _host(split), _host(st)
    for s in range(n_slots):
        want, tot, L, R = score_restated(g.hists[s], g.subsets[s], g)
        assert got[s].tobytes() == want.tobytes(), "slot %d: got %s want %s" % (s, got[s].view(SPLIT_DTYPE)[0], want[0])
        assert np.array_equal(stats[0, s], tot) and np.array_equal(stats[1, s], L) and np.array_equal(stats[2, s], R), s
    return got.view(SPLIT_DTYPE).reshape(n_slots), stats


def check_score_exact(g, rec, stats):
    """each non-leaf slot's choice (and, for 'sep' slots, its gain) against the exact reference"""
    for s, kind in enumerate(g.kinds):
        if kind == "restate" or rec["flags"][s] & 1:
            continue
        cands, bi, scale = _slot_exact(g, s)
        j = int(np.nonzero(g.subsets[s] == rec["feat"][s])[0][0])
        check_exact(cands, bi, scale, j, int(rec["bin_thr"][s]), stats[1, s], rec["mask"][s] if rec["kind"][s] else None,
                    float(rec["gain"][s]), kind == "sep")


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["m1_odd", "m4", "m5", "m41", "m41_large_S", "m41_small_S", "categorical", "categorical_small_S"])
def test_score_separated_and_categorical(name):
    g = _groups()[name]
    rec, stats = run_score(g)
    assert (rec["flags"] & 1 == 0).all()
    check_score_exact(g, rec, stats)
    if name.startswith("categorical"):
        assert np.any(rec["mask"][:, 1:] != 0) and (rec["kind"] == 1).any()


@pytest.mark.gpu
def test_score_ties():
    g = _groups()["ties"]
    rec, stats = run_score(g)
    check_score_exact(g, rec, stats)
    assert list(rec["feat"][:4]) == [3, 2, 1, 0]
    assert list(rec["bin_thr"][4:]) == [31, 40, 100, 5]
    g = _groups()["mirror"]
    rec, stats = run_score(g)
    check_score_exact(g, rec, stats)
    assert list(rec["bin_thr"]) == [0, 0] and list(rec["feat"]) == [0, 1] and rec["mask"][0][0] == 0b100


@pytest.mark.gpu
def test_score_equal_centroids_rank_stably():
    g = _groups()["equal_centroids_min_inst"]
    rec, stats = run_score(g)
    assert rec["flags"][0] == 1 and rec["gain"][0] == -DBL_MAX and (stats[1, 0] == 0).all()
    assert rec["flags"][1] & 1 == 0 and rec["mask"][1][0] == 0b011
    check_score_exact(g, rec, stats)


def _eps_slot(S, S2, num):
    """two bins: bin 0 holds one record of impurity num/4 EPSILON (q = 0, Σq2 = num 2^(S2 - 54)), bin 1 a hundred records of
    variance 1 around 1; the one split leaves bin 0 alone on the left"""
    h = np.zeros((1, 2, 3), np.int64)
    h[0, 0] = (1, 0, num * 2 ** (S2 - 54))
    h[0, 1] = (100, 100 * 2 ** S, 200 * 2 ** S2)
    return h


@pytest.mark.gpu
@pytest.mark.parametrize("edge", ["no_valid_split", "min_info_gain", "gain_zero", "level_eq_max", "last_level", "epsilon", "defaults"])
def test_score_leaf_rules(edge):
    S, S2 = 44, 54
    kw = dict(no_valid_split=dict(min_inst=10 ** 6), min_info_gain=dict(min_gain=1e6), level_eq_max=dict(level=5, max_depth=5),
              last_level=dict(level=4, max_depth=5), defaults=dict(level=1, max_depth=7)).get(edge, {})
    g = ScoreGroup([2], [0], 2, S, S2, **kw)
    for num in (3, 4, 5):                                   # left child impurity below, at and above MLUtils.EPSILON
        g.add(_eps_slot(S, S2, num), [0], "restate")
        g.add(_eps_slot(S, S2, num)[:, ::-1].copy(), [0], "restate")      # the same on the right
    if edge in ("gain_zero", "defaults"):                   # every residual 1/2 exactly: each impurity and gain is 0
        h = np.zeros((1, 2, 3), np.int64)
        h[0, 0] = (3, 3 * 2 ** (S - 1), 3 * 2 ** (S2 - 2)); h[0, 1] = (5, 5 * 2 ** (S - 1), 5 * 2 ** (S2 - 2))
        g.add(h, [0], "restate")
        g.add(np.zeros((1, 2, 3), np.int64), [0], "restate")   # an empty node
    rec, stats = run_score(g)
    flags = list(rec["flags"])
    if edge in ("no_valid_split", "min_info_gain"):
        assert flags == [1] * 6 and (rec["gain"] == -DBL_MAX).all() and (stats[1:] == 0).all()
    elif edge == "level_eq_max":
        assert flags == [1] * 6 and (rec["gain"] > 0).all() and (stats[1, :, 0] > 0).all()
    elif edge == "last_level":
        assert flags == [6] * 6
    else:
        assert flags[:6] == [2, 4, 0, 0, 0, 0]
        if edge != "epsilon":
            assert flags[6:] == [1, 1] and rec["gain"][6] == 0.0 and rec["gain"][7] == -DBL_MAX and stats[1, 6, 0] == 3


# ------------------------------------------------------------------------------------------------ leaf values
def _stats(rng, n):
    st = np.stack([rng.integers(0, 1 << 40, n), rng.integers(-(1 << 61), 1 << 61, n), rng.integers(0, 1 << 61, n)], 1)
    st[:3] = [(0, 0, 0), (0, 5, 7), (0, -5, 7)]             # empty nodes: 0/0 = NaN and ±inf
    st[3] = (1, (1 << 62) - 1, (1 << 62) - 1)
    return st.astype(np.int64)


def _leaf_value(st, weight, S):
    return go.leaf_value(dict(stats=st), weight, S)


@pytest.mark.gpu
@pytest.mark.parametrize("S", [44, -150, 200])
def test_gbt_leaf_values(S):
    rng = np.random.default_rng(S + 1000)
    n, T = 1000, 7
    st = _stats(rng, n)
    node_tree = rng.integers(0, T, n).astype(np.int32)
    tw = np.array([1.0, 0.1, 0.3, 1e-300, -2.5, 0.0, 1e300])
    out = torch.full((n,), 12.5, dtype=torch.float64, device=DEV)
    _call("b200flow_gbt_leaf_values", n, _dev(st), _dev(node_tree), _dev(tw), S, out)
    want = np.array([_leaf_value(st[i], tw[node_tree[i]], S) for i in range(n)])
    assert np.isnan(want[0])
    assert_same_f64(_host(out), want, "payload")


@pytest.mark.gpu
@pytest.mark.parametrize("S", [44, -150])
def test_gbr_leaf_values_only_its_tree(S):
    rng = np.random.default_rng(S + 2000)
    n = 700
    st = _stats(rng, n)
    node_tree = rng.integers(0, 4, n).astype(np.int32)
    node_tree[:4] = 2
    before = rng.standard_normal(n)
    out = _dev(before.copy())
    _call("b200flow_gbr_leaf_values", n, _dev(st), _dev(node_tree), 2, 0.1, S, out)
    want = np.where(node_tree == 2, [_leaf_value(st[i], 0.1, S) for i in range(n)], before)
    assert_same_f64(_host(out), want, "payload")


@pytest.mark.gpu
@pytest.mark.parametrize("width", [1, 2])
@pytest.mark.parametrize("S,S2", [(44, 44), (-140, -300)])
def test_reg_leaf_table(width, S, S2):
    rng = np.random.default_rng(width * 10 + abs(S))
    n = 600
    st = _stats(rng, n)
    st[4] = (1, 3, 1)                                       # count 1
    st[5] = (7, 0, 0)
    table = torch.full((n, width), 3.25, dtype=torch.float64, device=DEV)
    _call("b200flow_reg_leaf_table", n, _dev(st), S, S2, table, width)
    got = _host(table)
    assert_same_f64(got[:, 0], [_leaf_value(st[i], 1.0, S) for i in range(n)], "mean")
    if width == 2:
        assert_same_f64(got[:, 1], go.variance(st[:, 0], st[:, 1], st[:, 2], S, S2), "variance")


@pytest.mark.gpu
@pytest.mark.parametrize("d", [3.0, 7.0, -0.1])
def test_reg_divide(d):
    rng = np.random.default_rng(int(abs(d) * 10))
    x = rng.standard_normal(1000) * 10.0 ** rng.integers(-300, 300, 1000)
    x[:4] = [0.0, -0.0, np.inf, np.nan]
    t = _dev(x.copy())
    _call("b200flow_reg_divide", t, len(x), d, t)            # in place, as the forest's mean calls it
    with np.errstate(all="ignore"):
        assert_same_f64(_host(t), x / d, "quotient")


# ------------------------------------------------------------------------------------------------ tree pools and walks
def random_tree(rng, fb, fk, depth):
    """{nid: node} in gbt_oracle's form; categorical masks draw bits in all four words"""
    nodes = {}

    def grow(nid, d):
        if d == depth or (d > 1 and rng.random() < 0.2):
            nodes[nid] = dict(leaf=True, feat=-1, kind=0, bin_thr=0, mask=np.zeros(4, np.uint64))
            return
        f = int(rng.integers(0, len(fb)))
        if fk[f]:
            mask = rng.integers(0, 1 << 63, 4, dtype=np.uint64) | (rng.integers(0, 2, 4, dtype=np.uint64) << np.uint64(63))
            nodes[nid] = dict(leaf=False, feat=f, kind=1, bin_thr=int(rng.integers(0, 255)), mask=mask)
        else:
            nodes[nid] = dict(leaf=False, feat=f, kind=0, bin_thr=int(rng.integers(0, fb[f])), mask=np.zeros(4, np.uint64))
        grow(2 * nid, d + 1)
        grow(2 * nid + 1, d + 1)

    grow(1, 0)
    return nodes


def build_pool(trees):
    """trees [root index] -> (nodes NODE_DTYPE [P], node_mask uint64 [P][4], {(root, nid): pool index}); roots first,
    then each split's two children as an adjacent pair"""
    R = len(trees)
    order = [(r, 1) for r in range(R)]
    index = {(r, 1): r for r in range(R)}
    nxt = R
    i = 0
    while i < len(order):
        r, nid = order[i]
        if not trees[r][nid]["leaf"]:
            for c in (2 * nid, 2 * nid + 1):
                index[(r, c)] = nxt; nxt += 1; order.append((r, c))
        i += 1
    nodes = np.zeros(nxt, NODE_DTYPE)
    mask = np.zeros((nxt, 4), np.uint64)
    for (r, nid), p in index.items():
        nd = trees[r][nid]
        nodes[p]["nid"] = nid
        if nd["leaf"]:
            nodes[p]["feat"] = -1
            continue
        nodes[p]["feat"] = nd["feat"]
        nodes[p]["kind_bin"] = (nd["kind"] << 16) | nd["bin_thr"]
        nodes[p]["left"] = index[(r, 2 * nid)]
        mask[p] = nd["mask"]
    return nodes, mask, index


def leaf_index(trees, index, root, bins):
    return np.array([index[(root, int(nid))] for nid in go.walk(trees[root], bins)], np.int64)


def walk_case(rng, n, F, n_trees, depth=7):
    """records over F features (256-bin categoricals and continuous features of several widths) and n_trees trees"""
    fb = np.array(([256, 256, 130, 70, 256, 2, 17] * 3)[:F], np.int32)
    fk = np.array(([1, 0, 1, 0, 1, 0, 1] * 3)[:F], np.int32)
    bins = np.stack([rng.integers(0, b, n) for b in fb], 1).astype(np.uint8)
    trees = [random_tree(rng, fb, fk, depth) for _ in range(n_trees)]
    nodes, mask, index = build_pool(trees)
    return bins, trees, nodes, mask, index


# ------------------------------------------------------------------------------------------------ gbt_update / _classes / output
def _records(bins, labels, F):
    tp = np.zeros((bins.shape[0], fr.tp_stride(F)), np.uint8)
    tp[:, :F] = bins
    tp[:, F] = labels
    return tp


@pytest.mark.gpu
def test_gbt_update_walk_nan_and_exp_range():
    rng = np.random.default_rng(5)
    n, F, T = 5000, 12, 3
    bins, trees, nodes, mask, index = walk_case(rng, n, F, T)
    labels = rng.integers(0, 2, n).astype(np.uint8)
    y = np.where(labels > 0, 1.0, -1.0)
    payload = rng.standard_normal(len(nodes)) * 0.5
    leaf1 = leaf_index(trees, index, 1, bins)
    nan_leaf = next(int(v) for v in leaf1[40:] if v not in set(leaf1[10:40].tolist()))
    payload[nan_leaf] = np.nan                              # an empty tree's 0/0 leaf
    margin0 = rng.standard_normal(n)
    margin0[10:20] = 400.0 * y[10:20]                       # 2yF > 709.78: exp overflows, r = ±0
    margin0[20:30] = -400.0 * y[20:30]                      # 2yF < -745.13: exp underflows, r = 4y
    margin0[30:40] = -payload[leaf1[30:40]]                 # F = 0: r = 2y
    S, S2 = go.grid_shift(n)
    tp = _dev(_records(bins, labels, F))
    margin = _dev(margin0.copy())
    rq = torch.full((n, 2), SENTINEL, dtype=torch.int64, device=DEV)
    _call("b200flow_gbt_update", tp, tp.shape[1], F, n, _dev(nodes.view(np.uint8)), _dev(mask), _dev(payload), 1, S, S2, margin, rq)
    Fm = margin0 + payload[leaf1]
    q, q2 = go.to_grid(go.residual(y, Fm), S, S2)
    assert_same_f64(_host(margin), Fm, "margin")
    got = _host(rq)
    assert np.array_equal(got[:, 0], q) and np.array_equal(got[:, 1], q2)
    assert np.isnan(Fm[leaf1 == nan_leaf]).all() and (got[leaf1 == nan_leaf] == 0).all()
    assert (got[10:20] == 0).all() and np.array_equal(got[20:30, 0], (4.0 * y[20:30] * 2.0 ** S).astype(np.int64))
    # root < 0: F = +0.0 and r = y
    _call("b200flow_gbt_update", tp, tp.shape[1], F, n, None, None, None, -1, S, S2, margin, rq)
    q, q2 = go.to_grid(y, S, S2)
    assert_same_f64(_host(margin), np.zeros(n), "margin")
    got = _host(rq)
    assert np.array_equal(got[:, 0], q) and np.array_equal(got[:, 1], q2)


@pytest.mark.gpu
@pytest.mark.parametrize("root,S,S2", [(0, -2, 10), (-1, -1, 10), (-1, 0, -1), (0, 0, -3)])
def test_gbt_update_grid_half_way(root, S, S2):
    # q and q2 exactly half-way between two integers on both signs: rint rounds to even (0 here), not away from zero.
    # root 0 is one leaf of payload 0, so F = 0 and r = 2y; root < 0 gives r = y.
    n = 64
    labels = (np.arange(n) % 2).astype(np.uint8)
    y = np.where(labels > 0, 1.0, -1.0)
    nodes = np.zeros(1, NODE_DTYPE); nodes["feat"] = -1; nodes["nid"] = 1
    tp = _dev(_records(np.zeros((n, 1), np.uint8), labels, 1))
    margin = _dev(np.zeros(n))
    rq = torch.full((n, 2), SENTINEL, dtype=torch.int64, device=DEV)
    _call("b200flow_gbt_update", tp, tp.shape[1], 1, n, _dev(nodes.view(np.uint8)), _dev(np.zeros((1, 4), np.uint64)),
          _dev(np.zeros(1)), root, S, S2, margin, rq)
    r = go.residual(y, np.zeros(n)) if root >= 0 else y
    q, q2 = go.to_grid(r, S, S2)
    got = _host(rq)
    assert np.array_equal(got[:, 0], q) and np.array_equal(got[:, 1], q2)
    assert (np.abs(r * 2.0 ** S) == 0.5).all() or (np.abs(q.astype(np.float64) * 2.0 ** -S) ** 2 * 2.0 ** S2 == 0.5).all()
    assert (got[:, 1] == 0).all() and (S >= 0 or (got[:, 0] == 0).all())


@pytest.mark.gpu
@pytest.mark.parametrize("K", [1, 3, 23])
def test_gbt_update_classes(K):
    rng = np.random.default_rng(K + 50)
    n, F, T, t = 1500, 9, 2, 1
    bins, trees, nodes, mask, index = walk_case(rng, n, F, K * T, depth=6)
    labels = rng.integers(0, max(K, 2), n).astype(np.uint8)     # K = 1: labels 1 are "rest" rows of the only class
    payload = rng.standard_normal(len(nodes))
    payload[index[(1 * T + t, 1)] if K > 1 else 0] = 700.0   # class 1's root split: its leaves are others, left as drawn
    margin0 = rng.standard_normal((K, n)) * 3.0
    margin0[:, :8] = 500.0
    S, S2 = go.grid_shift(n)
    tp = _dev(_records(bins, labels, F))
    margin = _dev(margin0.copy())
    rq = torch.full((K * n, 2), SENTINEL, dtype=torch.int64, device=DEV)
    _call("b200flow_gbt_update_classes", tp, tp.shape[1], F, n, K, _dev(nodes.view(np.uint8)), _dev(mask), _dev(payload), t, T,
          S, S2, margin, rq)
    got_m, got_q = _host(margin), _host(rq).reshape(K, n, 2)
    for k in range(K):
        y = np.where(labels == k, 1.0, -1.0)
        Fm = margin0[k] + payload[leaf_index(trees, index, k * T + t, bins)]
        q, q2 = go.to_grid(go.residual(y, Fm), S, S2)
        assert_same_f64(got_m[k], Fm, "margin of class %d" % k)
        assert np.array_equal(got_q[k, :, 0], q) and np.array_equal(got_q[k, :, 1], q2), k
    _call("b200flow_gbt_update_classes", tp, tp.shape[1], F, n, K, None, None, None, -1, T, S, S2, margin, rq)
    got_m, got_q = _host(margin), _host(rq).reshape(K, n, 2)
    assert (_bits(got_m) == 0).all()
    for k in range(K):
        q, q2 = go.to_grid(np.where(labels == k, 1.0, -1.0), S, S2)
        assert np.array_equal(got_q[k, :, 0], q) and np.array_equal(got_q[k, :, 1], q2)


@pytest.mark.gpu
@pytest.mark.parametrize("want", list(itertools.product([0, 1], repeat=3)))
def test_gbt_output(want):
    rng = np.random.default_rng(9)
    n = 777
    F = rng.standard_normal(n) * 10.0 ** rng.integers(-5, 3, n)
    F[:8] = [0.0, -0.0, np.nan, np.inf, -np.inf, 400.0, -400.0, 5e-324]
    outs = [torch.full((n, 2), 9.0, dtype=torch.float64, device=DEV) if want[0] else None,
            torch.full((n, 2), 9.0, dtype=torch.float64, device=DEV) if want[1] else None,
            torch.full((n,), 9.0, dtype=torch.float64, device=DEV) if want[2] else None]
    _call("b200flow_gbt_output", _dev(F), n, *outs)
    with np.errstate(all="ignore"):
        p0 = 1.0 / (1.0 + go.pexp(-2.0 * -F))
        refs = [np.stack([-F, F], 1), np.stack([p0, 1.0 - p0], 1), (F > 0.0).astype(np.float64)]
    for o, ref, name in zip(outs, refs, ("raw", "probability", "prediction")):
        if o is not None:
            assert_same_f64(_host(o), ref, name)


# ------------------------------------------------------------------------------------------------ regression trainer kernels
@pytest.mark.gpu
@pytest.mark.parametrize("n,in_record", [(1, True), (31, True), (5000, False), (300001, True)])
def test_reg_labels(n, in_record):
    rng = np.random.default_rng(n)
    F = 20                                                  # the label bytes start at F + 1 = 21: not 8-aligned
    y = rng.standard_normal(n) * 10.0 ** rng.integers(-300, 300, n)
    bad_at = rng.random(n) < 0.01
    y[bad_at] = rng.choice([np.nan, np.inf, -np.inf], int(bad_at.sum()))
    if n >= 31:
        y[:3] = [np.nan, -np.inf, -0.0]
    stride = fr.tp_stride(F)
    host = rng.integers(0, 256, (n, stride)).astype(np.uint8)
    tp = _dev(host)
    out = _dev(np.array([5, 0], np.int64))
    _call("b200flow_reg_labels", _dev(y), n, tp if in_record else None, stride, F + 1, out)
    got = _host(out)
    fin = np.isfinite(y)
    assert got[0] == 5 + int((~fin).sum())
    assert got[1] == (int(np.abs(y[fin]).max().view(np.int64)) if fin.any() and np.abs(y[fin]).max() > 0 else 0)
    want = host.copy()
    if in_record:
        want[:, F + 1:F + 9] = y.view(np.uint8).reshape(n, 8)
    assert np.array_equal(_host(tp), want)


@pytest.mark.gpu
@pytest.mark.parametrize("E", [ro.E_MIN, -3, 0, 40, ro.E_MAX])
def test_reg_grid_record_and_vector(E):
    rng = np.random.default_rng(E + 400)
    n, F = 3000, 20
    S, S2 = 61 - 12, 61 - 12
    y = rng.uniform(-1.0, 1.0, n) * 2.0 ** E
    y[:6] = [2.0 ** E, -(2.0 ** E), 0.0, -0.0, 2.0 ** (E - S) * 1.5, -(2.0 ** (E - S)) * 2.5]   # |y'| = 1, half-way q
    y[6:9] = [2.0 ** E * 3 * 2.0 ** -S, 5 * 2.0 ** (E - S), 2.0 ** (E - S)]               # q = 3, 5, 1
    stride = fr.tp_stride(F)
    host = np.zeros((n, stride), np.uint8)
    host[:, F + 1:F + 9] = y.view(np.uint8).reshape(n, 8)
    want_q, want_q2 = ro.to_grid(y, E, S, S2)
    for S2_ in (S2, 2 * S - 1):                             # S2 = 2S - 1: q2 = q² / 2 is half-way for odd q
        if S2_ > 62:
            S2_ = 62
        want_q, want_q2 = ro.to_grid(y, E, S, S2_)
        got = []
        for from_record in (True, False):
            rq = torch.full((n, 2), SENTINEL, dtype=torch.int64, device=DEV)
            _call("b200flow_reg_grid", _dev(host) if from_record else None, stride, F + 1, None if from_record else _dev(y), n, E, S,
                  S2_, rq)
            got.append(_host(rq))
        assert np.array_equal(got[0], got[1])
        assert np.array_equal(got[0][:, 0], want_q) and np.array_equal(got[0][:, 1], want_q2)
    assert list(want_q[:6]) == [1 << S, -(1 << S), 0, 0, 2, -2]


@pytest.mark.gpu
@pytest.mark.parametrize("T,U", [(1, 1), (3, 100003), (5, 255), (2, 16384 * 3 + 7)])
def test_reg_tree_weights(T, U):
    rng = np.random.default_rng(T * U)
    W = rng.integers(0, 1 << 20, (T, U)).astype(np.int32)
    W[:, rng.random(U) < 0.3] = 0
    totals = _dev(np.arange(T, dtype=np.int64) * 11)
    _call("b200flow_reg_tree_weights", _dev(W), T, U, totals)
    assert [int(v) for v in _host(totals)] == [11 * t + sum(int(v) for v in W[t]) for t in range(T)]


# ------------------------------------------------------------------------------------------------ gbr_update
@pytest.mark.gpu
@pytest.mark.parametrize("loss", ["squared", "absolute"])
@pytest.mark.parametrize("label_src", ["record", "vector"])
def test_gbr_update(loss, label_src):
    rng = np.random.default_rng(3 if loss == "squared" else 4)
    n, F, T = 6000, 20, 2
    bins, trees, nodes, mask, index = walk_case(rng, n, F, T)
    y = rng.standard_normal(n) * 3.0
    payload = rng.standard_normal(len(nodes))
    leaf = leaf_index(trees, index, 1, bins)
    margin0 = rng.standard_normal(n)
    margin0[20:40] = 0.0; payload[leaf[20:40]] = 0.0        # (leaves shared with other rows: they get F = margin + 0.0)
    y[20:40] = -0.0                                         # difference -0.0 - +0.0 = -0.0
    nan_leaf = next(int(v) for v in leaf[40:] if v not in set(leaf[:40].tolist()))
    payload[nan_leaf] = np.nan                              # an empty tree's leaf: r becomes 0 (squared)
    y[:20] = margin0[:20] + payload[leaf[:20]]              # difference exactly 0
    stride = fr.tp_stride(F)
    host = np.zeros((n, stride), np.uint8)
    host[:, :F] = bins
    host[:, F + 1:F + 9] = y.view(np.uint8).reshape(n, 8)
    tp = _dev(host)
    yv = _dev(y) if label_src == "vector" else None
    margin, resid = _dev(margin0.copy()), torch.full((n,), 9.0, dtype=torch.float64, device=DEV)
    mx = _dev(np.zeros(1, np.int64))
    code = 0 if loss == "squared" else 1
    _call("b200flow_gbr_update", tp, stride, F + 1, yv, n, _dev(nodes.view(np.uint8)), _dev(mask), _dev(payload), 1, code, margin,
          resid, mx)
    Fm = margin0 + payload[leaf]
    r = gro.residual(y, Fm, loss)
    assert_same_f64(_host(margin), Fm, "margin")
    assert_same_f64(_host(resid), r, "residual")
    assert int(_host(mx)[0]) == int(np.abs(r).max().view(np.int64))
    assert (r[:20] == (0.0 if loss == "squared" else 1.0)).all()
    if loss == "absolute":
        assert (r[20:40] == 1.0).all()
    else:
        assert (_bits(r[20:40]) == _bits(-0.0)).all()
    assert r[leaf == nan_leaf].tolist() == [0.0 if loss == "squared" else 1.0] * int((leaf == nan_leaf).sum())
    # root < 0: F = +0.0, r = y
    mx.zero_()
    _call("b200flow_gbr_update", tp, stride, F + 1, yv, n, None, None, None, -1, code, margin, resid, mx)
    assert (_bits(_host(margin)) == 0).all()
    assert_same_f64(_host(resid), y, "residual")
    assert int(_host(mx)[0]) == int(np.abs(y).max().view(np.int64))


# ------------------------------------------------------------------------------------------------ evaluator
def eval_terms(y, p, mode, m):
    with np.errstate(all="ignore"):
        if mode == 0:
            d = y - p
            return [y, y * y, d * d, np.abs(d)]
        return [(y - m) * (y - m), (p - m) * (p - m)]


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("n,scale,shape", [(1, 1.0, "mixed"), (31, 1.0, "mixed"), (31, 1e40, "negative"),
                                           (300001, 1.0, "negative"), (300001, 3e45, "mixed"), (5000, 1e-200, "mixed")])
def test_reg_eval(mode, n, scale, shape):
    # 'negative': every label below -1, so term 0's limbs carry through every word; scale 1e40 / 3e45: sh < 0
    rng = np.random.default_rng(n + mode)
    y = rng.standard_normal(n) * scale
    if shape == "negative":
        y = -np.abs(y) - scale
    p = y + rng.standard_normal(n) * scale * 0.1
    if n > 100:
        y[:3] = [np.nan, np.inf, 1.0]; p[3:5] = [-np.inf, np.nan]
        y[5] = 1e300 if scale < 1e100 else 1e160            # a term overflows: the row is skipped and counted
    m = float(rng.standard_normal()) * scale
    terms = eval_terms(y, p, mode, m)
    ok = np.isfinite(y) & np.isfinite(p)
    for t in terms:
        ok &= np.isfinite(t)
    K = len(terms)
    head = _dev(np.zeros(5, np.int64))
    yd, pd = _dev(y), _dev(p)
    _call("b200flow_reg_eval_max", yd, pd, n, mode, m, head)
    h = _host(head)
    assert h[0] == int((~ok).sum())
    mxs = [float(np.abs(t[ok]).max()) if ok.any() else 0.0 for t in terms]
    assert [int(v) for v in h[1:1 + K]] == [int(np.float64(v).view(np.int64)) for v in mxs] and (h[1 + K:] == 0).all()
    sh = [ro.fixed_shift(v, n) for v in mxs] + [0] * (4 - K)
    assert shape != "negative" or mode != 0 or scale < 1e30 or sh[0] < 0
    limbs = _dev(np.zeros((4, 4), np.int64))
    _call("b200flow_reg_eval_sums", yd, pd, n, mode, m, sh[0], sh[1], sh[2], sh[3], limbs)
    L = _host(limbs)
    for k in range(K):
        total = sum(int(v) << (32 * j) for j, v in enumerate(L[k]))
        want = sum(int(v) for v in np.rint(np.ldexp(terms[k][ok], sh[k])).tolist())
        assert total == want, k
        got_v = (total / (1 << sh[k]) if sh[k] >= 0 else float(total * (1 << -sh[k]))) if total else 0.0
        assert got_v == ro.exact_sum(terms[k][ok], n)
    assert (L[K:] == 0).all()
    if shape == "negative" and mode == 0:
        assert L[0, :3].max() >= 1 << 32                    # the low limbs carried
