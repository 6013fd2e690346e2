"""Launch paths of the tree-preparation kernels (csrc/treeprep.cu) that the end-to-end forest tests never reach, each called through the C ABI and compared exactly with the CPU oracle or numpy.

exclusive scan: the single-CTA kernel (n <= 16 * 4096) and the three-launch path, including the totals kernel's loop over
1024-block chunks (n > 1024 * 4096), with block sums near 2^31 and grand totals past 2^32.  group_rows: ids colliding in
the per-CTA 256-line cache, hot groups over many CTAs, more rows than the persistent grid covers in one trip.  bag_weights:
the identity, uid-merged and grouped paths, the whole-CTA fast path inside a hot group (and a final partial CTA that must
not take it), T not a multiple of 4, row offsets across 2^32, Poisson CDFs of several rates, GBT's Bernoulli CDF and no
bootstrap; bag_count / bag_fill with U not a multiple of 1024.  The Philox draw 0xFFFFFFFF, which passes every saturated
threshold of the CDF head: pinned rows where it occurs.  dedup_rows: load exactly 0.5, strides 16 to 256, key_bytes = F
and F + 1.  bin_rows: thresholds in global memory, the strided-feature path (F > 256), ld > F, NaN, +-inf, +-0 and values on
a threshold.  find_splits: the 16384 / 16385 switch between the shared- and global-memory kernels, possible == numSplits,
one and two samples, +-inf.  (The batch predictor's cases are in test_predict_forest.py.)"""
import numpy as np
import pytest
import torch

import oracle
from b200flow import _lib, forest as fr, gbt
from b200flow._lib import call, ptr

DEV = "cuda"
SAT = 0xFFFFFFFF


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


# ------------------------------------------------------------------------------- exclusive scan
SCAN_N = [0, 1, 4095, 4096, 4097, 65535, 65536, 65537, 17 * 4096, 1024 * 4096, 1024 * 4096 + 1, 5_000_000]


@pytest.mark.gpu
@pytest.mark.parametrize("with_total", [True, False])
@pytest.mark.parametrize("n", SCAN_N)
def test_exclusive_scan(n, with_total):
    # the block scan is int32: every 4096-element block must sum below 2^31, while the int64 totals pass 2^32
    top = (2 ** 31 - 1) // 4096
    rng = np.random.default_rng(n)
    v = rng.integers(0, top + 1, n, dtype=np.int32)
    v[: min(n, 4096)] = top                                 # a first block summing to 4096 * top = 2^31 - 4096
    if n > 3 * 4096:
        v[-4096:] = top                                     # ... and the last full block
    want = np.zeros(n + 1, np.int64)
    np.cumsum(v, dtype=np.int64, out=want[1:])
    if n > 3 * 4096:
        assert want[-1] > 2 ** 32
    inp = _dev(v if n else np.zeros(1, np.int32))           # n = 0 still needs a real pointer
    out = torch.full((n + 2,), -7, dtype=torch.int64, device=DEV)
    total = torch.full((1,), -7, dtype=torch.int64, device=DEV) if with_total else None
    call("b200flow_exclusive_scan_i32_to_i64", ptr(inp), n, ptr(out), ptr(total))
    got = out.cpu().numpy()
    assert np.array_equal(got[: n + 1], want)
    assert got[n + 1] == -7                                 # nothing written past out[n]
    if with_total:
        assert int(total.item()) == want[-1]


# ------------------------------------------------------------------------------- group rows
def _group_ids(case):
    rng = np.random.default_rng(len(case))
    if case == "collide":                    # 3000 ids over 200 000 rows: lines of the 256-entry cache are shared ~12 ways
        return rng.integers(0, 3000, 200_000).astype(np.int32), 3000
    if case == "hot":                        # two hot ids on the same cache line (5 and 261) over many CTAs, plus singletons
        n, U = 1_000_003, 300_000
        uid = rng.integers(0, U, n)
        r = rng.random(n)
        uid[r < 0.4] = 5
        uid[(r >= 0.4) & (r < 0.6)] = 261
        return uid.astype(np.int32), U
    # KDD-full size: more rows than the persistent grid covers in one trip, ~1 M ids, a third of the rows on one id
    n, U = 5_000_000, 1_000_000
    uid = rng.integers(0, U, n)
    uid[rng.random(n) < 0.33] = 777
    return uid.astype(np.int32), U


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["collide", "hot", "kdd_full"])
def test_group_rows(case):
    uid, U = _group_ids(case)
    n = uid.shape[0]
    uid_d = _dev(uid)
    gsize = torch.empty(U, dtype=torch.int32, device=DEV); cursor = torch.empty(U, dtype=torch.int32, device=DEV)
    goff = torch.empty(U + 1, dtype=torch.int64, device=DEV)
    perm = torch.empty(n, dtype=torch.int32, device=DEV); uperm = torch.empty(n, dtype=torch.int32, device=DEV)
    call("b200flow_group_rows", ptr(uid_d), n, U, ptr(gsize), ptr(goff), ptr(cursor), ptr(perm), ptr(uperm))
    cnt = np.bincount(uid, minlength=U)
    assert np.array_equal(gsize.cpu().numpy(), cnt)
    want_off = np.zeros(U + 1, np.int64); np.cumsum(cnt, out=want_off[1:])
    assert np.array_equal(goff.cpu().numpy(), want_off)
    p, up = perm.cpu().numpy(), uperm.cpu().numpy()
    assert np.array_equal(np.sort(p), np.arange(n))                          # a permutation of the rows
    assert (np.diff(up) >= 0).all() and np.array_equal(up, uid[p])          # grouped by id (order inside a group is free)


# ------------------------------------------------------------------------------- bagging
CDFS = {
    "poisson1": lambda: fr.poisson_cdf_table(1.0),
    "poisson0.5": lambda: fr.poisson_cdf_table(0.5),
    "poisson0.07": lambda: fr.poisson_cdf_table(0.07),
    "poisson0.05": lambda: fr.poisson_cdf_table(0.05),
    "poisson0.01": lambda: fr.poisson_cdf_table(0.01),
    "gbt0.5": lambda: gbt.subsample_cdf(0.5),
    "none": lambda: None,
}


def _bag(seed, T, row_offset, n, cdf, uid=None, perm=None, U=None):
    """b200flow_bag_weights -> W [T, U] (uint32 as int64).  uid in position order when perm is given, else in row order."""
    U = n if U is None else U
    W = torch.zeros(T * U, dtype=torch.int32, device=DEV)
    cdf_d = None if cdf is None else _dev(cdf.view(np.int32))
    uid_d = None if uid is None else _dev(uid.astype(np.int32))
    perm_d = None if perm is None else _dev(perm.astype(np.int32))
    call("b200flow_bag_weights", seed, T, row_offset, n, ptr(cdf_d), None if cdf is None else cdf.ctypes.data,
         ptr(uid_d), ptr(perm_d), U, ptr(W))
    return W, W.cpu().numpy().view(np.uint32).astype(np.int64).reshape(T, U)


def _want_bag(seed, T, row_offset, n, cdf, uid_rows, U):
    """oracle weights of every (tree, row), summed per unique id"""
    w = oracle.bag_weights(seed, T, n, cdf, row_offset).astype(np.int64)
    return np.stack([np.bincount(uid_rows, weights=w[t], minlength=U).astype(np.int64) for t in range(T)])


def _layout(rng, sizes, shuffle):
    """rows of groups with the given sizes in position order -> (uid by row, perm, uid by position, U)"""
    uperm = np.repeat(np.arange(len(sizes)), sizes).astype(np.int32)
    n = uperm.shape[0]
    perm = rng.permutation(n).astype(np.int32) if shuffle else np.arange(n, dtype=np.int32)
    uid = np.empty(n, np.int32); uid[perm] = uperm
    return uid, perm, uperm, len(sizes)


def _bag_sizes(rng):
    # positions 0..2347: small groups; a hot group from 2348 (mid CTA 2) to 6943 covers CTAs 3, 4 and 5 entirely (the
    # whole-CTA fast path) and meets the merged path at its two ends; more small groups; then a last group that starts in
    # CTA 10 and runs to n = 11 * 1024 + 700, so the final partial CTA lies inside one group and must not take the fast path
    head = list(rng.integers(1, 9, 600))
    while sum(head) > 2348:
        head.pop()
    head.append(2348 - sum(head))
    mid = list(rng.integers(1, 5, 2000))
    rest = 10 * 1024 + 300 - 6944
    while sum(mid) > rest:
        mid.pop()
    mid.append(rest - sum(mid))
    sizes = [s for s in head if s] + [4596] + [s for s in mid if s] + [11 * 1024 + 700 - 10 * 1024 - 300]
    assert sum(sizes) == 11 * 1024 + 700
    return sizes


def test_bag_layout():
    # the fixture's position layout: which 1024-position CTAs lie inside one group (those take the whole-CTA fast path)
    for shuffle in (False, True):
        rng = np.random.default_rng(3 * 7 + shuffle)
        _, perm, uperm, U = _layout(rng, _bag_sizes(rng), shuffle)
        n = uperm.shape[0]
        assert n % 1024 == 700 and U % 1024
        inside = [bool(uperm[c * 1024] == uperm[min(n, c * 1024 + 1024) - 1]) for c in range((n + 1023) // 1024)]
        assert inside == [False] * 3 + [True] * 3 + [False] * 5 + [True]     # CTA 11: partial, inside the last group
        assert uperm[2347] != uperm[2348] and uperm[6943] != uperm[6944]      # the hot group starts and ends mid CTA
        assert (np.diff(uperm) >= 0).all() and np.array_equal(np.sort(perm), np.arange(n))


def _entries(W, T, U):
    """b200flow_bag_count + scan + b200flow_bag_fill on device W [T * U] -> entries [E, 2] (record, weight)"""
    nb = (U + 1023) // 1024
    blk_cnt = torch.full((T * nb,), -1, dtype=torch.int32, device=DEV)
    blk_off = torch.empty(T * nb + 1, dtype=torch.int64, device=DEV)
    total = torch.zeros(1, dtype=torch.int64, device=DEV)
    call("b200flow_bag_count", ptr(W), T, U, ptr(blk_cnt))
    call("b200flow_exclusive_scan_i32_to_i64", ptr(blk_cnt), T * nb, ptr(blk_off), ptr(total))
    E = int(total.item())
    ent = torch.full((E + 1, 2), -1, dtype=torch.int32, device=DEV)
    call("b200flow_bag_fill", ptr(W), T, U, ptr(blk_off), ptr(ent))
    e = ent.cpu().numpy().view(np.uint32)
    assert (e[E] == SAT).all()                                              # nothing past the counted entries
    return e[:E].astype(np.int64)


def _want_entries(Wh):
    out = []
    for t in range(Wh.shape[0]):
        u = np.nonzero(Wh[t])[0]
        out.append(np.stack([u, Wh[t][u]], 1))
    return np.concatenate(out) if out else np.zeros((0, 2), np.int64)


@pytest.mark.gpu
@pytest.mark.parametrize("cdf_name", ["poisson1", "poisson0.5", "poisson0.05", "poisson0.01", "gbt0.5", "none"])
@pytest.mark.parametrize("T", [1, 3, 4, 5, 37])
def test_bag_weights_paths(T, cdf_name):
    cdf = CDFS[cdf_name]()
    seed = 1000 + T
    for shuffle, row_offset in ((False, 0), (True, 2 ** 32 - 5000)):        # the second batch straddles global row 2^32
        rng = np.random.default_rng(T * 7 + shuffle)
        uid, perm, uperm, U = _layout(rng, _bag_sizes(rng), shuffle)
        n = uid.shape[0]
        want_rows = oracle.bag_weights(seed, T, n, cdf, row_offset).astype(np.int64)
        _, got = _bag(seed, T, row_offset, n, cdf)                          # identity: one entry per row
        assert np.array_equal(got, want_rows), "identity"
        want = _want_bag(seed, T, row_offset, n, cdf, uid, U)
        Wd, got = _bag(seed, T, row_offset, n, cdf, uid=uid, U=U)          # uid in row order: merged inside warps
        assert np.array_equal(got, want), "uid-merged"
        Wg, got = _bag(seed, T, row_offset, n, cdf, uid=uperm, perm=perm, U=U)   # grouped: the fast path in CTAs 3..5
        assert np.array_equal(got, want), "grouped"
        assert np.array_equal(_entries(Wg, T, U), _want_entries(want))
    # the identity path's W (U = n = 3000)
    Wi, got = _bag(seed, T, 0, 3000, cdf)
    assert np.array_equal(got, oracle.bag_weights(seed, T, 3000, cdf).astype(np.int64))
    assert np.array_equal(_entries(Wi, T, 3000), _want_entries(got))


# ------------------------------------------------------------------------------- the saturated-head draw
# Rows whose Philox bagging word is 0xFFFFFFFF for seed SAT_SEED: (global row, tree).  Found once by an exhaustive search
# over the rows with the oracle's Philox; the search is not part of the suite, the self-check below pins the fixture.
SAT_SEED = 7
SAT_DRAWS = [(201_425_420, 3), (4_315_415_842, 2), (4_348_036_984, 1)]
# weight of the draw 0xFFFFFFFF = the number of non-saturated thresholds: the spec (orc_bag_weights) never counts a saturated one
SAT_CDFS = {"poisson1": 12, "poisson0.07": 5, "poisson0.05": 5, "poisson0.01": 4, "gbt0.5": 1}


def test_saturated_draw_fixture():
    for g, t in SAT_DRAWS:
        r = oracle.philox(SAT_SEED, oracle.PURPOSE_BAG, g & 0xFFFFFFFF, g >> 32, t >> 2, 0)
        assert int(r[t & 3]) == SAT, (g, t)
        for name, w in SAT_CDFS.items():
            assert int(oracle.bag_weights(SAT_SEED, t + 1, 1, CDFS[name](), g)[t, 0]) == w, (g, t, name)


def test_which_rates_saturate_the_cdf_head():
    # the first saturated threshold of each CDF: inside the six-entry head of bag_weights for small rates and for GBT
    first = lambda c: int(np.nonzero(c == SAT)[0][0])
    assert first(fr.poisson_cdf_table(1.0)) == 12 and first(fr.poisson_cdf_table(0.5)) == 9
    assert first(fr.poisson_cdf_table(0.1)) == 6
    assert first(fr.poisson_cdf_table(0.07)) == 5 and first(fr.poisson_cdf_table(0.05)) == 5
    assert first(fr.poisson_cdf_table(0.01)) == 4
    assert first(gbt.subsample_cdf(0.5)) == 1 and first(gbt.subsample_cdf(0.9)) == 1
    for rate in (1.0, 0.5, 0.07, 0.01):
        assert np.array_equal(fr.poisson_cdf_table(rate), oracle.poisson_cdf_table(rate))
        c = fr.poisson_cdf_table(rate)
        assert (np.diff(c.astype(np.int64)) >= 0).all() and (c[first(c):] == SAT).all()


@pytest.mark.gpu
@pytest.mark.parametrize("cdf_name", list(SAT_CDFS))
@pytest.mark.parametrize("draw", range(len(SAT_DRAWS)))
def test_bag_weights_saturated_draw(draw, cdf_name):
    g, t = SAT_DRAWS[draw]
    cdf = CDFS[cdf_name]()
    T = 5
    # 4096 rows with the drawn row at local index 1500; by position: 100 singletons, one group over positions 100..3999
    # (CTAs 1 and 2 whole: the fast path), 96 singletons.  The drawn row sits at position 1500 of the grouped order.
    n, loc = 4096, 1500
    sizes = [1] * 100 + [3900] + [1] * 96
    uperm = np.repeat(np.arange(len(sizes)), sizes).astype(np.int32)
    U = len(sizes)
    rng = np.random.default_rng(draw)
    perm = rng.permutation(n).astype(np.int32)
    j = int(np.nonzero(perm == loc)[0][0])
    perm[[j, 1500]] = perm[[1500, j]]                                       # row `loc` at position 1500
    uid = np.empty(n, np.int32); uid[perm] = uperm
    row_offset = g - loc
    want_rows = oracle.bag_weights(SAT_SEED, T, n, cdf, row_offset).astype(np.int64)
    assert want_rows[t, loc] == SAT_CDFS[cdf_name]
    _, got = _bag(SAT_SEED, T, row_offset, n, cdf)
    assert got[t, loc] == SAT_CDFS[cdf_name] and np.array_equal(got, want_rows), "identity"
    want = _want_bag(SAT_SEED, T, row_offset, n, cdf, uid, U)
    _, got = _bag(SAT_SEED, T, row_offset, n, cdf, uid=uid, U=U)
    assert np.array_equal(got, want), "uid-merged"
    _, got = _bag(SAT_SEED, T, row_offset, n, cdf, uid=uperm, perm=perm, U=U)
    assert np.array_equal(got, want), "grouped (whole-CTA fast path)"


# ------------------------------------------------------------------------------- de-duplication
def _dedup_records(n, F, stride, with_label, seed):
    rng = np.random.default_rng(seed)
    tp = np.zeros((n, stride), np.uint8)
    tp[:, :F] = rng.integers(0, 256, (n, F))
    if with_label:
        tp[:, F] = rng.integers(0, 7, n)
    hot = tp[0].copy()
    tp[rng.random(n) < 0.5] = hot                                             # a hot group over half the rows
    # near-duplicates of the hot record: one differing byte at every position of the key, the last one included
    key = F + 1 if with_label else F
    for j in range(min(key, n // 4)):
        i = int(rng.integers(0, n))
        tp[i] = hot; tp[i, j] ^= 1 + (j % 255)
    if n >= 4:
        tp[n - 1] = tp[1]                                                       # a duplicate pair, representative row 1
    return tp


@pytest.mark.gpu
@pytest.mark.parametrize("with_label", [True, False])
@pytest.mark.parametrize("F", [15, 41, 255])
@pytest.mark.parametrize("n", [1, 255, 257, 2 ** 16, 2 ** 16 + 1])
def test_dedup_rows(n, F, with_label):
    # key_bytes = F + 1: the fit (bins + label); key_bytes = F: predict (binned without labels, the label byte is 0).
    # Strides 16 (F = 15), 48 and 256; n = 2^16 fills the hash table to exactly one half.
    stride = oracle.tp_stride(F)
    key = F + 1 if with_label else F
    tp = _dedup_records(n, F, stride, with_label, n * 3 + F)
    _, first, inv = np.unique(tp.view(np.dtype((np.void, stride))).ravel(), return_index=True, return_inverse=True)
    rank = np.empty(first.shape[0], np.int64); rank[np.argsort(first)] = np.arange(first.shape[0])
    want_uid = rank[inv.ravel()]                                              # ids in first-occurrence order
    tpd = _dev(tp)
    tpu, uid, U = fr.dedup_rows(tpd, key)
    assert U == first.shape[0]
    u = uid.cpu().numpy()
    assert np.array_equal(u, want_uid)
    assert np.array_equal(tpu.cpu().numpy()[u], tp)
    _, uid2, U2 = fr.dedup_rows(tpd, key)
    assert U2 == U and np.array_equal(uid2.cpu().numpy(), u)
    # rows that differ in a key byte never share an id
    keys = tp[:, :key].view(np.dtype((np.void, key))).ravel()
    _, kinv = np.unique(keys, return_inverse=True)
    per_id = np.zeros(U, np.int64) - 1
    per_id[u] = kinv.ravel()
    assert np.array_equal(per_id[u], kinv.ravel())


# ------------------------------------------------------------------------------- binning
def _bin_case(name):
    """-> (x [n, ld] f64 whose first F columns are the features, F, arity, max_bins, thresholds [F, max_bins-1], n_thr)"""
    rng = np.random.default_rng(len(name))
    F, mb, ld, n_cat = {"global_thr": (78, 256, 78, 0), "wide": (300, 32, 300, 20), "wide_global": (300, 64, 300, 0),
                        "ld": (41, 70, 50, 3), "tiny": (5, 2, 5, 1)}[name]
    n = 5003
    arity = np.zeros(F, np.int32)
    arity[F - n_cat:] = rng.integers(2, min(mb, 255) + 1, n_cat)
    thr = np.zeros((F, mb - 1)); n_thr = np.zeros(F, np.int32)
    for f in range(F - n_cat):
        k = int(rng.integers(0, mb)) if f % 5 else mb - 1
        t = np.unique(rng.normal(0, 10, k))
        if f % 7 == 1 and t.size:
            t[-1] = np.inf                                                    # a sample with +inf had a +inf midpoint
        if f % 7 == 2 and t.size:
            t[0] = -np.inf
        thr[f, : t.size] = t; n_thr[f] = t.size
    x = np.empty((n, ld))
    x[:] = rng.normal(0, 12, (n, ld))
    for f in range(F - n_cat):
        if n_thr[f]:                                                           # values exactly on a threshold
            on = rng.random(n) < 0.2
            x[on, f] = thr[f, rng.integers(0, n_thr[f], on.sum())]
    special = np.array([np.nan, np.inf, -np.inf, 0.0, -0.0])
    sp = rng.random((n, F - n_cat)) < 0.03
    x[:, : F - n_cat][sp] = special[rng.integers(0, special.size, sp.sum())]
    for f in range(F - n_cat, F):                                             # categories, and cells that are none
        x[:, f] = rng.integers(0, arity[f], n)
        bad = rng.random(n) < 0.02
        x[bad, f] = np.array([np.nan, np.inf, -np.inf, -1.0, 2.5, -0.5, float(arity[f]), 3e9, -0.0])[rng.integers(0, 9, bad.sum())]
    return x, F, arity, mb, thr, n_thr


def _bad_cells(x, arity):
    cat = x[:, arity > 0]; ar = arity[arity > 0]
    with np.errstate(invalid="ignore"):
        ok = (np.floor(cat) == cat) & (cat >= 0) & (cat < ar)
    return int((~ok).sum())


@pytest.mark.gpu
@pytest.mark.parametrize("with_labels", [True, False])
@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
@pytest.mark.parametrize("name", ["global_thr", "wide", "wide_global", "ld", "tiny"])
def test_bin_rows(name, dtype, with_labels):
    x, F, arity, mb, thr, n_thr = _bin_case(name)
    n, ld = x.shape
    xd = torch.from_numpy(x).to(dtype).to(DEV)                              # a [n, ld] buffer: the features are its first F columns
    xs = xd.double().cpu().numpy()[:, :F]                                   # the values the kernel sees, widened
    labels = np.random.default_rng(1).integers(0, 23, n).astype(np.int32) if with_labels else None
    stride = fr.tp_stride(F)
    tp = torch.full((n, stride), 0xAB, dtype=torch.uint8, device=DEV)
    bad = torch.zeros(1, dtype=torch.int32, device=DEV)
    thr_d, n_thr_d, arity_d = _dev(thr), _dev(n_thr), _dev(arity)
    lab_d = None if labels is None else _dev(labels)
    call("b200flow_bin_rows", ptr(xd), _lib.dtype_code(xd), n, F, ld, ptr(thr_d), ptr(n_thr_d), ptr(arity_d), mb, ptr(lab_d),
         ptr(tp), stride, ptr(bad))
    want, _ = oracle.bin_rows(xs, thr, n_thr, arity, mb, labels)
    got = tp.cpu().numpy()
    assert np.array_equal(got[:, : F + 1], want[:, : F + 1])                # label byte 0 without labels
    assert not got[:, F + 1:].any()                                         # pad bytes zero
    assert int(bad.item()) == _bad_cells(xs, arity)                         # the kernel counts bad cells, not rows


# ------------------------------------------------------------------------------- find_splits
def _split_columns(n_s, mb, rng):
    cols = [rng.normal(size=n_s)]                                             # all distinct
    for k in (mb, mb + 1, mb - 1):                                            # possible = numSplits, numSplits + 1, numSplits - 1
        vals = np.sort(rng.normal(size=k)) * 3
        c = vals[rng.integers(0, k, n_s)]
        c[: min(k, n_s)] = vals[: min(k, n_s)]
        cols.append(rng.permutation(c))
    ties = rng.integers(0, 40, n_s).astype(np.float64)                        # heavy ties, with +-inf
    ties[rng.random(n_s) < 0.05] = np.inf
    ties[rng.random(n_s) < 0.05] = -np.inf
    ties[0] = 7.0                                                             # -inf and +inf never adjacent (no NaN midpoint)
    cols.append(ties)
    cols.append(np.full(n_s, 2.5))                                            # constant
    cols.append(rng.integers(0, 4, n_s).astype(np.float64))                  # a categorical column: no thresholds
    return np.stack(cols)


@pytest.mark.gpu
@pytest.mark.parametrize("count_on_device", [False, True])
@pytest.mark.parametrize("mb", [32, 256])
@pytest.mark.parametrize("n_s", [1, 2, 300, 16383, 16384, 16385, 40000])
def test_find_splits(n_s, mb, count_on_device):
    rng = np.random.default_rng(n_s + mb)
    cols = _split_columns(n_s, mb, rng)
    F = cols.shape[0]
    arity = np.zeros(F, np.int32); arity[-1] = 4
    n_pad = 1
    while n_pad < n_s:
        n_pad <<= 1
    cap = n_pad + 16
    sample = torch.zeros((F, cap), dtype=torch.float64, device=DEV)
    sample[:, :n_s] = torch.from_numpy(cols)
    thr = torch.zeros((F, mb - 1), dtype=torch.float64, device=DEV)
    n_thr = torch.full((F,), -1, dtype=torch.int32, device=DEV)
    arity_d = _dev(arity)
    if count_on_device:      # the fit's single-GPU call: the host passes an upper bound, the count stays on the device
        n_s_dev = torch.tensor([n_s], dtype=torch.int32, device=DEV)
        call("b200flow_find_splits", ptr(sample), cap, n_pad, F, ptr(arity_d), mb, ptr(thr), ptr(n_thr), ptr(n_s_dev))
    else:
        call("b200flow_find_splits", ptr(sample), cap, n_s, F, ptr(arity_d), mb, ptr(thr), ptr(n_thr), None)
    got_thr, got_n = thr.cpu().numpy(), n_thr.cpu().numpy()
    assert got_n[-1] == 0
    for f in range(F - 1):
        want = oracle.find_splits_1d(cols[f], mb - 1)
        assert got_n[f] == want.size, f
        assert np.array_equal(got_thr[f, : want.size].view(np.uint64), want.view(np.uint64)), f   # bit for bit
    if n_s >= mb:
        assert got_n[1] == mb - 1                                             # possible == numSplits: every midpoint
