"""The three kernels of one forest level (csrc/forest.cu) called one by one through the C ABI, on synthetic records, entries
and splits whose edges are placed on purpose, against the plain restatement in tests/level_oracle.py:

  route_hist_level  every launch shape x histogram update (the subset width picks it: the rotated update up to 12 features a
                    pass, the generic loop above), byte and 16/32/48/64-byte packed records, subset widths 1..41 and feature
                    passes, 2..200 classes, segment lengths around the chunk size, one-sided and dropped children,
                    categorical masks in all four words, hot counters with large weights;
  partition_level + next_segments (the unfused routing);
  score_level       ragged and serial prefix scans, exact ties, ordered categoricals up to 255 categories, unordered ones with
                    as few bins as categories, feature batches, and every leaf rule;
  grow_level        more than one scan block, every flag combination, pool overflow.

Histograms, cursors and counts are compared exactly, routed entries as multisets per side (their order within a side
depends on the atomics), split records byte for byte.  The first test needs no GPU: it checks the restatement of
binsToBestSplit against the C++ oracle's root nodes before it judges the kernels."""
import zlib

import numpy as np
import pytest
import torch

import oracle
from b200flow import _lib, forest as fr
from b200flow._lib import NODE_DTYPE, SPLIT_DTYPE
from level_oracle import grow_ref, route_ref, score_ref
from util import forests_equal

DEV = "cuda"
SHAPES = ["8x2", "8x1", "16x2", "16x1", "32x1"]
SENTINEL = -7
WIDTHS = ["narrow", "wide", "all"]


def _width(name, narrow, F):
    """subset width of each histogram update: `narrow` (rotated), `wide` = 13 (the generic loop: a pass wider than 12) or
    every feature (featureSubsetStrategy="all"; feature passes where the child histograms do not fit at once)"""
    return {"narrow": narrow, "wide": 13, "all": F}[name]


def unordered_features(n, C, seed):
    """unordered categoricals of arity 4, 5 and 6 whose category subsets carry the label, and continuous columns with 2, 3
    and 4 distinct values: the widest feature has at most 6 bins while an unordered one lists up to 31 subsets."""
    rng = np.random.default_rng(seed)
    arity = [4, 5, 6, 0, 0, 0]
    cats = [rng.integers(0, a, n) for a in arity[:3]]
    cont = [rng.integers(0, k, n) * 0.75 - 1.0 for k in (2, 3, 4)]
    x = np.stack(cats + cont, 1).astype(np.float64)
    look = [rng.integers(0, C, a) for a in arity[:3]]
    y = (look[0][cats[0]] + look[1][cats[1]] * (cats[2] % 2) + (cont[2] > 0)) % C
    noise = rng.random(n) < 0.15
    y = np.where(noise, rng.integers(0, C, n), y).astype(np.int32)
    return x, y, arity


# ------------------------------------------------------------------------------------------------ host-only self-check
@pytest.mark.parametrize("seed,C,max_bins,trees", [(1, 3, 32, 1), (2, 5, 32, 3), (3, 3, 70, 3), (4, 5, 70, 1), (5, 2, 32, 3)])
def test_score_ref_equals_oracle_roots(seed, C, max_bins, trees):
    x, y, arity = unordered_features(3000, C, seed)
    fo, meta = oracle.fit_forest(x, y, C, arity, num_trees=trees, max_bins=max_bins, max_depth=1, seed=seed)
    fb, kind, n_bins, m = meta["feat_bins"], meta["feat_kind"], meta["n_bins"], meta["m"]
    if C > 2:
        assert (kind == 2).any() and max((1 << (b - 1)) - 1 for b, k in zip(fb, kind) if k == 2) > n_bins
    ex = fo.export()
    F = x.shape[1]
    for t in range(trees):
        rows = np.nonzero(meta["w"][t])[0]
        sub = oracle.feature_subset(seed, t, 1, F, m)
        hist = oracle.hist_node(meta["tp"], F, rows, meta["w"][t][rows], sub, n_bins, C)
        sp, tot, L, R = score_ref(hist, sub, fb, kind, 0, 1, 1, 0.0)
        r = np.nonzero((ex["tree"] == t) & (ex["nid"] == 1))[0][0]
        assert int(sp["flags"] & 1) == ex["is_leaf"][r]
        assert (sp["feat"], sp["kind"], sp["bin_thr"]) == (ex["feat"][r], ex["kind"][r], ex["bin_thr"][r])
        assert np.array_equal(sp["mask"], ex["mask"][r]) and np.array_equal(tot, ex["counts"][r])
        assert sp["gain"] == ex["gain"][r] and sp["impurity"] == ex["impurity"][r]
        if not ex["is_leaf"][r]:
            for nid, want in ((2, L), (3, R)):
                c = np.nonzero((ex["tree"] == t) & (ex["nid"] == nid))[0][0]
                assert np.array_equal(ex["counts"][c], want)


# ------------------------------------------------------------------------------------------------ helpers
_alive = []


@pytest.fixture(autouse=True)
def _keep_arguments_alive():
    # the kernels run asynchronously on device pointers: a tensor freed after its pointer was taken would hand its block to
    # the next argument of the same size, so every tensor _dev makes lives until the test has synchronised
    yield
    if _alive:
        torch.cuda.synchronize()
        _alive.clear()


def _dev(a):
    a = np.ascontiguousarray(a)
    if a.dtype in (np.uint32, np.uint64):                  # same bits as the signed type torch handles everywhere
        a = a.view(np.int32 if a.dtype == np.uint32 else np.int64)
    t = torch.from_numpy(a).to(DEV)
    _alive.append(t)
    return t


def _scan(counts):
    off = np.zeros(len(counts) + 1, np.int64)
    off[1:] = np.cumsum(counts)
    return off


def _pack(bins, labels, desc, rec_bytes):
    """bit-packed records as b200flow_packed_layout describes them: field f at (word d & 0xff, shift (d >> 8) & 0xff)."""
    n, F = bins.shape
    words = np.zeros((n, rec_bytes // 4), np.uint32)
    fields = np.concatenate([bins, labels[:, None]], 1).astype(np.uint32)
    for f in range(F + 1):
        d = int(desc[f])
        words[:, d & 0xFF] |= (fields[:, f] & np.uint32(d >> 16)) << np.uint32((d >> 8) & 0xFF)
    return words


class RouteCase:
    """records, parents, splits and child subsets of one routing pass.  lens = entries per parent; parents are laid out with
    gaps of unused entries between them.  Splits: parent 0 at threshold 0, parent 1 at its feature's last bin (everything
    goes left), then categorical masks (every cat_every-th parent) and random thresholds.  With six parents or more, parent 2
    keeps only its right child, parent 3 only its left one, and parent 4 is a leaf without routing chunks."""

    def __init__(self, rng, feat_bins, C, lens, m, n_rec=3000, hot=False, max_w=3, cat_every=3):
        F = len(feat_bins)
        self.F, self.C, self.m, self.feat_bins = F, C, m, np.asarray(feat_bins, np.int32)
        self.n_bins = int(self.feat_bins.max())
        self.bins = np.stack([rng.integers(0, b, n_rec) for b in feat_bins], 1).astype(np.uint8)
        self.labels = rng.integers(0, C, n_rec).astype(np.uint8)
        S = len(lens)
        gaps = rng.integers(0, 4, S + 1)
        self.seg_begin = np.zeros(S, np.int64); self.seg_end = np.zeros(S, np.int64)
        pos = int(gaps[0])
        for s, n in enumerate(lens):
            self.seg_begin[s] = pos; self.seg_end[s] = pos + n; pos += n + int(gaps[s + 1])
        E = pos
        rec = rng.integers(0, n_rec, E)
        w = rng.integers(1, max_w + 1, E)
        if hot:                                            # one record (one counter per feature) takes most entries
            sel = rng.random(E) < 0.8
            rec[sel] = 0
            w[sel] = rng.integers(40000, 50000, int(sel.sum()))
        self.ent = np.stack([rec, w], 1).astype(np.int32)
        split = np.zeros(S, SPLIT_DTYPE)
        for s in range(S):
            f = int(rng.integers(0, F))
            split[s]["feat"] = f
            if s >= 2 and s % cat_every == 0:
                split[s]["kind"] = 1
                split[s]["mask"] = rng.integers(0, 2 ** 63, 4, dtype=np.uint64) | rng.integers(0, 2, 4, dtype=np.uint64) << np.uint64(63)
            else:
                nb = int(self.feat_bins[f])
                split[s]["bin_thr"] = 0 if s == 0 else nb - 1 if s == 1 else int(rng.integers(0, nb))
            split[s]["flags"] = 0
        self.split = split
        child = np.full(2 * S, -1, np.int64)
        self.n_chunks_keep = np.ones(S, bool)
        nxt = 0
        for s in range(S):
            for side in (0, 1):
                if S >= 6 and (s, side) in ((2, 0), (3, 1)):      # one-sided parents
                    continue
                if S >= 6 and s == 4:                            # a leaf parent: no chunks, its entries stay where they are
                    self.n_chunks_keep[s] = False
                    continue
                child[2 * s + side] = nxt; nxt += 1
        perm = rng.permutation(max(nxt, 1))
        self.child_slot = np.where(child >= 0, perm[np.maximum(child, 0)], -1).astype(np.int32)
        self.n_next = max(nxt, 1)
        self.subset_next = np.stack([np.sort(rng.choice(F, m, replace=False)) for _ in range(self.n_next)]).astype(np.int16)


def _run_route(case, packed, route=True, extra_chunks=37, shape=None, monkeypatch=None):
    """b200flow_route_hist_level on the case; returns (hist, ent_out, cursors, config)."""
    if shape is not None:
        monkeypatch.setenv("B200FLOW_ROUTE_SHAPE", shape)
    F, C, m, n_bins = case.F, case.C, case.m, case.n_bins
    if packed:
        desc, rec_bytes = _lib.packed_layout(case.feat_bins, C)
        assert rec_bytes > 0
        tp = _dev(_pack(case.bins, case.labels, desc, rec_bytes).view(np.uint8))
        desc_d, stride = _dev(desc), rec_bytes
        dev_packed = torch.empty_like(tp)                  # the library's packer writes the same words
        bytes_tp = np.zeros((case.bins.shape[0], fr.tp_stride(F)), np.uint8)
        bytes_tp[:, :F] = case.bins; bytes_tp[:, F] = case.labels
        _lib.call("b200flow_pack_records", _lib.ptr(_dev(bytes_tp)), fr.tp_stride(F), bytes_tp.shape[0], F, _lib.ptr(desc_d),
                  rec_bytes, _lib.ptr(dev_packed))
        assert torch.equal(dev_packed, tp)
    else:
        rec_bytes, desc_d, stride = 0, None, fr.tp_stride(F)
        host = np.zeros((case.bins.shape[0], stride), np.uint8)
        host[:, :F] = case.bins; host[:, F] = case.labels
        tp = _dev(host)
    cfg = _lib.route_hist_config(F, m, n_bins, C, rec_bytes)
    assert cfg is not None
    ch, m_pass = cfg
    if shape is not None:
        nw, ks = map(int, shape.split("x"))
        assert ch == nw * ks * 32
    lens = case.seg_end - case.seg_begin
    nch = np.where(case.n_chunks_keep, (lens + ch - 1) // ch, 0)
    off = _scan(nch)
    S = len(lens)
    cmax = int(off[-1]) + extra_chunks
    scratch = torch.empty(max(cmax, 1) * 4, dtype=torch.int32, device=DEV)
    hist = torch.zeros(case.n_next * m * n_bins * C, dtype=torch.int32, device=DEV)
    ent = _dev(case.ent)
    ent_out = torch.full_like(ent, SENTINEL) if route else None
    cursors = torch.zeros(2 * S, dtype=torch.int32, device=DEV) if route else None
    off_d = _dev(off)
    _lib.call("b200flow_route_hist_level", _lib.ptr(tp), stride, F, _lib.ptr(desc_d), _lib.ptr(ent), _lib.ptr(ent_out), S,
              _lib.ptr(_dev(case.seg_begin)), _lib.ptr(_dev(case.seg_end)), _lib.ptr(off_d), _lib.ptr(off_d[S:]), cmax, ch,
              _lib.ptr(_dev(case.split.view(np.uint8))), _lib.ptr(_dev(case.child_slot)), _lib.ptr(cursors), _lib.ptr(scratch),
              _lib.ptr(_dev(case.subset_next)), m, n_bins, C, _lib.ptr(hist), 1 if route else 0)
    torch.cuda.synchronize()
    out = (hist.cpu().numpy().view(np.uint32).reshape(case.n_next, m, n_bins, C),
           ent_out.cpu().numpy() if route else None, cursors.cpu().numpy().reshape(S, 2) if route else None)
    return out + ((ch, m_pass, nch),)


def _key(pairs):
    p = np.asarray(pairs, np.int64)
    return np.sort((p[:, 0] << 32) | (p[:, 1] & 0xFFFFFFFF)) if len(p) else np.zeros(0, np.int64)


def _check_entries(case, ent_out, cursors, left, right, cur_ref):
    assert np.array_equal(cursors, cur_ref)
    untouched = np.ones(len(ent_out), bool)
    for s in range(len(case.seg_begin)):
        sb, se = int(case.seg_begin[s]), int(case.seg_end[s])
        L, R = len(left[s]), len(right[s])
        assert np.array_equal(_key(ent_out[sb:sb + L]), _key(left[s])), "left entries of parent %d" % s
        assert np.array_equal(_key(ent_out[se - R:se]), _key(right[s])), "right entries of parent %d" % s
        untouched[sb:sb + L] = False; untouched[se - R:se] = False
    assert (ent_out[untouched] == SENTINEL).all()


def _check_route(case, got, route=True):
    hist, ent_out, cursors, (ch, m_pass, nch) = got
    want, left, right, cur = route_ref(case.bins, case.labels, case.ent, case.seg_begin, case.seg_end, nch, ch, case.split,
                                       case.child_slot, case.subset_next, case.n_bins, case.C, case.n_next)
    assert want.max() < 2 ** 32
    assert np.array_equal(hist.astype(np.int64), want)
    if route:
        _check_entries(case, ent_out, cursors, left, right, cur)


def _lens(ch):
    return [0, 1, ch - 1, ch, ch + 1, 2 * ch + 3, 5, 700, 64, 3 * ch]


# byte and packed record formats: (F, feat_bins, expected packed bytes; 0 = byte records)
FORMATS = {
    "bytes41": (41, [70] * 38 + [3, 66, 11], 0),
    "bytes78": (78, [78] * 78, 0),
    "bytes200": (200, [5, 17, 33, 2] * 50, 0),
    "packed16": (20, [2] * 20, 16),
    "packed32": (41, [32] * 41, 32),
    "packed48": (78, [16] * 78, 48),
    "packed64": (90, [32] * 90, 64),
}


def _format(name):
    F, fb, want = FORMATS[name]
    assert _lib.packed_layout(fb, 5)[1] == want or not want
    return F, fb, want > 0


# ------------------------------------------------------------------------------------------------ route_hist_level
@pytest.mark.gpu
@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("width", WIDTHS)
@pytest.mark.parametrize("fmt", ["bytes41", "packed32"])
def test_route_variant_x_shape(fmt, width, shape, monkeypatch):
    F, fb, packed = _format(fmt)
    m = _width(width, 7, F)
    nw, ks = map(int, shape.split("x"))
    rng = np.random.default_rng(zlib.crc32((fmt + width + shape).encode()))
    case = RouteCase(rng, fb, 5, _lens(nw * ks * 32), m)
    got = _run_route(case, packed, shape=shape, monkeypatch=monkeypatch)
    assert got[3][1] == m                                 # one pass of 7 (rotated), 13 or 41 (generic loop) features
    _check_route(case, got)


@pytest.mark.gpu
@pytest.mark.parametrize("width", WIDTHS)
@pytest.mark.parametrize("fmt", list(FORMATS))
def test_route_record_formats(fmt, width, monkeypatch):
    F, fb, packed = _format(fmt)
    mm = _width(width, 9, F)
    rng = np.random.default_rng(len(fmt) * 7 + F + mm)
    ch = _lib.route_hist_config(F, mm, max(fb), 5, FORMATS[fmt][2])[0]
    case = RouteCase(rng, fb, 5, _lens(ch), mm)
    _check_route(case, _run_route(case, packed, monkeypatch=monkeypatch))


@pytest.mark.gpu
@pytest.mark.parametrize("m", list(range(1, 42)) + ["passes"])
def test_route_subset_width(m, monkeypatch):
    # every width of a 41-feature record in one pass: the rotated update compiled for 1..12, the generic loop from 13
    rng = np.random.default_rng(100 + (m if m != "passes" else 99))
    if m == "passes":                                     # child histograms too wide for one pass: only pass 0 routes
        F, fb, C, mm = 78, [64] * 78, 23, 36
        ch, m_pass = _lib.route_hist_config(F, mm, 64, C, 0)
        assert m_pass < mm and m_pass <= 12
    else:
        F, fb, C, mm = 41, [70] * 38 + [3, 66, 11], 5, m
        ch, m_pass = _lib.route_hist_config(F, mm, 70, C, 0)
        assert m_pass == mm
    case = RouteCase(rng, fb, C, _lens(ch), mm)
    got = _run_route(case, False, monkeypatch=monkeypatch)
    assert got[3][1] == m_pass
    _check_route(case, got)


@pytest.mark.gpu
@pytest.mark.parametrize("width", WIDTHS)
@pytest.mark.parametrize("C", [2, 23, 200])
def test_route_classes(C, width, monkeypatch):
    # C = 200: the wider subsets run in feature passes
    m = _width(width, 5, 30)
    rng = np.random.default_rng(C + m)
    fb = [16] * 30
    case = RouteCase(rng, fb, C, _lens(_lib.route_hist_config(30, m, 16, C, 0)[0]), m)
    _check_route(case, _run_route(case, False, monkeypatch=monkeypatch))


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ["bytes41", "packed48"])
@pytest.mark.parametrize("width", WIDTHS)
def test_route_hot_counter_large_weights(width, fmt, monkeypatch):
    F, fb, packed = _format(fmt)
    mm = _width(width, 6, F)
    rng = np.random.default_rng(7)
    ch = _lib.route_hist_config(F, mm, max(fb), 5, FORMATS[fmt][2])[0]
    case = RouteCase(rng, fb, 5, [0, 3 * ch + 17, ch, 11, 2 * ch, 40, 900], mm, hot=True)
    _check_route(case, _run_route(case, packed, monkeypatch=monkeypatch))


@pytest.mark.gpu
@pytest.mark.parametrize("width", WIDTHS)
def test_route_masks_in_all_words(width, monkeypatch):
    # 256-bin categorical splits: mask words 1-3 decide for bins 64-255
    m = _width(width, 4, 15)
    rng = np.random.default_rng(256)
    fb = [256] * 12 + [200, 130, 65]
    ch = _lib.route_hist_config(15, m, 256, 3, 0)[0]
    case = RouteCase(rng, fb, 3, _lens(ch), m, cat_every=1)
    assert (case.split["kind"][2:] == 1).all()
    _check_route(case, _run_route(case, False, monkeypatch=monkeypatch))


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ["bytes78", "packed16"])
def test_route_many_parents_and_spare_chunks(fmt, monkeypatch):
    F, fb, packed = _format(fmt)
    rng = np.random.default_rng(300)
    ch = _lib.route_hist_config(F, 9, max(fb), 5, FORMATS[fmt][2])[0]
    lens = list(rng.integers(0, 2 * ch, 300))
    case = RouteCase(rng, fb, 5, lens, 9)
    _check_route(case, _run_route(case, packed, extra_chunks=100000, monkeypatch=monkeypatch))


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ["bytes41", "packed64"])
def test_route_histograms_only(fmt, monkeypatch):
    # flags = 0: no entries written, ent_out and cursors are NULL
    F, fb, packed = _format(fmt)
    rng = np.random.default_rng(11)
    ch = _lib.route_hist_config(F, 7, max(fb), 5, FORMATS[fmt][2])[0]
    case = RouteCase(rng, fb, 5, _lens(ch), 7)
    _check_route(case, _run_route(case, packed, route=False, monkeypatch=monkeypatch), route=False)


# ------------------------------------------------------------------------------------------------ partition_level
@pytest.mark.gpu
@pytest.mark.parametrize("chunk_rows", [2048, 777])
def test_partition_level_and_next_segments(chunk_rows):
    rng = np.random.default_rng(chunk_rows)
    F, fb = 41, [70] * 38 + [3, 66, 11]
    case = RouteCase(rng, fb, 5, _lens(chunk_rows) + list(rng.integers(0, 3000, 40)), 1)
    S = len(case.seg_begin)
    # partition_level keeps a side by the split's flags: bit 0 leaf parent, bit 1 / 2 left / right child is a leaf
    split = case.split.copy()
    flags = np.zeros(S, np.int32)
    flags[4] = 1; flags[2] = 2; flags[3] = 4; flags[7] = 6; flags[12:20:3] = 1
    split["flags"] = flags
    keep = np.full(2 * S, -1, np.int32)
    for s in range(S):
        for side in (0, 1):
            if not (flags[s] & 1) and not (flags[s] & (2 << side)):
                keep[2 * s + side] = 0
    stride = fr.tp_stride(F)
    host = np.zeros((case.bins.shape[0], stride), np.uint8)
    host[:, :F] = case.bins; host[:, F] = case.labels
    lens = case.seg_end - case.seg_begin
    nch = (lens + chunk_rows - 1) // chunk_rows
    off = _scan(nch)
    ent = _dev(case.ent)
    ent_out = torch.full_like(ent, SENTINEL)
    cursors = torch.zeros(2 * S, dtype=torch.int32, device=DEV)
    sb, se = _dev(case.seg_begin), _dev(case.seg_end)
    _lib.call("b200flow_partition_level", _lib.ptr(_dev(host)), stride, _lib.ptr(ent), _lib.ptr(ent_out), S, _lib.ptr(sb),
              _lib.ptr(se), _lib.ptr(_dev(off)), int(off[-1]), chunk_rows, _lib.ptr(_dev(split.view(np.uint8))), _lib.ptr(cursors))
    _, left, right, cur = route_ref(case.bins, case.labels, case.ent, case.seg_begin, case.seg_end, nch, chunk_rows, split, keep,
                                    None, case.n_bins, case.C, 0)
    cur_got = cursors.cpu().numpy().reshape(S, 2)
    _check_entries(case, ent_out.cpu().numpy(), cur_got, left, right, cur)
    # next level's segments: the kept children in slot order; n_next_dev below the host bound leaves the tail untouched
    parents = np.array([2 * s + side for s in range(S) for side in (0, 1) if keep[2 * s + side] >= 0], np.int32)
    n = len(parents)
    for n_dev in (None, n - 5):
        nb_ = torch.full((n,), -1, dtype=torch.int64, device=DEV); ne_ = torch.full((n,), -1, dtype=torch.int64, device=DEV)
        cnt = None if n_dev is None else _dev(np.array([n_dev], np.int64))
        _lib.call("b200flow_next_segments", n, _lib.ptr(cnt), _lib.ptr(_dev(parents)), _lib.ptr(sb), _lib.ptr(se), _lib.ptr(cursors),
                  _lib.ptr(nb_), _lib.ptr(ne_))
        lim = n if n_dev is None else n_dev
        b_, e_ = nb_.cpu().numpy(), ne_.cpu().numpy()
        for i, p in enumerate(parents[:lim]):
            s, side = p >> 1, p & 1
            want = (case.seg_begin[s], case.seg_begin[s] + cur[s, 0]) if side == 0 else (case.seg_end[s] - cur[s, 1], case.seg_end[s])
            assert (b_[i], e_[i]) == want
        assert (b_[lim:] == -1).all() and (e_[lim:] == -1).all()


# ------------------------------------------------------------------------------------------------ score_level
def _node_hist(rng, n, feat_bins, subset, C, skew=None, pure=False, dup=None):
    """histogram [m][n_bins][C] of n random records (consistent over features: every feature sums to the node's counts).
    skew = (feature, strength): that feature's bin decides the label with the given probability.  dup = (j1, j2): subset
    position j2 gets the bins of position j1 (identical histograms)."""
    n_bins = int(max(feat_bins))
    m = len(subset)
    bins = np.stack([rng.integers(0, feat_bins[f], n) for f in subset], 1) if n else np.zeros((0, m), np.int64)
    lab = rng.integers(0, C, n)
    if pure:
        lab[:] = int(rng.integers(0, C))
    if skew is not None and n:
        j, p = skew
        sel = rng.random(n) < p
        lab[sel] = (bins[sel, j] * 7 + 3) % C
    if dup is not None:
        bins[:, dup[1]] = bins[:, dup[0]]
    w = rng.integers(1, 4, n)
    h = np.zeros((m, n_bins, C), np.int64)
    for j in range(m):
        np.add.at(h[j], (bins[:, j], lab), w)
    return h


def _run_score(hists, subsets, feat_bins, feat_kind, C, level=0, max_depth=5, min_inst=1, min_gain=0.0):
    S, m, n_bins, _ = hists.shape
    assert hists.max(initial=0) < 2 ** 32
    split = torch.zeros((S, 64), dtype=torch.uint8, device=DEV)
    nc, lc, rc = (torch.full((S, C), SENTINEL, dtype=torch.int32, device=DEV) for _ in range(3))
    _lib.call("b200flow_score_level", _lib.ptr(_dev(hists.astype(np.uint32))), S, _lib.ptr(_dev(np.asarray(subsets, np.int16))),
              m, n_bins, C, _lib.ptr(_dev(np.asarray(feat_bins, np.int32))), _lib.ptr(_dev(np.asarray(feat_kind, np.int32))),
              level, max_depth, min_inst, float(min_gain), _lib.ptr(split), _lib.ptr(nc), _lib.ptr(lc), _lib.ptr(rc))
    got = split.cpu().numpy()
    nc, lc, rc = (t.cpu().numpy().view(np.uint32).astype(np.int64) for t in (nc, lc, rc))
    for s in range(S):
        want, tot, L, R = score_ref(hists[s], subsets[s], feat_bins, feat_kind, level, max_depth, min_inst, min_gain)
        w = np.zeros(1, SPLIT_DTYPE); w[0] = want
        assert got[s].tobytes() == w.tobytes(), "slot %d: got %s want %s" % (s, got[s].view(SPLIT_DTYPE)[0], want)
        assert np.array_equal(nc[s], tot) and np.array_equal(lc[s], L) and np.array_equal(rc[s], R), "counts of slot %d" % s
    return got.view(SPLIT_DTYPE).reshape(S)


def _mixed_features(rng, n_feats, n_bins, C):
    """continuous features of 1, 2, ... n_bins bins, ordered categoricals, and unordered ones (multiclass, <= 6 categories)."""
    fb = rng.integers(1, n_bins + 1, n_feats)
    fb[0], fb[1], fb[2] = n_bins, 1, 2
    kind = np.zeros(n_feats, np.int32)
    kind[3::4] = 1
    if C > 2:
        kind[5::6] = 2
        fb[kind == 2] = np.minimum(np.maximum(fb[kind == 2], 2), 6)
    return fb.astype(np.int32), kind


@pytest.mark.gpu
@pytest.mark.parametrize("n_bins", [13, 37])
@pytest.mark.parametrize("C", [2, 3, 16, 17, 23])
def test_score_classes_and_scans(C, n_bins):
    # C <= 16: the segmented prefix scan (32 / C lane segments, ragged when nb is no multiple of them); C > 16: serial
    rng = np.random.default_rng(C * 100 + n_bins)
    F, m = 24, 9
    fb, kind = _mixed_features(rng, F, n_bins, C)
    hists, subsets = [], []
    for s in range(14):
        sub = np.sort(rng.choice(F, m, replace=False)) if s % 3 else np.arange(m)
        n = [0, 1, 2, 50, 400, 3000][s % 6]
        skew = (int(rng.integers(0, m)), 0.7) if s % 2 else None
        hists.append(_node_hist(rng, n, fb, sub, C, skew=skew, pure=(s == 7)))
        subsets.append(sub)
    _run_score(np.stack(hists), np.stack(subsets), fb, kind, C)


@pytest.mark.gpu
@pytest.mark.parametrize("kind_of_dup", [0, 1, 2])
def test_score_exact_ties(kind_of_dup):
    # two identical features: the first in subset order wins; equal splits inside a feature: the first split wins
    rng = np.random.default_rng(40 + kind_of_dup)
    C, F = 3, 10
    fb = np.full(F, 12 if kind_of_dup != 2 else 6, np.int32)
    kind = np.full(F, kind_of_dup, np.int32)
    hists, subsets = [], []
    n_split_ties = 0
    for s in range(8):
        sub = np.arange(F)
        h = _node_hist(rng, 500 + 50 * s, fb, sub, C, skew=(4, 0.8), dup=(4, 8))
        if kind_of_dup == 0 and s % 2:
            # empty the bin after the best threshold b (its entries move one bin up): split b + 1 now has exactly b's gain
            best = score_ref(h, sub, fb, kind, 0, 5, 1, 0.0)[0]
            b = int(best["bin_thr"])
            if best["feat"] == 4 and b + 2 < fb[4]:
                for j in (4, 8):
                    h[j, b + 2] += h[j, b + 1]; h[j, b + 1] = 0
                n_split_ties += 1
        hists.append(h); subsets.append(sub)
    got = _run_score(np.stack(hists), np.stack(subsets), fb, kind, C)
    assert (got["feat"] == 4).all()
    assert kind_of_dup != 0 or n_split_ties >= 2


@pytest.mark.gpu
@pytest.mark.parametrize("n_cat", [200, 255])
@pytest.mark.parametrize("C", [2, 23])
def test_score_ordered_categoricals_wide(C, n_cat):
    # 200-255 categories: the chosen ranks reach mask words 0-3; tied centroids (equal and empty categories) rank stably
    rng = np.random.default_rng(n_cat + C)
    F, m = 6, 6
    fb = np.array([n_cat, n_cat, 255, 40, n_cat, 7], np.int32)
    kind = np.array([1, 1, 1, 0, 1, 1], np.int32)
    hists, subsets = [], []
    for s in range(6):
        sub = np.arange(m)
        h = _node_hist(rng, 20000, fb, sub, C, skew=(s % m, 0.6))
        for j in np.nonzero(fb >= 200)[0]:                  # every feature keeps the node's class counts
            pool = h[j, 10:30].sum(0)
            h[j, 10:30] = pool // 20                        # categories 10-28: tied centroids
            h[j, 29] += pool - 20 * (pool // 20)
            h[j, 60] += h[j, 100:140].sum(0)
            h[j, 100:140] = 0                               # forty empty categories: ranked last, in index order
        hists.append(h); subsets.append(sub)
    got = _run_score(np.stack(hists), np.stack(subsets), fb, kind, C)
    assert np.any(got["mask"][:, 1:] != 0)


@pytest.mark.gpu
@pytest.mark.parametrize("C", [3, 5])
@pytest.mark.parametrize("nb", [2, 3, 4, 5, 6, 7, 8])
def test_score_unordered_with_few_bins(nb, C):
    # an unordered feature of nb categories has 2^(nb-1) - 1 candidate subsets, more than n_bins = nb from nb = 4 on;
    # every other feature of the node lists its own candidates next to it
    rng = np.random.default_rng(nb * 10 + C)
    F, m = 8, 8
    fb = np.full(F, nb, np.int32)
    kind = np.array([2, 0, 2, 0, 1, 2, 0, 2], np.int32)
    fb[1] = max(nb - 1, 1)
    hists, subsets = [], []
    for s in range(10):
        sub = np.arange(m)
        hists.append(_node_hist(rng, [0, 5, 300, 4000][s % 4], fb, sub, C, skew=(int(rng.integers(0, m)), 0.5)))
        subsets.append(sub)
    got = _run_score(np.stack(hists), np.stack(subsets), fb, kind, C)
    assert (got["feat"] >= 0).sum() >= 5


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["m80", "wide"])
def test_score_feature_batches(shape):
    # m > 64, or n_bins * C so large that only a few features fit: the scorer stages the features in batches; the best
    # split lies in a later batch, and its twin in an earlier batch wins the tie
    rng = np.random.default_rng(80 if shape == "m80" else 81)
    if shape == "m80":
        F, n_bins, C = 80, 16, 3
    else:
        F, n_bins, C = 9, 256, 23
    fb = np.full(F, n_bins, np.int32)
    kind = np.zeros(F, np.int32)
    late = F - 3
    hists, subsets = [], []
    for s in range(4):
        sub = np.arange(F)
        dup = (late, 1) if s % 2 else None                   # slot 1, 3: position 1 copies the late feature
        h = _node_hist(rng, 6000, fb, sub, C, skew=(late, 0.9))
        if dup is not None:
            h[1] = h[late]
        hists.append(h); subsets.append(sub)
    got = _run_score(np.stack(hists), np.stack(subsets), fb, kind, C)
    assert list(got["feat"]) == [late, 1, late, 1]


@pytest.mark.gpu
@pytest.mark.parametrize("edge", ["min_instances", "min_info_gain", "level_eq_max", "last_level", "pure_child", "defaults"])
def test_score_leaf_rules(edge):
    rng = np.random.default_rng(5)
    C, F, m = 4, 12, 12
    fb, kind = _mixed_features(rng, F, 20, C)
    hists, subsets = [], []
    for s in range(10):
        sub = np.arange(m)
        n = [0, 1, 2, 40, 2000][s % 5]
        h = _node_hist(rng, n, fb, sub, C, skew=(0, 0.95), pure=(s == 9))
        if s == 8:                                          # the only valid split of the node has a pure left child
            h[:] = 0
            h[0, 0, 1] = 500; h[0, 1] = [300, 0, 300, 300]
            h[1:, 0] = h[0].sum(0)
        hists.append(h); subsets.append(sub)
    kw = dict(min_instances=dict(min_inst=10 ** 6), min_info_gain=dict(min_gain=2.0), level_eq_max=dict(level=5, max_depth=5),
              last_level=dict(level=4, max_depth=5), pure_child=dict(), defaults=dict(level=1, max_depth=7))[edge]
    got = _run_score(np.stack(hists), np.stack(subsets), fb, kind, C, **kw)
    if edge in ("min_instances", "min_info_gain"):
        assert (got["flags"] == 1).all() and (got["gain"] == -np.finfo(np.float64).max).all()
    if edge == "level_eq_max":
        assert (got["flags"] == 1).all()
    if edge == "last_level":
        assert set(got["flags"]) <= {1, 6}
    if edge == "pure_child":
        assert got["flags"][8] & 2


# ------------------------------------------------------------------------------------------------ grow_level
@pytest.mark.gpu
@pytest.mark.parametrize("with_mask", [True, False])
@pytest.mark.parametrize("capacity", ["enough", "one_short"])
def test_grow_level(capacity, with_mask):
    rng = np.random.default_rng(3 if with_mask else 4)
    S, P0, C = 700, 2000, 5
    cap_alloc = P0 + 2 * S + 10
    split = np.zeros(S, SPLIT_DTYPE)
    split["flags"] = rng.choice([1, 0, 2, 4, 6], S)
    split["feat"] = rng.integers(0, 41, S); split["kind"] = rng.integers(0, 2, S); split["bin_thr"] = rng.integers(0, 256, S)
    split["mask"] = rng.integers(0, 2 ** 63, (S, 4), dtype=np.uint64)
    slot_node = rng.permutation(P0)[:S].astype(np.int32)
    slot_tree = rng.integers(0, 50, S).astype(np.int32)
    slot_nid = rng.integers(1, 2 ** 31, S).astype(np.uint32)
    slot_nid[:3] = [1, 2 ** 31 + 5, 0xFFFFFFFF]
    node_counts, left_counts, right_counts = (rng.integers(0, 2 ** 32, (S, C), dtype=np.uint32) for _ in range(3))
    nodes = rng.integers(0, 256, (cap_alloc, 16), dtype=np.uint8).view(NODE_DTYPE).reshape(cap_alloc)
    node_mask = rng.integers(0, 2 ** 63, (cap_alloc, 4), dtype=np.uint64) if with_mask else None
    pool_counts = rng.integers(0, 2 ** 32, (cap_alloc, C), dtype=np.uint32)
    node_tree = rng.integers(0, 50, cap_alloc).astype(np.int32)
    n_split = int(((split["flags"] & 1) == 0).sum())
    pool_capacity = P0 + 2 * n_split - (1 if capacity == "one_short" else 0)
    nblk = (S + 255) // 256
    assert nblk > 1
    counters = np.full(8 + nblk + 1, -3, np.int64); counters[0] = P0
    d = {k: _dev(v) for k, v in dict(nodes=nodes.view(np.uint8), pool_counts=pool_counts, node_tree=node_tree, counters=counters).items()}
    d_mask = _dev(node_mask) if with_mask else None
    nxt = [torch.full((2 * S,), SENTINEL, dtype=torch.int32, device=DEV) for _ in range(5)]
    _lib.call("b200flow_grow_level", S, _lib.ptr(_dev(slot_tree)), _lib.ptr(_dev(slot_nid)), _lib.ptr(_dev(slot_node)),
              _lib.ptr(_dev(split.view(np.uint8))), _lib.ptr(_dev(node_counts)), _lib.ptr(_dev(left_counts)), _lib.ptr(_dev(right_counts)),
              C, _lib.ptr(d["nodes"]), _lib.ptr(d_mask), _lib.ptr(d["pool_counts"]), _lib.ptr(d["node_tree"]), pool_capacity,
              *[_lib.ptr(t) for t in nxt], _lib.ptr(d["counters"]))
    w_nodes, w_mask, w_pc, w_nt = nodes.copy(), (node_mask.copy() if with_mask else None), pool_counts.copy(), node_tree.copy()
    cnt, n_tree, n_nid, n_node, n_parent, child_slot = grow_ref(slot_tree, slot_nid, slot_node, split, node_counts, left_counts,
                                                                right_counts, w_nodes, w_mask, w_pc, w_nt, P0, pool_capacity)
    got_cnt = d["counters"].cpu().numpy()
    assert tuple(got_cnt[:4]) == cnt
    assert cnt[2] == (1 if capacity == "one_short" else 0)
    assert d["nodes"].cpu().numpy().tobytes() == w_nodes.tobytes()
    assert np.array_equal(d["pool_counts"].cpu().numpy().view(np.uint32), w_pc)
    assert np.array_equal(d["node_tree"].cpu().numpy(), w_nt)
    if with_mask:
        assert np.array_equal(d_mask.cpu().numpy().view(np.uint64), w_mask)
    got_next = [t.cpu().numpy() for t in nxt]
    n = cnt[1]
    for got, want in zip(got_next[:4], (n_tree, n_nid, n_node, n_parent)):
        assert np.array_equal(got[:n].view(np.uint32).astype(np.int64) if got is got_next[1] else got[:n], want)
        assert (got[n:] == SENTINEL).all()
    if child_slot is None:
        assert (got_next[4] == SENTINEL).all()
    else:
        assert np.array_equal(got_next[4], child_slot)


# ------------------------------------------------------------------------------------------------ forest guard
@pytest.mark.gpu
@pytest.mark.parametrize("max_bins", [32, 70])
@pytest.mark.parametrize("C", [3, 5])
@pytest.mark.parametrize("trees", [1, 8])
def test_forest_unordered_features_few_bins(trees, C, max_bins):
    # the widest feature has 6 bins while an unordered categorical lists up to 31 candidate subsets
    x, y, arity = unordered_features(6000, C, 17 * C + max_bins + trees)
    p = fr.ForestParams(num_trees=trees, max_bins=max_bins, max_depth=6, seed=2019, bootstrap=trees > 1)
    model = fr.fit_forest(_dev(x), _dev(y), C, arity, p)
    fo, meta = oracle.fit_forest(x, y, C, arity, num_trees=trees, max_bins=max_bins, max_depth=6, seed=2019)
    fb, kind = meta["feat_bins"], meta["feat_kind"]
    assert max((1 << (b - 1)) - 1 for b, k in zip(fb, kind) if k == 2) > meta["n_bins"]
    ex = model.export()
    assert forests_equal(ex, fo.export()) == []
    assert np.isin(ex["feat"][ex["is_leaf"] == 0], np.nonzero(kind == 2)[0]).any()
    tp_o, _ = oracle.bin_rows(x, meta["thresholds"], meta["n_thr"], meta["arity"], meta["max_bins"])
    raw_o, prob_o, pred_o = fo.predict(tp_o, dt_mode=trees == 1)
    raw, prob, pred = model.predict(_dev(x))
    assert np.array_equal(pred.cpu().numpy(), pred_o)
    assert np.array_equal(raw.cpu().numpy(), raw_o) and np.array_equal(prob.cpu().numpy(), prob_o)
