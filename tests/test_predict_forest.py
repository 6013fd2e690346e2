"""The batch predictor over the per-tree compact layout (b200flow_forest_layout_size, b200flow_build_forest_layout,
b200flow_predict_forest) against a numpy walk of the same forest: raw, prob and pred bit for bit.  The forests are random
level-major pools (roots first, children appended in pairs level by level, as grow_level writes them) with continuous and
categorical splits, and forests fitted by fit_forest.  Cases: C = 2, 5, 23, 64, 180 and 250, both vote modes, T = 1,
stumps, an empty batch, row counts that are not a multiple of a block's rows and that take several rounds of the
persistent grid, and trees larger than the shared-memory buffer (one over 65,535 nodes), whose deep nodes and leaf votes
are read from global memory.  The layout itself is checked against a numpy restatement."""
import numpy as np
import pytest
import torch

from b200flow import forest as fr
from b200flow._lib import NODE_DTYPE, call, ptr

DEV = "cuda"
F = 41


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _make_pool(depths, C, seed, p_split=0.7, p_cat=0.3, bins=40, interleave=True):
    """level-major pool of len(depths) trees; tree t keeps a spine down to depths[t], other nodes split with p_split.
    Continuous splits take a threshold below `bins`; interleave: trees interleave within a level."""
    rng = np.random.default_rng(seed)
    T = len(depths)
    feat, kb, left, nid, tree = [-1] * T, [0] * T, [-1] * T, [1] * T, list(range(T))
    queue = [(t, 0, depths[t], True) for t in range(T)]
    while queue:
        nxt = []
        for i, d, D, spine in queue:
            if d >= D or not (spine or rng.random() < p_split):
                continue
            li = len(feat)
            feat[i] = int(rng.integers(0, F))
            kb[i] = (65536 | int(rng.integers(0, 32))) if rng.random() < p_cat else int(rng.integers(0, bins))
            left[i] = li
            feat += [-1, -1]; kb += [0, 0]; left += [-1, -1]; nid += [2 * nid[i], 2 * nid[i] + 1]; tree += [tree[i]] * 2
            go = int(rng.integers(0, 2))
            nxt += [(li, d + 1, D, spine and go == 0), (li + 1, d + 1, D, spine and go == 1)]
        if interleave:
            rng.shuffle(nxt)
        queue = nxt
    nodes = np.zeros(len(feat), NODE_DTYPE)
    nodes["feat"], nodes["kind_bin"], nodes["left"], nodes["nid"] = feat, kb, left, nid
    mask = rng.integers(0, 2 ** 63, (len(feat), 4), dtype=np.int64).view(np.uint64)
    leaf_prob = rng.random((len(feat), C))
    counts = rng.integers(0, 5000, (len(feat), C)).astype(np.uint32)
    return nodes, mask, leaf_prob, counts, np.asarray(tree, np.int32)


def _rows(n, seed, bins=48):
    rng = np.random.default_rng(seed)
    tp = np.zeros((n, fr.tp_stride(F)), np.uint8)
    tp[:, :F] = rng.integers(0, bins, (n, F))
    tp[:, :8] = rng.integers(0, 256, (n, 8))                                  # bins in every word of a categorical mask
    return tp


def _walk(tp, nodes, mask, payload, T):
    """votes of every row: payload of its leaf in each tree, added in tree order from 0.0 as the kernel does"""
    n = tp.shape[0]
    feat, kb, left = nodes["feat"].astype(np.int64), nodes["kind_bin"].astype(np.int64), nodes["left"].astype(np.int64)
    votes = np.zeros((n, payload.shape[1]))
    rows = np.arange(n)
    for t in range(T):
        idx = np.full(n, t, np.int64)
        act = rows[feat[idx] >= 0]
        while act.size:
            nd = idx[act]
            b = tp[act, feat[nd]].astype(np.int64)
            cont = kb[nd] < 65536
            bit = (mask[nd, b >> 6] >> (b & 63).astype(np.uint64)) & np.uint64(1)
            right = np.where(cont, b > kb[nd], bit == 0).astype(np.int64)
            idx[act] = left[nd] + right
            act = act[feat[idx[act]] >= 0]
        votes += payload[idx]
    return votes


def _want_predict(votes):
    s = np.zeros(votes.shape[0])
    for k in range(votes.shape[1]):                                           # sequential, class order
        s = s + votes[:, k]
    with np.errstate(invalid="ignore", divide="ignore"):
        prob = np.where(s[:, None] != 0, votes / s[:, None], 0.0)
    return votes, prob, np.argmax(votes, 1).astype(np.float64)              # first maximum


def _layout(nodes_d, mask_d, prob_d, counts_d, tree_d, P, T, C, dt):
    scratch = torch.empty(2 * P + 4 * T, dtype=torch.int32, device=DEV)
    tree_off = torch.empty(T + 1, dtype=torch.int64, device=DEV)
    call("b200flow_forest_layout_size", ptr(nodes_d), ptr(tree_d), P, T, C, ptr(scratch), ptr(tree_off))
    layout = torch.empty(max(int(tree_off[T].item()), 2), dtype=torch.int64, device=DEV)
    call("b200flow_build_forest_layout", ptr(nodes_d), ptr(mask_d), ptr(prob_d), ptr(counts_d), ptr(tree_d), P, T, C, dt,
         ptr(scratch), ptr(tree_off), ptr(layout))
    return layout, tree_off


def _predict(pool, T, C, dt, tp):
    """b200flow_predict_forest outputs over the layout built from the pool, and the layout"""
    nodes, mask, leaf_prob, counts, tree = pool
    P, n = nodes.shape[0], tp.shape[0]
    nodes_d = _dev(nodes.view(np.uint8).reshape(-1, 16))
    mask_d, prob_d, counts_d, tree_d = _dev(mask.view(np.int64)), _dev(leaf_prob), _dev(counts.view(np.int32)), _dev(tree)
    tp_d = _dev(tp) if n else torch.empty((0, tp.shape[1]), dtype=torch.uint8, device=DEV)
    raw = torch.full((n, C), -1.0, dtype=torch.float64, device=DEV); prob = torch.full_like(raw, -1.0)
    pred = torch.full((n,), -1.0, dtype=torch.float64, device=DEV)
    layout, tree_off = _layout(nodes_d, mask_d, prob_d, counts_d, tree_d, P, T, C, dt)
    call("b200flow_predict_forest", ptr(tp_d), tp.shape[1], F, n, ptr(layout), ptr(tree_off), T, C, ptr(raw), ptr(prob),
         ptr(pred))
    got = tuple(a.cpu().numpy() for a in (raw, prob, pred))
    return got, (layout.cpu().numpy().view(np.uint64), tree_off.cpu().numpy())


def _assert_walk(got, pool, T, dt, tp, what):
    nodes, mask, leaf_prob, counts, _ = pool
    want = _want_predict(_walk(tp, nodes, mask, counts.astype(np.float64) if dt else leaf_prob, T))
    for g, w, name in zip(got, want, ("raw", "prob", "pred")):
        assert g.shape == w.shape and np.array_equal(g.view(np.uint64), w.view(np.uint64)), (what, name)


def _want_layout(pool, T, C, dt):
    """numpy restatement of the layout: per tree, node records in pool order, categorical records, leaf votes, padded to
    an even word count -> (words, tree offsets, unpadded block sizes)"""
    nodes, mask, leaf_prob, counts, tree = pool
    payload = counts.astype(np.float64) if dt else leaf_prob
    blocks, sizes, local = [], [], np.full(nodes.shape[0], -1, np.int64)
    for t in range(T):
        idx = np.flatnonzero(tree == t)
        local[idx] = np.arange(idx.size)
    for t in range(T):
        idx = np.flatnonzero(tree == t)
        leaves = [i for i in idx if nodes["feat"][i] < 0]
        cats = [i for i in idx if nodes["feat"][i] >= 0 and nodes["kind_bin"][i] >= 65536]
        n_t, c_t = idx.size, len(cats)
        size = n_t + 5 * c_t + len(leaves) * C
        words = np.zeros(size + (size & 1), np.uint64)
        for i in idx:
            f, kbin, lc = int(nodes["feat"][i]), int(nodes["kind_bin"][i]), int(nodes["left"][i])
            if f < 0:
                a, b = 1 << 31, n_t + 5 * c_t + leaves.index(i) * C
                words[b:b + C] = payload[i].view(np.uint64)
            elif kbin >= 65536:
                a, b = f | (1 << 30), n_t + 5 * cats.index(i)
                words[b] = local[lc]
                words[b + 1:b + 5] = mask[i]
            else:
                a, b = f | (min(kbin, 255) << 16), local[lc]
            words[local[i]] = np.uint64(a) | (np.uint64(b) << np.uint64(32))
        blocks.append(words)
        sizes.append(size)
    off = np.concatenate([[0], np.cumsum([b.size for b in blocks])]).astype(np.int64)
    return np.concatenate(blocks), off, sizes


DEPTHS = [0, 1, 3, 9, 12, 0, 14, 6]
# a second fixture: stumps, shallow trees and trees deeper than 8 and 10 levels, continuous thresholds below 32, trees
# appended level by level without interleaving
PRED_DEPTHS = [0, 1, 3, 9, 12, 0, 14]
PRED_C = [2, 23, 64, 180, 250]


def _pred_pool(C):
    return _make_pool(PRED_DEPTHS, C, seed=C, bins=32, interleave=False)


@pytest.mark.gpu
@pytest.mark.parametrize("C", [2, 5, 23, 250])
@pytest.mark.parametrize("dt", [0, 1])
def test_predict_forest_matches_walk(C, dt):
    pool = _make_pool(DEPTHS, C, seed=C + dt)
    n = 600_001 if C == 2 else 1037                                            # several grid rounds / one partial block
    tp = _rows(n, C)
    got, (layout, off) = _predict(pool, len(DEPTHS), C, dt, tp)
    _assert_walk(got, pool, len(DEPTHS), dt, tp, (C, dt))
    want_layout, want_off, sizes = _want_layout(pool, len(DEPTHS), C, dt)
    assert np.array_equal(off, want_off)
    for t, w in enumerate(sizes):                                             # the padding word of an odd block is not written
        assert np.array_equal(layout[off[t]:off[t] + w], want_layout[want_off[t]:want_off[t] + w]), t


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [0, 1])
def test_predict_forest_single_tree_stumps_and_empty_match_walk(dt):
    one, stumps = _make_pool([10], 5, seed=3), _make_pool([0, 0, 0], 5, seed=4)
    for what, pool, T, tp in (("T=1", one, 1, _rows(4099, 9)),
                              ("empty", one, 1, _rows(0, 9)),                 # empty batch: nothing written, no error
                              ("stumps", stumps, 3, _rows(333, 2))):
        got, _ = _predict(pool, T, 5, dt, tp)
        _assert_walk(got, pool, T, dt, tp, (what, dt))


@pytest.mark.gpu
@pytest.mark.parametrize("C", [5, 23])
def test_predict_forest_large_tree_matches_walk(C):
    # a dense depth-17 tree of ~100k nodes (past 65,535: offsets are 32-bit) beside small ones: its blocks run far past the
    # shared-memory buffer, so deep nodes, most leaf votes and its categorical records come from global memory
    pool = _make_pool([17, 4, 16], C, seed=C, p_split=0.93)
    sizes = np.bincount(pool[4])
    assert sizes[0] > 65_535 and sizes[2] > 20_000
    tp = _rows(50_003, C)
    got, (_, off) = _predict(pool, 3, C, 0, tp)
    assert off[1] - off[0] > 65_535
    _assert_walk(got, pool, 3, 0, tp, ("large", C))


def test_predict_pool_shapes():
    # the second fixture's forests: every tree reaches its depth (a spine)
    nodes, _, _, _, tree = _pred_pool(23)
    depth = np.floor(np.log2(nodes["nid"].astype(np.float64))).astype(int)
    assert [int(depth[tree == t].max()) for t in range(len(PRED_DEPTHS))] == PRED_DEPTHS


@pytest.mark.gpu
@pytest.mark.parametrize("C", PRED_C)
def test_predict_against_walk(C):
    # many classes (C = 250: a row's bins and votes leave little shared memory for the tree buffers); n is never a multiple
    # of a block's rows, and C = 2 with 600,001 rows loops the grid
    pool, T = _pred_pool(C), len(PRED_DEPTHS)
    n = 1037 if C != 2 else 600_001
    tp = _rows(n, C + n, bins=40)
    for dt in (0, 1):
        got, _ = _predict(pool, T, C, dt, tp)
        _assert_walk(got, pool, T, dt, tp, (C, dt))


@pytest.mark.gpu
@pytest.mark.parametrize("num_trees,depth", [(12, 10), (1, 16)])
def test_predict_forest_fitted_model_matches_walk(num_trees, depth):
    # forests grown by fit_forest on rows with categorical features (left-set splits); ForestModel.predict_binned walks the
    # compact layout, numpy the model's host copy of the pool
    rng = np.random.default_rng(7)
    n = 60_000
    x = rng.normal(size=(n, 6))
    cat = rng.integers(0, 9, (n, 2)).astype(np.float64)
    x = np.concatenate([x, cat], 1)
    y = ((x[:, 0] > 0.2).astype(int) + (cat[:, 0] % 3 == 1) + (x[:, 1] * x[:, 2] > 0.3)).astype(np.int32)
    C = int(y.max()) + 1
    arity = [0] * 6 + [9, 9]
    params = fr.ForestParams(num_trees=num_trees, max_depth=depth, max_bins=32, seed=11,
                             bootstrap=num_trees > 1)
    model = fr.fit_forest(_dev(x), _dev(y), C, arity, params)
    P = model.n_nodes
    assert bool((model.nodes[:P, 1] >= 65536).any()), "no categorical split"
    tp, _ = model.bin(_dev(x))
    got = tuple(a.cpu().numpy() for a in model.predict_binned(tp))
    dt = 1 if model.dt_mode else 0
    pool = (model.nodes[:P].cpu().numpy().view(NODE_DTYPE).reshape(-1), model.node_mask[:P].cpu().numpy().view(np.uint64),
            model.leaf_prob[:P].cpu().numpy(), model.pool_counts[:P].cpu().numpy().view(np.uint32) if dt else None, None)
    _assert_walk(got, pool, model.T, dt, tp.cpu().numpy(), (num_trees, depth))
