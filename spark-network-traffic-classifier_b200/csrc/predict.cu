// predict.cu — batch prediction (SURVEY.md §8a R9, HOT LOOP C), the confusion-matrix kernel of
// MulticlassMetrics (R10) and the two relational steps either side of the path (§8f rank 1):
// randomSplit and stable row compaction.
// Reference call sites: model.transform(test_set) kdd99.py:82 / cicids17.py:86; evaluator.evaluate
// kdd99.py:86-91; randomSplit kdd99.py:52; where / handleInvalid="skip" cicids17.py:30-35,41.
#include <type_traits>

#include "common.cuh"

namespace b200flow {

// ------------------------------------------------------------------ R9 predict over the per-tree compact layout
// A walk through the pool is bound by L1 tag lookups: below the first few levels every lane of a warp is at a different
// node, so every node load (and, at the leaf, each of its C vote loads) is a separate request.  A KDD tree is small once
// compacted (~1,900 nodes: ~15 KB of 8-byte nodes plus ~37 KB of C = 5 fp64 leaf votes), so the whole tree is staged in
// shared memory and every walk step and vote add becomes a scattered LDS.
//
// Layout (8-byte words), built once per model: tree t owns words [tree_off[t], tree_off[t+1]), padded to an even count.
//   [0, n_t)            node records in pool order (the pool is level-major, so this is the tree's BFS order), uint2 {a, b}:
//                         a = feat | min(bin_thr, 255) << 16 | kCat | kLeaf, b = word offset in the tree's block of
//                         the left child (continuous split), of the categorical record (categorical split) or of the C
//                         fp64 votes (leaf).  The root is word 0; a node's right child is its left child + 1.
//   [n_t, ...)          one 5-word record per categorical split: left child, then the 4-word left-set mask
//   [..., end)          the leaves' C fp64 votes (leaf_prob, or pool_counts as fp64 in dt_mode), in leaf order
// The categorical records, read at every categorical step, come before the votes, read once per walk: a tree larger than
// the shared-memory buffer leaves its votes in global memory first.
// All offsets are 32-bit, so a tree of any size is exact.
constexpr uint32_t kLayoutLeaf = 1u << 31, kLayoutCat = 1u << 30;
constexpr int kLayoutCatWords = 5;
constexpr int kLayoutRankBlock = 1024, kLayoutRankPer = 4;
constexpr int kVoteBatch = 8;                                                 // leaf votes loaded together (C = 5 on KDD99)
constexpr int kPredForestRegC = 8;                                           // classes whose votes accumulate in registers
constexpr int kPredForestRegThreads = 896;                                   // its block bound: 72 registers, no spills

// block-wide exclusive scan of one uint64 per thread (blockDim == kLayoutRankBlock); sh holds 33 words
__device__ __forceinline__ unsigned long long block_exclusive_scan_u64(unsigned long long v, unsigned long long* sh,
                                                                      unsigned long long* total) {
    const unsigned long long inc = warp_inclusive_scan(v);
    if (lane_id() == 31) sh[warp_id()] = inc;
    __syncthreads();
    if (warp_id() == 0) {
        const unsigned long long w = sh[lane_id()];
        const unsigned long long winc = warp_inclusive_scan(w);
        sh[lane_id()] = winc - w;
        if (lane_id() == 31) sh[32] = winc;
    }
    __syncthreads();
    const unsigned long long res = inc - v + sh[warp_id()];
    *total = sh[32];
    __syncthreads();                                                          // sh is reused by the next chunk
    return res;
}

// one CTA per tree t: scans the pool in order and gives each of t's nodes its rank in the tree (local[i]) and its rank
// among the tree's leaves or categorical splits (ord[i]); cnt[t] = {nodes, leaves, categorical splits}, words[t] = the
// tree's block size.  Counts travel packed in 21-bit fields of one uint64 (a chunk holds 4096 nodes).
__global__ void __launch_bounds__(kLayoutRankBlock) layout_rank_kernel(const int4* __restrict__ nodes,
                                                                        const int32_t* __restrict__ node_tree, int64_t n, int C,
                                                                        int32_t* local, int32_t* ord, int32_t* cnt, int32_t* words) {
    __shared__ unsigned long long sh[33];
    const int t = blockIdx.x;
    constexpr unsigned long long kOne = 1ull, kLeafOne = 1ull << 21, kCatOne = 1ull << 42, kField = (1ull << 21) - 1;
    int64_t base_n = 0, base_l = 0, base_c = 0;
    for (int64_t c0 = 0; c0 < n; c0 += (int64_t)kLayoutRankBlock * kLayoutRankPer) {
        const int64_t i0 = c0 + (int64_t)threadIdx.x * kLayoutRankPer;
        unsigned long long inc[kLayoutRankPer], v = 0;
#pragma unroll
        for (int j = 0; j < kLayoutRankPer; ++j) {
            inc[j] = 0;
            const int64_t i = i0 + j;
            if (i < n && node_tree[i] == t) {
                const int4 nd = __ldg(nodes + i);
                inc[j] = kOne | (nd.x < 0 ? kLeafOne : ((uint32_t)nd.y >= 65536u ? kCatOne : 0ull));
            }
            v += inc[j];
        }
        unsigned long long total;
        unsigned long long pre = block_exclusive_scan_u64(v, sh, &total);
#pragma unroll
        for (int j = 0; j < kLayoutRankPer; ++j) {
            if (inc[j]) {
                const int64_t i = i0 + j;
                local[i] = (int32_t)(base_n + (pre & kField));
                ord[i] = (int32_t)((inc[j] & kLeafOne) ? base_l + ((pre >> 21) & kField)
                                                       : base_c + ((pre >> 42) & kField));
            }
            pre += inc[j];
        }
        base_n += total & kField; base_l += (total >> 21) & kField; base_c += (total >> 42) & kField;
    }
    if (threadIdx.x == 0) {
        cnt[3 * t] = (int32_t)base_n; cnt[3 * t + 1] = (int32_t)base_l; cnt[3 * t + 2] = (int32_t)base_c;
        const int64_t w = base_n + base_l * C + base_c * kLayoutCatWords;
        words[t] = (int32_t)((w + 1) & ~1ll);                                 // even: every tree block starts 16-byte aligned
    }
}

// one thread per pool node of trees [0, T): its node record, and its votes or categorical record
__global__ void __launch_bounds__(256) layout_fill_kernel(const int4* __restrict__ nodes,
                                                          const unsigned long long* __restrict__ node_mask,
                                                          const double* __restrict__ leaf_prob,
                                                          const uint32_t* __restrict__ pool_counts,
                                                          const int32_t* __restrict__ node_tree, int64_t n, int T, int C,
                                                          int dt_mode, const int32_t* __restrict__ local,
                                                          const int32_t* __restrict__ ord, const int32_t* __restrict__ cnt,
                                                          const int64_t* __restrict__ tree_off, uint2* layout) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int t = node_tree[i];
    if (t < 0 || t >= T) return;
    uint2* blk = layout + tree_off[t];
    const int4 nd = nodes[i];
    const uint32_t n_t = (uint32_t)cnt[3 * t], c_t = (uint32_t)cnt[3 * t + 2];
    uint2 rec;
    if (nd.x < 0) {
        const uint32_t vo = n_t + c_t * kLayoutCatWords + (uint32_t)ord[i] * (uint32_t)C;
        rec = make_uint2(kLayoutLeaf, vo);
        double* v = (double*)(blk + vo);
        if (dt_mode) { for (int k = 0; k < C; ++k) v[k] = (double)pool_counts[i * C + k]; }
        else { for (int k = 0; k < C; ++k) v[k] = leaf_prob[i * C + k]; }
    } else if ((uint32_t)nd.y >= 65536u) {
        const uint32_t co = n_t + (uint32_t)ord[i] * kLayoutCatWords;
        rec = make_uint2((uint32_t)nd.x | kLayoutCat, co);
        blk[co] = make_uint2((uint32_t)local[nd.z], 0u);
        unsigned long long* m = (unsigned long long*)(blk + co + 1);
        for (int q = 0; q < 4; ++q) m[q] = node_mask ? node_mask[i * 4 + q] : 0ull;
    } else {
        const uint32_t thr = (uint32_t)nd.y < 255u ? (uint32_t)nd.y : 255u;   // bins are bytes: a threshold >= 255 sends all left
        rec = make_uint2((uint32_t)nd.x | (thr << 16), (uint32_t)local[nd.z]);
    }
    blk[local[i]] = rec;
}

// A CTA owns a block of rows (one per thread; bins transposed in shared memory, word k of thread t at [k*blockDim + t],
// conflict-free) and walks them through the trees in order.  Tree t's block is staged with cp.async into one of two buffers while tree t-1 is walked; a
// word at offset o of the block is read from shared memory when o < cap (the buffer size) and from global memory otherwise,
// so a tree larger than the buffer keeps its first (top-level) nodes in shared memory.  A tree that fits is walked by the
// same code compiled without the bound check, which saves the compare and select on every load.  The last tree of a round
// stages tree 0 of the next.  Votes add in fp64, in tree order, from 0.0.
// kRegC > 0 (C <= kRegC): the votes accumulate in registers, not in shared memory: no shared-memory read-modify-write per
// class and leaf, and 8·C more bytes per row for the tree buffers (every KDD99 tree then fits).  The bin of feature f is one
// byte load from the thread's column: byte f & 3 of word f >> 2, at (f >> 2)·4·bd + (f & 3) = (f & ~3)·bd + (f & 3).
template <int kRegC>
__global__ void __launch_bounds__(kRegC ? kPredForestRegThreads : 1024, 1)
predict_forest_kernel(const uint8_t* __restrict__ tp, int stride, int fwords, int64_t n, const uint2* __restrict__ layout,
                      const int64_t* __restrict__ tree_off, int T, int C, int cap, double* raw, double* prob, double* pred) {
    extern __shared__ __align__(16) uint8_t sm[];
    const int bd = blockDim.x, tid = threadIdx.x;
    uint32_t* binw = (uint32_t*)sm;                                           // [fwords][bd]
    double* votes = (double*)(sm + (size_t)fwords * bd * 4);                  // [C][bd] (kRegC == 0)
    uint2* tbuf = (uint2*)(votes + (kRegC ? 0 : (size_t)C * bd));             // [2][cap]
    auto stage = [&](int t, int buf) {
        if (t >= 0) {
            const int64_t o = tree_off[t];
            const int64_t w = tree_off[t + 1] - o < cap ? tree_off[t + 1] - o : cap;
            const uint4* src = (const uint4*)(layout + o);
            uint4* dst = (uint4*)(tbuf + (size_t)buf * cap);
            for (int i = tid; i < (int)(w >> 1); i += bd) cp_async16(dst + i, src + i);
        }
        cp_async_commit();
    };
    const int64_t round_rows = (int64_t)gridDim.x * bd;
    const uint8_t* bb = (const uint8_t*)(binw + tid);                         // this thread's column of the transposed bins
    double* vt = votes + tid;
    int g = 0;                                                                // trees walked by this CTA: buffer parity
    if ((int64_t)blockIdx.x * bd < n) stage(0, 0);
    for (int64_t base = (int64_t)blockIdx.x * bd; base < n; base += round_rows) {
        const int64_t row = base + tid;
        const bool live = row < n;
        if (live) {
            const uint4* src = (const uint4*)(tp + row * stride);
            for (int q = 0; q < fwords / 4; ++q) {
                const uint4 v = ld_stream_u4(src + q);
                binw[(4 * q + 0) * bd + tid] = v.x; binw[(4 * q + 1) * bd + tid] = v.y;
                binw[(4 * q + 2) * bd + tid] = v.z; binw[(4 * q + 3) * bd + tid] = v.w;
            }
        }
        double acc[kRegC > 0 ? kRegC : 1];
#pragma unroll
        for (int k = 0; k < (kRegC > 0 ? kRegC : 1); ++k) acc[k] = 0.0;
        if (!kRegC) for (int k = 0; k < C; ++k) vt[k * bd] = 0.0;
        for (int t = 0; t < T; ++t, ++g) {
            cp_async_wait_all();
            __syncthreads();                                                // tree t landed; everybody left tree t-1
            stage(t + 1 < T ? t + 1 : (base + round_rows < n ? 0 : -1), (g + 1) & 1);
            const uint2* tb = tbuf + (size_t)(g & 1) * cap;
            const uint2* gb = layout + tree_off[t];
            const bool whole = tree_off[t + 1] - tree_off[t] <= cap;
            auto walk = [&](auto whole_tag) {
                constexpr bool kWhole = decltype(whole_tag)::value;
                auto word = [&](uint32_t o) -> uint2 { return (kWhole || o < (uint32_t)cap) ? tb[o] : __ldg(gb + o); };
                if (!live) return;
                uint2 nd = word(0);
                while (!(nd.x & kLayoutLeaf)) {
                    const uint32_t f = nd.x & 0xffff;
                    const uint32_t bin = bb[(f & ~3u) * bd + (f & 3u)];
                    uint32_t next;
                    if (nd.x & kLayoutCat) {
                        const uint2 m = word(nd.y + 1 + (bin >> 6));
                        next = word(nd.y).x + !((((bin & 32) ? m.y : m.x) >> (bin & 31)) & 1u);
                    } else {
                        next = nd.y + (bin > ((nd.x >> 16) & 0xff));
                    }
                    nd = word(next);
                }
                if (kRegC) {
#pragma unroll
                    for (int k = 0; k < kRegC; ++k)
                        if (k < C) { const uint2 w = word(nd.y + k); acc[k] += __hiloint2double((int)w.y, (int)w.x); }
                } else {
                    for (int k0 = 0; k0 < C; k0 += kVoteBatch) {                // the batch's loads issue before its adds
                        uint2 w[kVoteBatch];
#pragma unroll
                        for (int j = 0; j < kVoteBatch; ++j) if (k0 + j < C) w[j] = word(nd.y + k0 + j);
#pragma unroll
                        for (int j = 0; j < kVoteBatch; ++j)
                            if (k0 + j < C) vt[(k0 + j) * bd] += __hiloint2double((int)w[j].y, (int)w[j].x);
                    }
                }
            };
            if (whole) walk(std::integral_constant<bool, true>()); else walk(std::integral_constant<bool, false>());
        }
        if (!live) continue;
        if (kRegC) {
            double s = 0.0; int arg = 0; double best = acc[0];
#pragma unroll
            for (int k = 0; k < kRegC; ++k) if (k < C) { s += acc[k]; if (acc[k] > best) { best = acc[k]; arg = k; } }
#pragma unroll
            for (int k = 0; k < kRegC; ++k) if (k < C) {
                if (raw) raw[row * C + k] = acc[k];
                if (prob) prob[row * C + k] = s != 0.0 ? acc[k] / s : 0.0;
            }
            pred[row] = (double)arg;
        } else {
            double s = 0.0; int arg = 0; double best = vt[0];
            for (int k = 0; k < C; ++k) { const double v = vt[k * bd]; s += v; if (v > best) { best = v; arg = k; } }
            for (int k = 0; k < C; ++k) {
                const double v = vt[k * bd];
                if (raw) raw[row * C + k] = v;
                if (prob) prob[row * C + k] = s != 0.0 ? v / s : 0.0;
            }
            pred[row] = (double)arg;
        }
    }
    cp_async_wait_all();                                                    // nothing in flight when the CTA exits
}

// ------------------------------------------------------------------ row gather (predictions of unique records -> rows)
__global__ void __launch_bounds__(256) gather_rows_kernel(const uint32_t* __restrict__ src, int words, const int32_t* __restrict__ idx,
                                                          int64_t n, uint32_t* out) {
    const int64_t total = n * words;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = e / words; const int w = (int)(e - r * words);
        out[e] = __ldg(src + (int64_t)idx[r] * words + w);
    }
}

// ------------------------------------------------------------------ R10 confusion matrix
__global__ void __launch_bounds__(256) confusion_kernel(const double* __restrict__ pred, const double* __restrict__ label,
                                                        int64_t n, int C, unsigned long long* cm, int use_smem) {
    extern __shared__ uint32_t sh_cm[];
    if (use_smem) { for (int i = threadIdx.x; i < C * C; i += blockDim.x) sh_cm[i] = 0; __syncthreads(); }
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int l = (int)label[i], p = (int)pred[i];
        if (l >= 0 && l < C && p >= 0 && p < C) {
            if (use_smem) atomicAdd(&sh_cm[l * C + p], 1u); else atomicAdd(&cm[l * C + p], 1ull);
        }
    }
    if (use_smem) {
        __syncthreads();
        for (int i = threadIdx.x; i < C * C; i += blockDim.x) if (sh_cm[i]) atomicAdd(&cm[i], (unsigned long long)sh_cm[i]);
    }
}

// ------------------------------------------------------------------ grid prediction -> confusion matrices (model selection)
// For fixed other params, the forest fitted with (T, d) is the first T trees of the (T_max, d_max) forest cut at depth d
// (DESIGN.md §5a).  One thread owns one UNIQUE validation record (label at byte F, multiplicity mult[row]; its bins in
// transposed smem, word k of thread t at [k*blockDim + t]) and walks each tree once through the pool's 16-byte nodes, down
// to a leaf or to the deepest depth cut of this launch.  The node met at depth cut j (or the leaf the walk ended on above
// it) adds its payload to votes[j] in tree order, from 0.0: the fp64 adds of predicting with the truncated forest.  After
// tree T_i - 1 the first argmax of every votes[j] (the `v > best` rule of predict_forest_kernel) is counted into
// cm[i][j][label][pred].  A launch covers depth cuts [j0, j0 + jn) of J.
//
// What bounds the walk is the L1: below the first few levels every lane of a warp is at a different node, so each level
// costs 32 separate sector requests per warp.  The top `top_levels` levels of the CURRENT tree (2^K - 1 nodes,
// heap-indexed by MLlib's node id; build_top_kernel) are therefore staged in shared memory, double-buffered with cp.async
// one tree ahead: a scattered LDS.128 costs a handful of bank wavefronts instead of 32 tag lookups, and only the levels
// below K go to the L1/L2.

// top[tree][nid] = the tree's node with MLlib id nid, for nid < 2^K (entry 0 unused)
__global__ void __launch_bounds__(256) build_top_kernel(const int4* __restrict__ nodes, const int32_t* __restrict__ node_tree,
                                                        int64_t n_nodes, int K, int4* top) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_nodes) return;
    const int4 nd = nodes[i];
    if ((uint32_t)nd.w < (1u << K)) top[((int64_t)node_tree[i] << K) + nd.w] = nd;
}

constexpr int kGridMaxTreeCuts = 256;
constexpr int kGridMaxDepthCuts = 31;                 // depths 0..30
struct GridCuts { int32_t tree[kGridMaxTreeCuts]; int32_t depth[kGridMaxDepthCuts]; };

// kScores: instead of counting argmaxes, write votes[1] of every (tree cut, depth cut) to scores[i][j][row] — rawPrediction[1]
// of that truncated forest, the score BinaryClassificationEvaluator reads (mult and cm are not used).
template <bool kScores>
__global__ void __launch_bounds__(128) predict_grid_kernel(const uint8_t* __restrict__ tp, int stride, int F, int64_t n,
                                                           const int32_t* __restrict__ mult,
                                                           const b200flow_node* __restrict__ nodes,
                                                           const unsigned long long* __restrict__ node_mask,
                                                           const double* __restrict__ leaf_prob,
                                                           const uint32_t* __restrict__ pool_counts, int C, int dt_mode,
                                                           const int4* __restrict__ top, int K, const GridCuts cuts, int I,
                                                           int J, int j0, int jn, int L, unsigned long long* cm, int use_smem,
                                                           double* scores) {
    extern __shared__ __align__(16) uint8_t sm[];
    const int bd = blockDim.x, tid = threadIdx.x;
    const int words = stride / 4;
    uint32_t* binw = (uint32_t*)sm;                                           // [words][bd]
    double* votes = (double*)(sm + (size_t)words * bd * 4);                   // [jn][C][bd]
    const int topn = top ? (1 << K) : 0;
    int4* topbuf = (int4*)(votes + (size_t)jn * C * bd);                      // [2][topn] when the top table is given
    unsigned long long* sh_cm = (unsigned long long*)(topbuf + 2 * topn);     // [I][jn][L][L] when use_smem
    const int T = cuts.tree[I - 1];
    const int cm_cells = I * jn * L * L;
    if (use_smem) { for (int i = tid; i < cm_cells; i += bd) sh_cm[i] = 0ull; __syncthreads(); }
    auto stage_top = [&](int t, int buf) {
        if (t < T) for (int i = tid; i < topn; i += bd) cp_async16(topbuf + (size_t)buf * topn + i, top + ((int64_t)t << K) + i);
        cp_async_commit();
    };
    const int4* nodes4 = (const int4*)nodes;                                  // {feat, kind<<16|bin, left, nid}
    const uint32_t* bw = binw + tid;                                          // this thread's column of the transposed bins
    double* vt = votes + tid;
    for (int64_t base = (int64_t)blockIdx.x * bd; base < n; base += (int64_t)gridDim.x * bd) {
        const int64_t row = base + tid;
        const bool live = row < n;
        int lab = 0; unsigned long long w = 0;
        if (live) {
            const uint4* src = (const uint4*)(tp + row * stride);
            for (int q = 0; q < words / 4; ++q) {
                const uint4 v = ld_stream_u4(src + q);
                binw[(4 * q + 0) * bd + tid] = v.x; binw[(4 * q + 1) * bd + tid] = v.y;
                binw[(4 * q + 2) * bd + tid] = v.z; binw[(4 * q + 3) * bd + tid] = v.w;
            }
            if (!kScores) {
                lab = tp[row * stride + F];
                w = (unsigned long long)mult[row];
            }
        }
        for (int k = 0; k < jn * C; ++k) vt[(size_t)k * bd] = 0.0;
        if (top) stage_top(0, 0);
        int ic = 0;                                                           // next tree cut
        for (int t = 0; t < T; ++t) {
            const int4* tb = topbuf + (size_t)(t & 1) * topn;
            if (top) {
                cp_async_wait_all();
                __syncthreads();                                              // table of tree t landed; everybody left tree t-1
                stage_top(t + 1, (t + 1) & 1);
            }
            if (live) {
                int idx = t; uint32_t nid = 1u; int4 nd = top ? tb[1] : __ldg(nodes4 + t);
                int depth = 0, jj = 0;
                auto add = [&](int node, int j) {
                    double* v = vt + (size_t)j * C * bd;
                    if (dt_mode) { for (int k = 0; k < C; ++k) v[(size_t)k * bd] += (double)pool_counts[(int64_t)node * C + k]; }
                    else { for (int k = 0; k < C; ++k) v[(size_t)k * bd] += leaf_prob[(int64_t)node * C + k]; }
                };
                while (true) {
                    if (cuts.depth[j0 + jj] == depth) { add(idx, jj); ++jj; }  // cuts ascend: at most one per depth
                    if (jj == jn || nd.x < 0) break;
                    const int f = nd.x;
                    const int bin = (bw[(f >> 2) * bd] >> ((f & 3) * 8)) & 0xff;
                    const int right = nd.y < 65536 ? (bin > nd.y)
                                                    : !((node_mask[(int64_t)idx * 4 + (bin >> 6)] >> (bin & 63)) & 1ull);
                    idx = nd.z + right;
                    nid = 2u * nid + (uint32_t)right;
                    ++depth;
                    nd = nid < (uint32_t)topn ? tb[nid] : __ldg(nodes4 + idx);
                }
                for (; jj < jn; ++jj) add(idx, jj);                           // a leaf above the remaining cuts
            }
            if (t + 1 == cuts.tree[ic]) {
                if (kScores) {
                    if (live) {
                        double* out = scores + ((int64_t)ic * J + j0) * n + row;
                        for (int j = 0; j < jn; ++j) out[(int64_t)j * n] = vt[((size_t)j * C + 1) * bd];
                    }
                } else if (live && lab < L) {
                    for (int j = 0; j < jn; ++j) {
                        const double* v = vt + (size_t)j * C * bd;
                        int arg = 0; double best = v[0];
                        for (int k = 0; k < C; ++k) { const double x = v[(size_t)k * bd]; if (x > best) { best = x; arg = k; } }
                        const int64_t cell = (((int64_t)ic * jn + j) * L + lab) * L + arg;
                        if (use_smem) atomicAdd(&sh_cm[cell], w);
                        else atomicAdd(&cm[((((int64_t)ic * J + j0 + j) * L + lab) * L) + arg], w);
                    }
                }
                ++ic;
            }
        }
        if (top) { cp_async_wait_all(); __syncthreads(); }                  // the look-ahead copy of the last tree is a no-op commit
    }
    if (use_smem) {
        __syncthreads();
        for (int c = tid; c < cm_cells; c += bd) {
            const unsigned long long v = sh_cm[c];
            if (!v) continue;
            const int p = c % L, l = (c / L) % L, j = (c / (L * L)) % jn, i = c / (L * L * jn);
            atomicAdd(&cm[(((int64_t)i * J + j0 + j) * L + l) * L + p], v);
        }
    }
}

// ------------------------------------------------------------------ randomSplit
constexpr int kMaxSplits = 32;                     // randomSplit weights / CrossValidator folds
struct SplitBounds { double cum[kMaxSplits]; int n; };

__global__ void __launch_bounds__(256) random_split_kernel(uint64_t seed, int64_t row_offset, int64_t n, SplitBounds bnd,
                                                           uint8_t* out) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const uint64_t g = (uint64_t)(row_offset + i);
        const uint4 r = philox_keyed(seed, PURPOSE_RSPLIT, (uint32_t)g, (uint32_t)(g >> 32), 0u, 0u);
        const double u = (double)r.x * 2.3283064365386963e-10;     // 2^-32
        int k = 0;
        while (k < bnd.n - 1 && !(u < bnd.cum[k])) ++k;
        out[i] = (uint8_t)k;
    }
}

// ------------------------------------------------------------------ stable row compaction
constexpr int kCompactRows = 1024;

__global__ void __launch_bounds__(256) compact_count_kernel(const uint8_t* __restrict__ flag, int64_t n, int want, int32_t* blk_cnt) {
    __shared__ int cnt;
    if (threadIdx.x == 0) cnt = 0;
    __syncthreads();
    int c = 0;
    const int64_t rb = (int64_t)blockIdx.x * kCompactRows + threadIdx.x * 4;
#pragma unroll
    for (int k = 0; k < 4; ++k) if (rb + k < n && (flag[rb + k] != 0) == (want != 0)) ++c;
    c = warp_sum(c);
    if (lane_id() == 0 && c) atomicAdd(&cnt, c);
    __syncthreads();
    if (threadIdx.x == 0) blk_cnt[blockIdx.x] = cnt;
}

__global__ void __launch_bounds__(256) compact_scatter_kernel(const uint8_t* __restrict__ rows, int64_t n, int row_bytes,
                                                              const uint8_t* __restrict__ flag, int want,
                                                              const int64_t* __restrict__ blk_off, uint8_t* out) {
    __shared__ int sh[33];
    __shared__ int src_of[kCompactRows];                 // kept rows of this block, in order
    const int64_t rb0 = (int64_t)blockIdx.x * kCompactRows;
    const int64_t rb = rb0 + threadIdx.x * 4;
    int keep[4], c = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) { keep[k] = (rb + k < n && (flag[rb + k] != 0) == (want != 0)) ? 1 : 0; c += keep[k]; }
    int tot;
    int pos = block_exclusive_scan(c, sh, &tot);
#pragma unroll
    for (int k = 0; k < 4; ++k) if (keep[k]) src_of[pos++] = threadIdx.x * 4 + k;
    __syncthreads();
    const int words = row_bytes / 4;
    const uint32_t* src = (const uint32_t*)(rows + rb0 * row_bytes);
    uint32_t* dst = (uint32_t*)(out + blk_off[blockIdx.x] * row_bytes);
    for (int64_t i = threadIdx.x; i < (int64_t)tot * words; i += blockDim.x) {
        int r = (int)(i / words), wd = (int)(i - (int64_t)r * words);
        dst[i] = src[(int64_t)src_of[r] * words + wd];
    }
}

}  // namespace b200flow

using namespace b200flow;

extern "C" int b200flow_build_top_nodes(const b200flow_node* nodes, const int32_t* node_tree, int64_t n_nodes, int32_t T,
                                        int32_t top_levels, void* top, void* stream) {
    B2F_REQUIRE(nodes && node_tree && top && T > 0 && top_levels >= 1 && top_levels <= 10 && ((uintptr_t)top & 15) == 0, "build_top_nodes: bad arguments");
    if (n_nodes <= 0) return B200FLOW_OK;
    build_top_kernel<<<(unsigned)((n_nodes + 255) / 256), 256, 0, (cudaStream_t)stream>>>((const int4*)nodes, node_tree, n_nodes, top_levels, (int4*)top);
    return check_launch("build_top_nodes");
}

extern "C" int b200flow_forest_layout_size(const b200flow_node* nodes, const int32_t* node_tree, int64_t n_nodes, int32_t T,
                                           int32_t C, int32_t* scratch, int64_t* tree_off, void* stream) {
    B2F_REQUIRE(nodes && node_tree && scratch && tree_off && T > 0 && C > 0 && n_nodes >= T, "forest_layout_size: bad arguments");
    // every offset in a tree's block is 32-bit and the rank kernel counts at most 2^21 per chunk field: bound the words
    B2F_REQUIRE(n_nodes * ((int64_t)C + kLayoutCatWords + 1) < ((int64_t)1 << 31), "forest_layout_size: forest too large for 32-bit offsets");
    cudaStream_t st = (cudaStream_t)stream;
    int32_t* local = scratch; int32_t* ord = scratch + n_nodes; int32_t* cnt = ord + n_nodes; int32_t* words = cnt + 3 * (int64_t)T;
    layout_rank_kernel<<<T, kLayoutRankBlock, 0, st>>>((const int4*)nodes, node_tree, n_nodes, C, local, ord, cnt, words);
    const int rc = check_launch("forest_layout_size");
    if (rc) return rc;
    return b200flow_exclusive_scan_i32_to_i64(words, T, tree_off, tree_off + T, stream);
}

extern "C" int b200flow_build_forest_layout(const b200flow_node* nodes, const uint64_t* node_mask, const double* leaf_prob,
                                            const uint32_t* pool_counts, const int32_t* node_tree, int64_t n_nodes, int32_t T,
                                            int32_t C, int32_t dt_mode, const int32_t* scratch, const int64_t* tree_off,
                                            uint64_t* layout, void* stream) {
    B2F_REQUIRE(nodes && node_tree && scratch && tree_off && layout && T > 0 && C > 0 && n_nodes >= T && ((uintptr_t)layout & 15) == 0,
                "build_forest_layout: bad arguments");
    B2F_REQUIRE(dt_mode ? pool_counts != nullptr : leaf_prob != nullptr, "build_forest_layout: missing leaf payload");
    const int32_t* local = scratch; const int32_t* ord = scratch + n_nodes; const int32_t* cnt = ord + n_nodes;
    layout_fill_kernel<<<(unsigned)((n_nodes + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
        (const int4*)nodes, (const unsigned long long*)node_mask, leaf_prob, pool_counts, node_tree, n_nodes, T, C, dt_mode,
        local, ord, cnt, tree_off, (uint2*)layout);
    return check_launch("build_forest_layout");
}

// shared memory of predict_forest_kernel: the rows take at most half of kPredForestSmem, the two tree buffers the rest
constexpr size_t kPredForestSmem = 227 * 1024;              // the H100's opt-in maximum per CTA

extern "C" int b200flow_predict_forest(const uint8_t* tp, int32_t tp_stride, int32_t F, int64_t n_rows, const uint64_t* layout,
                                       const int64_t* tree_off, int32_t T, int32_t C, double* raw, double* prob, double* pred,
                                       void* stream) {
    if (n_rows <= 0) return B200FLOW_OK;            // empty batch: nothing to do (pointers may be NULL)
    B2F_REQUIRE(tp && layout && tree_off && pred && T > 0 && C > 0 && F > 0 && F < 65536 && F <= tp_stride && (tp_stride & 15) == 0,
                "predict_forest: bad arguments");
    B2F_REQUIRE(((uintptr_t)tp & 15) == 0 && ((uintptr_t)layout & 15) == 0, "predict_forest: tp and layout must be 16-byte aligned");
    const bool reg = C <= kPredForestRegC;          // votes in registers
    const int fwords = (F + 15) / 16 * 4;           // bin words a row keeps (whole 16-byte loads; <= tp_stride / 4)
    const size_t row_bytes = (size_t)fwords * 4 + (reg ? 0 : (size_t)C * 8);
    const int64_t max_bd = reg ? kPredForestRegThreads : 1024;
    int64_t bd = (int64_t)(kPredForestSmem / 2 / row_bytes) / 32 * 32;
    if (bd > max_bd) bd = max_bd;
    if (bd < 32) bd = 32;
    B2F_REQUIRE((size_t)bd * row_bytes + 16 <= kPredForestSmem, "predict_forest: too many classes/features for shared memory");
    // as few rounds as the widest block allows, with the rows spread evenly over them and the SMs
    const int64_t rounds = (n_rows + (int64_t)kNumSMs * bd - 1) / ((int64_t)kNumSMs * bd);
    const int64_t want = (n_rows + (int64_t)kNumSMs * rounds - 1) / ((int64_t)kNumSMs * rounds);
    bd = (want + 31) / 32 * 32 < bd ? (want + 31) / 32 * 32 : bd;
    const int grid = grid_for(n_rows, (int)bd, kNumSMs);
    const size_t rows_smem = (size_t)bd * row_bytes;
    const int cap = (int)((kPredForestSmem - rows_smem) / 16) & ~1;   // words per tree buffer, even
    const size_t smem = rows_smem + (size_t)2 * cap * 8;
    const void* fn = reg ? (const void*)predict_forest_kernel<kPredForestRegC> : (const void*)predict_forest_kernel<0>;
    cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) { set_error("predict_forest: %s", cudaGetErrorString(e)); return B200FLOW_ERR_CUDA; }
    if (reg) predict_forest_kernel<kPredForestRegC><<<grid, (int)bd, smem, (cudaStream_t)stream>>>(tp, tp_stride, fwords, n_rows,
                                                                  (const uint2*)layout, tree_off, T, C, cap, raw, prob, pred);
    else predict_forest_kernel<0><<<grid, (int)bd, smem, (cudaStream_t)stream>>>(tp, tp_stride, fwords, n_rows,
                                                                  (const uint2*)layout, tree_off, T, C, cap, raw, prob, pred);
    return check_launch("predict_forest");
}

extern "C" int b200flow_gather_rows(const void* src, int32_t row_bytes, const int32_t* idx, int64_t n_rows, void* out, void* stream) {
    if (n_rows <= 0) return B200FLOW_OK;
    B2F_REQUIRE(src && idx && out && row_bytes > 0 && (row_bytes & 3) == 0, "gather_rows: bad arguments");
    const int words = row_bytes / 4;
    gather_rows_kernel<<<grid_for(n_rows * words, 256 * 4, kNumSMs * 8), 256, 0, (cudaStream_t)stream>>>((const uint32_t*)src, words, idx, n_rows, (uint32_t*)out);
    return check_launch("gather_rows");
}

extern "C" int b200flow_confusion(const double* pred, const double* label, int64_t n_rows, int32_t C, int64_t* cm, void* stream) {
    if (n_rows <= 0) return B200FLOW_OK;            // empty batch: nothing to do (pointers may be NULL)
    B2F_REQUIRE(pred && label && cm && C > 0 && C <= 1024, "confusion: bad arguments");
    int use_smem = (size_t)C * C * 4 <= 64 * 1024;
    size_t smem = use_smem ? (size_t)C * C * 4 : 0;
    if (smem > 48 * 1024) cudaFuncSetAttribute(confusion_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    int grid = grid_for(n_rows, 256 * 8, kNumSMs * 4);
    confusion_kernel<<<grid, 256, smem, (cudaStream_t)stream>>>(pred, label, n_rows, C, (unsigned long long*)cm, use_smem);
    return check_launch("confusion");
}

// the launches of predict_grid_kernel<kScores> (confusion matrices, or scores) over the depth cuts
template <bool kScores>
static int predict_grid_launch(const char* what, const uint8_t* tp, int32_t tp_stride, int32_t F, int64_t n_rows, const int32_t* mult,
                               const b200flow_node* nodes, const uint64_t* node_mask, const double* leaf_prob,
                               const uint32_t* pool_counts, int32_t T, int32_t C, int32_t dt_mode,
                               const void* top_nodes, int32_t top_levels, const int32_t* tree_cuts_host,
                               int32_t n_tree_cuts, const int32_t* depth_cuts_host, int32_t n_depth_cuts,
                               int32_t cm_side, int32_t max_depth_cuts_per_launch, int64_t* cm, double* scores, void* stream) {
    const int I = n_tree_cuts, J = n_depth_cuts, L = cm_side;
    B2F_REQUIRE(tree_cuts_host && depth_cuts_host && I >= 1 && I <= kGridMaxTreeCuts && J >= 1 && J <= kGridMaxDepthCuts,
                "%s: 1..%d tree cuts and 1..%d depth cuts", what, kGridMaxTreeCuts, kGridMaxDepthCuts);
    GridCuts cuts;
    for (int i = 0; i < I; ++i) {
        B2F_REQUIRE(tree_cuts_host[i] >= 1 && tree_cuts_host[i] <= T && (i == 0 || tree_cuts_host[i] > tree_cuts_host[i - 1]),
                    "%s: tree cuts must ascend strictly within [1, %d]", what, T);
        cuts.tree[i] = tree_cuts_host[i];
    }
    for (int j = 0; j < J; ++j) {
        B2F_REQUIRE(depth_cuts_host[j] >= 0 && depth_cuts_host[j] <= 30 && (j == 0 || depth_cuts_host[j] > depth_cuts_host[j - 1]),
                    "%s: depth cuts must ascend strictly within [0, 30]", what);
        cuts.depth[j] = depth_cuts_host[j];
    }
    if (n_rows <= 0) return B200FLOW_OK;            // empty shard: nothing to count (pointers may be NULL)
    if (kScores) B2F_REQUIRE(tp && nodes && scores && T > 0 && C >= 2 && F >= 0 && F < tp_stride && (tp_stride & 15) == 0,
                             "predict_grid_scores: bad arguments (C >= 2: the score is votes[1])");
    else B2F_REQUIRE(tp && mult && nodes && cm && T > 0 && C > 0 && L >= C && F >= 0 && F < tp_stride && (tp_stride & 15) == 0,
                     "predict_grid_confusion: bad arguments");
    B2F_REQUIRE(dt_mode ? pool_counts != nullptr : leaf_prob != nullptr, "%s: missing leaf payload", what);
    B2F_REQUIRE(((uintptr_t)tp & 15) == 0, "%s: tp must be 16-byte aligned", what);
    B2F_REQUIRE(!top_nodes || (top_levels >= 1 && top_levels <= 10 && ((uintptr_t)top_nodes & 15) == 0),
                "%s: bad top table", what);
    // shared memory per launch: transposed bins + votes of jc depth cuts per thread, the top table, and the confusion
    // matrices of the launch when they fit as well.  The widest block that holds every depth cut is taken; when not even 32
    // threads hold them, the depth cuts are split over launches (each launch walks the trees again; counts do not change).
    const size_t kBudget = 200 * 1024;
    const size_t top_bytes = top_nodes ? (size_t)2 * 16 * ((size_t)1 << top_levels) : 0;
    const int want = max_depth_cuts_per_launch > 0 && max_depth_cuts_per_launch < J ? max_depth_cuts_per_launch : J;
    auto cuts_that_fit = [&](int bd) -> int {
        const size_t fixed = (size_t)bd * tp_stride + top_bytes;
        if (fixed >= kBudget) return 0;
        const size_t per_cut = (size_t)bd * C * 8;
        return (int)((kBudget - fixed) / per_cut < (size_t)want ? (kBudget - fixed) / per_cut : (size_t)want);
    };
    int bd = 128;
    while (bd > 32 && cuts_that_fit(bd) < want) bd >>= 1;
    const int jc = cuts_that_fit(bd);
    B2F_REQUIRE(jc >= 1, "%s: too many classes/features for shared memory", what);
    const int grid = grid_for(n_rows, bd, kNumSMs * 16);
    for (int j0 = 0; j0 < J; j0 += jc) {
        const int jn = J - j0 < jc ? J - j0 : jc;
        size_t smem = (size_t)bd * ((size_t)tp_stride + (size_t)jn * C * 8) + top_bytes;
        const size_t cm_bytes = kScores ? 0 : (size_t)I * jn * L * L * 8;
        const int use_smem = !kScores && smem + cm_bytes <= kBudget;
        if (use_smem) smem += cm_bytes;
        cudaError_t e = cudaFuncSetAttribute(predict_grid_kernel<kScores>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) { set_error("%s: %s", what, cudaGetErrorString(e)); return B200FLOW_ERR_CUDA; }
        predict_grid_kernel<kScores><<<grid, bd, smem, (cudaStream_t)stream>>>(tp, tp_stride, F, n_rows, mult, nodes,
                                                                               (const unsigned long long*)node_mask, leaf_prob,
                                                                               pool_counts, C, dt_mode, (const int4*)top_nodes,
                                                                               top_levels, cuts, I, J, j0, jn, L,
                                                                               (unsigned long long*)cm, use_smem, scores);
        const int rc = check_launch(what);
        if (rc) return rc;
    }
    return B200FLOW_OK;
}

extern "C" int b200flow_predict_grid_confusion(const uint8_t* tp, int32_t tp_stride, int32_t F, int64_t n_rows, const int32_t* mult,
                                               const b200flow_node* nodes, const uint64_t* node_mask, const double* leaf_prob,
                                               const uint32_t* pool_counts, int32_t T, int32_t C, int32_t dt_mode,
                                               const void* top_nodes, int32_t top_levels, const int32_t* tree_cuts_host,
                                               int32_t n_tree_cuts, const int32_t* depth_cuts_host, int32_t n_depth_cuts,
                                               int32_t cm_side, int32_t max_depth_cuts_per_launch, int64_t* cm, void* stream) {
    return predict_grid_launch<false>("predict_grid_confusion", tp, tp_stride, F, n_rows, mult, nodes, node_mask, leaf_prob,
                                      pool_counts, T, C, dt_mode, top_nodes, top_levels, tree_cuts_host, n_tree_cuts,
                                      depth_cuts_host, n_depth_cuts, cm_side, max_depth_cuts_per_launch, cm, nullptr, stream);
}

extern "C" int b200flow_predict_grid_scores(const uint8_t* tp, int32_t tp_stride, int32_t F, int64_t n_rows,
                                            const b200flow_node* nodes, const uint64_t* node_mask, const double* leaf_prob,
                                            const uint32_t* pool_counts, int32_t T, int32_t C, int32_t dt_mode,
                                            const void* top_nodes, int32_t top_levels, const int32_t* tree_cuts_host,
                                            int32_t n_tree_cuts, const int32_t* depth_cuts_host, int32_t n_depth_cuts,
                                            int32_t max_depth_cuts_per_launch, double* scores, void* stream) {
    return predict_grid_launch<true>("predict_grid_scores", tp, tp_stride, F, n_rows, nullptr, nodes, node_mask, leaf_prob,
                                     pool_counts, T, C, dt_mode, top_nodes, top_levels, tree_cuts_host, n_tree_cuts,
                                     depth_cuts_host, n_depth_cuts, C, max_depth_cuts_per_launch, nullptr, scores, stream);
}

extern "C" int b200flow_random_split(uint64_t seed, int64_t row_offset, int64_t n_rows, const double* cum_bounds_host,
                                     int32_t n_splits, uint8_t* split_id, void* stream) {
    if (n_rows <= 0) return B200FLOW_OK;            // empty batch: nothing to do (pointers may be NULL)
    B2F_REQUIRE(cum_bounds_host && split_id && n_splits >= 1 && n_splits <= kMaxSplits, "random_split: bad arguments");
    SplitBounds b; b.n = n_splits;
    for (int i = 0; i < kMaxSplits; ++i) b.cum[i] = i < n_splits ? cum_bounds_host[i] : 2.0;
    int grid = grid_for(n_rows, 256 * 4, kNumSMs * 8);
    random_split_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(seed, row_offset, n_rows, b, split_id);
    return check_launch("random_split");
}

extern "C" int b200flow_compact_rows(const void* rows, int64_t n_rows, int32_t row_bytes, const uint8_t* flag, int32_t want,
                                     void* out_rows, int64_t* scratch, int64_t* n_kept, void* stream) {
    B2F_REQUIRE(rows && flag && out_rows && scratch && n_kept && row_bytes > 0 && (row_bytes & 3) == 0, "compact_rows: bad arguments");
    B2F_REQUIRE(((uintptr_t)rows & 3) == 0 && ((uintptr_t)out_rows & 3) == 0, "compact_rows: buffers must be 4-byte aligned");
    if (n_rows <= 0) { cudaMemsetAsync(n_kept, 0, 8, (cudaStream_t)stream); return check_launch("compact_rows"); }
    const int64_t nb = (n_rows + kCompactRows - 1) / kCompactRows;
    // scratch: int64 off[nb+1] first (8-aligned), then int32 cnt[nb]
    int64_t* off = scratch;
    int32_t* cnt = (int32_t*)(scratch + nb + 1);
    compact_count_kernel<<<(unsigned)nb, 256, 0, (cudaStream_t)stream>>>(flag, n_rows, want, cnt);
    int rc = b200flow_exclusive_scan_i32_to_i64(cnt, nb, off, n_kept, stream);
    if (rc) return rc;
    compact_scatter_kernel<<<(unsigned)nb, 256, 0, (cudaStream_t)stream>>>((const uint8_t*)rows, n_rows, row_bytes, flag, want, off, (uint8_t*)out_rows);
    return check_launch("compact_rows");
}
