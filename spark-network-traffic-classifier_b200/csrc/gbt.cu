// gbt.cu — GBTClassifier (binary, LogLoss) on the device, DESIGN.md §5e: the regression-tree level loop's variance
// histograms and split scoring, the leaf values, and the per-iteration margin / residual update.
//
// Residuals live on a fixed-point grid: record u carries q_u = rint(r_u 2^S) and q2_u = rint((q_u 2^-S)^2 2^S2) (int64,
// S = 60 - ceil(log2 n), S2 = 58 - ceil(log2 n)), so every histogram cell {Σw, Σw·q, Σw·q2} is an exact int64 sum below 2^62:
// the all-reduce over ranks, the shared- and global-memory atomics and the order of the entries cannot change a bit.
// The tree structure reuses the forest's: b200flow_split records, b200flow_partition_level, b200flow_next_segments,
// b200flow_grow_level (the three int64 stats travel as 6 opaque words per node) and b200flow_predict_forest (C = 1
// over the payloads).  OneVsRest(GBTClassifier) grows the K binary problems' trees side by side (DESIGN.md §5f): the _classes entry
// points read each slot's residuals from its class's block and update every (class, record) pair.  Compiled with -fmad=false: every fp64 expression below is restated operation for operation by the test oracle.
#include <float.h>

#include "common.cuh"
#include "portable_exp.h"
#include "tree_walk.cuh"

namespace b200flow {

constexpr int kGbtHistThreads = 256;
constexpr size_t kGbtHistSmem = 112 * 1024;          // per CTA: two CTAs (16 warps) per SM
constexpr int kGbtScoreThreads = 128;
constexpr double kGbtEpsilon = 2.220446049250313e-16; // MLUtils.EPSILON (2^-52): a child this pure is a leaf

// ------------------------------------------------------------------ variance histograms (the hot loop)
// One CTA per chunk of one slot's entries (the chunk table of hist_level).  Each entry's record, q and q2 are gathered once
// per feature pass, and every subset feature of the pass adds {w, w·q, w·q2} to the slot's shared-memory histogram with
// 64-bit shared atomics; the histogram is flushed with sparse global REDs.  Wide nodes go in feature passes of m_pass.
// kClasses (OneVsRest, DESIGN.md §5f): the residuals are rq [K][class_rows] and slot s reads the block of its class
// slot_class[s]; the records and entries are the ones all classes share.  The binary instantiation ignores both arguments,
// which come last so that its parameter layout and SASS are those of the kernel before classes existed.
template <bool kClasses>
__global__ void __launch_bounds__(kGbtHistThreads, 2) gbt_hist_level_kernel(
    const uint8_t* __restrict__ tp, int stride, const b2f_entry* __restrict__ ent, const longlong2* __restrict__ rq, int n_slots,
    const int64_t* __restrict__ seg_begin, const int64_t* __restrict__ seg_end, const int64_t* __restrict__ chunk_off,
    int chunk_rows, const uint16_t* __restrict__ subset, int m, int n_bins, int m_pass, unsigned long long* hist,
    const int32_t* __restrict__ slot_class, int64_t class_rows) {
    extern __shared__ unsigned long long sh_h[];        // [m_pass][n_bins][3]
    __shared__ int sh_feat[256];
    const int64_t c = blockIdx.x;
    const int s = find_slot(chunk_off, n_slots, c);
    if (kClasses) rq += (int64_t)slot_class[s] * class_rows;
    const int64_t b = seg_begin[s] + (c - chunk_off[s]) * chunk_rows;
    const int64_t e = min(seg_end[s], b + chunk_rows);
    const int nb3 = n_bins * 3;
    for (int j = threadIdx.x; j < m; j += blockDim.x) sh_feat[j] = subset[(int64_t)s * m + j];
    unsigned long long* gh = hist + (int64_t)s * m * nb3;
    for (int j0 = 0; j0 < m; j0 += m_pass) {
        const int mp = min(m_pass, m - j0);
        const int hsz = mp * nb3;
        __syncthreads();
        for (int i = threadIdx.x; i < hsz; i += blockDim.x) sh_h[i] = 0ull;
        __syncthreads();
        for (int64_t i = b + threadIdx.x; i < e; i += blockDim.x) {
            const b2f_entry en = ent[i];
            const longlong2 v = __ldg(rq + en.x);
            const unsigned long long w = en.y;
            const unsigned long long wq = w * (unsigned long long)v.x, wq2 = w * (unsigned long long)v.y;   // two's complement
            const uint8_t* rec = tp + (int64_t)en.x * stride;
            for (int j = 0; j < mp; ++j) {
                unsigned long long* cell = sh_h + (j * n_bins + rec[sh_feat[j0 + j]]) * 3;
                atomicAdd(cell, w); atomicAdd(cell + 1, wq); atomicAdd(cell + 2, wq2);
            }
        }
        __syncthreads();
        for (int i = threadIdx.x; i < hsz; i += blockDim.x) {
            const unsigned long long v = sh_h[i];
            if (v) atomicAdd(gh + (int64_t)j0 * nb3 + i, v);
        }
    }
}

// ------------------------------------------------------------------ split scoring (Variance)
struct GbtScale { double s1, s2; };                    // 2^-S, 2^-S2

// shared-memory bytes of one scoring warp: {raw, cum} int64 [n_bins][3], centroids f64 [n_bins], order int32 [n_bins];
// rounded up to 16 bytes so that every warp's int64 block stays 8-byte aligned for odd n_bins
__host__ __device__ __forceinline__ size_t gbt_score_per_warp(int n_bins) { return ((size_t)n_bins * (24 + 24 + 8 + 4) + 15) & ~(size_t)15; }

// Variance.calculate(count, sum, sumSq): (sumSq - sum * sum / count) / count, 0 for an empty side
__device__ __forceinline__ double gbt_variance(long long w, long long wq, long long wq2, GbtScale sc) {
    const double cnt = (double)w;
    if (cnt == 0.0) return 0.0;
    const double sum = (double)wq * sc.s1, sq = (double)wq2 * sc.s2;
    return (sq - sum * sum / cnt) / cnt;
}

// calculateImpurityStats: -DBL_MAX marks an invalid split (minInstancesPerNode / minInfoGain)
__device__ __forceinline__ double gbt_gain(const long long* L, const long long* tot, double parent_imp, GbtScale sc,
                                           int min_inst, double min_gain) {
    const double lc = (double)L[0], rc = (double)(tot[0] - L[0]);
    if (lc < (double)min_inst || rc < (double)min_inst) return -DBL_MAX;
    const double il = gbt_variance(L[0], L[1], L[2], sc);
    const double ir = gbt_variance(tot[0] - L[0], tot[1] - L[1], tot[2] - L[2], sc);
    const double t = lc + rc;
    const double lw = lc / t, rw = rc / t;
    const double g = parent_imp - lw * il - rw * ir;
    return g < min_gain ? -DBL_MAX : g;
}

// One CTA per slot, one warp per subset feature: the bins (continuous: in bin order; categorical: stably sorted by
// centroid sum / count, empty categories last) are prefix-summed in int64 by three lanes, then the warp scores the
// nb - 1 candidate splits.  The winner is the first maximum under (gain desc, feature position asc, split asc) — MLlib's
// maxBy over splits, then over features.
__global__ void __launch_bounds__(kGbtScoreThreads) gbt_score_level_kernel(
    const long long* __restrict__ hist, const uint16_t* __restrict__ subset, int m, int n_bins,
    const int32_t* __restrict__ feat_bins, const int32_t* __restrict__ feat_kind, GbtScale sc, int level, int max_depth,
    int min_inst, double min_gain, b200flow_split* split, long long* node_stats, long long* left_stats, long long* right_stats) {
    extern __shared__ __align__(8) uint8_t sm_raw[];
    constexpr int NW = kGbtScoreThreads / 32;
    const int s = blockIdx.x, tid = threadIdx.x, w = warp_id(), lane = lane_id();
    const int nb3 = n_bins * 3;
    const size_t per_warp = gbt_score_per_warp(n_bins);
    uint8_t* wb = sm_raw + per_warp * w;
    long long* raw = (long long*)wb;                   // [n_bins][3] this feature's cells
    long long* cum = raw + nb3;                        // [n_bins][3] prefix sums in split order
    double* cen = (double*)(cum + nb3);                // [n_bins]
    int* order = (int*)(cen + n_bins);                 // [n_bins] category at each rank
    __shared__ long long tot[3];
    __shared__ double sh_g[NW];
    __shared__ int sh_j[NW], sh_s[NW], sh_kind[NW];
    __shared__ long long sh_L[NW][3];
    __shared__ unsigned long long sh_mask[NW][4];

    const long long* h0 = hist + (int64_t)s * m * nb3;
    if (tid < 3) { long long a = 0; for (int b = 0; b < n_bins; ++b) a += h0[b * 3 + tid]; tot[tid] = a; }
    __syncthreads();
    const double parent_imp = gbt_variance(tot[0], tot[1], tot[2], sc);

    double wg = -DBL_MAX; int wj = -1, wsp = -1;       // this warp's best so far (lane 0's copy is authoritative)
    for (int jj = w; jj < m; jj += NW) {
        const int f = subset[(int64_t)s * m + jj];
        const int nb = feat_bins[f], cat = feat_kind[f] != 0;
        for (int i = lane; i < nb * 3; i += 32) raw[i] = h0[(int64_t)jj * nb3 + i];
        __syncwarp();
        if (cat) {
            for (int c = lane; c < nb; c += 32) {
                const long long cnt = raw[c * 3];
                cen[c] = cnt == 0 ? DBL_MAX : ((double)raw[c * 3 + 1] * sc.s1) / (double)cnt;
            }
            __syncwarp();
            for (int c = lane; c < nb; c += 32) {      // stable rank by centroid
                const double ce = cen[c]; int rk = 0;
                for (int c2 = 0; c2 < nb; ++c2) { const double o = cen[c2]; rk += (o < ce || (o == ce && c2 < c)) ? 1 : 0; }
                order[rk] = c;
            }
        } else {
            for (int c = lane; c < nb; c += 32) order[c] = c;
        }
        __syncwarp();
        if (lane < 3) { long long a = 0; for (int i = 0; i < nb; ++i) { a += raw[order[i] * 3 + lane]; cum[i * 3 + lane] = a; } }
        __syncwarp();
        double g = -DBL_MAX; int sp_best = -1;
        for (int sp = lane; sp < nb - 1; sp += 32) {
            const double gg = gbt_gain(cum + sp * 3, tot, parent_imp, sc, min_inst, min_gain);
            if (gg != -DBL_MAX && (sp_best < 0 || gg > g)) { g = gg; sp_best = sp; }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const double og = __shfl_xor_sync(0xffffffffu, g, o); const int os = __shfl_xor_sync(0xffffffffu, sp_best, o);
            if (os >= 0 && (sp_best < 0 || og > g || (og == g && os < sp_best))) { g = og; sp_best = os; }
        }
        if (lane == 0 && sp_best >= 0 && (wj < 0 || g > wg)) {   // features ascend within a warp: ties keep the earlier one
            wg = g; wj = jj; wsp = sp_best;
            sh_kind[w] = cat;
            for (int k = 0; k < 3; ++k) sh_L[w][k] = cum[sp_best * 3 + k];
            unsigned long long mk[4] = {0ull, 0ull, 0ull, 0ull};
            if (cat) for (int i = 0; i <= sp_best; ++i) { const int c = order[i]; mk[c >> 6] |= 1ull << (c & 63); }
            for (int q = 0; q < 4; ++q) sh_mask[w][q] = mk[q];
        }
        __syncwarp();
    }
    if (lane == 0) { sh_g[w] = wg; sh_j[w] = wj; sh_s[w] = wsp; }
    __syncthreads();
    if (tid != 0) return;
    int bw = -1;
    for (int q = 0; q < NW; ++q) {
        if (sh_j[q] < 0) continue;
        if (bw < 0 || sh_g[q] > sh_g[bw] || (sh_g[q] == sh_g[bw] && sh_j[q] < sh_j[bw])) bw = q;
    }
    const bool has = bw >= 0;
    const double bg = has ? sh_g[bw] : -DBL_MAX;
    long long L[3] = {0, 0, 0};
    if (has) for (int k = 0; k < 3; ++k) L[k] = sh_L[bw][k];
    for (int k = 0; k < 3; ++k) {
        node_stats[(int64_t)s * 3 + k] = tot[k];
        left_stats[(int64_t)s * 3 + k] = L[k];
        right_stats[(int64_t)s * 3 + k] = has ? tot[k] - L[k] : 0;
    }
    b200flow_split o;
    o.gain = bg; o.impurity = parent_imp;
    const bool leaf = !(has && bg > 0.0) || level >= max_depth;
    int flags = leaf ? 1 : 0;
    o.feat = -1; o.kind = 0; o.bin_thr = 0;
    o.mask[0] = o.mask[1] = o.mask[2] = o.mask[3] = 0;
    if (!leaf) {
        o.feat = subset[(int64_t)s * m + sh_j[bw]]; o.kind = sh_kind[bw]; o.bin_thr = sh_s[bw];
        for (int q = 0; q < 4; ++q) o.mask[q] = sh_mask[bw][q];
        const double il = gbt_variance(L[0], L[1], L[2], sc), ir = gbt_variance(tot[0] - L[0], tot[1] - L[1], tot[2] - L[2], sc);
        if (level + 1 == max_depth || fabs(il) < kGbtEpsilon) flags |= 2;
        if (level + 1 == max_depth || fabs(ir) < kGbtEpsilon) flags |= 4;
    }
    o.flags = flags;
    split[s] = o;
}

// ------------------------------------------------------------------ leaf values, margin and residual update
// payload[i] = tree_weight[tree of i] * (sum / count) of node i's stats (LeafNode prediction x tree weight)
__global__ void gbt_leaf_values_kernel(int64_t n_nodes, const long long* __restrict__ stats, const int32_t* __restrict__ node_tree,
                                       const double* __restrict__ tree_weight, GbtScale sc, double* payload) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_nodes) return;
    payload[i] = tree_weight[node_tree[i]] * (((double)stats[3 * i + 1] * sc.s1) / (double)stats[3 * i]);
}

// r -> {q, q2} on the fixed-point grid
__device__ __forceinline__ longlong2 gbt_grid(double r, int S, int S2) {
    const long long q = __double2ll_rn(r * pexp_pow2(S));
    const double rh = (double)q * pexp_pow2(-S);
    return make_longlong2(q, __double2ll_rn(rh * rh * pexp_pow2(S2)));
}

// root < 0: F = +0.0 and the targets of tree 0 (r = y itself).  root >= 0: walk the tree whose root is pool node `root`,
// F += its payload, then r = -LogLoss.gradient = 4y / (1 + exp(2yF)), y = 2 label - 1.  A NaN margin (only reachable through
// an empty tree, whose leaf value is 0/0) gives r = 0, so that q stays defined.
__device__ __forceinline__ void gbt_update_record(const uint8_t* rec, double y, const int4* __restrict__ nodes,
                                                  const unsigned long long* __restrict__ node_mask,
                                                  const double* __restrict__ payload, int root, int S, int S2, double* margin,
                                                  longlong2* rq) {
    if (root < 0) {
        *margin = 0.0;
        *rq = gbt_grid(y, S, S2);
        return;
    }
    const int idx = variance_tree_leaf(rec, nodes, node_mask, root);
    const double Fm = *margin + payload[idx];
    *margin = Fm;
    double r = 4.0 * y / (1.0 + portable_exp(2.0 * y * Fm));
    if (r != r) r = 0.0;
    *rq = gbt_grid(r, S, S2);
}

__global__ void gbt_update_kernel(const uint8_t* __restrict__ tp, int stride, int F, int64_t n, const int4* __restrict__ nodes,
                                  const unsigned long long* __restrict__ node_mask, const double* __restrict__ payload, int tree,
                                  int S, int S2, double* margin, longlong2* rq) {
    const int64_t u = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= n) return;
    const uint8_t* rec = tp + u * stride;
    gbt_update_record(rec, rec[F] ? 1.0 : -1.0, nodes, node_mask, payload, tree, S, S2, margin + u, rq + u);
}

// OneVsRest: thread i = (class k, record u), k = i / n.  Class k's tree of iteration `tree` is pool node k T + tree, its
// label is (label == k), and margin / rq are [K][n]: the operations of gbt_update_kernel on the relabelled record.
__global__ void gbt_update_classes_kernel(const uint8_t* __restrict__ tp, int stride, int F, int64_t n, int K,
                                          const int4* __restrict__ nodes, const unsigned long long* __restrict__ node_mask,
                                          const double* __restrict__ payload, int tree, int T, int S, int S2, double* margin,
                                          longlong2* rq) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n * K) return;
    const int k = (int)(i / n);
    const uint8_t* rec = tp + (i - (int64_t)k * n) * stride;
    gbt_update_record(rec, rec[F] == k ? 1.0 : -1.0, nodes, node_mask, payload, tree < 0 ? -1 : k * T + tree, S, S2, margin + i,
                      rq + i);
}

// GBTClassificationModel output: raw = [-F, F], probability[0] = 1 / (1 + exp(-2 raw[0])), probability[1] = 1 - that,
// prediction = F > 0
__global__ void gbt_output_kernel(const double* __restrict__ margin, int64_t n, double* raw, double* prob, double* pred) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double Fm = margin[i];
    const double r0 = -Fm;
    if (raw) { raw[2 * i] = r0; raw[2 * i + 1] = Fm; }
    if (prob) { const double p0 = 1.0 / (1.0 + portable_exp(-2.0 * r0)); prob[2 * i] = p0; prob[2 * i + 1] = 1.0 - p0; }
    if (pred) pred[i] = Fm > 0.0 ? 1.0 : 0.0;
}

static GbtScale gbt_scale(int S, int S2) { GbtScale sc; sc.s1 = ldexp(1.0, -S); sc.s2 = ldexp(1.0, -S2); return sc; }

}  // namespace b200flow

using namespace b200flow;

template <bool kClasses>
static int gbt_hist_level_launch(const char* name, const uint8_t* tp, int32_t tp_stride, const void* ent, const int64_t* rq,
                                 const int32_t* slot_class, int64_t class_rows, int32_t n_slots, const int64_t* seg_begin,
                                 const int64_t* seg_end, const int64_t* chunk_off, int64_t n_chunks, int32_t chunk_rows,
                                 const uint16_t* subset, int32_t m, int32_t n_bins, int64_t* hist, void* stream) {
    B2F_REQUIRE(tp && ent && rq && seg_begin && seg_end && chunk_off && subset && hist, "%s: null pointer", name);
    B2F_REQUIRE(m > 0 && m <= 256 && n_bins > 0 && n_bins <= 256 && chunk_rows > 0, "%s: bad shape", name);
    B2F_REQUIRE(((uintptr_t)rq & 15) == 0, "%s: rq must be 16-byte aligned", name);
    const size_t per_feat = (size_t)n_bins * 24;
    int m_pass = (int)(kGbtHistSmem / per_feat);
    if (m_pass > m) m_pass = m;
    const size_t smem = per_feat * m_pass;
    if (n_slots <= 0 || n_chunks <= 0) return B200FLOW_OK;
    B2F_REQUIRE(n_chunks < ((int64_t)1 << 31), "%s: too many chunks", name);
    cudaError_t e = cudaFuncSetAttribute(gbt_hist_level_kernel<kClasses>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) { (void)cudaGetLastError(); set_error("%s: %s", name, cudaGetErrorString(e)); return B200FLOW_ERR_CUDA; }
    gbt_hist_level_kernel<kClasses><<<(unsigned)n_chunks, kGbtHistThreads, smem, (cudaStream_t)stream>>>(
        tp, tp_stride, (const b2f_entry*)ent, (const longlong2*)rq, n_slots, seg_begin, seg_end, chunk_off, chunk_rows, subset, m,
        n_bins, m_pass, (unsigned long long*)hist, slot_class, class_rows);
    return check_launch(name);
}

extern "C" int b200flow_gbt_hist_level(const uint8_t* tp, int32_t tp_stride, const void* ent, const int64_t* rq, int32_t n_slots,
                                       const int64_t* seg_begin, const int64_t* seg_end, const int64_t* chunk_off, int64_t n_chunks,
                                       int32_t chunk_rows, const uint16_t* subset, int32_t m, int32_t n_bins, int64_t* hist,
                                       void* stream) {
    return gbt_hist_level_launch<false>("gbt_hist_level", tp, tp_stride, ent, rq, nullptr, 0, n_slots, seg_begin, seg_end,
                                        chunk_off, n_chunks, chunk_rows, subset, m, n_bins, hist, stream);
}

extern "C" int b200flow_gbt_hist_level_classes(const uint8_t* tp, int32_t tp_stride, const void* ent, const int64_t* rq,
                                               int64_t class_rows, const int32_t* slot_class, int32_t n_slots,
                                               const int64_t* seg_begin, const int64_t* seg_end, const int64_t* chunk_off,
                                               int64_t n_chunks, int32_t chunk_rows, const uint16_t* subset, int32_t m,
                                               int32_t n_bins, int64_t* hist, void* stream) {
    B2F_REQUIRE(slot_class && class_rows >= 0, "gbt_hist_level_classes: bad class table");
    return gbt_hist_level_launch<true>("gbt_hist_level_classes", tp, tp_stride, ent, rq, slot_class, class_rows, n_slots,
                                       seg_begin, seg_end, chunk_off, n_chunks, chunk_rows, subset, m, n_bins, hist, stream);
}

extern "C" int b200flow_gbt_score_level(const int64_t* hist, int32_t n_slots, const uint16_t* subset, int32_t m, int32_t n_bins,
                                        const int32_t* feat_bins, const int32_t* feat_kind, int32_t S, int32_t S2, int32_t level,
                                        int32_t max_depth, int32_t min_instances, double min_info_gain, b200flow_split* split,
                                        int64_t* node_stats, int64_t* left_stats, int64_t* right_stats, void* stream) {
    B2F_REQUIRE(hist && subset && feat_bins && feat_kind && split && node_stats && left_stats && right_stats, "gbt_score_level: null pointer");
    B2F_REQUIRE(m > 0 && n_bins > 0 && n_bins <= 256 && S > -1000 && S < 1000 && S2 > -1000 && S2 < 1000, "gbt_score_level: bad shape");
    if (n_slots <= 0) return B200FLOW_OK;
    const size_t smem = gbt_score_per_warp(n_bins) * (kGbtScoreThreads / 32);
    cudaError_t e = cudaFuncSetAttribute(gbt_score_level_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) { (void)cudaGetLastError(); set_error("gbt_score_level: %s", cudaGetErrorString(e)); return B200FLOW_ERR_CUDA; }
    gbt_score_level_kernel<<<n_slots, kGbtScoreThreads, smem, (cudaStream_t)stream>>>(
        (const long long*)hist, subset, m, n_bins, feat_bins, feat_kind, gbt_scale(S, S2), level, max_depth, min_instances,
        min_info_gain, split, (long long*)node_stats, (long long*)left_stats, (long long*)right_stats);
    return check_launch("gbt_score_level");
}

extern "C" int b200flow_gbt_leaf_values(int64_t n_nodes, const int64_t* stats, const int32_t* node_tree, const double* tree_weight,
                                        int32_t S, double* payload, void* stream) {
    B2F_REQUIRE(stats && node_tree && tree_weight && payload, "gbt_leaf_values: null pointer");
    if (n_nodes <= 0) return B200FLOW_OK;
    gbt_leaf_values_kernel<<<(unsigned)((n_nodes + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
        n_nodes, (const long long*)stats, node_tree, tree_weight, gbt_scale(S, S), payload);
    return check_launch("gbt_leaf_values");
}

extern "C" int b200flow_gbt_update(const uint8_t* tp, int32_t tp_stride, int32_t F, int64_t n_rows, const b200flow_node* nodes,
                                   const uint64_t* node_mask, const double* payload, int32_t tree, int32_t S, int32_t S2,
                                   double* margin, int64_t* rq, void* stream) {
    B2F_REQUIRE(tp && margin && rq && (tree < 0 || (nodes && payload)), "gbt_update: null pointer");
    B2F_REQUIRE(((uintptr_t)rq & 15) == 0, "gbt_update: rq must be 16-byte aligned");
    if (n_rows <= 0) return B200FLOW_OK;
    gbt_update_kernel<<<(unsigned)((n_rows + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
        tp, tp_stride, F, n_rows, (const int4*)nodes, (const unsigned long long*)node_mask, payload, tree, S, S2, margin, (longlong2*)rq);
    return check_launch("gbt_update");
}

extern "C" int b200flow_gbt_update_classes(const uint8_t* tp, int32_t tp_stride, int32_t F, int64_t n_rows, int32_t n_classes,
                                           const b200flow_node* nodes, const uint64_t* node_mask, const double* payload,
                                           int32_t tree, int32_t n_iter, int32_t S, int32_t S2, double* margin, int64_t* rq,
                                           void* stream) {
    B2F_REQUIRE(tp && margin && rq && (tree < 0 || (nodes && payload)), "gbt_update_classes: null pointer");
    B2F_REQUIRE(n_classes >= 1 && n_classes <= 256 && (tree < 0 || tree < n_iter), "gbt_update_classes: bad shape");
    B2F_REQUIRE(((uintptr_t)rq & 15) == 0, "gbt_update_classes: rq must be 16-byte aligned");
    if (n_rows <= 0) return B200FLOW_OK;
    const int64_t total = n_rows * n_classes;
    gbt_update_classes_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
        tp, tp_stride, F, n_rows, n_classes, (const int4*)nodes, (const unsigned long long*)node_mask, payload, tree, n_iter, S, S2,
        margin, (longlong2*)rq);
    return check_launch("gbt_update_classes");
}

extern "C" int b200flow_gbt_output(const double* margin, int64_t n_rows, double* raw, double* prob, double* pred, void* stream) {
    B2F_REQUIRE(margin, "gbt_output: null pointer");
    if (n_rows <= 0) return B200FLOW_OK;
    gbt_output_kernel<<<(unsigned)((n_rows + 255) / 256), 256, 0, (cudaStream_t)stream>>>(margin, n_rows, raw, prob, pred);
    return check_launch("gbt_output");
}
