// forest.cu — the RandomForest level loop (SURVEY.md §8a R7, R7r, R8): per-node per-feature
// integer histograms (HOT LOOP A), Gini split scoring (HOT LOOP B), pool growth and row routing.
// Reference call sites: classifiers[c].fit(train_set) kdd99.py:79 / cicids17.py:83; upstream
// algorithm: ml/tree/impl/RandomForest.scala findBestSplits/binsToBestSplit (restated in A.5).
//
// Data layout in HBM
//   tp        [n_rows][stride] uint8   TreePoint: bin per feature, label at byte F (row = 3..5 x 16 B)
//   ent_row/w [E] int32/uint8          bagged entries of all trees; a node owns a contiguous segment
//   hist      [slots][m][n_bins][C] uint32   exact integer counts (weights are integer Poisson draws)
// The row -> node relation is kept by PARTITIONING the entry array level by level (no per-row tree
// walk as in MLlib); histograms are accumulated in shared memory per (node, chunk) and flushed
// with sparse global REDs, so the multi-GPU all-reduce sees one dense uint32 buffer per level.
#include <float.h>
#include <stdlib.h>

#include "common.cuh"

namespace b200flow {

// ------------------------------------------------------------------ feature subsets
constexpr int kMaxSubset = 128;

__global__ void __launch_bounds__(128) feature_subsets_kernel(uint64_t seed, int n_slots, const int32_t* __restrict__ slot_tree,
                                                              const uint32_t* __restrict__ slot_nid, int F, int m,
                                                              uint16_t* subset) {
    int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_slots) return;
    uint16_t* out = subset + (int64_t)s * m;
    if (m >= F) { for (int i = 0; i < F; ++i) out[i] = (uint16_t)i; return; }
    // virtual partial Fisher-Yates: only touched positions are materialised (pos[], val[])
    uint16_t pos[kMaxSubset], val[kMaxSubset], pick[kMaxSubset];
    int nt = 0;
    const int tree = slot_tree[s]; const uint32_t nid = slot_nid[s];
    uint4 r = make_uint4(0, 0, 0, 0);
    for (int i = 0; i < m; ++i) {
        if ((i & 3) == 0) r = philox_keyed(seed, PURPOSE_FEAT, (uint32_t)tree, nid, (uint32_t)(i >> 2), 0u);
        uint32_t w = (i & 3) == 0 ? r.x : (i & 3) == 1 ? r.y : (i & 3) == 2 ? r.z : r.w;
        int j = i + (int)(w % (uint32_t)(F - i));
        int vi = i, vj = j, ki = -1, kj = -1;
        for (int k = 0; k < nt; ++k) { if (pos[k] == i) { vi = val[k]; ki = k; } if (pos[k] == j) { vj = val[k]; kj = k; } }
        pick[i] = (uint16_t)vj;                       // perm[i] <- old perm[j]
        if (j != i) {                                  // perm[j] <- old perm[i]
            if (kj >= 0) val[kj] = (uint16_t)vi; else { pos[nt] = (uint16_t)j; val[nt] = (uint16_t)vi; ++nt; }
        }
        (void)ki;
    }
    for (int i = 1; i < m; ++i) {                      // insertion sort ascending
        uint16_t x = pick[i]; int k = i - 1;
        while (k >= 0 && pick[k] > x) { pick[k + 1] = pick[k]; --k; }
        pick[k + 1] = x;
    }
    for (int i = 0; i < m; ++i) out[i] = pick[i];
}

// ------------------------------------------------------------------ R7 histogram build (HOT LOOP A)
__global__ void __launch_bounds__(256) hist_level_kernel(const uint8_t* __restrict__ tp, int stride, int F,
                                                         const b2f_entry* __restrict__ ent, int n_slots, const int64_t* __restrict__ seg_begin,
                                                         const int64_t* __restrict__ seg_end, const int64_t* __restrict__ chunk_off,
                                                         int chunk_rows, const uint16_t* __restrict__ subset, int m, int n_bins,
                                                         int C, int m_pass, uint32_t* hist) {
    extern __shared__ uint32_t sh_hist[];              // [m][n_bins][C]
    __shared__ int sh_feat[256];
    const int64_t c = blockIdx.x;
    const int s = find_slot(chunk_off, n_slots, c);
    const int64_t b = seg_begin[s] + (c - chunk_off[s]) * chunk_rows;
    const int64_t e = min(seg_end[s], b + chunk_rows);
    const int nbC = n_bins * C;
    for (int j = threadIdx.x; j < m; j += blockDim.x) sh_feat[j] = subset[(int64_t)s * m + j];
    uint32_t* gh = hist + (int64_t)s * m * nbC;
    // features are processed m_pass at a time so that the shared histogram fits (wide nodes: DecisionTree, many classes)
    for (int j0 = 0; j0 < m; j0 += m_pass) {
        const int mp = min(m_pass, m - j0);
        const int hsz = mp * nbC;
        __syncthreads();
        for (int i = threadIdx.x; i < hsz; i += blockDim.x) sh_hist[i] = 0;
        __syncthreads();
        for (int64_t i = b + threadIdx.x; i < e; i += blockDim.x) {
            const b2f_entry en = ent[i];
            const uint32_t w = en.y;
            const uint8_t* rec = tp + (int64_t)en.x * stride;
            const int lab = rec[F];
            for (int j = 0; j < mp; ++j) {
                const int bin = rec[sh_feat[j0 + j]];
                atomicAdd(&sh_hist[j * nbC + bin * C + lab], w);
            }
        }
        __syncthreads();
        for (int i = threadIdx.x; i < hsz; i += blockDim.x) {
            uint32_t v = sh_hist[i];
            if (v) atomicAdd(gh + (int64_t)j0 * nbC + i, v);
        }
    }
}

// ------------------------------------------------------------------ R8 split scoring (HOT LOOP B)
// Correctly rounded a / b with the reciprocal y = RN(1/b) shared by all numerators over the same denominator (Markstein:
// q = RN(a*y), r = a - b*q exact by FMA, RN(q + r*y) = RN(a/b) when b's significand is not all ones — b is an integer
// below 2^33 here).  Bit-identical to the oracle's `/`, at 3 fp64 instructions per quotient instead of a full division;
// tests/test_oracle_known_answers.py checks the identity exhaustively for small b and on 10^8 random pairs.
__device__ __forceinline__ double div_rn(double a, double b, double y) {
    const double q = __dmul_rn(a, y);
    return __fma_rn(__fma_rn(-b, q, a), y, q);
}

__device__ __forceinline__ double gini_u32(const uint32_t* c, int C, double tot) {
    if (tot == 0.0) return 0.0;
    const double y = __drcp_rn(tot);
    double imp = 1.0;
    for (int k = 0; k < C; ++k) { double f = div_rn((double)c[k], tot, y); imp -= f * f; }
    return imp;
}

// gain of one candidate split; L = left class counts (smem), tot = node class counts (smem). A.5
__device__ __forceinline__ double split_gain(const uint32_t* L, const uint32_t* tot, int C, double parent_imp,
                                             int min_inst, double min_gain) {
    double lc = 0.0, rc = 0.0;
    for (int k = 0; k < C; ++k) { lc += (double)L[k]; rc += (double)(tot[k] - L[k]); }
    if (lc < (double)min_inst || rc < (double)min_inst) return -DBL_MAX;
    const double t = lc + rc;
    double gl = 1.0, gr = 1.0;
    if (lc == 0.0) gl = 0.0; else { const double y = __drcp_rn(lc); for (int k = 0; k < C; ++k) { double f = div_rn((double)L[k], lc, y); gl -= f * f; } }
    if (rc == 0.0) gr = 0.0; else { const double y = __drcp_rn(rc); for (int k = 0; k < C; ++k) { double f = div_rn((double)(tot[k] - L[k]), rc, y); gr -= f * f; } }
    const double yt = __drcp_rn(t);
    const double lw = div_rn(lc, t, yt), rw = div_rn(rc, t, yt);
    const double gain = parent_imp - lw * gl - rw * gr;
    if (gain < min_gain) return -DBL_MAX;
    return gain;
}

constexpr int kScoreThreads = 128;

// One CTA per slot.  The slot's histogram block is staged ONCE (all loads in flight together), then
//   B. per feature of the node's subset (a warp each): class-wise prefix sums over its bins in shared memory, split into
//      32/C lane segments (continuous); or the centroid ranking + prefix sums in ranked order (ordered categorical); or the
//      raw per-category counts (unordered categorical).  The warp also lists the candidate splits that can win: a split
//      whose left counts equal the previous split's (empty bin / category in between) has exactly the previous gain and
//      "first max" never picks it, so only as many fp64 evaluations remain as there are occupied bins.
//   C. ALL listed candidates of ALL staged features form one flat list (feature-major, split-minor = MLlib's scan order);
//      thread t evaluates candidates t, t+256, ... in fp64 (calculateImpurityStats, no FMA) and keeps its first maximum;
//      a shuffle/smem reduction under (gain desc, feature asc, split asc) reproduces "first max over splits, then first
//      max over features".
// Features are staged in batches when m * n_bins * C exceeds the shared-memory budget (DecisionTree: all features).
__global__ void __launch_bounds__(kScoreThreads) score_level_kernel(
    const uint32_t* __restrict__ hist, int n_slots, const uint16_t* __restrict__ subset, int m, int n_bins, int C,
    const int32_t* __restrict__ feat_bins, const int32_t* __restrict__ feat_kind, int level, int max_depth, int min_inst,
    double min_gain, int batch, b200flow_split* split, uint32_t* node_counts, uint32_t* left_counts, uint32_t* right_counts) {
    extern __shared__ __align__(8) uint8_t sm_raw[];
    const int s = blockIdx.x;
    const int tid = threadIdx.x, w = warp_id(), lane = lane_id(), nw = kScoreThreads / 32;
    const int nbC = n_bins * C;
    // layout: tot[C] | bestL[C] | per-warp {cen[n_bins] f64, raw[nbC] u32} (8-byte multiples) | cum[batch][nbC] | order[batch][n_bins]
    //         | cand[batch][n_bins] u8 (continuous and ordered features; an unordered feature's candidates are all its subsets)
    uint32_t* tot = (uint32_t*)sm_raw;
    uint32_t* bestL = tot + C;
    const size_t per_warp = ((size_t)n_bins * 8 + (size_t)nbC * 4 + 7) & ~(size_t)7;
    uint8_t* wbase = (uint8_t*)(bestL + C);
    double* cen = (double*)(wbase + per_warp * w);
    uint32_t* raw = (uint32_t*)(cen + n_bins);
    uint32_t* cum_all = (uint32_t*)(wbase + per_warp * nw);
    int* order_all = (int*)(cum_all + (size_t)batch * nbC);
    uint8_t* cand_all = (uint8_t*)(order_all + (size_t)batch * n_bins);
    __shared__ int sh_ncand[64], sh_kind[64], sh_nb[64];
    __shared__ double sh_wg[kScoreThreads / 32];
    __shared__ int sh_wj[kScoreThreads / 32], sh_ws[kScoreThreads / 32];
    __shared__ double sh_best_gain; __shared__ int sh_best_j, sh_best_s, sh_best_kind;
    __shared__ unsigned long long sh_best_mask[4];

    const uint32_t* h0 = hist + (int64_t)s * m * nbC;
    if (tid == 0) { sh_best_gain = -DBL_MAX; sh_best_j = -1; sh_best_s = -1; sh_best_kind = 0; }
    double parent_imp = 0.0;

    for (int j0 = 0; j0 < m; j0 += batch) {
        const int nb_feats = min(batch, m - j0);
        // ---- A: stage the batch's histograms (contiguous in global memory)
        {
            const uint32_t* src = h0 + (int64_t)j0 * nbC;
            const int nwords = nb_feats * nbC;
            for (int i = tid; i < nwords; i += kScoreThreads) cum_all[i] = __ldg(src + i);
        }
        __syncthreads();
        // ---- B: prefix sums + candidate lists, one warp per feature
        for (int jj = w; jj < nb_feats; jj += nw) {
            const int f = subset[(int64_t)s * m + j0 + jj];
            const int nb = feat_bins[f], kind = feat_kind[f];
            uint32_t* cum = cum_all + (size_t)jj * nbC;
            int* order = order_all + (size_t)jj * n_bins;
            if (lane == 0) { sh_kind[jj] = kind; sh_nb[jj] = nb; }
            if (kind == 1) {
                for (int i = lane; i < nb * C; i += 32) raw[i] = cum[i];
                __syncwarp();
                for (int c = lane; c < nb; c += 32) {            // centroid per category
                    double cnt = 0.0;
                    for (int k = 0; k < C; ++k) cnt += (double)raw[c * C + k];
                    cen[c] = cnt == 0.0 ? DBL_MAX : (C > 2 ? gini_u32(raw + c * C, C, cnt) : (double)raw[c * C + 1]);
                }
                __syncwarp();
                for (int c = lane; c < nb; c += 32) {            // stable rank by centroid
                    const double ce = cen[c]; int rk = 0;
                    for (int c2 = 0; c2 < nb; ++c2) { const double o = cen[c2]; rk += (o < ce || (o == ce && c2 < c)) ? 1 : 0; }
                    order[rk] = c;
                }
                __syncwarp();
                for (int k = lane; k < C; k += 32) { uint32_t a = 0; for (int i = 0; i < nb; ++i) { a += raw[order[i] * C + k]; cum[i * C + k] = a; } }
            } else if (kind == 0) {
                if (C <= 16) {                                   // lane = (class k, bin segment): 32/C segments scanned side by side
                    const int nseg = 32 / C, seg_len = (nb + nseg - 1) / nseg;
                    const int k = lane % C, seg = lane / C;
                    const bool act = seg < nseg;
                    const int b0 = min(nb, seg * seg_len), b1 = act ? min(nb, b0 + seg_len) : b0;
                    uint32_t a = 0;
                    for (int b = b0; b < b1; ++b) a += cum[b * C + k];
                    uint32_t run = 0;
                    for (int s2 = 0; s2 < nseg; ++s2) { const uint32_t v = __shfl_sync(0xffffffffu, a, s2 * C + k); if (s2 < seg) run += v; }
                    for (int b = b0; b < b1; ++b) { run += cum[b * C + k]; cum[b * C + k] = run; }
                } else {
                    for (int k = lane; k < C; k += 32) { uint32_t a = 0; for (int b = 0; b < nb; ++b) { a += cum[b * C + k]; cum[b * C + k] = a; } }
                }
            }                                                    // kind 2: raw per-category counts stay; subsets are summed per candidate
            __syncwarp();
            if (j0 == 0 && jj == 0) {                            // node class counts = all bins of the first subset feature
                for (int k = lane; k < C; k += 32) {
                    uint32_t a;
                    if (kind == 2) { a = 0; for (int c = 0; c < nb; ++c) a += cum[c * C + k]; }
                    else a = cum[(nb - 1) * C + k];
                    tot[k] = a;
                }
            }
            // the candidate row holds at most nb - 1 <= n_bins - 1 splits of a continuous / ordered feature.  An unordered
            // feature keeps all of its 2^(nb-1) - 1 subsets, which can outnumber n_bins (nb = 5 categories, n_bins = 5): its
            // list is implicitly 0, 1, ..., ns - 1 and is never written to the row
            int n_cand = 0;
            if (kind == 2) {
                n_cand = (1 << (nb - 1)) - 1;
            } else {
                uint8_t* cand = cand_all + (size_t)jj * n_bins;
                const int ns = nb - 1;
                for (int sp0 = 0; sp0 < ns; sp0 += 32) {
                    const int sp = sp0 + lane;
                    bool keep = sp < ns;
                    if (keep && sp > 0) {
                        keep = false;
                        for (int k = 0; k < C; ++k) keep |= cum[sp * C + k] != cum[(sp - 1) * C + k];
                    }
                    const uint32_t mk = __ballot_sync(0xffffffffu, keep);
                    if (keep) cand[n_cand + __popc(mk & ((1u << lane) - 1u))] = (uint8_t)sp;
                    n_cand += __popc(mk);
                }
            }
            if (lane == 0) sh_ncand[jj] = n_cand;
        }
        __syncthreads();
        if (j0 == 0) {                                           // parent impurity: once per warp, broadcast
            double pi = 0.0;
            if (lane == 0) { double ptot = 0.0; for (int k = 0; k < C; ++k) ptot += (double)tot[k]; pi = gini_u32(tot, C, ptot); }
            parent_imp = __shfl_sync(0xffffffffu, pi, 0);
        }
        // ---- C: every listed candidate of the batch, flat over the CTA
        int n_items = 0;
        for (int jj = 0; jj < nb_feats; ++jj) n_items += sh_ncand[jj];
        double tbest = -DBL_MAX; int tj = -1, ts = -1;
        for (int it = tid; it < n_items; it += kScoreThreads) {
            int jj = 0, o = 0;
            while (it >= o + sh_ncand[jj]) { o += sh_ncand[jj]; ++jj; }
            const int sp = sh_kind[jj] == 2 ? it - o : cand_all[(size_t)jj * n_bins + (it - o)];
            const uint32_t* cum = cum_all + (size_t)jj * nbC;
            double g;
            if (sh_kind[jj] != 2) {
                g = split_gain(cum + sp * C, tot, C, parent_imp, min_inst, min_gain);
            } else {
                // unordered: left = sum of the categories whose bit is set in (sp + 1); evaluated without materialising L
                const unsigned bits = (unsigned)(sp + 1); const int nb = sh_nb[jj];
                double lc = 0.0, rc = 0.0;
                for (int k = 0; k < C; ++k) { uint32_t a = 0; for (int c = 0; c < nb; ++c) if ((bits >> c) & 1u) a += cum[c * C + k]; lc += (double)a; rc += (double)(tot[k] - a); }
                if (lc < (double)min_inst || rc < (double)min_inst) g = -DBL_MAX;
                else {
                    const double t = lc + rc; double gl = 1.0, gr = 1.0;
                    if (lc == 0.0) gl = 0.0; else { const double y = __drcp_rn(lc); for (int k = 0; k < C; ++k) { uint32_t a = 0; for (int c = 0; c < nb; ++c) if ((bits >> c) & 1u) a += cum[c * C + k]; const double fq = div_rn((double)a, lc, y); gl -= fq * fq; } }
                    if (rc == 0.0) gr = 0.0; else { const double y = __drcp_rn(rc); for (int k = 0; k < C; ++k) { uint32_t a = 0; for (int c = 0; c < nb; ++c) if ((bits >> c) & 1u) a += cum[c * C + k]; const double fq = div_rn((double)(tot[k] - a), rc, y); gr -= fq * fq; } }
                    const double yt = __drcp_rn(t);
                    const double lw = div_rn(lc, t, yt), rw = div_rn(rc, t, yt);
                    g = parent_imp - lw * gl - rw * gr;
                    if (g < min_gain) g = -DBL_MAX;
                }
            }
            if (g > tbest) { tbest = g; tj = j0 + jj; ts = sp; }      // items ascend in (feature, split): strict > keeps the first
        }
        // CTA argmax under (gain desc, feature asc, split asc); threads without a valid candidate carry tj = -1
        double g = tbest; int bj = tj, bs = ts;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const double og = __shfl_xor_sync(0xffffffffu, g, o); const int oj = __shfl_xor_sync(0xffffffffu, bj, o), os = __shfl_xor_sync(0xffffffffu, bs, o);
            if (oj >= 0 && (bj < 0 || og > g || (og == g && (oj < bj || (oj == bj && os < bs))))) { g = og; bj = oj; bs = os; }
        }
        if (lane == 0) { sh_wg[w] = g; sh_wj[w] = bj; sh_ws[w] = bs; }
        __syncthreads();
        if (tid == 0) {
            double bg = sh_best_gain; int gj = sh_best_j, gs = sh_best_s; bool improved = false;
            for (int q = 0; q < nw; ++q) {
                if (sh_wj[q] < 0) continue;
                if (sh_wg[q] > bg) { bg = sh_wg[q]; gj = sh_wj[q]; gs = sh_ws[q]; improved = true; }
                else if (improved && sh_wg[q] == bg && (sh_wj[q] < gj || (sh_wj[q] == gj && sh_ws[q] < gs))) { gj = sh_wj[q]; gs = sh_ws[q]; }
            }
            if (improved) {                                           // earlier batches win ties (their features come first)
                sh_best_gain = bg; sh_best_j = gj; sh_best_s = gs;
                const int jj = gj - j0; const int kind = sh_kind[jj], nb = sh_nb[jj];
                const uint32_t* cum = cum_all + (size_t)jj * nbC;
                sh_best_kind = kind;
                unsigned long long mk[4] = {0, 0, 0, 0};
                if (kind == 2) {
                    const unsigned bits = (unsigned)(gs + 1);
                    for (int k = 0; k < C; ++k) { uint32_t a = 0; for (int c = 0; c < nb; ++c) if ((bits >> c) & 1u) a += cum[c * C + k]; bestL[k] = a; }
                    mk[0] = bits;
                } else {
                    for (int k = 0; k < C; ++k) bestL[k] = cum[gs * C + k];
                    if (kind == 1) { const int* order = order_all + (size_t)jj * n_bins; for (int i = 0; i <= gs; ++i) { const int c = order[i]; mk[c >> 6] |= 1ull << (c & 63); } }
                }
                for (int q = 0; q < 4; ++q) sh_best_mask[q] = mk[q];
            }
        }
        __syncthreads();
    }
    // ---- outputs
    const bool has = sh_best_j >= 0;
    for (int k = tid; k < C; k += kScoreThreads) {
        node_counts[(int64_t)s * C + k] = tot[k];
        const uint32_t l = has ? bestL[k] : 0u;
        left_counts[(int64_t)s * C + k] = l;
        right_counts[(int64_t)s * C + k] = has ? tot[k] - l : 0u;
    }
    if (tid == 0) {
        b200flow_split o;
        const double bg = sh_best_gain;
        o.gain = has ? bg : -DBL_MAX; o.impurity = parent_imp;
        const bool leaf = !(has && bg > 0.0) || level >= max_depth;
        int flags = leaf ? 1 : 0;
        o.feat = -1; o.kind = 0; o.bin_thr = 0;
        o.mask[0] = o.mask[1] = o.mask[2] = o.mask[3] = 0;
        if (!leaf) {
            o.feat = subset[(int64_t)s * m + sh_best_j]; o.kind = sh_best_kind == 0 ? 0 : 1; o.bin_thr = sh_best_s;
            for (int q = 0; q < 4; ++q) o.mask[q] = sh_best_mask[q];
            double lc = 0.0, rc = 0.0, gl = 1.0, gr = 1.0;
            for (int k = 0; k < C; ++k) { lc += (double)bestL[k]; rc += (double)(tot[k] - bestL[k]); }
            if (lc == 0.0) gl = 0.0; else for (int k = 0; k < C; ++k) { const double fq = (double)bestL[k] / lc; gl -= fq * fq; }
            if (rc == 0.0) gr = 0.0; else for (int k = 0; k < C; ++k) { const double fq = (double)(tot[k] - bestL[k]) / rc; gr -= fq * fq; }
            if (level + 1 == max_depth || gl == 0.0) flags |= 2;
            if (level + 1 == max_depth || gr == 0.0) flags |= 4;
        }
        o.flags = flags;
        split[s] = o;
    }
}

// ------------------------------------------------------------------ pool growth (3 kernels: count, scan, write)
constexpr int kGrowBlock = 256;

__device__ __forceinline__ void grow_flags(const b200flow_split* __restrict__ split, int s, int n_slots, int* is_split, int* n_next) {
    int fl = s < n_slots ? split[s].flags : 1;
    *is_split = (fl & 1) ? 0 : 1;
    *n_next = (fl & 1) ? 0 : ((fl & 2) ? 0 : 1) + ((fl & 4) ? 0 : 1);
}

__global__ void __launch_bounds__(kGrowBlock) grow_count_kernel(int n_slots, const b200flow_split* __restrict__ split, int32_t* blk) {
    __shared__ int sh[2];
    if (threadIdx.x < 2) sh[threadIdx.x] = 0;
    __syncthreads();
    int is, nn; grow_flags(split, blockIdx.x * kGrowBlock + threadIdx.x, n_slots, &is, &nn);
    is = warp_sum(is); nn = warp_sum(nn);
    if (lane_id() == 0) { if (is) atomicAdd(&sh[0], is); if (nn) atomicAdd(&sh[1], nn); }
    __syncthreads();
    if (threadIdx.x < 2) blk[2 * blockIdx.x + threadIdx.x] = sh[threadIdx.x];
}

// single CTA: exclusive scan of the interleaved (split, next) block counts, in place; updates counters
__global__ void __launch_bounds__(1024) grow_scan_kernel(int n_blocks, int32_t* blk, int64_t* counters, int64_t pool_capacity) {
    __shared__ int sh[33];
    __shared__ int carry[2];
    if (threadIdx.x < 2) carry[threadIdx.x] = 0;
    __syncthreads();
    for (int base = 0; base < n_blocks; base += 1024) {
        int i = base + threadIdx.x;
        int a = i < n_blocks ? blk[2 * i] : 0, b = i < n_blocks ? blk[2 * i + 1] : 0;
        int ta, tb;
        int ea = block_exclusive_scan(a, sh, &ta);
        __syncthreads();
        int eb = block_exclusive_scan(b, sh, &tb);
        if (i < n_blocks) { blk[2 * i] = carry[0] + ea; blk[2 * i + 1] = carry[1] + eb; }
        __syncthreads();
        if (threadIdx.x == 0) { carry[0] += ta; carry[1] += tb; }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        int64_t pool = counters[0];
        counters[3] = pool;                               // pool size before this level (base for grow_write)
        int64_t grown = pool + 2 * (int64_t)carry[0];
        counters[2] = grown > pool_capacity ? 1 : 0;      // overflow flag: nothing is written then
        counters[0] = grown > pool_capacity ? pool : grown;
        counters[1] = grown > pool_capacity ? 0 : carry[1];
    }
}

__global__ void __launch_bounds__(kGrowBlock) grow_write_kernel(
    int n_slots, const int32_t* __restrict__ slot_tree, const uint32_t* __restrict__ slot_nid,
    const int32_t* __restrict__ slot_node, const b200flow_split* __restrict__ split,
    const uint32_t* __restrict__ node_counts, const uint32_t* __restrict__ left_counts,
    const uint32_t* __restrict__ right_counts, int C, b200flow_node* nodes, uint64_t* node_mask, uint32_t* pool_counts,
    int32_t* node_tree, const int32_t* __restrict__ blk, const int64_t* __restrict__ counters, int32_t* next_tree,
    uint32_t* next_nid, int32_t* next_node, int32_t* next_parent, int32_t* child_slot) {
    __shared__ int sh[33];
    if (counters[2]) return;
    const int s = blockIdx.x * kGrowBlock + threadIdx.x;
    int is, nn; grow_flags(split, s, n_slots, &is, &nn);
    int t0, t1;
    int e0 = block_exclusive_scan(is, sh, &t0);
    __syncthreads();
    int e1 = block_exclusive_scan(nn, sh, &t1);
    if (s >= n_slots) return;
    const b200flow_split sp = split[s];
    const int node = slot_node[s];
    const uint32_t nid = slot_nid[s];
    const int tree = slot_tree[s];
    b200flow_node nd;
    nd.nid = nid; nd.feat = -1; nd.kind_bin = 0; nd.left = -1;
    int csl = -1, csr = -1;
    for (int k = 0; k < C; ++k) pool_counts[(int64_t)node * C + k] = node_counts[(int64_t)s * C + k];
    if (is) {
        const int64_t child = counters[3] + 2 * ((int64_t)blk[2 * blockIdx.x] + e0);
        nd.feat = sp.feat; nd.kind_bin = (sp.kind << 16) | (sp.bin_thr & 0xffff); nd.left = (int32_t)child;
        if (node_mask) for (int q = 0; q < 4; ++q) node_mask[(int64_t)node * 4 + q] = sp.mask[q];
        b200flow_node ch; ch.feat = -1; ch.kind_bin = 0; ch.left = -1;
        ch.nid = nid * 2u;     nodes[child] = ch;
        ch.nid = nid * 2u + 1; nodes[child + 1] = ch;
        node_tree[child] = tree; node_tree[child + 1] = tree;
        for (int k = 0; k < C; ++k) {
            pool_counts[child * C + k] = left_counts[(int64_t)s * C + k];
            pool_counts[(child + 1) * C + k] = right_counts[(int64_t)s * C + k];
        }
        int64_t ns = (int64_t)blk[2 * blockIdx.x + 1] + e1;
        if (!(sp.flags & 2)) { next_tree[ns] = tree; next_nid[ns] = nid * 2u; next_node[ns] = (int32_t)child; next_parent[ns] = s * 2; csl = (int)ns; ++ns; }
        if (!(sp.flags & 4)) { next_tree[ns] = tree; next_nid[ns] = nid * 2u + 1; next_node[ns] = (int32_t)child + 1; next_parent[ns] = s * 2 + 1; csr = (int)ns; }
    }
    if (child_slot) { child_slot[2 * s] = csl; child_slot[2 * s + 1] = csr; }
    nodes[node] = nd;
}

// per-slot routing plan of a scored level: how many routing chunks each parent needs (0 when it is a leaf or both children
// are leaves) and, on the side, the node's gain for featureImportances — one launch instead of a dozen elementwise ones
__global__ void __launch_bounds__(256) plan_route_kernel(int n_slots, const b200flow_split* __restrict__ split,
                                                         const int64_t* __restrict__ seg_begin, const int64_t* __restrict__ seg_end,
                                                         int chunk_rows, const int32_t* __restrict__ slot_node, double* node_gain,
                                                         int32_t* n_chunks, int32_t* cursors) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_slots) return;
    if (cursors) { cursors[2 * s] = 0; cursors[2 * s + 1] = 0; }          // the routing pass counts into them
    const int flags = split[s].flags;
    const bool routed = !(flags & 1) && (flags & 6) != 6;
    const int64_t len = seg_end[s] - seg_begin[s];
    n_chunks[s] = routed ? (int32_t)((len + chunk_rows - 1) / chunk_rows) : 0;
    if (node_gain) node_gain[slot_node[s]] = split[s].gain;
}

// ------------------------------------------------------------------ row routing
constexpr int kPartPerThread = 8;      // chunk_rows <= 256 * 8

__global__ void __launch_bounds__(256) partition_level_kernel(
    const uint8_t* __restrict__ tp, int stride, const b2f_entry* __restrict__ ent, b2f_entry* ent_out, int n_slots,
    const int64_t* __restrict__ seg_begin, const int64_t* __restrict__ seg_end, const int64_t* __restrict__ chunk_off,
    int chunk_rows, const b200flow_split* __restrict__ split, int32_t* cursors) {
    const int64_t c = blockIdx.x;
    const int s = find_slot(chunk_off, n_slots, c);
    const b200flow_split sp = split[s];
    if (sp.flags & 1) return;                          // leaf: its entries are dropped
    const bool keepL = !(sp.flags & 2), keepR = !(sp.flags & 4);
    if (!keepL && !keepR) return;
    const int64_t sb = seg_begin[s], se = seg_end[s];
    const int64_t b = sb + (c - chunk_off[s]) * chunk_rows;
    const int64_t e = min(se, b + chunk_rows);
    const int lane = lane_id();
    b2f_entry ents[kPartPerThread]; uint32_t dec = 0;  // dec: 2 bits per entry (1 = left kept, 2 = right kept)
    int nL = 0, nR = 0;
#pragma unroll
    for (int k = 0; k < kPartPerThread; ++k) {
        const int64_t i = b + threadIdx.x + (int64_t)k * blockDim.x;
        int d = 0; ents[k] = make_uint2(0u, 0u);
        if (i < e) {
            ents[k] = ent[i];
            const int bin = tp[(int64_t)ents[k].x * stride + sp.feat];
            const bool left = sp.kind == 0 ? (bin <= sp.bin_thr) : ((sp.mask[bin >> 6] >> (bin & 63)) & 1ull);
            d = left ? (keepL ? 1 : 0) : (keepR ? 2 : 0);
        }
        dec |= (uint32_t)d << (2 * k);
        nL += __popc(__ballot_sync(0xffffffffu, d == 1));
        nR += __popc(__ballot_sync(0xffffffffu, d == 2));
    }
    int baseL = 0, baseR = 0;                           // one cursor reservation per warp and side
    if (lane == 0) { if (nL) baseL = atomicAdd(&cursors[2 * s], nL); if (nR) baseR = atomicAdd(&cursors[2 * s + 1], nR); }
    baseL = __shfl_sync(0xffffffffu, baseL, 0); baseR = __shfl_sync(0xffffffffu, baseR, 0);
#pragma unroll
    for (int k = 0; k < kPartPerThread; ++k) {
        const int d = (dec >> (2 * k)) & 3;
        const uint32_t mL = __ballot_sync(0xffffffffu, d == 1), mR = __ballot_sync(0xffffffffu, d == 2);
        const uint32_t lt = (1u << lane) - 1u;
        if (d == 1) ent_out[sb + baseL + __popc(mL & lt)] = ents[k];
        else if (d == 2) ent_out[se - 1 - (baseR + __popc(mR & lt))] = ents[k];
        baseL += __popc(mL); baseR += __popc(mR);
    }
}

// ------------------------------------------------------------------ fused row routing + next-level histogram
// Persistent CTAs (a multiple of 132), each owning a contiguous range of chunks (<= CH entries of one SPLIT parent).
// Software pipeline per WARP, all copies asynchronous (LDGSTS, no register staging):
//     entries(t+2)  -->  record gather(t+1)  -->  route + histogram(t)
//   * the gather brings each entry's TreePoint record (the 64-byte-aligned byte record, or its bit-packed copy when that
//     saves a 16-byte granule: KDD's 32 bytes) into a shared-memory tile, ONCE per entry per level — partition_level +
//     hist_level gathered it twice and were bound by exactly that;
//   * every entry is routed by the parent's split and accumulated into its CHILD's histogram (child feature subset)
//     in shared memory with shared atomics; lane i takes the child's subset features in the ROTATED order (i + t) % m, so
//     that one warp instruction spreads over all m features: the byte reads of the tile fall on random banks instead of
//     a guaranteed 4-way conflict (48-byte pitch), and at most 32 / m lanes can meet on one hot counter;
//   * kept entries go to the child's range (left grows up from seg_begin, right grows down from seg_end; one cursor
//     reservation per warp step and side); the two child histograms stay in shared memory while consecutive chunks
//     belong to the same parent and are flushed with sparse global REDs when the parent changes.
// Launch shapes (route_cfg below): NW warps per CTA x KS entries per lane and step; a chunk is NW * KS * 32 entries.
// Narrow nodes (KDD 5-class: 2 x 9.8 KB of child histograms) run 3 CTAs x 8 warps x 64 entries per SM; wide nodes
// (KDD 23-class: 2 x 45 KB, CICIDS 15-class: 2 x 42 KB) trade tile bytes for histogram bytes — 2 CTAs x 16 warps x 32
// entries, or 1 CTA x 32 warps.  Nodes whose two child histograms exceed shared
// memory altogether (DecisionTree: every feature of every node) are processed in FEATURE PASSES: pass p accumulates
// subset positions [j0, j0 + m_pass) and only pass 0 routes.
#ifndef B2F_EVICT_FIRST
#define B2F_EVICT_FIRST 1
#endif
#ifndef B2F_GRAN
#define B2F_GRAN 16
#endif
constexpr int kGran = B2F_GRAN;                       // bytes per LDGSTS granule of the record gather (16, 8 or 4)
// granules per staged record, and the tile's record pitch in granules (odd for 8 / 4-byte granules: fewer LDS.U8 bank conflicts)
__host__ __device__ inline int route_granules(int F) { return (F + 1 + kGran - 1) / kGran; }
__host__ __device__ inline int route_pitch(int F) { return kGran == 16 ? route_granules(F) : (route_granules(F) | 1); }
constexpr bool kEvictFirst = B2F_EVICT_FIRST != 0;   // entry stream with L2::evict_first (records stay L2-resident)

// Bit-packed TreePoint records (b200flow_packed_layout): field f of a record is (word[d & 0xff] >> ((d >> 8) & 0xff)) &
// (d >> 16) with d = desc[f]; the label is field F.  Records are 16 to 64 bytes, always gathered in 16-byte granules.
// In the staged tile the granules of entry i are swizzled (granule g stored at g ^ sw) so that one word read by a whole
// warp falls on 8 banks (at most 4-way conflicts), as it does for the 48-byte pitch of KDD's byte records: a plain
// 32-byte pitch would put every 4th entry on the same bank (8-way), a 64-byte pitch every 2nd (16-way).
constexpr int kPackedMaxBytes = 64;
__device__ __forceinline__ int packed_swizzle_words(int i, int nq) {      // word-index XOR of entry i (granule swizzle x 4)
    return nq == 2 ? ((i >> 2) & 1) << 2 : nq == 4 ? ((i >> 1) & 3) << 2 : 0;
}

struct RouteChunk { int32_t slot; int32_t n; long long begin; };   // 16 bytes, one per chunk

__global__ void route_chunks_kernel(const int64_t* __restrict__ chunk_off, int n_slots, const int64_t* __restrict__ n_chunks_dev,
                                    const int64_t* __restrict__ seg_begin, const int64_t* __restrict__ seg_end, int CH,
                                    RouteChunk* out) {
    int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= *n_chunks_dev) return;                            // the count lives on the device: the host never waits for it
    const int s = find_slot(chunk_off, n_slots, c);
    RouteChunk rc; rc.slot = s; rc.begin = seg_begin[s] + (c - chunk_off[s]) * CH;
    rc.n = (int)(min(seg_end[s], (int64_t)rc.begin + CH) - rc.begin);
    out[c] = rc;
}

struct RouteArgs {
    const uint8_t* tp; int stride; int F;
    const int32_t* field_desc;                  // packed records: F + 1 field descriptors (NULL: byte records)
    const b2f_entry* ent; b2f_entry* ent_out;
    const RouteChunk* chunks; const int64_t* n_chunks_dev;
    const int64_t* seg_begin; const int64_t* seg_end;
    const b200flow_split* split; const int32_t* child_slot; int32_t* cursors;
    const uint16_t* subset_next; int m_total;   // subset width of a slot (stride of subset_next and of a slot's histogram)
    int j0; int m;                              // this pass accumulates subset positions [j0, j0 + m)
    int n_bins; int C; uint32_t* hist_next;
    int route;                                  // 1: write the routed entries + cursors (first pass of a routed level)
};

// M = compile-time number of subset features of the pass (rotated shared atomics); M = 0: generic path (passes wider than 12).
// Barrier-free inner loop: a chunk is NW sub-chunks of KS * 32 entries, one per warp.  Per warp and step t:
//     entries(t+2) -> registers (prefetch) | record gather(t) -> private tile (LDGSTS; hidden by the other resident warps)
//     write-out of step t-1 (its cursor reservation, a global atomic issued one step earlier, has landed by now)
//     route + histogram of step t from the tile
// CTA-wide barriers happen only when the parent slot changes (flush + re-zero of the two child histograms).
// Packed records with the rotated update read each (entry, feature) through a per-lane descriptor table, built once per
// parent slot: entry [side][t][lane] describes the feature lane `lane` visits at step t for that side (subset position
// j = (lane % M + t) % M), with the granule swizzle of the lane's entries already applied.  .x = byte offset of the field's
// word in the staged record, .y = shift (bits 0-4, read by a wrapping funnel shift) | value mask << 8 | word index of the
// (side, j) histogram << 16.  The lane-major layout keeps every table read conflict-free.
__host__ __device__ inline size_t route_tab_bytes(int mp, bool packed) { return packed && mp <= 12 ? (size_t)2 * mp * 32 * 8 : 0; }

template <int M, int NW, int KS, int NQ>   // M > 0: rotated features, M = 0: plain shared atomics (runtime m); NQ: 16-byte
                                          // granules of a bit-packed record (a.field_desc, a.stride == 16 * NQ), 0: byte records
__global__ void __launch_bounds__(NW * 32, NW == 8 ? 3 : (NW == 16 ? 2 : 1)) route_hist_level_kernel(const RouteArgs a) {
    extern __shared__ __align__(16) uint32_t sm_u32[];
    constexpr bool PACKED = NQ > 0;
    constexpr bool kTab = PACKED && M > 0;                   // histogram update through the per-lane descriptor table
    constexpr int kThreads = NW * 32, kSub = KS * 32;
    constexpr int gran = PACKED ? 16 : kGran;
    const int m = M > 0 ? M : a.m;
    const int F = a.F;
    const int tid = threadIdx.x, lane = lane_id(), wid = warp_id();
    const int nq = PACKED ? NQ : route_granules(F);            // staged granules (16-byte quads by default) per record
    const int rs = PACKED ? NQ * 16 : route_pitch(F) * kGran;  // bytes per staged record
    const int nbC = a.n_bins * a.C, hsz = m * nbC;
    const int tile_words = rs * kSub / 4;
    uint32_t* tile = sm_u32 + (size_t)wid * tile_words;      // this warp's [kSub][nq] quad tile (entry-major)
    uint32_t* sh_hist = sm_u32 + (size_t)NW * tile_words;    // [2][hsz]
    int* sh_fpos = (int*)(sh_hist + 2 * hsz);                // [2][m]: byte offset (packed: descriptor) of the feature in a record
    uint2* sh_tab = (uint2*)(sh_fpos + 2 * m);               // kTab: [2][M][32] descriptor table (route_tab_bytes)
    __shared__ b200flow_split sh_split;
    __shared__ int sh_child[2], sh_route_field;              // sh_route_field: byte offset / descriptor of the split feature

    const int64_t n_chunks = *a.n_chunks_dev;
    const int64_t c0 = n_chunks * blockIdx.x / gridDim.x, c1 = n_chunks * (blockIdx.x + 1) / gridDim.x;
    if (c0 >= c1) return;
    auto flush = [&]() {
        for (int side = 0; side < 2; ++side) {
            const int cs = sh_child[side];
            if (cs < 0) continue;
            uint32_t* gh = a.hist_next + ((int64_t)cs * a.m_total + a.j0) * nbC;
            uint32_t* sh = sh_hist + side * hsz;
            for (int i = tid; i < hsz; i += kThreads) { const uint32_t v = sh[i]; if (v) { atomicAdd(gh + i, v); sh[i] = 0; } }   // flush + re-zero
        }
    };
    for (int i = tid; i < 2 * hsz; i += kThreads) sh_hist[i] = 0;     // zero once; every flush leaves the histograms zeroed
    auto desc_at = [&](int64_t c) { return c < c1 ? __ldg((const int4*)(a.chunks + c)) : make_int4(-1, 0, 0, 0); };
    auto count_of = [&](const int4& d) { return min(kSub, d.y - wid * kSub); };
    auto entries_of = [&](const int4& d, b2f_entry* x) {
        const int cn = count_of(d);
        const b2f_entry* ep = a.ent + (((long long)(uint32_t)d.z) | ((long long)d.w << 32)) + wid * kSub;
#pragma unroll
        for (int k = 0; k < KS; ++k) x[k] = lane + 32 * k < cn ? (kEvictFirst ? ld_evict_first_u2(ep + 32 * k + lane) : __ldg(ep + 32 * k + lane)) : make_uint2(0u, 0u);
    };
    // The tile is entry-major ([kSub entries][nq quads]) and its kSub * nq 16-byte chunks are copied in linear order, lane
    // after lane: neighbouring lanes fetch neighbouring quads of the SAME record (same 32-byte sector) into neighbouring
    // shared addresses, which the L1 can fill with fewer wavefronts than one scattered 16-byte fill per lane.
    // Packed records: the KS * NQ granule copies of a lane are unrolled with the geometry known at compile time, so entry,
    // granule and swizzle fold to per-lane constants plus an immediate per copy, and each copy shuffles its record index out
    // of one known x[k] (entry 32k starts at granule 32k * NQ, a multiple of 32).  For NQ = 2 and 4 a copy covers 32 / NQ
    // whole entries and the swizzle of entry it * 32 / NQ + lane / NQ depends on the lane alone.
    constexpr int kNQ = PACKED ? NQ : 1;
    constexpr bool kPow2 = (kNQ & (kNQ - 1)) == 0;
    const int g_e0 = kPow2 ? lane / kNQ : 0, g_q0 = kPow2 ? lane % kNQ : 0;
    const int g_sw = packed_swizzle_words(g_e0, NQ) >> 2;
    const uint8_t* g_src = a.tp + g_q0 * 16;
    uint8_t* g_dst = (uint8_t*)tile + g_e0 * rs + (g_q0 ^ g_sw) * 16;
    const uint32_t inv_nq = (1u << 20) / (uint32_t)nq + 1u;     // c / nq == (c * inv_nq) >> 20 for c * nq < 2^20
    auto issue_gather = [&](const int4& d, const b2f_entry* x) {
        const int cn = count_of(d);
        if (PACKED) {
#pragma unroll
            for (int it = 0; it < KS * kNQ; ++it) {
                const int k = it / kNQ;
                if (kPow2) {
                    const int e = it * (32 / kNQ) + g_e0;
                    const uint32_t r = __shfl_sync(0xffffffffu, x[k].x, e & 31);
                    if (e < cn) cp_async16(g_dst + it * 512, g_src + (size_t)r * (kNQ * 16));
                } else {                                        // NQ = 3: a copy straddles entries, divide by the constant
                    const int c = it * 32 + lane, e = c / kNQ, q = c - e * kNQ;
                    const uint32_t r = __shfl_sync(0xffffffffu, x[k].x, e & 31);
                    if (e < cn) cp_async16((uint8_t*)tile + e * rs + q * 16, a.tp + (size_t)r * (kNQ * 16) + q * 16);
                }
            }
        } else {
            for (int c = lane; c < kSub * nq; c += 32) {       // uniform trip count (KS * nq)
                const int e = (int)(((uint32_t)c * inv_nq) >> 20), q = c - e * nq;
                uint32_t r = __shfl_sync(0xffffffffu, x[0].x, e & 31);
                if (KS == 2) { const uint32_t r1 = __shfl_sync(0xffffffffu, x[KS - 1].x, e & 31); r = e < 32 ? r : r1; }
                if (e < cn) {
                    uint8_t* dst = (uint8_t*)tile + e * rs + q * gran;
                    const uint8_t* src = a.tp + (int64_t)r * a.stride + q * gran;
                    if (gran == 16) cp_async16(dst, src); else if (gran == 8) cp_async8(dst, src); else cp_async4(dst, src);
                }
            }
        }
        cp_async_commit();
    };
    // pending write of the previous step (registers only)
    bool pending = false;
    b2f_entry p_e[KS]; uint32_t p_dec = 0; int p_bl = 0, p_br = 0; int64_t p_sb = 0, p_se = 0;
#pragma unroll
    for (int k = 0; k < KS; ++k) p_e[k] = make_uint2(0u, 0u);
    const uint32_t lt = (1u << lane) - 1u;
    auto write_pending = [&]() {
        int baseL = __shfl_sync(0xffffffffu, p_bl, 0), baseR = __shfl_sync(0xffffffffu, p_br, 0);
#pragma unroll
        for (int k = 0; k < KS; ++k) {
            const int d = (p_dec >> (2 * k)) & 3;
            const uint32_t mL = __ballot_sync(0xffffffffu, d == 1), mR = __ballot_sync(0xffffffffu, d == 2);
            if (d == 1) { if (kEvictFirst) st_evict_first_u2(a.ent_out + p_sb + baseL + __popc(mL & lt), p_e[k]); else a.ent_out[p_sb + baseL + __popc(mL & lt)] = p_e[k]; }
            else if (d == 2) { if (kEvictFirst) st_evict_first_u2(a.ent_out + p_se - 1 - (baseR + __popc(mR & lt)), p_e[k]); else a.ent_out[p_se - 1 - (baseR + __popc(mR & lt))] = p_e[k]; }
            baseL += __popc(mL); baseR += __popc(mR);
        }
        pending = false;
    };

    int4 d0 = desc_at(c0), d1 = desc_at(c0 + 1), d2 = desc_at(c0 + 2);
    b2f_entry e[KS], f[KS], g[KS];                             // entries of steps t, t+1, t+2
    entries_of(d0, e);
    entries_of(d1, f);
    int cur_slot = -1;
    const int lab_pos = PACKED ? __ldg(a.field_desc + F) : F;  // byte (packed: descriptor) of the label inside a staged record
    const uint8_t* tile8 = (const uint8_t*)tile;               // [kSub entries][nq * 16 bytes]
    // field of staged entry i at byte offset / descriptor d
    auto field = [&](int i, int d) -> uint32_t {
        if (!PACKED) return tile8[d + i * rs];
        const uint32_t v = tile[i * (rs >> 2) + ((d & 0xff) ^ packed_swizzle_words(i, nq))];
        return (v >> ((d >> 8) & 0xff)) & (uint32_t)(d >> 16);
    };
    for (int64_t c = c0; c < c1; ++c) {
        entries_of(d2, g);                                     // prefetch, consumed two steps later
        const int4 d3 = desc_at(c + 3);
        issue_gather(d0, e);                                   // single tile: latency hidden by the other resident warps
        if (pending) write_pending();
        cp_async_wait_all();
        __syncwarp();
        const int s = d0.x;
        if (s != cur_slot) {                                   // same decision in every warp: all iterate the same chunks
            __syncthreads();
            if (cur_slot >= 0) flush();                           // reads sh_child of the OLD slot: barrier before it is replaced
            __syncthreads();
            if (tid < 16) ((uint32_t*)&sh_split)[tid] = ((const uint32_t*)(a.split + s))[tid];
            if (tid < 2) sh_child[tid] = a.child_slot[2 * s + tid];
            if (tid == 0) { const int fs = max(a.split[s].feat, 0); sh_route_field = PACKED ? a.field_desc[fs] : fs; }
            if (kTab) {
                constexpr int kM = M > 0 ? M : 1;
                for (int idx = tid; idx < 2 * kM * 32; idx += kThreads) {
                    const int side = idx / (kM * 32), t = idx / 32 % kM, ln = idx % 32, j = (ln % kM + t) % kM;
                    const int cs = a.child_slot[2 * s + side];
                    const int fidx = cs >= 0 ? a.subset_next[(int64_t)cs * a.m_total + a.j0 + j] : 0;
                    const uint32_t d = (uint32_t)__ldg(a.field_desc + fidx);
                    const uint32_t word = (d & 0xffu) ^ (uint32_t)packed_swizzle_words(ln, NQ);   // lane swizzle == entry swizzle
                    sh_tab[idx] = make_uint2(word * 4u, ((d >> 8) & 31u) | ((d >> 16) << 8) | ((uint32_t)(side * hsz + j * nbC) << 16));
                }
            } else {
                for (int j = tid; j < 2 * m; j += kThreads) {
                    const int cs = a.child_slot[2 * s + (j >= m)];
                    const int fidx = cs >= 0 ? a.subset_next[(int64_t)cs * a.m_total + a.j0 + (j < m ? j : j - m)] : 0;
                    sh_fpos[j] = PACKED ? a.field_desc[fidx] : fidx;
                }
            }
            cur_slot = s;
            __syncthreads();
        }
        const int cnt = count_of(d0);
        if (cnt > 0) {
            const int cl = sh_child[0], cr = sh_child[1];
            const int fs = sh_route_field, kind = sh_split.kind, thr = sh_split.bin_thr;
            int nL = 0, nR = 0;
            uint32_t dec = 0;
#pragma unroll
            for (int k = 0; k < KS; ++k) {
                const int i = k * 32 + lane;
                int d = 0;
                if (i < cnt) {
                    const int bin = (int)field(i, fs);
                    const bool left = kind == 0 ? (bin <= thr) : ((sh_split.mask[bin >> 6] >> (bin & 63)) & 1ull);
                    d = left ? (cl >= 0 ? 1 : 0) : (cr >= 0 ? 2 : 0);
                }
                dec |= (uint32_t)d << (2 * k);
                const uint32_t mL = __ballot_sync(0xffffffffu, d == 1), mR = __ballot_sync(0xffffffffu, d == 2);
                nL += __popc(mL); nR += __popc(mR);
                if (d != 0) {
                    const int side = d - 1;
                    const int* fpos = sh_fpos + side * m;
                    uint32_t* hist = sh_hist + side * hsz;
                    const uint32_t lab = field(i, lab_pos);
                    const uint32_t w = e[k].y;
                    if (kTab) {
                        // rotated features through the descriptor table: one table read, one tile read, one shared atomic
                        const uint2* tab = sh_tab + side * (M * 32) + lane;
                        const uint8_t* rec = (const uint8_t*)tile + i * rs;
                        uint32_t* hl = sh_hist + lab;
#pragma unroll
                        for (int t = 0; t < M; ++t) {
                            const uint2 dd = tab[t * 32];
                            const uint32_t v = *(const uint32_t*)(rec + dd.x);
                            const uint32_t bin = __funnelshift_r(v, 0u, dd.y) & ((dd.y >> 8) & 0xffu);
                            atomicAdd(hl + (dd.y >> 16) + bin * a.C, w);
                        }
                    } else if (M > 0) {
                        // rotated features: lane i walks the subset positions in the order (i + t) % M, so that one warp
                        // instruction spreads over all M features — the lanes 8 apart (same bank for a 48-byte pitch) read
                        // different record words, and only ~32 / M lanes can meet on one hot counter.  Integer sums: same result.
                        int j = lane % M;
#pragma unroll
                        for (int t = 0; t < M; ++t) {
                            const int fp = fpos[j];
                            const uint32_t bin = field(i, fp);
                            atomicAdd(&hist[j * nbC + bin * a.C + lab], w);
                            j = j + 1 == M ? 0 : j + 1;
                        }
                    } else {
                        for (int j = 0; j < m; ++j) {
                            const int fp = fpos[j];
                            const uint32_t bin = field(i, fp);
                            atomicAdd(&hist[j * nbC + bin * a.C + lab], w);
                        }
                    }
                }
            }
            __syncwarp();
            // reserve output positions (one atomic pair per warp step); the result is consumed one step later
            if (a.route && (nL | nR)) {
                if (lane == 0) {   // both cursors of the slot in ONE 64-bit atomic (left count in the low word): the top levels' few hundred cursors are hot
                    const unsigned long long old = atomicAdd((unsigned long long*)(a.cursors + 2 * s), (unsigned long long)(uint32_t)nL | ((unsigned long long)(uint32_t)nR << 32));
                    p_bl = (int)(uint32_t)old; p_br = (int)(uint32_t)(old >> 32);
                }
#pragma unroll
                for (int k = 0; k < KS; ++k) p_e[k] = e[k];
                p_dec = dec; p_sb = a.seg_begin[s]; p_se = a.seg_end[s];
                pending = true;
            }
        }
        d0 = d1; d1 = d2; d2 = d3;
#pragma unroll
        for (int k = 0; k < KS; ++k) { e[k] = f[k]; f[k] = g[k]; }
    }
    if (pending) write_pending();
    cp_async_wait_all();
    __syncthreads();
    flush();
}

// ---- launch shape of the fused kernel
struct RouteCfg { int nw, ks, m_pass, per_sm; size_t smem; };
constexpr size_t kSmemPerSM = 227 * 1024;                  // 232,448 B usable per block on sm_90
constexpr size_t kSmemCtaOverhead = 1024 + 128;            // driver reservation per CTA + the kernel's static shared memory

// rs = bytes per staged record: route_pitch(F) * kGran for byte records, the record size for packed ones
static size_t route_hist_smem(int rs, bool packed, int mp, int n_bins, int C, int nw, int ks) {
    return (size_t)nw * ks * 32 * rs + 2 * (size_t)mp * n_bins * C * 4 + 2 * (size_t)mp * 4 + route_tab_bytes(mp, packed) + 64;
}
static int route_max_ctas(int nw) { return nw == 8 ? 3 : (nw == 16 ? 2 : 1); }   // __launch_bounds__ (8 warps: 3 CTAs, 85 registers)

// Picks (warps per CTA, entries per lane, features per pass): the fewest passes first (every extra pass gathers the
// records again), then the most entries in flight per SM (resident warps x entries per lane) up to 48, then the smallest
// chunk, then the most resident warps.  On an H100 (KDD99-full, level kernel per fit) 8x2 with 3 CTAs per SM took 26.6 ms,
// 16x2 with 64 entries in flight 30.5, 8x1 28.3, 16x1 28.4, and 8x2 with 4 CTAs per SM (64 registers: spills) 35.0.
static bool route_cfg(int F, int rs, bool packed, int m, int n_bins, int C, RouteCfg* out) {
    static const int cand[5][2] = {{8, 2}, {8, 1}, {16, 2}, {16, 1}, {32, 1}};
    int force_nw = 0, force_ks = 0;                         // tuning / test knob, read per call: B200FLOW_ROUTE_SHAPE=<warps>x<entries per lane>
    { const char* e = getenv("B200FLOW_ROUTE_SHAPE"); if (e && sscanf(e, "%dx%d", &force_nw, &force_ks) != 2) force_nw = force_ks = 0; }
    if (F <= 0 || F > 255 || m <= 0 || n_bins <= 0 || C <= 0) return false;
    auto fits = [&](int mp, int nw, int ks) { return route_hist_smem(rs, packed, mp, n_bins, C, nw, ks) + kSmemCtaOverhead <= kSmemPerSM; };
    int mp = m;
    while (mp >= 1 && !fits(mp, 8, 1)) --mp;                // (8, 1) has the smallest tiles
    if (mp < 1) return false;
    const int passes = (m + mp - 1) / mp;
    mp = (m + passes - 1) / passes;                          // balanced passes
    int best = -1; long best_key = -1;
    for (int i = 0; i < 5; ++i) {
        const int nw = cand[i][0], ks = cand[i][1];
        if (force_nw > 0 && (nw != force_nw || ks != force_ks)) continue;
        if (!fits(mp, nw, ks)) continue;
        const size_t smem = route_hist_smem(rs, packed, mp, n_bins, C, nw, ks);
        int per_sm = (int)(kSmemPerSM / (smem + kSmemCtaOverhead));
        if (per_sm > route_max_ctas(nw)) per_sm = route_max_ctas(nw);
        const int warps = per_sm * nw > 32 ? 32 : per_sm * nw;
        const long key = ((long)(warps * ks < 48 ? warps * ks : 48) << 20) + ((long)(1023 - nw * ks) << 10) + warps;
        if (key > best_key) { best_key = key; best = i; }
    }
    if (best < 0) return false;
    out->nw = cand[best][0]; out->ks = cand[best][1]; out->m_pass = mp;
    out->smem = route_hist_smem(rs, packed, mp, n_bins, C, out->nw, out->ks);
    out->per_sm = (int)(kSmemPerSM / (out->smem + kSmemCtaOverhead));
    if (out->per_sm > route_max_ctas(out->nw)) out->per_sm = route_max_ctas(out->nw);
    return true;
}

// M = 1..12: the rotated histogram update compiled for that pass width; any other M: the generic runtime loop
template <int NW, int KS, int NQ>
static cudaError_t route_launch(int M, unsigned grid_cap, size_t smem, int per_sm_hint, int waves, int64_t n_chunks_max,
                                const RouteArgs& a, cudaStream_t st) {
    cudaError_t e = cudaSuccess;
#define B2F_ROUTE_GO(KERNEL)                                                                                                   \
    {                                                                                                                          \
        e = cudaFuncSetAttribute(KERNEL, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);                             \
        if (e != cudaSuccess) return e;                                                                                        \
        int per_sm = 0;                                                                                                        \
        e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, KERNEL, NW * 32, smem);                                    \
        if (e != cudaSuccess) return e;                                                                                        \
        if (per_sm < 1) per_sm = per_sm_hint > 0 ? per_sm_hint : 1;                                                            \
        const int64_t want = (int64_t)kNumSMs * per_sm * waves;                                                                \
        unsigned grid = (unsigned)(n_chunks_max < want ? n_chunks_max : want);                                                 \
        if (grid_cap && grid > grid_cap) grid = grid_cap;                                                                      \
        KERNEL<<<grid, NW * 32, smem, st>>>(a);                                                                                \
    }
#define B2F_ROUTE_CASE(MM) case MM: B2F_ROUTE_GO((route_hist_level_kernel<MM, NW, KS, NQ>)) break;
    switch (M) {
        B2F_ROUTE_CASE(1) B2F_ROUTE_CASE(2) B2F_ROUTE_CASE(3) B2F_ROUTE_CASE(4) B2F_ROUTE_CASE(5) B2F_ROUTE_CASE(6)
        B2F_ROUTE_CASE(7) B2F_ROUTE_CASE(8) B2F_ROUTE_CASE(9) B2F_ROUTE_CASE(10) B2F_ROUTE_CASE(11) B2F_ROUTE_CASE(12)
        default: B2F_ROUTE_GO((route_hist_level_kernel<0, NW, KS, NQ>)) break;
    }
#undef B2F_ROUTE_CASE
#undef B2F_ROUTE_GO
    return cudaGetLastError();
}

template <int NQ>
static cudaError_t route_shape(const RouteCfg& cfg, int M, size_t smem, int waves, int64_t n_chunks_max, const RouteArgs& a,
                               cudaStream_t st) {
    if (cfg.nw == 8 && cfg.ks == 2) return route_launch<8, 2, NQ>(M, 0, smem, cfg.per_sm, waves, n_chunks_max, a, st);
    if (cfg.nw == 8) return route_launch<8, 1, NQ>(M, 0, smem, cfg.per_sm, waves, n_chunks_max, a, st);
    if (cfg.nw == 16 && cfg.ks == 2) return route_launch<16, 2, NQ>(M, 0, smem, cfg.per_sm, waves, n_chunks_max, a, st);
    if (cfg.nw == 16) return route_launch<16, 1, NQ>(M, 0, smem, cfg.per_sm, waves, n_chunks_max, a, st);
    return route_launch<32, 1, NQ>(M, 0, smem, cfg.per_sm, waves, n_chunks_max, a, st);
}

__global__ void next_segments_kernel(int n_next, const int64_t* __restrict__ n_next_dev, const int32_t* __restrict__ next_parent,
                                     const int64_t* __restrict__ seg_begin, const int64_t* __restrict__ seg_end,
                                     const int32_t* __restrict__ cursors, int64_t* next_begin, int64_t* next_end) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_next || (n_next_dev && i >= *n_next_dev)) return;
    const int p = next_parent[i], ps = p >> 1;
    if ((p & 1) == 0) { next_begin[i] = seg_begin[ps]; next_end[i] = seg_begin[ps] + cursors[2 * ps]; }
    else { next_begin[i] = seg_end[ps] - cursors[2 * ps + 1]; next_end[i] = seg_end[ps]; }
}

__global__ void finalize_forest_kernel(int64_t n_nodes, const uint32_t* __restrict__ pool_counts, int C, double* leaf_prob) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_nodes) return;
    double tot = 0.0;
    for (int k = 0; k < C; ++k) tot += (double)pool_counts[i * C + k];
    for (int k = 0; k < C; ++k) leaf_prob[i * C + k] = tot != 0.0 ? (double)pool_counts[i * C + k] / tot : 0.0;
}

}  // namespace b200flow

using namespace b200flow;

extern "C" int b200flow_feature_subsets(uint64_t seed, int32_t n_slots, const int32_t* slot_tree, const uint32_t* slot_nid,
                                        int32_t F, int32_t m, uint16_t* subset, void* stream) {
    B2F_REQUIRE(slot_tree && slot_nid && subset && F > 0 && F < 65536 && m > 0 && m <= F, "feature_subsets: bad arguments");
    B2F_REQUIRE(m == F || m <= kMaxSubset, "feature_subsets: subset size %d > %d not supported", m, kMaxSubset);
    if (n_slots <= 0) return B200FLOW_OK;
    feature_subsets_kernel<<<(n_slots + 127) / 128, 128, 0, (cudaStream_t)stream>>>(seed, n_slots, slot_tree, slot_nid, F, m, subset);
    return check_launch("feature_subsets");
}

extern "C" int b200flow_hist_level(const uint8_t* tp, int32_t tp_stride, int32_t F, const void* ent,
                                   int32_t n_slots, const int64_t* seg_begin, const int64_t* seg_end, const int64_t* chunk_off,
                                   int64_t n_chunks, int32_t chunk_rows, const uint16_t* subset, int32_t m, int32_t n_bins,
                                   int32_t C, uint32_t* hist, void* stream) {
    B2F_REQUIRE(tp && ent && seg_begin && seg_end && chunk_off && subset && hist, "hist_level: null pointer");
    B2F_REQUIRE(m > 0 && m <= 256 && n_bins > 0 && n_bins <= 256 && C > 0 && C <= 256 && chunk_rows > 0, "hist_level: bad shape");
    const size_t per_feat = (size_t)n_bins * C * 4;
    B2F_REQUIRE(per_feat <= 200 * 1024, "hist_level: one feature's histogram (%zu B) exceeds shared memory", per_feat);
    int m_pass = (int)((64 * 1024) / per_feat);            // <= 64 KB per CTA keeps >= 3 CTAs resident per SM
    if (m_pass < 1) m_pass = 1;
    if (m_pass > m) m_pass = m;
    size_t smem = per_feat * m_pass;
    if (n_slots <= 0 || n_chunks <= 0) return B200FLOW_OK;
    B2F_REQUIRE(n_chunks < ((int64_t)1 << 31), "hist_level: too many chunks");
    cudaError_t e = cudaFuncSetAttribute(hist_level_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) { set_error("hist_level: %s", cudaGetErrorString(e)); return B200FLOW_ERR_CUDA; }
    hist_level_kernel<<<(unsigned)n_chunks, 256, smem, (cudaStream_t)stream>>>(tp, tp_stride, F, (const b2f_entry*)ent, n_slots, seg_begin,
                                                                             seg_end, chunk_off, chunk_rows, subset, m, n_bins, C, m_pass, hist);
    return check_launch("hist_level");
}

extern "C" int b200flow_score_level(const uint32_t* hist, int32_t n_slots, const uint16_t* subset, int32_t m, int32_t n_bins,
                                    int32_t C, const int32_t* feat_bins, const int32_t* feat_kind, int32_t level, int32_t max_depth,
                                    int32_t min_instances, double min_info_gain, b200flow_split* split, uint32_t* node_counts,
                                    uint32_t* left_counts, uint32_t* right_counts, void* stream) {
    B2F_REQUIRE(hist && subset && feat_bins && feat_kind && split && node_counts && left_counts && right_counts, "score_level: null pointer");
    B2F_REQUIRE(m > 0 && n_bins > 0 && n_bins <= 256 && C > 0 && C <= 256, "score_level: bad shape");
    if (n_slots <= 0) return B200FLOW_OK;
    // shared memory: tot + bestL + per-feature {prefix sums, rank order} for a batch of features + per-warp scratch
    const size_t per_feat = (size_t)n_bins * C * 4 + (size_t)n_bins * 4 + (size_t)n_bins;
    const size_t per_warp = ((size_t)n_bins * 8 + (size_t)n_bins * C * 4 + 7) & ~(size_t)7;
    const size_t fixed = (size_t)2 * C * 4 + 16 + per_warp * (kScoreThreads / 32) + 16;
    int batch = m < 64 ? m : 64;
    while (batch > 1 && fixed + per_feat * batch > 160 * 1024) --batch;
    const size_t smem = fixed + per_feat * batch;
    B2F_REQUIRE(smem <= 200 * 1024, "score_level: scratch exceeds shared memory");
    cudaError_t e = cudaFuncSetAttribute(score_level_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) { set_error("score_level: %s", cudaGetErrorString(e)); return B200FLOW_ERR_CUDA; }
    score_level_kernel<<<n_slots, kScoreThreads, smem, (cudaStream_t)stream>>>(hist, n_slots, subset, m, n_bins, C, feat_bins, feat_kind, level,
                                                                              max_depth, min_instances, min_info_gain, batch, split,
                                                                              node_counts, left_counts, right_counts);
    return check_launch("score_level");
}

extern "C" int b200flow_grow_level(int32_t n_slots, const int32_t* slot_tree, const uint32_t* slot_nid, const int32_t* slot_node,
                                   const b200flow_split* split, const uint32_t* node_counts, const uint32_t* left_counts,
                                   const uint32_t* right_counts, int32_t C, b200flow_node* nodes, uint64_t* node_mask,
                                   uint32_t* pool_counts, int32_t* node_tree, int64_t pool_capacity, int32_t* next_tree,
                                   uint32_t* next_nid, int32_t* next_node, int32_t* next_parent, int32_t* child_slot,
                                   int64_t* counters, void* stream) {
    B2F_REQUIRE(slot_tree && slot_nid && slot_node && split && node_counts && left_counts && right_counts && nodes && pool_counts &&
                    node_tree && next_tree && next_nid && next_node && next_parent && counters, "grow_level: null pointer");
    if (n_slots <= 0) return B200FLOW_OK;
    // counters: int64[8] header {pool size, n_next, overflow flag, pool size before the level, 4 free for the caller}
    // followed by the int32 scratch for the per-block counts (2 * ceil(n_slots/256) ints), all caller-owned.
    const int nb = (n_slots + kGrowBlock - 1) / kGrowBlock;
    int32_t* blk = (int32_t*)(counters + 8);
    grow_count_kernel<<<nb, kGrowBlock, 0, (cudaStream_t)stream>>>(n_slots, split, blk);
    grow_scan_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(nb, blk, counters, pool_capacity);
    grow_write_kernel<<<nb, kGrowBlock, 0, (cudaStream_t)stream>>>(n_slots, slot_tree, slot_nid, slot_node, split, node_counts, left_counts,
                                                                  right_counts, C, nodes, node_mask, pool_counts, node_tree, blk, counters,
                                                                  next_tree, next_nid, next_node, next_parent, child_slot);
    return check_launch("grow_level");
}

extern "C" int b200flow_plan_route(int32_t n_slots, const b200flow_split* split, const int64_t* seg_begin, const int64_t* seg_end,
                                   int32_t chunk_rows, const int32_t* slot_node, double* node_gain, int32_t* n_chunks, int32_t* cursors,
                                   void* stream) {
    if (n_slots <= 0) return B200FLOW_OK;
    B2F_REQUIRE(split && seg_begin && seg_end && n_chunks && chunk_rows > 0 && (!node_gain || slot_node), "plan_route: bad arguments");
    plan_route_kernel<<<(n_slots + 255) / 256, 256, 0, (cudaStream_t)stream>>>(n_slots, split, seg_begin, seg_end, chunk_rows, slot_node, node_gain, n_chunks, cursors);
    return check_launch("plan_route");
}

extern "C" int b200flow_partition_level(const uint8_t* tp, int32_t tp_stride, const void* ent, void* ent_out, int32_t n_slots,
                                        const int64_t* seg_begin, const int64_t* seg_end, const int64_t* chunk_off, int64_t n_chunks,
                                        int32_t chunk_rows, const b200flow_split* split, int32_t* cursors, void* stream) {
    B2F_REQUIRE(tp && ent && ent_out && seg_begin && seg_end && chunk_off && split && cursors, "partition_level: null pointer");
    B2F_REQUIRE(chunk_rows > 0 && chunk_rows <= 256 * kPartPerThread, "partition_level: chunk_rows must be <= %d", 256 * kPartPerThread);
    if (n_slots <= 0 || n_chunks <= 0) return B200FLOW_OK;
    partition_level_kernel<<<(unsigned)n_chunks, 256, 0, (cudaStream_t)stream>>>(tp, tp_stride, (const b2f_entry*)ent, (b2f_entry*)ent_out, n_slots, seg_begin, seg_end,
                                                                               chunk_off, chunk_rows, split, cursors);
    return check_launch("partition_level");
}

extern "C" int b200flow_next_segments(int32_t n_next, const int64_t* n_next_dev, const int32_t* next_parent, const int64_t* seg_begin,
                                      const int64_t* seg_end, const int32_t* cursors, int64_t* next_begin, int64_t* next_end, void* stream) {
    B2F_REQUIRE(next_parent && seg_begin && seg_end && cursors && next_begin && next_end, "next_segments: null pointer");
    if (n_next <= 0) return B200FLOW_OK;
    next_segments_kernel<<<(n_next + 255) / 256, 256, 0, (cudaStream_t)stream>>>(n_next, n_next_dev, next_parent, seg_begin, seg_end, cursors, next_begin, next_end);
    return check_launch("next_segments");
}

extern "C" int b200flow_finalize_forest(int64_t n_nodes, const uint32_t* pool_counts, int32_t C, double* leaf_prob, void* stream) {
    B2F_REQUIRE(pool_counts && leaf_prob && C > 0, "finalize_forest: bad arguments");
    if (n_nodes <= 0) return B200FLOW_OK;
    finalize_forest_kernel<<<(unsigned)((n_nodes + 255) / 256), 256, 0, (cudaStream_t)stream>>>(n_nodes, pool_counts, C, leaf_prob);
    return check_launch("finalize_forest");
}

extern "C" int b200flow_packed_layout(int32_t F, const int32_t* feat_bins, int32_t C, int32_t* desc, int32_t* rec_bytes) {
    B2F_REQUIRE(feat_bins && desc && rec_bytes && F > 0 && C > 0 && C <= 256, "packed_layout: bad arguments");
    *rec_bytes = 0;
    if (F > 255) return B200FLOW_OK;                         // no fused level kernel for such records (route_cfg): keep bytes
    int width[256], order[256], used[256];
    auto bits = [](int v) { int b = 0; while (v > 0) { ++b; v >>= 1; } return b > 0 ? b : 1; };
    for (int f = 0; f <= F; ++f) {
        const int nb = f < F ? feat_bins[f] : C;
        B2F_REQUIRE(nb >= 1 && nb <= 256, "packed_layout: field %d has %d values", f, nb);
        width[f] = bits(nb - 1);
        order[f] = f;
    }
    for (int i = 1; i <= F; ++i) {                           // stable sort by width, widest first
        const int f = order[i]; int k = i - 1;
        while (k >= 0 && width[order[k]] < width[f]) { order[k + 1] = order[k]; --k; }
        order[k + 1] = f;
    }
    int nw = 0;
    for (int i = 0; i <= F; ++i) {                           // first fit: no field crosses a 32-bit word
        const int f = order[i];
        int w = 0;
        while (w < nw && used[w] + width[f] > 32) ++w;
        if (w == nw) used[nw++] = 0;
        desc[f] = w | (used[w] << 8) | (((1 << width[f]) - 1) << 16);
        used[w] += width[f];
    }
    const int bytes = (nw * 4 + 15) / 16 * 16;
    // packed only when it saves at least one 16-byte granule of the staged byte record, up to kPackedMaxBytes
    *rec_bytes = bytes <= kPackedMaxBytes && bytes + 16 <= route_pitch(F) * kGran ? bytes : 0;
    return B200FLOW_OK;
}

extern "C" int b200flow_route_hist_config(int32_t F, int32_t m, int32_t n_bins, int32_t C, int32_t rec_bytes, int32_t* chunk_rows,
                                          int32_t* m_pass) {
    RouteCfg cfg;
    if (rec_bytes < 0 || !route_cfg(F, rec_bytes > 0 ? rec_bytes : route_pitch(F) * kGran, rec_bytes > 0, m, n_bins, C, &cfg)) return 0;
    if (chunk_rows) *chunk_rows = cfg.nw * cfg.ks * 32;
    if (m_pass) *m_pass = cfg.m_pass;
    return 1;
}

extern "C" int b200flow_route_hist_level(const uint8_t* tp, int32_t tp_stride, int32_t F, const int32_t* field_desc,
                                         const void* ent, void* ent_out,
                                         int32_t n_slots, const int64_t* seg_begin, const int64_t* seg_end, const int64_t* chunk_off,
                                         const int64_t* n_chunks_dev, int64_t n_chunks_max, int32_t chunk_rows,
                                         const b200flow_split* split, const int32_t* child_slot,
                                         int32_t* cursors, void* chunk_scratch, const uint16_t* subset_next, int32_t m, int32_t n_bins,
                                         int32_t C, uint32_t* hist_next, int32_t flags, void* stream) {
    B2F_REQUIRE(tp && ent && seg_begin && seg_end && chunk_off && n_chunks_dev && split && child_slot && chunk_scratch &&
                    subset_next && hist_next, "route_hist_level: null pointer");
    const bool route = (flags & 1) != 0;
    B2F_REQUIRE(!route || (ent_out && cursors && ((uintptr_t)cursors & 7) == 0), "route_hist_level: routing needs ent_out and 8-byte aligned cursors");
    if (field_desc)
        B2F_REQUIRE((tp_stride & 15) == 0 && tp_stride > 0 && tp_stride <= kPackedMaxBytes && ((uintptr_t)tp & 15) == 0,
                    "route_hist_level: packed records must be 16-byte multiples up to %d bytes, 16-byte aligned", kPackedMaxBytes);
    else
        B2F_REQUIRE((tp_stride & 15) == 0 && tp_stride >= (F + 1 + 15) / 16 * 16 && ((uintptr_t)tp & 15) == 0, "route_hist_level: bad TreePoint stride/alignment");
    B2F_REQUIRE(((uintptr_t)chunk_scratch & 15) == 0, "route_hist_level: chunk_scratch must be 16-byte aligned");
    RouteCfg cfg;
    const int rs = field_desc ? tp_stride : route_pitch(F) * kGran;
    B2F_REQUIRE(route_cfg(F, rs, field_desc != nullptr, m, n_bins, C, &cfg), "route_hist_level: one feature's child histograms exceed shared memory (use partition_level + hist_level)");
    B2F_REQUIRE(chunk_rows == cfg.nw * cfg.ks * 32, "route_hist_level: chunk_rows must be the value of b200flow_route_hist_config (%d)", cfg.nw * cfg.ks * 32);
    if (n_slots <= 0 || n_chunks_max <= 0) return B200FLOW_OK;
    cudaStream_t st = (cudaStream_t)stream;
    RouteChunk* chunks = (RouteChunk*)chunk_scratch;
    route_chunks_kernel<<<(unsigned)((n_chunks_max + 255) / 256), 256, 0, st>>>(chunk_off, n_slots, n_chunks_dev, seg_begin,
                                                                             seg_end, chunk_rows, chunks);
    RouteArgs a;
    a.tp = tp; a.stride = tp_stride; a.F = F; a.field_desc = field_desc; a.ent = (const b2f_entry*)ent; a.ent_out = (b2f_entry*)ent_out; a.chunks = chunks; a.n_chunks_dev = n_chunks_dev;
    a.seg_begin = seg_begin; a.seg_end = seg_end; a.split = split; a.child_slot = child_slot; a.cursors = cursors;
    a.subset_next = subset_next; a.m_total = m; a.n_bins = n_bins; a.C = C; a.hist_next = hist_next;
    static int waves = -1;                                    // CTAs per resident slot: > 1 lets the block scheduler even out the tail
    if (waves < 0) { const char* e = getenv("B200FLOW_ROUTE_WAVES"); waves = e ? atoi(e) : 2; if (waves < 1) waves = 1; }
    for (int j0 = 0, pass = 0; j0 < m; j0 += cfg.m_pass, ++pass) {
        a.j0 = j0; a.m = m - j0 < cfg.m_pass ? m - j0 : cfg.m_pass; a.route = (route && pass == 0) ? 1 : 0;
        const int M = a.m <= 12 ? a.m : 0;
        const size_t smem = route_hist_smem(rs, field_desc != nullptr, a.m, n_bins, C, cfg.nw, cfg.ks);
        cudaError_t e;
        switch (field_desc ? tp_stride / 16 : 0) {               // packed: granules per record, a compile-time gather geometry
            case 1: e = route_shape<1>(cfg, M, smem, waves, n_chunks_max, a, st); break;
            case 2: e = route_shape<2>(cfg, M, smem, waves, n_chunks_max, a, st); break;
            case 3: e = route_shape<3>(cfg, M, smem, waves, n_chunks_max, a, st); break;
            case 4: e = route_shape<4>(cfg, M, smem, waves, n_chunks_max, a, st); break;
            default: e = route_shape<0>(cfg, M, smem, waves, n_chunks_max, a, st); break;
        }
        if (e != cudaSuccess) { set_error("route_hist_level: %s", cudaGetErrorString(e)); return B200FLOW_ERR_CUDA; }
    }
    return check_launch("route_hist_level");
}
