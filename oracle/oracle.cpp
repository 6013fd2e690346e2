// oracle.cpp — CPU restatement of the MLlib algorithms on the hot path.
//
// TEST INFRASTRUCTURE ONLY.  Nothing under spark-network-traffic-classifier_b200/
// may import, link or execute this file; only tests/, __graft_entry__.smoke() and
// bench.py's cpu_baseline / --impl reference legs use it, as the checker / CPU arm.
//
// PARITY UNPINNED: the reference (/root/reference/code/*.py) contains no arithmetic,
// no tests and no golden vectors; every number comes from Apache Spark MLlib (JVM,
// un-vendored, un-pinned, >= 2.4.0 because cicids17.py:41 uses
// VectorAssembler.setHandleInvalid).  There is no JVM/pyspark in this image, so the
// oracle is pinned only against the upstream doctest known answers listed in
// SURVEY.md §4 (tests/test_oracle_known_answers.py).  Each function cites the
// reference call site it serves and the upstream algorithm it restates
// (SURVEY.md Appendix A).
//
// RNG-dependent steps use the build's own counter-based spec (Philox4x32-10 keyed by
// (seed, purpose), counted by global row / (tree, node)), because Spark's streams
// (XORShiftRandom, commons-math Poisson, java.util.Random) are irreproducible outside
// a JVM (SURVEY.md §0 F9).
//
// Build: g++ -O2 -ffp-contract=off -fopenmp -shared -fPIC oracle.cpp -o _build/liboracle.so

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <limits>
#include <vector>
#ifdef _OPENMP
#include <omp.h>
#endif

namespace {

// ------------------------------------------------------------------ Philox4x32-10
struct U4 { uint32_t x, y, z, w; };

inline U4 philox(uint32_t k0, uint32_t k1, uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3) {
    const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
    for (int r = 0; r < 10; ++r) {
        uint64_t p0 = (uint64_t)M0 * c0, p1 = (uint64_t)M1 * c2;
        uint32_t hi0 = (uint32_t)(p0 >> 32), lo0 = (uint32_t)p0;
        uint32_t hi1 = (uint32_t)(p1 >> 32), lo1 = (uint32_t)p1;
        uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
        c0 = n0; c1 = n1; c2 = n2; c3 = n3;
        k0 += W0; k1 += W1;
    }
    return {c0, c1, c2, c3};
}

const uint32_t PURPOSE_SAMPLE = 0x53414D50u;  // 'SAMP' findSplits row sample
const uint32_t PURPOSE_BAG    = 0x42414747u;  // 'BAGG' Poisson bagging
const uint32_t PURPOSE_FEAT   = 0x46454154u;  // 'FEAT' per-node feature subset
const uint32_t PURPOSE_RSPLIT = 0x5253504Cu;  // 'RSPL' DataFrame.randomSplit

inline U4 philox_keyed(uint64_t seed, uint32_t purpose, uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3) {
    return philox((uint32_t)seed ^ purpose, (uint32_t)(seed >> 32), c0, c1, c2, c3);
}

struct Slot {           // mirrors b200flow_slot (include/b200flow.h) — layout only
    int32_t kind, src_off, lut_off, lut_len, hot, reserved;
    double mean, scale;
};

// Gini.calculate (spark: mllib/tree/impurity/Gini.scala): 1 - Σ (c_k/tot)², loop order kept
inline double gini(const double* c, int C, double tot) {
    if (tot == 0.0) return 0.0;
    double imp = 1.0;
    for (int k = 0; k < C; ++k) { double f = c[k] / tot; imp -= f * f; }
    return imp;
}

struct Node {
    int32_t tree; uint32_t nid;
    int32_t feat, kind, bin_thr, is_leaf;
    double gain, impurity;
    uint64_t mask[4];
    int32_t left, right;                  // indices into Forest::nodes
    std::vector<int64_t> counts;
};

struct Forest {
    int T, C, F;
    std::vector<Node> nodes;              // per tree contiguous, BFS order
    std::vector<int64_t> tree_begin;      // T+1
};

struct TrainParams {
    int F, C, stride, max_depth, min_instances, m, n_bins;
    double min_info_gain;
    uint64_t seed;
    const int32_t* feat_bins;
    const int32_t* feat_kind;             // 0 continuous, 1 ordered categorical, 2 unordered categorical
};

struct Best { int feat = -1, kind = 0, bin_thr = 0; double gain = -std::numeric_limits<double>::max();
              uint64_t mask[4] = {0, 0, 0, 0}; std::vector<double> L, R; };

// RandomForest.calculateImpurityStats (A.5): returns gain or -DBL_MAX when invalid
inline double impurity_gain(const double* L, const double* R, int C, double parent_imp,
                            int min_inst, double min_gain) {
    double lc = 0, rc = 0;
    for (int k = 0; k < C; ++k) { lc += L[k]; rc += R[k]; }
    if (lc < (double)min_inst || rc < (double)min_inst) return -std::numeric_limits<double>::max();
    double tot = lc + rc;
    double gl = gini(L, C, lc), gr = gini(R, C, rc);
    double lw = lc / tot, rw = rc / tot;
    double gain = parent_imp - lw * gl - rw * gr;
    if (gain < min_gain) return -std::numeric_limits<double>::max();
    return gain;
}

// RandomForest.binsToBestSplit (A.5) for one node. hist layout [m][n_bins][C] (counts as int64)
void best_split(const std::vector<int64_t>& hist, const std::vector<int>& subset,
                const TrainParams& P, const std::vector<double>& parent, double parent_imp, Best& best) {
    const int C = P.C, NB = P.n_bins;
    std::vector<double> L(C), R(C), cum((size_t)NB * C);
    for (size_t j = 0; j < subset.size(); ++j) {
        const int f = subset[j];
        const int nb = P.feat_bins[f], kind = P.feat_kind[f];
        const int64_t* h = &hist[j * (size_t)NB * C];
        double fbest = -std::numeric_limits<double>::max(); int fs = -1;
        uint64_t fmask[4] = {0, 0, 0, 0};
        std::vector<double> fL(C), fR(C);
        if (kind == 0) {                               // continuous: prefix over bins
            std::fill(L.begin(), L.end(), 0.0);
            for (int s = 0; s < nb - 1; ++s) {
                for (int k = 0; k < C; ++k) { L[k] += (double)h[s * C + k]; R[k] = parent[k] - L[k]; }
                double g = impurity_gain(L.data(), R.data(), C, parent_imp, P.min_instances, P.min_info_gain);
                if (g > fbest) { fbest = g; fs = s; fL = L; fR = R; }
            }
        } else if (kind == 1) {                        // ordered categorical: sort by centroid (stable)
            std::vector<double> cen(nb);
            std::vector<double> cs(C);
            for (int c = 0; c < nb; ++c) {
                double cnt = 0;
                for (int k = 0; k < C; ++k) { cs[k] = (double)h[c * C + k]; cnt += cs[k]; }
                if (cnt == 0) cen[c] = std::numeric_limits<double>::max();
                else if (C > 2) cen[c] = gini(cs.data(), C, cnt);   // multiclass: category impurity
                else cen[c] = cs[1];                                 // binary: count of class 1
            }
            std::vector<int> order(nb);
            for (int c = 0; c < nb; ++c) order[c] = c;
            std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return cen[a] < cen[b]; });
            std::fill(L.begin(), L.end(), 0.0);
            uint64_t m[4] = {0, 0, 0, 0};
            for (int s = 0; s < nb - 1; ++s) {
                int c = order[s];
                m[c >> 6] |= (uint64_t)1 << (c & 63);
                for (int k = 0; k < C; ++k) { L[k] += (double)h[c * C + k]; R[k] = parent[k] - L[k]; }
                double g = impurity_gain(L.data(), R.data(), C, parent_imp, P.min_instances, P.min_info_gain);
                if (g > fbest) { fbest = g; fs = s; fL = L; fR = R; memcpy(fmask, m, sizeof(m)); }
            }
        } else {                                       // unordered categorical: subset splits
            int ns = (1 << (nb - 1)) - 1;
            for (int s = 0; s < ns; ++s) {
                unsigned bits = (unsigned)(s + 1);
                for (int k = 0; k < C; ++k) L[k] = 0.0;
                for (int c = 0; c < nb; ++c)
                    if ((bits >> c) & 1u) for (int k = 0; k < C; ++k) L[k] += (double)h[c * C + k];
                for (int k = 0; k < C; ++k) R[k] = parent[k] - L[k];
                double g = impurity_gain(L.data(), R.data(), C, parent_imp, P.min_instances, P.min_info_gain);
                if (g > fbest) { fbest = g; fs = s; fL = L; fR = R; fmask[0] = bits; fmask[1] = fmask[2] = fmask[3] = 0; }
            }
        }
        if (fs >= 0 && fbest > best.gain) {            // first max over features (subset order)
            best.gain = fbest; best.feat = f; best.kind = (kind == 0) ? 0 : 1; best.bin_thr = fs;
            memcpy(best.mask, fmask, sizeof(fmask)); best.L = fL; best.R = fR;
        }
    }
}

void feature_subset(uint64_t seed, int tree, uint32_t nid, int F, int m, std::vector<int>& out) {
    out.resize(m);
    if (m >= F) { for (int i = 0; i < F; ++i) out[i] = i; return; }
    std::vector<int> perm(F);
    for (int i = 0; i < F; ++i) perm[i] = i;
    U4 r{0, 0, 0, 0};
    for (int i = 0; i < m; ++i) {
        if ((i & 3) == 0) r = philox_keyed(seed, PURPOSE_FEAT, (uint32_t)tree, nid, (uint32_t)(i >> 2), 0);
        uint32_t w = (i & 3) == 0 ? r.x : (i & 3) == 1 ? r.y : (i & 3) == 2 ? r.z : r.w;
        int j = i + (int)(w % (uint32_t)(F - i));
        std::swap(perm[i], perm[j]);
    }
    for (int i = 0; i < m; ++i) out[i] = perm[i];
    std::sort(out.begin(), out.end());
}

struct Entry { int32_t row; uint8_t w; };

void train_tree(int t, const uint8_t* tp, const std::vector<Entry>& bag, const TrainParams& P,
                std::vector<Node>& out) {
    const int C = P.C, NB = P.n_bins;
    struct Work { int node; std::vector<Entry> ent; int level; };
    std::vector<Work> cur, nxt;
    Node root{}; root.tree = t; root.nid = 1; root.feat = -1; root.is_leaf = 1; root.left = root.right = -1;
    root.counts.assign(C, 0);
    for (const Entry& e : bag) root.counts[tp[(size_t)e.row * P.stride + P.F]] += e.w;
    out.push_back(root);
    if (P.max_depth > 0) cur.push_back({0, bag, 0});
    else {
        std::vector<double> pc(C); double tot = 0;
        for (int k = 0; k < C; ++k) { pc[k] = (double)root.counts[k]; tot += pc[k]; }
        out[0].impurity = gini(pc.data(), C, tot);
    }
    std::vector<int> subset;
    while (!cur.empty()) {
        nxt.clear();
        for (Work& wk : cur) {
            feature_subset(P.seed, t, out[wk.node].nid, P.F, P.m, subset);
            std::vector<int64_t> hist(subset.size() * (size_t)NB * C, 0);
            for (const Entry& e : wk.ent) {            // HOT LOOP A: DTStatsAggregator.update
                const uint8_t* r = tp + (size_t)e.row * P.stride;
                int lab = r[P.F];
                for (size_t j = 0; j < subset.size(); ++j)
                    hist[(j * NB + r[subset[j]]) * C + lab] += e.w;
            }
            std::vector<double> parent(C); double tot = 0;
            for (int k = 0; k < C; ++k) { parent[k] = (double)out[wk.node].counts[k]; tot += parent[k]; }
            double pimp = gini(parent.data(), C, tot);
            Best b;
            best_split(hist, subset, P, parent, pimp, b);   // HOT LOOP B
            Node& nd = out[wk.node];
            nd.impurity = pimp; nd.gain = b.gain;
            bool leaf = !(b.gain > 0.0) || wk.level == P.max_depth;
            if (leaf) { nd.is_leaf = 1; nd.feat = -1; continue; }
            nd.is_leaf = 0; nd.feat = b.feat; nd.kind = b.kind; nd.bin_thr = b.bin_thr;
            memcpy(nd.mask, b.mask, sizeof(b.mask));
            double lc = 0, rc = 0;
            for (int k = 0; k < C; ++k) { lc += b.L[k]; rc += b.R[k]; }
            double gl = gini(b.L.data(), C, lc), gr = gini(b.R.data(), C, rc);
            bool lleaf = (wk.level + 1 == P.max_depth) || gl == 0.0;
            bool rleaf = (wk.level + 1 == P.max_depth) || gr == 0.0;
            Node l{}, r{};
            l.tree = r.tree = t; l.nid = nd.nid * 2; r.nid = nd.nid * 2 + 1;
            l.feat = r.feat = -1; l.is_leaf = r.is_leaf = 1; l.left = l.right = r.left = r.right = -1;
            l.impurity = gl; r.impurity = gr;
            l.counts.resize(C); r.counts.resize(C);
            for (int k = 0; k < C; ++k) { l.counts[k] = (int64_t)b.L[k]; r.counts[k] = (int64_t)b.R[k]; }
            int li = (int)out.size(), ri = li + 1;
            int feat = b.feat, kind = b.kind, thr = b.bin_thr;
            uint64_t mask[4]; memcpy(mask, b.mask, sizeof(mask));
            out[wk.node].left = li; out[wk.node].right = ri;
            out.push_back(l); out.push_back(r);        // invalidates nd
            Work wl{li, {}, wk.level + 1}, wr{ri, {}, wk.level + 1};
            for (const Entry& e : wk.ent) {
                int bin = tp[(size_t)e.row * P.stride + feat];
                bool goleft = kind == 0 ? (bin <= thr) : ((mask[bin >> 6] >> (bin & 63)) & 1u);
                if (goleft) { if (!lleaf) wl.ent.push_back(e); } else { if (!rleaf) wr.ent.push_back(e); }
            }
            if (!lleaf) nxt.push_back(std::move(wl));
            if (!rleaf) nxt.push_back(std::move(wr));
        }
        cur.swap(nxt);
    }
}

}  // namespace

extern "C" {

void orc_philox(uint64_t seed, uint32_t purpose, uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t* out4) {
    U4 r = philox_keyed(seed, purpose, c0, c1, c2, c3);
    out4[0] = r.x; out4[1] = r.y; out4[2] = r.z; out4[3] = r.w;
}

// explicit thread count: torchrun exports OMP_NUM_THREADS=1 to its workers, which would silently serialise the CPU arm
void orc_set_num_threads(int n) {
#ifdef _OPENMP
    if (n > 0) omp_set_num_threads(n);
#else
    (void)n;
#endif
}

int orc_num_threads() {
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}

// R1 StringIndexer.fit — counting half (kdd99.py:34-37): occurrences per dictionary code
void orc_category_counts(const uint8_t* records, int64_t n, int32_t row_bytes, int32_t src_off,
                         int32_t K, int64_t* counts) {
    for (int64_t i = 0; i < n; ++i) {
        int32_t code; memcpy(&code, records + i * row_bytes + src_off, 4);
        if (code >= 0 && code < K) counts[code]++;
    }
}

// R2+R3+R3b+R3c (kdd99.py:37,46; cicids17.py:42,46; A.7): index lookup, one-hot, scale, assemble
void orc_encode(const uint8_t* records, int64_t n, int32_t row_bytes, const Slot* plan, int32_t n_out,
                const int32_t* lut, int32_t label_off, int32_t label_lut_off, int32_t label_lut_len,
                int32_t check_nan, double* out, int32_t* label_out, uint8_t* valid_out) {
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < n; ++i) {
        const uint8_t* r = records + i * row_bytes;
        bool ok = true;
        for (int d = 0; d < n_out; ++d) {
            const Slot& s = plan[d];
            double v = 0.0;
            if (s.kind == 0) { float x; memcpy(&x, r + s.src_off, 4); v = (double)x; if (check_nan && std::isnan(v)) ok = false; }
            else if (s.kind == 1) { memcpy(&v, r + s.src_off, 8); if (check_nan && std::isnan(v)) ok = false; }
            else if (s.kind == 2) { int32_t x; memcpy(&x, r + s.src_off, 4); v = (double)x; }
            else {
                int32_t code; memcpy(&code, r + s.src_off, 4);
                int32_t rank = (code >= 0 && code < s.lut_len) ? lut[s.lut_off + code] : -1;
                if (rank < 0) ok = false;
                v = (s.kind == 3) ? (double)rank : (rank == s.hot ? 1.0 : 0.0);
            }
            out[i * n_out + d] = (v - s.mean) * s.scale;
        }
        if (label_off >= 0) {
            int32_t code; memcpy(&code, r + label_off, 4);
            int32_t rank = (code >= 0 && code < label_lut_len) ? lut[label_lut_off + code] : -1;
            if (rank < 0) ok = false;
            if (label_out) label_out[i] = rank;
        }
        if (valid_out) valid_out[i] = ok ? 1 : 0;
    }
}

// R3c StandardScaler.fit (A.7): mean and unbiased std per column, two-pass fp64
void orc_moments(const double* x, int64_t n, int32_t D, double* mean, double* stdev) {
    for (int d = 0; d < D; ++d) {
        double s = 0;
        for (int64_t i = 0; i < n; ++i) s += x[i * D + d];
        double mu = n ? s / (double)n : 0.0, m2 = 0, c = 0;
        for (int64_t i = 0; i < n; ++i) { double dlt = x[i * D + d] - mu; m2 += dlt * dlt; c += dlt; }
        m2 -= c * c / (double)(n ? n : 1);
        mean[d] = mu;
        stdev[d] = n > 1 ? std::sqrt(m2 / (double)(n - 1)) : 0.0;
    }
}

// R4 RandomForest.findSplits + findSplitsForContinuousFeature (A.2), fit call site kdd99.py:79
// x: dense [n][F] fp64; arity[f] == 0 continuous.  thresholds [F][max_bins-1], n_thr[F].
void orc_find_splits(const double* x, int64_t n, int32_t F, uint64_t seed, uint64_t keep_threshold,
                     int64_t row_offset, const int32_t* arity, int32_t max_bins,
                     double* thresholds, int32_t* n_thr, int32_t* n_sampled_out) {
    std::vector<int64_t> rows;
    for (int64_t i = 0; i < n; ++i) {
        uint64_t g = (uint64_t)(row_offset + i);
        U4 r = philox_keyed(seed, PURPOSE_SAMPLE, (uint32_t)g, (uint32_t)(g >> 32), 0, 0);
        if ((uint64_t)r.x < keep_threshold) rows.push_back(i);
    }
    if (n_sampled_out) *n_sampled_out = (int32_t)rows.size();
    const int num_splits = max_bins - 1;
    for (int f = 0; f < F; ++f) {
        n_thr[f] = 0;
        if (arity[f] > 0 || rows.empty()) continue;
        std::vector<double> v(rows.size());
        for (size_t i = 0; i < rows.size(); ++i) v[i] = x[rows[i] * F + f];
        std::sort(v.begin(), v.end());
        std::vector<double> val; std::vector<int64_t> cnt;
        for (double a : v) { if (!val.empty() && val.back() == a) cnt.back()++; else { val.push_back(a); cnt.push_back(1); } }
        int possible = (int)val.size() - 1;
        double* thr = thresholds + (size_t)f * num_splits;
        int nt = 0;
        if (possible == 0) { /* constant */ }
        else if (possible <= num_splits) {
            for (int i = 1; i <= possible; ++i) thr[nt++] = (val[i - 1] + val[i]) / 2.0;
        } else {
            double stride = (double)v.size() / (double)(num_splits + 1);
            double cur = (double)cnt[0], target = stride;
            for (size_t i = 1; i < val.size(); ++i) {
                double prev = cur; cur += (double)cnt[i];
                if (std::fabs(prev - target) < std::fabs(cur - target)) {
                    if (nt < num_splits) thr[nt++] = (val[i - 1] + val[i]) / 2.0;
                    target += stride;
                }
            }
        }
        n_thr[f] = nt;
    }
}

// R5 TreePoint.findBin (A.3)
void orc_bin_rows(const double* x, int64_t n, int32_t F, const double* thresholds, const int32_t* n_thr,
                  const int32_t* arity, int32_t max_bins, const int32_t* labels,
                  uint8_t* tp, int32_t stride, int32_t* bad_rows) {
    int bad = 0;
#pragma omp parallel for schedule(static) reduction(+ : bad)
    for (int64_t i = 0; i < n; ++i) {
        uint8_t* r = tp + i * stride;
        bool rowbad = false;
        for (int f = 0; f < F; ++f) {
            double v = x[i * F + f];
            if (arity[f] > 0) {
                int b = (int)v;
                if (!((double)b == v) || b < 0 || b >= arity[f]) { rowbad = true; b = arity[f] < 255 ? arity[f] : 255; }   // bin `arity` is no category when arity <= 255 (build_metadata refuses 256): not in any left set, goes right
                r[f] = (uint8_t)b;
            } else {
                const double* thr = thresholds + (size_t)f * (max_bins - 1);
                int lo = 0, hi = n_thr[f];                 // first b with v <= thr[b]
                while (lo < hi) { int mid = (lo + hi) >> 1; if (v <= thr[mid]) hi = mid; else lo = mid + 1; }
                r[f] = (uint8_t)lo;
            }
        }
        for (int f = F; f < stride; ++f) r[f] = 0;
        if (labels) r[F] = (uint8_t)labels[i];
        if (rowbad) bad++;
    }
    if (bad_rows) *bad_rows = bad;
}

// R6 BaggedPoint (A.4): w[t][i] = #{k : cdf[k] != 2^32-1 and r >= cdf[k]}, r = word tree%4 of philox(seed,'BAGG', global row, tree/4)
void orc_bag_weights(uint64_t seed, int32_t T, int64_t row_offset, int64_t n, const uint32_t* cdf, uint8_t* w) {
#pragma omp parallel for schedule(static)
    for (int t = 0; t < T; ++t)
        for (int64_t i = 0; i < n; ++i) {
            if (!cdf) { w[(size_t)t * n + i] = 1; continue; }
            uint64_t g = (uint64_t)(row_offset + i);
            U4 r4 = philox_keyed(seed, PURPOSE_BAG, (uint32_t)g, (uint32_t)(g >> 32), (uint32_t)(t >> 2), 0);   // one call serves 4 trees
            uint32_t r = (t & 3) == 0 ? r4.x : (t & 3) == 1 ? r4.y : (t & 3) == 2 ? r4.z : r4.w;
            int k = 0;
            for (int j = 0; j < 32; ++j) k += (cdf[j] != 0xFFFFFFFFu && r >= cdf[j]) ? 1 : 0;   // saturated thresholds are unreachable
            w[(size_t)t * n + i] = (uint8_t)k;
        }
}

void orc_feature_subset(uint64_t seed, int32_t tree, uint32_t nid, int32_t F, int32_t m, int32_t* out) {
    std::vector<int> s; feature_subset(seed, tree, nid, F, m, s);
    for (int i = 0; i < m; ++i) out[i] = s[i];
}

// one node's histogram (R7) for direct kernel tests: entries (row,w) -> hist[m][n_bins][C]
void orc_hist_node(const uint8_t* tp, int32_t stride, int32_t F, const int32_t* rows, const uint8_t* w,
                   int64_t n_ent, const int32_t* subset, int32_t m, int32_t n_bins, int32_t C, int64_t* hist) {
    for (int64_t e = 0; e < n_ent; ++e) {
        const uint8_t* r = tp + (size_t)rows[e] * stride;
        for (int j = 0; j < m; ++j) hist[((size_t)j * n_bins + r[subset[j]]) * C + r[F]] += w[e];
    }
}

// R7+R8 RandomForest.run (A.1, A.5): level-wise growth of T trees on binned rows; w[T][n] bag weights
void* orc_rf_train(const uint8_t* tp, int64_t n, int32_t F, int32_t stride, int32_t C, int32_t T,
                   const uint8_t* w, const int32_t* feat_bins, const int32_t* feat_kind, int32_t n_bins,
                   int32_t m, int32_t max_depth, int32_t min_instances, double min_info_gain, uint64_t seed) {
    Forest* fo = new Forest; fo->T = T; fo->C = C; fo->F = F;
    TrainParams P{F, C, stride, max_depth, min_instances, m, n_bins, min_info_gain, seed, feat_bins, feat_kind};
    std::vector<std::vector<Node>> per(T);
#pragma omp parallel for schedule(dynamic, 1)
    for (int t = 0; t < T; ++t) {
        std::vector<Entry> bag;
        for (int64_t i = 0; i < n; ++i) { uint8_t wi = w[(size_t)t * n + i]; if (wi) bag.push_back({(int32_t)i, wi}); }
        train_tree(t, tp, bag, P, per[t]);
    }
    fo->tree_begin.push_back(0);
    for (int t = 0; t < T; ++t) {
        int64_t base = (int64_t)fo->nodes.size();
        for (Node& nd : per[t]) { if (nd.left >= 0) { nd.left += (int32_t)base; nd.right += (int32_t)base; } fo->nodes.push_back(std::move(nd)); }
        fo->tree_begin.push_back((int64_t)fo->nodes.size());
    }
    return fo;
}

int64_t orc_forest_num_nodes(void* h) { return (int64_t)((Forest*)h)->nodes.size(); }

// canonical export, nodes ordered by (tree, nid)
void orc_forest_export(void* h, int32_t* tree, uint32_t* nid, int32_t* feat, int32_t* kind, int32_t* bin_thr,
                       int32_t* is_leaf, double* gain, double* impurity, uint64_t* mask, int64_t* counts) {
    Forest* fo = (Forest*)h;
    for (size_t i = 0; i < fo->nodes.size(); ++i) {
        const Node& nd = fo->nodes[i];
        tree[i] = nd.tree; nid[i] = nd.nid; feat[i] = nd.feat; kind[i] = nd.kind; bin_thr[i] = nd.bin_thr;
        is_leaf[i] = nd.is_leaf; gain[i] = nd.gain; impurity[i] = nd.impurity;
        for (int k = 0; k < 4; ++k) mask[i * 4 + k] = nd.is_leaf ? 0 : nd.mask[k];
        for (int k = 0; k < fo->C; ++k) counts[i * fo->C + k] = nd.counts[k];
    }
}

// R9 predictRaw / raw2probability / raw2prediction (A.6), call site kdd99.py:82
void orc_rf_predict(void* h, const uint8_t* tp, int64_t n, int32_t stride, int32_t dt_mode,
                    double* raw, double* prob, double* pred) {
    Forest* fo = (Forest*)h; const int C = fo->C;
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < n; ++i) {
        const uint8_t* r = tp + i * stride;
        std::vector<double> votes(C, 0.0);
        for (int t = 0; t < fo->T; ++t) {
            const Node* nd = &fo->nodes[fo->tree_begin[t]];
            while (!nd->is_leaf) {
                int bin = r[nd->feat];
                bool goleft = nd->kind == 0 ? (bin <= nd->bin_thr) : ((nd->mask[bin >> 6] >> (bin & 63)) & 1u);
                nd = &fo->nodes[goleft ? nd->left : nd->right];
            }
            double tot = 0; for (int k = 0; k < C; ++k) tot += (double)nd->counts[k];
            if (dt_mode) { for (int k = 0; k < C; ++k) votes[k] += (double)nd->counts[k]; }
            else if (tot != 0) { for (int k = 0; k < C; ++k) votes[k] += (double)nd->counts[k] / tot; }
        }
        double s = 0; int arg = 0;
        for (int k = 0; k < C; ++k) { s += votes[k]; if (votes[k] > votes[arg]) arg = k; }
        for (int k = 0; k < C; ++k) {
            if (raw) raw[i * C + k] = votes[k];
            if (prob) prob[i * C + k] = s != 0 ? votes[k] / s : 0.0;
        }
        pred[i] = (double)arg;
    }
}

void orc_forest_free(void* h) { delete (Forest*)h; }

// R10 MulticlassMetrics (A.8) from a confusion matrix cm[label*C+pred]:
// out = {accuracy, weightedPrecision, weightedRecall, weightedF1, macroF1}
void orc_metrics(const int64_t* cm, int32_t C, double* out) {
    double N = 0, tp_sum = 0, wp = 0, wr = 0, wf = 0, mf = 0; int nlab = 0;
    for (int i = 0; i < C * C; ++i) N += (double)cm[i];
    for (int l = 0; l < C; ++l) {
        double sup = 0, predl = 0, tp = (double)cm[l * C + l];
        for (int k = 0; k < C; ++k) { sup += (double)cm[l * C + k]; predl += (double)cm[k * C + l]; }
        if (sup == 0) continue;                          // labels = distinct TRUE labels
        double p = predl == 0 ? 0.0 : tp / predl, r = tp / sup;
        double f1 = (p + r == 0) ? 0.0 : 2.0 * p * r / (p + r);
        tp_sum += tp; wp += p * sup / N; wr += r * sup / N; wf += f1 * sup / N; mf += f1; nlab++;
    }
    out[0] = N ? tp_sum / N : 0; out[1] = wp; out[2] = wr; out[3] = wf; out[4] = nlab ? mf / nlab : 0;
}

void orc_confusion(const double* pred, const double* label, int64_t n, int32_t C, int64_t* cm) {
    for (int64_t i = 0; i < n; ++i) {
        int l = (int)label[i], p = (int)pred[i];
        if (l >= 0 && l < C && p >= 0 && p < C) cm[l * C + p]++;
    }
}

// A.9 DataFrame.randomSplit (build rule): split = first k with u < cum[k], u = r * 2^-32
void orc_random_split(uint64_t seed, int64_t row_offset, int64_t n, const double* cum, int32_t n_splits, uint8_t* out) {
    for (int64_t i = 0; i < n; ++i) {
        uint64_t g = (uint64_t)(row_offset + i);
        U4 r = philox_keyed(seed, PURPOSE_RSPLIT, (uint32_t)g, (uint32_t)(g >> 32), 0, 0);
        double u = (double)r.x * 2.3283064365386963e-10;
        int k = 0; while (k < n_splits - 1 && !(u < cum[k])) ++k;
        out[i] = (uint8_t)k;
    }
}

// single-feature split finder for the known-answer tests (SURVEY §4)
int32_t orc_find_splits_1d(const double* samples, int32_t n, int32_t num_splits, double* thr) {
    std::vector<double> x(samples, samples + n);
    std::vector<int32_t> ar(1, 0); int32_t nt = 0;
    std::vector<double> t(num_splits > 0 ? num_splits : 1);
    orc_find_splits(x.data(), n, 1, 0, (uint64_t)1 << 32, 0, ar.data(), num_splits + 1, t.data(), &nt, nullptr);
    for (int i = 0; i < nt; ++i) thr[i] = t[i];
    return nt;
}

// Checks the identity the CUDA split scorer relies on (forest.cu div_rn): for integers 0 <= a <= b, with y = RN(1/b),
// q = RN(a*y), RN(q + (a - b*q)*y) == RN(a/b) (std::fma = one rounding).  Exhaustive for b <= small_b, then n_random random
// pairs below 2^32 and their a/(a+b) forms.  Returns the number of mismatches (0 expected).
int64_t orc_check_shared_reciprocal_division(int32_t small_b, int64_t n_random) {
    auto mdiv = [](double a, double b, double y) { double q = a * y; double r = std::fma(-b, q, a); return std::fma(r, y, q); };
    int64_t bad = 0;
#pragma omp parallel for reduction(+ : bad) schedule(dynamic, 16)
    for (int32_t b = 1; b <= small_b; ++b) {
        const double y = 1.0 / (double)b;
        for (int32_t a = 0; a <= b; ++a) bad += mdiv(a, b, y) != (double)a / (double)b;
    }
#pragma omp parallel for reduction(+ : bad) schedule(static)
    for (int64_t i = 0; i < n_random; ++i) {
        U4 r = philox_keyed(0x1234, 0x44495653u, (uint32_t)i, (uint32_t)(i >> 32), 0, 0);
        uint32_t bb = r.x >> (r.z & 31); if (!bb) bb = 1;
        const uint32_t aa = (uint32_t)(((uint64_t)r.y * ((uint64_t)bb + 1)) >> 32);
        const double a = aa, b = bb, t = a + b;
        bad += mdiv(a, b, 1.0 / b) != a / b;
        bad += mdiv(a, t, 1.0 / t) != a / t;
        bad += mdiv(b, t, 1.0 / t) != b / t;
    }
    return bad;
}

}  // extern "C"
