// treeprep.cu — what RandomForest.run does before the level loop (SURVEY.md §8a R4, R5, R6):
//   findSplits sample + findSplitsForContinuousFeature, TreePoint binning, Poisson bagging.
// Reference call sites: classifiers[c].fit(train_set) kdd99.py:79 / cicids17.py:83.
#include <math.h>

#include "common.cuh"

namespace b200flow {

// ------------------------------------------------------------------ exclusive scan
// Small inputs: one CTA.  Large inputs: three launches without extra scratch — (1) every 4096-element block writes its local
// exclusive scan and parks its total in the first slot of the NEXT block (whose local value is always 0), (2) one CTA scans
// those parked totals in place (they become the final value of that slot), (3) every block adds its offset to the rest.
constexpr int kScanBlock = 4096;

__global__ void __launch_bounds__(1024) scan_i32_i64_kernel(const int32_t* __restrict__ in, int64_t n, int64_t* out,
                                                            int64_t* total) {
    __shared__ int sh[33];
    __shared__ long long carry;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (int64_t base = 0; base < n; base += kScanBlock) {
        int64_t i0 = base + (int64_t)threadIdx.x * 4;
        int v[4]; int s = 0;
#pragma unroll
        for (int k = 0; k < 4; ++k) { v[k] = (i0 + k < n) ? in[i0 + k] : 0; s += v[k]; }
        int tot;
        int ex = block_exclusive_scan(s, sh, &tot);
        long long c = carry + ex;
#pragma unroll
        for (int k = 0; k < 4; ++k) { if (i0 + k < n) out[i0 + k] = c; c += v[k]; }
        __syncthreads();
        if (threadIdx.x == 0) carry += tot;
        __syncthreads();
    }
    if (threadIdx.x == 0) { out[n] = carry; if (total) *total = carry; }
}

__global__ void __launch_bounds__(1024) scan_local_kernel(const int32_t* __restrict__ in, int64_t n, int64_t* out) {
    __shared__ int sh[33];
    const int64_t base = (int64_t)blockIdx.x * kScanBlock;
    const int64_t i0 = base + (int64_t)threadIdx.x * 4;
    int v[4]; int s = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) { v[k] = (i0 + k < n) ? in[i0 + k] : 0; s += v[k]; }
    int tot;
    const int ex = block_exclusive_scan(s, sh, &tot);
    long long c = ex;
#pragma unroll
    for (int k = 0; k < 4; ++k) { if (i0 + k < n && (threadIdx.x | k)) out[i0 + k] = c; c += v[k]; }   // slot 0 belongs to the previous block's total
    if (threadIdx.x == 0) {
        if (blockIdx.x == 0) out[0] = 0;
        const int64_t park = min(n, base + kScanBlock);       // first slot of the next block, or out[n] for the last block
        out[park] = tot;
    }
}
__global__ void __launch_bounds__(1024) scan_totals_kernel(int64_t n, int64_t n_blocks, int64_t* out, int64_t* total) {
    __shared__ long long sh_w[32];
    __shared__ long long carry;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (int64_t b0 = 0; b0 < n_blocks; b0 += 1024) {
        const int64_t b = b0 + threadIdx.x;
        const int64_t idx = min(n, (b + 1) * (int64_t)kScanBlock);
        long long v = b < n_blocks ? out[idx] : 0;
        long long inc = v;                                     // warp inclusive scan (64-bit)
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { long long u = __shfl_up_sync(0xffffffffu, inc, o); if (lane_id() >= o) inc += u; }
        if (lane_id() == 31) sh_w[warp_id()] = inc;
        __syncthreads();
        long long woff = 0;
        for (int q = 0; q < warp_id(); ++q) woff += sh_w[q];
        if (b < n_blocks) out[idx] = carry + woff + inc;       // inclusive prefix = offset of block b+1 (= grand total for the last)
        __syncthreads();
        if (threadIdx.x == 1023) carry += woff + inc;
        __syncthreads();
    }
    if (threadIdx.x == 0 && total) *total = out[n];
}
__global__ void __launch_bounds__(1024) scan_add_kernel(int64_t n, int64_t* out) {
    const int64_t base = (int64_t)(blockIdx.x + 1) * kScanBlock;    // block 0 needs no offset
    const long long off = out[base];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int64_t i = base + (int64_t)threadIdx.x * 4 + k;
        if (i < n && (threadIdx.x | k)) out[i] += off;
    }
}

// ------------------------------------------------------------------ R4 sample rows
template <typename T>
__global__ void __launch_bounds__(256) sample_rows_kernel(const T* __restrict__ x, int64_t n, int F, int64_t ld,
                                                          uint64_t seed, uint64_t keep_thr, int64_t row_offset,
                                                          double* sample, int64_t cap, int32_t* n_sampled) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        uint64_t g = (uint64_t)(row_offset + i);
        uint4 r = philox_keyed(seed, PURPOSE_SAMPLE, (uint32_t)g, (uint32_t)(g >> 32), 0u, 0u);
        if ((uint64_t)r.x < keep_thr) {
            int slot = atomicAdd(n_sampled, 1);
            if (slot < cap)
                for (int f = 0; f < F; ++f) sample[(int64_t)f * cap + slot] = (double)x[i * ld + f];
        }
    }
}

// ------------------------------------------------------------------ R4 findSplitsForContinuousFeature
// One CTA per feature: bitonic sort of the (padded to pow2 with +inf) sample column in global/L2,
// then one thread walks the distinct values with MLlib's stride rule.
__global__ void __launch_bounds__(1024) find_splits_kernel(double* sample, int64_t cap, int n_s, int n_pad,
                                                           const int32_t* __restrict__ arity, int max_bins,
                                                           double* thresholds, int32_t* n_thr, const int32_t* __restrict__ n_s_dev) {
    const int f = blockIdx.x;
    if (n_s_dev) n_s = min(*n_s_dev, n_pad);               // the count stays on the device: the host did not wait for it
    __shared__ int sh_distinct;
    if (arity[f] > 0 || n_s <= 0) { if (threadIdx.x == 0) n_thr[f] = 0; return; }
    double* v = sample + (int64_t)f * cap;
    for (int i = n_s + threadIdx.x; i < n_pad; i += blockDim.x) v[i] = INFINITY;
    if (threadIdx.x == 0) sh_distinct = 0;
    __syncthreads();
    for (int k = 2; k <= n_pad; k <<= 1)
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = threadIdx.x; i < n_pad; i += blockDim.x) {
                int p = i ^ j;
                if (p > i) {
                    double a = v[i], b = v[p];
                    bool up = (i & k) == 0;
                    if ((a > b) == up) { v[i] = b; v[p] = a; }
                }
            }
            __syncthreads();
        }
    int local = 0;
    for (int i = 1 + threadIdx.x; i < n_s; i += blockDim.x) local += (v[i] != v[i - 1]) ? 1 : 0;
    local = warp_sum(local);
    if (lane_id() == 0 && local) atomicAdd(&sh_distinct, local);
    __syncthreads();
    if (threadIdx.x != 0) return;
    const int possible = sh_distinct;            // #distinct - 1
    const int num_splits = max_bins - 1;
    double* thr = thresholds + (int64_t)f * num_splits;
    int nt = 0;
    if (possible == 0) {
    } else if (possible <= num_splits) {
        for (int i = 1; i < n_s; ++i)
            if (v[i] != v[i - 1]) thr[nt++] = (v[i - 1] + v[i]) / 2.0;
    } else {
        const double stride = (double)n_s / (double)(num_splits + 1);
        double target = stride;
        // run-length walk: cur = cumulative count up to and including the current distinct value
        int i = 1;
        while (i < n_s && v[i] == v[0]) ++i;
        double cur = (double)i;                   // count of the first distinct value
        while (i < n_s) {
            int j = i + 1;
            while (j < n_s && v[j] == v[i]) ++j;
            const double prev = cur;
            cur += (double)(j - i);
            if (fabs(prev - target) < fabs(cur - target)) {
                if (nt < num_splits) thr[nt++] = (v[i - 1] + v[i]) / 2.0;
                target += stride;
            }
            i = j;
        }
    }
    n_thr[f] = nt;
}

// Shared-memory version (n_pad <= kFindSplitsSmemMax): the column is sorted in shared memory, the run boundaries are
// compacted in parallel, and the stride walk only visits the boundaries it takes: for the current target the predicate
// "|prev - target| < |cur - target|" (prev/cur = cumulative counts before/after a run) is monotone along the boundary list
// (2*target - prev - cur decreases), so the first boundary that satisfies it is found by bisection and then re-checked
// backwards with the very same fp64 predicate — identical thresholds to the sequential walk, ~100x fewer dependent steps.
constexpr int kFindSplitsSmemMax = 16384;

__global__ void __launch_bounds__(1024) find_splits_smem_kernel(const double* __restrict__ sample, int64_t cap, int n_s, int n_pad,
                                                                const int32_t* __restrict__ arity, int max_bins,
                                                                double* thresholds, int32_t* n_thr, const int32_t* __restrict__ n_s_dev) {
    extern __shared__ __align__(8) uint8_t fs_raw[];
    if (n_s_dev) n_s = min(*n_s_dev, n_pad);               // the count stays on the device: the host did not wait for it
    double* v = (double*)fs_raw;                           // [n_pad]
    int* B = (int*)(v + n_pad);                            // [n_pad] start index of every run but the first
    __shared__ int sh[33];
    const int f = blockIdx.x, tid = threadIdx.x, nt_threads = blockDim.x;
    if (arity[f] > 0 || n_s <= 0) { if (tid == 0) n_thr[f] = 0; return; }
    const double* src = sample + (int64_t)f * cap;
    for (int i = tid; i < n_pad; i += nt_threads) v[i] = i < n_s ? src[i] : INFINITY;
    __syncthreads();
    for (int k = 2; k <= n_pad; k <<= 1)
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int t = tid; t < (n_pad >> 1); t += nt_threads) {
                const int i = ((t & ~(j - 1)) << 1) | (t & (j - 1));      // the lower index of the t-th compare-exchange pair
                const int p = i | j;
                const double a = v[i], b = v[p];
                const bool up = (i & k) == 0;
                if ((a > b) == up) { v[i] = b; v[p] = a; }
            }
            __syncthreads();
        }
    // run boundaries, compacted in index order: thread t owns the contiguous slice [t*per, (t+1)*per)
    const int per = (n_s + nt_threads - 1) / nt_threads;
    const int lo = max(1, tid * per), hi = min(n_s, (tid + 1) * per);
    int local = 0;
    for (int i = lo; i < hi; ++i) local += v[i] != v[i - 1] ? 1 : 0;
    int possible;
    int pos = block_exclusive_scan(local, sh, &possible);   // possible = #distinct - 1
    for (int i = lo; i < hi; ++i) if (v[i] != v[i - 1]) B[pos++] = i;
    __syncthreads();
    if (tid != 0) return;
    const int num_splits = max_bins - 1;
    double* thr = thresholds + (int64_t)f * num_splits;
    int nt = 0;
    if (possible == 0) {
    } else if (possible <= num_splits) {
        for (int k = 0; k < possible; ++k) { const int i = B[k]; thr[nt++] = (v[i - 1] + v[i]) / 2.0; }
    } else {
        const double stride = (double)n_s / (double)(num_splits + 1);
        double target = stride;
        auto pred = [&](int k) {                            // run k+1 starts at B[k]: prev = B[k], cur = its end
            const double prev = (double)B[k], cur = (double)(k + 1 < possible ? B[k + 1] : n_s);
            return fabs(prev - target) < fabs(cur - target);
        };
        int k0 = 0;
        while (k0 < possible && nt < num_splits) {
            int a = k0, b = possible;                       // first k in [k0, possible) with pred(k), or possible
            while (a < b) { const int mid = (a + b) >> 1; if (pred(mid)) b = mid; else a = mid + 1; }
            int k = a;
            while (k > k0 && pred(k - 1)) --k;              // fp64 re-check: never skip an earlier boundary the walk would take
            while (k < possible && !pred(k)) ++k;
            if (k >= possible) break;
            const int i = B[k];
            thr[nt++] = (v[i - 1] + v[i]) / 2.0;
            target += stride;
            k0 = k + 1;
        }
    }
    n_thr[f] = nt;
}

// ------------------------------------------------------------------ R5 TreePoint binning
// thread -> (row, feature) with a fixed feature per thread; bins staged in smem, written as 16-byte words.
template <typename T>
__global__ void __launch_bounds__(256) bin_rows_kernel(const T* __restrict__ x, int64_t n, int F, int64_t ld,
                                                       const double* __restrict__ thresholds,
                                                       const int32_t* __restrict__ n_thr, const int32_t* __restrict__ arity,
                                                       int max_bins, const int32_t* __restrict__ labels, uint8_t* tp,
                                                       int stride, int32_t* bad_rows, int R, int thr_in_smem) {
    extern __shared__ __align__(16) uint8_t sm[];
    uint8_t* tile = sm;                                   // [R][stride]
    double* thr_sh = (double*)(sm + (((size_t)R * stride + 15) & ~(size_t)15));
    const int tid = threadIdx.x, bd = blockDim.x, ns = max_bins - 1;
    if (thr_in_smem) for (int i = tid; i < F * ns; i += bd) thr_sh[i] = thresholds[i];
    const double* thr_all = thr_in_smem ? thr_sh : thresholds;
    const int64_t n_tiles = (n + R - 1) / R;
    const bool fixed = F <= bd;
    const int rp = fixed ? bd / F : 1;
    for (int64_t t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        const int64_t rb = t * R;
        const int rows = (int)min((int64_t)R, n - rb);
        __syncthreads();                                  // previous tile written out (and thr_sh ready)
        for (int i = tid; i < rows * stride / 4; i += bd) ((uint32_t*)tile)[i] = 0;   // pad bytes
        __syncthreads();
        if (!fixed || tid < rp * F) {
            for (int f = fixed ? tid % F : tid; f < F; f += fixed ? F : bd) {
                const int ar = arity[f];
                const int nt = n_thr[f];
                const double* thr = thr_all + (int64_t)f * ns;
                for (int r = fixed ? tid / F : 0; r < rows; r += rp) {
                    const double v = (double)x[(rb + r) * ld + f];
                    int b;
                    if (ar > 0) {
                        b = (int)v;
                        if (!((double)b == v) || b < 0 || b >= ar) { b = ar < 255 ? ar : 255; atomicAdd(bad_rows, 1); }   // bin `arity` is no category (arity <= 255, build_metadata): no left-set mask contains it, it routes right
                    } else {
                        int lo = 0, hi = nt;              // lower_bound: first b with v <= thr[b]
                        while (lo < hi) { int mid = (lo + hi) >> 1; if (v <= thr[mid]) hi = mid; else lo = mid + 1; }
                        b = lo;
                    }
                    tile[r * stride + f] = (uint8_t)b;
                }
            }
        }
        if (labels) for (int r = tid; r < rows; r += bd) tile[r * stride + F] = (uint8_t)labels[rb + r];
        __syncthreads();
        uint4* dst = (uint4*)(tp + rb * stride);
        for (int i = tid; i < rows * stride / 16; i += bd) st_stream_u4(dst + i, ((const uint4*)tile)[i]);
    }
}

// ------------------------------------------------------------------ row de-duplication
// Flow records repeat massively (KDD99: 4.9 M rows, ~1.07 M distinct; the smurf/neptune floods are literally the same
// record).  After binning, rows with identical TreePoint records (bins + label) are interchangeable for the trees, so the
// level loop runs on UNIQUE records carrying the summed bag weight of their duplicates — same integer histograms, same
// forest, several times fewer entries.  Open-addressing hash table keyed by the record bytes; the representative of a
// group is its smallest row index (deterministic), unique ids are assigned in representative-row order.
__device__ __forceinline__ uint64_t mix64(uint64_t h, uint64_t v) {
    h ^= v * 0x9E3779B97F4A7C15ull; h ^= h >> 29; h *= 0xBF58476D1CE4E5B9ull; h ^= h >> 32;
    return h;
}
__device__ __forceinline__ bool records_equal(const uint4* a, const uint4* b, int nq) {
    bool eq = true;
    for (int q = 0; q < nq; ++q) { const uint4 x = __ldg(a + q), y = __ldg(b + q); eq = eq && x.x == y.x && x.y == y.y && x.z == y.z && x.w == y.w; }
    return eq;
}

__global__ void __launch_bounds__(256) dedup_insert_kernel(const uint8_t* __restrict__ tp, int64_t n, int stride, int nq,
                                                           int32_t* table, uint32_t cap_mask, int32_t* slot_of) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint4* rec = (const uint4*)(tp + i * stride);
    uint64_t h = 0x243F6A8885A308D3ull;
    for (int q = 0; q < nq; ++q) { const uint4 v = __ldg(rec + q); h = mix64(h, ((uint64_t)v.y << 32) | v.x); h = mix64(h, ((uint64_t)v.w << 32) | v.z); }
    uint32_t slot = (uint32_t)(h ^ (h >> 32)) & cap_mask;
    while (true) {
        int cur = table[slot];
        if (cur < 0) { cur = atomicCAS(&table[slot], -1, (int)i); if (cur < 0) { slot_of[i] = (int)slot; return; } }
        if (records_equal(rec, (const uint4*)(tp + (int64_t)cur * stride), nq)) { slot_of[i] = (int)slot; return; }
        slot = (slot + 1) & cap_mask;
    }
}
__global__ void __launch_bounds__(256) dedup_min_kernel(int64_t n, const int32_t* __restrict__ slot_of, int32_t* minrow) {
    // warp-aggregated: the lowest lane of a duplicate group holds the group's smallest row of this warp, and only it goes to
    // memory — the smurf flood alone is a third of KDD99, i.e. ~10 lanes of every warp hammering ONE address otherwise
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int lane = lane_id();
    const int sl = i < n ? slot_of[i] : -1 - lane;
    const uint32_t g = __match_any_sync(0xffffffffu, sl);
    // a plain read first: once a small row index sits in the slot, later (larger) candidates skip the atomic altogether, so the
    // hot slots (smurf, neptune) take a few hundred atomics instead of one per warp
    if (i < n && (int)(__ffs(g) - 1) == lane && (int)i < *(volatile const int32_t*)&minrow[sl]) atomicMin(&minrow[sl], (int)i);
}
__global__ void __launch_bounds__(256) dedup_flag_kernel(int64_t n, const int32_t* __restrict__ slot_of, const int32_t* __restrict__ minrow,
                                                         int32_t* rep, int32_t* flag) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) { const int r = minrow[slot_of[i]]; rep[i] = r; flag[i] = r == (int)i ? 1 : 0; }
}
__global__ void __launch_bounds__(256) dedup_emit_kernel(const uint8_t* __restrict__ tp, int64_t n, int stride, const int32_t* __restrict__ rep,
                                                         const int64_t* __restrict__ pos, int32_t* uid, uint8_t* tpu) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int r = rep[i];
    const int64_t u = pos[r];
    uid[i] = (int32_t)u;
    if (r == (int)i) {
        const uint4* src = (const uint4*)(tp + i * stride); uint4* dst = (uint4*)(tpu + u * stride);
        for (int q = 0; q < stride / 16; ++q) dst[q] = __ldg(src + q);
    }
}

// rows grouped by unique id (counting sort): perm[p] = row, uperm[p] = its unique id, non-decreasing in p.  With the rows of
// a duplicate group adjacent, bag_weights merges a whole group inside a warp and issues ONE global RED per (warp-run, tree)
// instead of one per row.  Atomics on the group counters are warp-aggregated (match.any on the id).
constexpr int kGroupTab = 256;          // per-CTA direct-mapped (unique id -> pending count) cache of group_count

__global__ void __launch_bounds__(256) group_count_kernel(const int32_t* __restrict__ uid, int64_t n, int32_t* gsize) {
    // persistent CTAs; the warp leaders of a duplicate group add into a small shared-memory cache keyed by the unique id, and
    // only evictions and the final flush touch global memory: a hot group (a third of KDD99 is one smurf record) costs one global
    // atomic per CTA instead of one per warp
    __shared__ int tab_key[kGroupTab];
    __shared__ int tab_cnt[kGroupTab];
    for (int k = threadIdx.x; k < kGroupTab; k += blockDim.x) { tab_key[k] = -1; tab_cnt[k] = 0; }
    __syncthreads();
    const int lane = lane_id();
    const int64_t n_pad = (n + 255) & ~(int64_t)255;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_pad; i += (int64_t)gridDim.x * blockDim.x) {
        const int u = i < n ? uid[i] : -1 - lane;
        const uint32_t g = __match_any_sync(0xffffffffu, u);
        if (i < n && (int)(__ffs(g) - 1) == lane) {
            const int c = __popc(g), h = u & (kGroupTab - 1);
            const int old = atomicCAS(&tab_key[h], -1, u);                 // claim an empty line, or find who owns it
            if (old == -1 || old == u) atomicAdd(&tab_cnt[h], c);
            else atomicAdd(&gsize[u], c);                                   // line taken by another id: straight to global
        }
    }
    __syncthreads();
    for (int k = threadIdx.x; k < kGroupTab; k += blockDim.x)
        if (tab_key[k] >= 0 && tab_cnt[k]) atomicAdd(&gsize[tab_key[k]], tab_cnt[k]);
}
__global__ void __launch_bounds__(256) group_fill_kernel(const int32_t* __restrict__ uid, int64_t n, const int64_t* __restrict__ goff,
                                                         int32_t* cursor, int32_t* perm, int32_t* uperm) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int lane = lane_id();
    const int u = i < n ? uid[i] : -1 - lane;
    const uint32_t g = __match_any_sync(0xffffffffu, u);
    const int leader = __ffs(g) - 1;
    int base = 0;
    if (i < n && leader == lane) base = atomicAdd(&cursor[u], __popc(g));
    base = __shfl_sync(0xffffffffu, base, leader);
    if (i < n) { const int64_t p = goff[u] + base + __popc(g & ((1u << lane) - 1u)); perm[p] = (int32_t)i; uperm[p] = u; }
}

// ------------------------------------------------------------------ R6 bagging
constexpr int kBagBlockRows = 1024;

// W[tree][uid[row]] += Poisson weight of (tree, row).  grid = row blocks of 1024; a thread owns 4 positions and loops over
// the tree quads (one Philox call per row yields the weights of a quad's 4 trees; the duplicate-group search is per row, not per tree).  Lanes whose rows belong to the same duplicate
// group are merged first (match.any on the unique id + three ballots for the weights 1..3), so a hot group — the smurf
// flood is a third of KDD99 — costs one global RED per warp and tree instead of one per row.
// First thresholds of the inverse CDF, passed by value (uniform registers).  n = how many of them are not saturated
// (0xFFFFFFFF): a saturated threshold is unreachable, yet r = 0xFFFFFFFF passes `r >= c[k]`, so the count is clamped to n.
// Small subsampling rates saturate inside the head (Poisson 0.07: c[5]; GBT's Bernoulli CDF: c[1..]).
struct CdfHead { uint32_t c[6]; uint32_t n; };

__device__ __forceinline__ uint32_t poisson_weight_fast(uint32_t r, const CdfHead& h, const uint32_t* cdf_sh) {
    uint32_t k = (r >= h.c[0]) + (r >= h.c[1]) + (r >= h.c[2]) + (r >= h.c[3]) + (r >= h.c[4]) + (r >= h.c[5]);   // increasing thresholds
    k = min(k, h.n);
    if (k == 6) while (k < 32 && cdf_sh[k] != 0xFFFFFFFFu && r >= cdf_sh[k]) ++k;                                 // P(w >= 6) = 6e-4 at lambda = 1
    return k;
}

__global__ void __launch_bounds__(256) bag_weights_kernel(uint64_t seed, int T, int64_t row_offset, int64_t n,
                                                          const uint32_t* __restrict__ cdf, const CdfHead head,
                                                          const int32_t* __restrict__ uid, const int32_t* __restrict__ perm,
                                                          int64_t U, uint32_t* W) {
    __shared__ uint32_t cdf_sh[32];
    const int lane = lane_id();
    if (threadIdx.x < 32) cdf_sh[threadIdx.x] = cdf ? cdf[threadIdx.x] : 0;
    __syncthreads();
    const int n_quads = (T + 3) >> 2;
    // Fast path for the hot duplicate groups: with the rows grouped (perm given, uid sorted along the positions) a CTA whose first
    // and last position carry the same unique id lies entirely inside ONE group — the smurf and neptune floods span thousands of
    // CTAs.  Its 1024 weights per tree are summed in registers, by shuffles and through shared memory, and ONE global RED per tree
    // leaves the CTA (31 x fewer same-address REDs than one per 32-position run).
    {
        const int64_t p_first = (int64_t)blockIdx.x * kBagBlockRows, p_last = min(n, p_first + kBagBlockRows) - 1;
        if (perm && uid && cdf && p_last - p_first + 1 == kBagBlockRows && uid[p_first] == uid[p_last]) {
            __shared__ uint32_t part[8][4];
            const int64_t u = uid[p_first];
            uint64_t grow[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) grow[k] = (uint64_t)(row_offset + (int64_t)perm[p_first + k * 256 + threadIdx.x]);
            for (int tq = 0; tq < n_quads; ++tq) {
                uint32_t w[4] = {0u, 0u, 0u, 0u};
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    const uint4 r = bag_draw4(seed, tq, grow[k]);
                    w[0] += poisson_weight_fast(r.x, head, cdf_sh); w[1] += poisson_weight_fast(r.y, head, cdf_sh);
                    w[2] += poisson_weight_fast(r.z, head, cdf_sh); w[3] += poisson_weight_fast(r.w, head, cdf_sh);
                }
#pragma unroll
                for (int q = 0; q < 4; ++q) w[q] = warp_sum(w[q]);
                if (lane == 0) { part[threadIdx.x >> 5][0] = w[0]; part[threadIdx.x >> 5][1] = w[1]; part[threadIdx.x >> 5][2] = w[2]; part[threadIdx.x >> 5][3] = w[3]; }
                __syncthreads();
                if (threadIdx.x < 4 && tq * 4 + (int)threadIdx.x < T) {
                    uint32_t tot = 0;
                    for (int q = 0; q < 8; ++q) tot += part[q][threadIdx.x];
                    if (tot) atomicAdd(&W[(int64_t)(tq * 4 + threadIdx.x) * U + u], tot);
                }
                __syncthreads();
            }
            return;
        }
    }
    // position p of the (optionally grouped) order: lane-consecutive positions so that a duplicate group is a run of lanes
    const int64_t pb = (int64_t)blockIdx.x * kBagBlockRows + (threadIdx.x >> 5) * 128 + lane;
    for (int k = 0; k < 4; ++k) {
        const int64_t p = pb + k * 32;
        const bool live = p < n;
        const int64_t i = live ? (perm ? (int64_t)perm[p] : p) : 0;          // the row behind position p
        const int64_t u = live ? (uid ? (int64_t)uid[p] : i) : 0;            // uid is given in POSITION order when perm is
        // the row's duplicate group inside this warp step, found ONCE for all trees (dead lanes form singleton groups)
        const uint32_t g = uid ? __match_any_sync(0xffffffffu, live ? (int)u : -1 - lane) : (1u << lane);
        const bool merged = uid && !__all_sync(0xffffffffu, g == (1u << lane));
        const uint64_t grow = (uint64_t)(row_offset + i);
        for (int tq = 0; tq < n_quads; ++tq) {
            uint32_t w[4] = {0u, 0u, 0u, 0u};
            if (live) {
                if (cdf) {
                    const uint4 r = bag_draw4(seed, tq, grow);
                    w[0] = poisson_weight_fast(r.x, head, cdf_sh); w[1] = poisson_weight_fast(r.y, head, cdf_sh);
                    w[2] = poisson_weight_fast(r.z, head, cdf_sh); w[3] = poisson_weight_fast(r.w, head, cdf_sh);
                } else { w[0] = w[1] = w[2] = w[3] = 1u; }
            }
            if (merged) {
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const uint32_t b1 = __ballot_sync(0xffffffffu, w[q] == 1), b2 = __ballot_sync(0xffffffffu, w[q] == 2),
                                   b3 = __ballot_sync(0xffffffffu, w[q] == 3);
                    if (tq * 4 + q >= T || !w[q]) continue;
                    uint32_t* addr = &W[(int64_t)(tq * 4 + q) * U + u];
                    const uint32_t gg = g & (b1 | b2 | b3);
                    if (w[q] > 3) atomicAdd(addr, w[q]);
                    else if ((int)(__ffs(gg) - 1) == lane) atomicAdd(addr, (uint32_t)(__popc(gg & b1) + 2 * __popc(gg & b2) + 3 * __popc(gg & b3)));
                }
            } else {
#pragma unroll
                for (int q = 0; q < 4; ++q)
                    if (tq * 4 + q < T && w[q]) atomicAdd(&W[(int64_t)(tq * 4 + q) * U + u], w[q]);
            }
        }
    }
}

// entries of every tree = its non-zero (unique record, weight) pairs, in unique-id order: count per block, scan, fill
__global__ void __launch_bounds__(256) bag_count_kernel(const uint32_t* __restrict__ W, int64_t U, int32_t* blk_cnt, int64_t n_blocks) {
    __shared__ int cnt_sh;
    const int t = blockIdx.y;
    if (threadIdx.x == 0) cnt_sh = 0;
    __syncthreads();
    const int64_t ub = (int64_t)blockIdx.x * kBagBlockRows + threadIdx.x * 4;
    int c = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) if (ub + k < U && W[(int64_t)t * U + ub + k]) ++c;
    c = warp_sum(c);
    if (lane_id() == 0 && c) atomicAdd(&cnt_sh, c);
    __syncthreads();
    if (threadIdx.x == 0) blk_cnt[(int64_t)t * n_blocks + blockIdx.x] = cnt_sh;
}

__global__ void __launch_bounds__(256) bag_fill_kernel(const uint32_t* __restrict__ W, int64_t U, const int64_t* __restrict__ blk_off,
                                                       int64_t n_blocks, b2f_entry* ent) {
    __shared__ int sh[33];
    const int t = blockIdx.y;
    const int64_t ub = (int64_t)blockIdx.x * kBagBlockRows + threadIdx.x * 4;
    uint32_t w[4]; int c = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) { w[k] = (ub + k < U) ? W[(int64_t)t * U + ub + k] : 0u; c += w[k] ? 1 : 0; }
    int tot;
    const int ex = block_exclusive_scan(c, sh, &tot);
    int64_t pos = blk_off[(int64_t)t * n_blocks + blockIdx.x] + ex;
#pragma unroll
    for (int k = 0; k < 4; ++k)
        if (w[k]) { ent[pos] = make_uint2((uint32_t)(ub + k), w[k]); ++pos; }
}

// byte TreePoint records -> bit-packed records (layout of b200flow_packed_layout): one thread per (record, 32-bit word) ORs in
// the fields placed in its word; the F + 1 bytes of a record are read by the rw threads of that record together.
__global__ void __launch_bounds__(256) pack_records_kernel(const uint8_t* __restrict__ tp, int stride, int64_t n_rows, int F,
                                                           const int32_t* __restrict__ desc, int rw, uint32_t* packed) {
    __shared__ int32_t sh_desc[256];
    for (int f = threadIdx.x; f <= F; f += blockDim.x) sh_desc[f] = desc[f];
    __syncthreads();
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_rows * rw) return;
    const int64_t r = t / rw; const int w = (int)(t - r * rw);
    const uint8_t* rec = tp + r * stride;
    uint32_t v = 0;
    for (int f = 0; f <= F; ++f) {
        const int d = sh_desc[f];
        if ((d & 0xff) == w) v |= ((uint32_t)__ldg(rec + f) & (uint32_t)(d >> 16)) << ((d >> 8) & 0xff);
    }
    packed[t] = v;
}

}  // namespace b200flow

using namespace b200flow;

extern "C" int b200flow_pack_records(const uint8_t* tp, int32_t tp_stride, int64_t n_rows, int32_t F, const int32_t* desc,
                                     int32_t rec_bytes, uint32_t* packed, void* stream) {
    if (n_rows <= 0) return B200FLOW_OK;
    B2F_REQUIRE(tp && desc && packed, "pack_records: null pointer");
    B2F_REQUIRE(F > 0 && F <= 255 && tp_stride >= F + 1 && rec_bytes > 0 && (rec_bytes & 15) == 0, "pack_records: bad shape");
    const int rw = rec_bytes / 4;
    pack_records_kernel<<<(unsigned)((n_rows * rw + 255) / 256), 256, 0, (cudaStream_t)stream>>>(tp, tp_stride, n_rows, F, desc, rw, packed);
    return check_launch("pack_records");
}

extern "C" int b200flow_exclusive_scan_i32_to_i64(const int32_t* in, int64_t n, int64_t* out, int64_t* total, void* stream) {
    B2F_REQUIRE(in && out && n >= 0, "scan: bad arguments");
    if (n <= 16 * kScanBlock) {
        scan_i32_i64_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(in, n, out, total);
    } else {
        const int64_t nb = (n + kScanBlock - 1) / kScanBlock;
        scan_local_kernel<<<(unsigned)nb, 1024, 0, (cudaStream_t)stream>>>(in, n, out);
        scan_totals_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(n, nb, out, total);
        scan_add_kernel<<<(unsigned)(nb - 1), 1024, 0, (cudaStream_t)stream>>>(n, out);
    }
    return check_launch("exclusive_scan");
}

extern "C" int b200flow_sample_rows(const void* x, int32_t dtype, int64_t n_rows, int32_t F, int64_t ld, uint64_t seed,
                                    uint64_t keep_threshold, int64_t row_offset, double* sample, int64_t cap,
                                    int32_t* n_sampled, void* stream) {
    if (n_rows <= 0) return B200FLOW_OK;            // empty batch: nothing to do (pointers may be NULL)
    B2F_REQUIRE(x && sample && n_sampled && F > 0 && ld >= F && cap > 0, "sample_rows: bad arguments");
    int grid = grid_for(n_rows, 256 * 4, kNumSMs * 8);
    if (dtype == B200FLOW_F32)
        sample_rows_kernel<float><<<grid, 256, 0, (cudaStream_t)stream>>>((const float*)x, n_rows, F, ld, seed, keep_threshold, row_offset, sample, cap, n_sampled);
    else if (dtype == B200FLOW_F64)
        sample_rows_kernel<double><<<grid, 256, 0, (cudaStream_t)stream>>>((const double*)x, n_rows, F, ld, seed, keep_threshold, row_offset, sample, cap, n_sampled);
    else { set_error("sample_rows: bad dtype"); return B200FLOW_ERR_ARG; }
    return check_launch("sample_rows");
}

extern "C" int b200flow_find_splits(double* sample, int64_t cap, int32_t n_s, int32_t F, const int32_t* arity,
                                    int32_t max_bins, double* thresholds, int32_t* n_thr, const int32_t* n_s_dev, void* stream) {
    B2F_REQUIRE(sample && arity && thresholds && n_thr && F > 0 && max_bins >= 2 && max_bins <= 256, "find_splits: bad arguments");
    B2F_REQUIRE(n_s >= 0 && n_s <= cap, "find_splits: n_s exceeds cap");
    int n_pad = 1; while (n_pad < n_s) n_pad <<= 1;         // with n_s_dev, n_s is the host's upper bound (the kernels clamp to n_pad)
    B2F_REQUIRE(n_pad <= cap, "find_splits: cap must be >= pow2ceil(n_s)");
    if (n_pad <= kFindSplitsSmemMax) {
        const size_t smem = (size_t)n_pad * 12;
        cudaError_t e = cudaFuncSetAttribute(find_splits_smem_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) { set_error("find_splits: %s", cudaGetErrorString(e)); return B200FLOW_ERR_CUDA; }
        find_splits_smem_kernel<<<F, 1024, smem, (cudaStream_t)stream>>>(sample, cap, n_s, n_pad, arity, max_bins, thresholds, n_thr, n_s_dev);
    } else {
        find_splits_kernel<<<F, 1024, 0, (cudaStream_t)stream>>>(sample, cap, n_s, n_pad, arity, max_bins, thresholds, n_thr, n_s_dev);
    }
    return check_launch("find_splits");
}

extern "C" int b200flow_bin_rows(const void* x, int32_t dtype, int64_t n_rows, int32_t F, int64_t ld,
                                 const double* thresholds, const int32_t* n_thr, const int32_t* arity, int32_t max_bins,
                                 const int32_t* labels, uint8_t* tp, int32_t tp_stride, int32_t* bad_rows, void* stream) {
    if (n_rows <= 0) return B200FLOW_OK;            // empty batch: nothing to do (pointers may be NULL)
    B2F_REQUIRE(x && thresholds && n_thr && arity && tp && bad_rows, "bin_rows: null pointer");
    B2F_REQUIRE(F > 0 && F < 65536 && ld >= F && tp_stride >= F + 1 && (tp_stride & 15) == 0 && max_bins >= 2 && max_bins <= 256,
                "bin_rows: bad shape (F=%d stride=%d max_bins=%d)", F, tp_stride, max_bins);
    B2F_REQUIRE(((uintptr_t)tp & 15) == 0, "bin_rows: tp must be 16-byte aligned");
    size_t thr_bytes = (size_t)F * (max_bins - 1) * 8;
    int thr_in_smem = thr_bytes <= 96 * 1024;
    int R = 4096 / tp_stride; if (R < 8) R = 8; if (R > 128) R = 128;
    size_t smem = (((size_t)R * tp_stride + 15) & ~(size_t)15) + (thr_in_smem ? thr_bytes : 0);
    int64_t n_tiles = (n_rows + R - 1) / R;
    int per_sm = (int)((200 * 1024) / (smem + 1024)); if (per_sm < 1) per_sm = 1; if (per_sm > 8) per_sm = 8;
    int grid = (int)(n_tiles < (int64_t)kNumSMs * per_sm ? n_tiles : (int64_t)kNumSMs * per_sm);
    cudaError_t e;
    if (dtype == B200FLOW_F32) {
        e = cudaFuncSetAttribute(bin_rows_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e == cudaSuccess) bin_rows_kernel<float><<<grid, 256, smem, (cudaStream_t)stream>>>((const float*)x, n_rows, F, ld, thresholds, n_thr, arity, max_bins, labels, tp, tp_stride, bad_rows, R, thr_in_smem);
    } else if (dtype == B200FLOW_F64) {
        e = cudaFuncSetAttribute(bin_rows_kernel<double>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e == cudaSuccess) bin_rows_kernel<double><<<grid, 256, smem, (cudaStream_t)stream>>>((const double*)x, n_rows, F, ld, thresholds, n_thr, arity, max_bins, labels, tp, tp_stride, bad_rows, R, thr_in_smem);
    } else { set_error("bin_rows: bad dtype"); return B200FLOW_ERR_ARG; }
    if (e != cudaSuccess) { set_error("bin_rows: %s", cudaGetErrorString(e)); return B200FLOW_ERR_CUDA; }
    return check_launch("bin_rows");
}

extern "C" int b200flow_dedup_rows(const uint8_t* tp, int64_t n_rows, int32_t tp_stride, int32_t key_bytes, int32_t* table,
                                   int32_t* minrow, int64_t table_cap, int32_t* slot_of, int32_t* rep, int32_t* flag, int64_t* pos,
                                   int64_t* n_unique, int32_t* uid, uint8_t* tp_unique, void* stream) {
    if (n_rows <= 0) return B200FLOW_OK;
    B2F_REQUIRE(tp && table && minrow && slot_of && rep && flag && pos && n_unique && uid && tp_unique, "dedup_rows: null pointer");
    B2F_REQUIRE((tp_stride & 15) == 0 && key_bytes > 0 && key_bytes <= tp_stride && ((uintptr_t)tp & 15) == 0 && ((uintptr_t)tp_unique & 15) == 0,
                "dedup_rows: bad stride/alignment");
    B2F_REQUIRE(table_cap >= 2 * n_rows && (table_cap & (table_cap - 1)) == 0 && table_cap <= ((int64_t)1 << 31), "dedup_rows: table_cap must be a power of two >= 2*n_rows");
    B2F_REQUIRE(n_rows < ((int64_t)1 << 31), "dedup_rows: too many rows");
    cudaStream_t st = (cudaStream_t)stream;
    cudaMemsetAsync(table, 0xFF, (size_t)table_cap * 4, st);            // -1 = empty
    cudaMemsetAsync(minrow, 0x7F, (size_t)table_cap * 4, st);           // 0x7F7F7F7F > any row index
    const unsigned grid = (unsigned)((n_rows + 255) / 256);
    const int nq = (key_bytes + 15) / 16;                               // pad bytes of a TreePoint are zero: whole quads compare equal
    dedup_insert_kernel<<<grid, 256, 0, st>>>(tp, n_rows, tp_stride, nq, table, (uint32_t)(table_cap - 1), slot_of);
    dedup_min_kernel<<<grid, 256, 0, st>>>(n_rows, slot_of, minrow);
    dedup_flag_kernel<<<grid, 256, 0, st>>>(n_rows, slot_of, minrow, rep, flag);
    int rc = b200flow_exclusive_scan_i32_to_i64(flag, n_rows, pos, n_unique, stream);
    if (rc) return rc;
    dedup_emit_kernel<<<grid, 256, 0, st>>>(tp, n_rows, tp_stride, rep, pos, uid, tp_unique);
    return check_launch("dedup_rows");
}

extern "C" int b200flow_group_rows(const int32_t* uid, int64_t n_rows, int64_t n_unique, int32_t* gsize, int64_t* goff, int32_t* cursor,
                                   int32_t* perm, int32_t* uperm, void* stream) {
    if (n_rows <= 0) return B200FLOW_OK;
    B2F_REQUIRE(uid && gsize && goff && cursor && perm && uperm && n_unique > 0, "group_rows: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    cudaMemsetAsync(gsize, 0, (size_t)n_unique * 4, st);
    cudaMemsetAsync(cursor, 0, (size_t)n_unique * 4, st);
    const unsigned grid = (unsigned)((n_rows + 255) / 256);
    group_count_kernel<<<grid_for(n_rows, 256 * 16, kNumSMs * 8), 256, 0, st>>>(uid, n_rows, gsize);
    int rc = b200flow_exclusive_scan_i32_to_i64(gsize, n_unique, goff, nullptr, stream);
    if (rc) return rc;
    group_fill_kernel<<<grid, 256, 0, st>>>(uid, n_rows, goff, cursor, perm, uperm);
    return check_launch("group_rows");
}

extern "C" int b200flow_bag_weights(uint64_t seed, int32_t T, int64_t row_offset, int64_t n_rows, const uint32_t* poisson_cdf,
                                    const uint32_t* poisson_cdf_host, const int32_t* uid, const int32_t* perm, int64_t n_unique,
                                    uint32_t* W, void* stream) {
    if (n_rows <= 0) return B200FLOW_OK;
    B2F_REQUIRE(W && T > 0 && T <= 65535 * 4 && n_unique > 0, "bag_weights: bad arguments");
    B2F_REQUIRE((poisson_cdf == nullptr) == (poisson_cdf_host == nullptr), "bag_weights: pass the CDF table both as device and host pointer");
    CdfHead head;
    head.n = 0;
    for (int k = 0; k < 6; ++k) {
        head.c[k] = poisson_cdf_host ? poisson_cdf_host[k] : 0xFFFFFFFFu;
        if (head.c[k] != 0xFFFFFFFFu && head.n == (uint32_t)k) ++head.n;        // leading non-saturated thresholds
    }
    const int64_t nb = (n_rows + kBagBlockRows - 1) / kBagBlockRows;
    bag_weights_kernel<<<(unsigned)nb, 256, 0, (cudaStream_t)stream>>>(seed, T, row_offset, n_rows, poisson_cdf, head, uid, perm, n_unique, W);
    return check_launch("bag_weights");
}

extern "C" int b200flow_bag_count(const uint32_t* W, int32_t T, int64_t n_unique, int32_t* blk_cnt, void* stream) {
    B2F_REQUIRE(W && blk_cnt && T > 0 && T <= 65535 && n_unique >= 0, "bag_count: bad arguments");
    if (n_unique == 0) return B200FLOW_OK;
    const int64_t nb = (n_unique + kBagBlockRows - 1) / kBagBlockRows;
    bag_count_kernel<<<dim3((unsigned)nb, (unsigned)T), 256, 0, (cudaStream_t)stream>>>(W, n_unique, blk_cnt, nb);
    return check_launch("bag_count");
}

extern "C" int b200flow_bag_fill(const uint32_t* W, int32_t T, int64_t n_unique, const int64_t* blk_off, void* ent, void* stream) {
    B2F_REQUIRE(W && blk_off && ent && T > 0 && T <= 65535 && n_unique >= 0 && ((uintptr_t)ent & 7) == 0, "bag_fill: bad arguments");
    if (n_unique == 0) return B200FLOW_OK;
    const int64_t nb = (n_unique + kBagBlockRows - 1) / kBagBlockRows;
    bag_fill_kernel<<<dim3((unsigned)nb, (unsigned)T), 256, 0, (cudaStream_t)stream>>>(W, n_unique, blk_off, nb, (b2f_entry*)ent);
    return check_launch("bag_fill");
}
