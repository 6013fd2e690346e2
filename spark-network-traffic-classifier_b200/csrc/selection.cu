// selection.cu — the chi-square, ANOVA and F-value tests behind feature selection, DESIGN.md §5i.
//
// b200flow_distinct_values: each warp stages 32 rows x 16 columns in shared memory, then walks the columns with one row per
// lane.  Lanes holding the same key (__match_any_sync) send one of them to the table, and the slot is read before the CAS,
// so a one-hot or indexed column, whose lanes nearly always agree, costs one load per 32 rows once its keys are in.
// b200flow_contingency_counts: one thread per (row, column) value finds the value's index in its column's sorted dictionary
// by binary search (dictionaries in shared memory when they fit) and counts it into [value][label]; the counters are
// privatised in shared memory when the table is small and flushed with 64-bit atomics, else counted in global memory.
// b200flow_group_centered_moments: one CTA per (4096-row global chunk, slab of columns); a thread owns a column and walks
// the chunk's rows in order, so every sum is sequential in row order.  The group accumulators and centres of the slab sit
// in shared memory.
#include "common.cuh"

namespace b200flow {

namespace {

constexpr int kChunkRows = 4096;
constexpr int kSelMaxW = 256;
constexpr int kSelMaxGroups = 256;
constexpr int kDvSlots = 1 << 15;                 // per column: more than three times the 10000 keys a column may hold
constexpr int kDvMaxKeys = 10000;                 // mllib's maxCategories
constexpr unsigned long long kDvEmpty = 0xFFFFFFFFFFFFFFFFull;
constexpr int kDvWarps = 8, kDvCols = 16;
constexpr int kCtThreads = 256;
constexpr int64_t kCtMaxCells = 1ll << 26;        // 512 MiB of int64 counters
constexpr int kCtPrivBytes = 64 << 10;            // counters privatised in shared memory up to this size
constexpr int kGmSmemBytes = 96 << 10;            // accumulators + centres of one slab

__device__ __forceinline__ unsigned long long value_key(double v) {
    const unsigned long long k = (unsigned long long)__double_as_longlong(v);
    return k == 0x8000000000000000ull ? 0ull : k;  // -0.0 and +0.0 are one category
}

__device__ __forceinline__ void dv_insert(unsigned long long* tab, unsigned long long key, int* count, int* overflow) {
    unsigned s = (unsigned)((key * 0x9E3779B97F4A7C15ull) >> 49);
    for (int probe = 0; probe < kDvSlots; ++probe, s = (s + 1) & (kDvSlots - 1)) {
        unsigned long long cur = *(volatile unsigned long long*)(tab + s);   // look before the CAS
        if (cur == key) return;
        if (cur == kDvEmpty) {
            cur = atomicCAS(tab + s, kDvEmpty, key);
            if (cur == kDvEmpty) {
                if (atomicAdd(count, 1) >= kDvMaxKeys) atomicExch(overflow, 1);
                return;
            }
            if (cur == key) return;
        }
    }
    atomicExch(overflow, 1);                      // every slot holds another key
}

__global__ void __launch_bounds__(kDvWarps * 32) distinct_values_kernel(const double* __restrict__ x, int64_t n, int W, int64_t ld,
                                                                         unsigned long long* tables, int* counts, int* overflow) {
    __shared__ double tile[kDvWarps][32][kDvCols + 1];
    const int lane = lane_id(), wp = warp_id();
    const int64_t n_tiles = (n + 31) / 32;
    for (int64_t t = (int64_t)blockIdx.x * kDvWarps + wp; t < n_tiles; t += (int64_t)gridDim.x * kDvWarps) {
        const int64_t r0 = t * 32;
        const int rows = n - r0 < 32 ? (int)(n - r0) : 32;
        for (int c0 = 0; c0 < W; c0 += kDvCols) {
            const int wc = W - c0 < kDvCols ? W - c0 : kDvCols;
            __syncwarp();                         // the previous columns' reads of the tile are done
            for (int e = lane; e < rows * wc; e += 32) {
                const int r = e / wc, c = e - r * wc;
                tile[wp][r][c] = x[(r0 + r) * ld + c0 + c];
            }
            __syncwarp();
            for (int c = 0; c < wc; ++c) {
                const int w = c0 + c;
                const unsigned long long key = lane < rows ? value_key(tile[wp][lane][c]) : kDvEmpty;
                const unsigned peers = __match_any_sync(0xffffffffu, key);
                const bool leader = key != kDvEmpty && (peers & ((1u << lane) - 1u)) == 0;
                if (leader && !*(volatile int*)(overflow + w))
                    dv_insert(tables + (int64_t)w * kDvSlots, key, counts + w, overflow + w);
            }
        }
    }
}

// first index j in [lo, hi) with d[j] >= v, or hi
__device__ __forceinline__ int lower_bound(const double* d, int lo, int hi, double v) {
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (d[mid] < v) lo = mid + 1; else hi = mid;
    }
    return lo;
}

__global__ void __launch_bounds__(256) dictionary_ids_kernel(const double* __restrict__ v, int64_t n, int64_t ld,
                                                             const double* __restrict__ dict, int L, int* __restrict__ ids) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const double x = v[i * ld];
        const int j = lower_bound(dict, 0, L, x);
        ids[i] = j < L && dict[j] == x ? j : -1;
    }
}

__global__ void __launch_bounds__(kCtThreads) contingency_counts_kernel(const double* __restrict__ x, int64_t n, int W, int64_t ld,
                                                                        const int* __restrict__ label_ids, int L,
                                                                        const double* __restrict__ dicts,
                                                                        const int* __restrict__ dict_off, int n_values,
                                                                        bool dicts_shared, bool priv,
                                                                        unsigned long long* __restrict__ counts) {
    extern __shared__ double ct_sm[];
    unsigned* sc = (unsigned*)ct_sm;              // [n_values][L] when priv
    double* sd = ct_sm + (priv ? ((int64_t)n_values * L + 1) / 2 : 0);   // [n_values] when dicts_shared
    int* so = (int*)(sd + (dicts_shared ? n_values : 0));                 // [W + 1] when dicts_shared
    const int cells = n_values * L;
    if (priv)
        for (int c = threadIdx.x; c < cells; c += kCtThreads) sc[c] = 0u;
    if (dicts_shared) {
        for (int j = threadIdx.x; j < n_values; j += kCtThreads) sd[j] = dicts[j];
        for (int j = threadIdx.x; j <= W; j += kCtThreads) so[j] = dict_off[j];
    }
    __syncthreads();
    const double* d = dicts_shared ? sd : dicts;
    const int* off = dicts_shared ? so : dict_off;
    const int64_t total = n * W;
    for (int64_t e = (int64_t)blockIdx.x * kCtThreads + threadIdx.x; e < total; e += (int64_t)gridDim.x * kCtThreads) {
        const int64_t r = e / W;
        const int w = (int)(e - r * W);
        const int l = label_ids[r];
        if (l < 0 || l >= L) continue;
        const double v = x[r * ld + w];
        const int lo = off[w], hi = off[w + 1];
        const int j = lower_bound(d, lo, hi, v);
        if (j == hi || d[j] != v) continue;
        const int cell = j * L + l;
        if (priv) atomicAdd(sc + cell, 1u);
        else atomicAdd(counts + cell, 1ull);
    }
    if (priv) {
        __syncthreads();
        for (int c = threadIdx.x; c < cells; c += kCtThreads)
            if (sc[c]) atomicAdd(counts + c, (unsigned long long)sc[c]);
    }
}

__global__ void group_centered_moments_kernel(const double* __restrict__ x, int64_t n, int W, int64_t ld,
                                              const int* __restrict__ ids, int G, const double* __restrict__ centers,
                                              const double* __restrict__ y, double yc, int64_t row_offset, int S,
                                              double* __restrict__ partials) {
    extern __shared__ double gm_sm[];
    const int w0 = blockIdx.y * S, ns = W - w0 < S ? W - w0 : S;
    const int t = threadIdx.x, w = w0 + t;
    const int64_t c0 = (row_offset / kChunkRows + blockIdx.x) * kChunkRows - row_offset;   // local index of the chunk's row 0
    const int64_t lo = c0 > 0 ? c0 : 0, hi = c0 + kChunkRows < n ? c0 + kChunkRows : n;
    if (y) {                                      // G == 1: [sq | cross | yy] in registers
        const int Wp = 2 * W + 1;
        double* part = partials + (int64_t)blockIdx.x * Wp;
        if (t < ns) {
            const double c = centers[w];
            double sq = 0.0, cr = 0.0;
            for (int64_t r = lo; r < hi; ++r) {
                const double dx = x[r * ld + w] - c, dy = y[r] - yc;
                sq = sq + dx * dx;
                cr = cr + dx * dy;
            }
            part[w] = sq;
            part[W + w] = cr;
        } else if (t == ns && blockIdx.y == 0) {
            double yy = 0.0;
            for (int64_t r = lo; r < hi; ++r) {
                const double dy = y[r] - yc;
                yy = yy + dy * dy;
            }
            part[2 * W] = yy;
        }
        return;
    }
    double* acc = gm_sm;                          // [G][S]
    double* cs = gm_sm + G * S;                   // [G][S]
    for (int e = t; e < G * S; e += blockDim.x) {
        const int g = e / S, j = e - g * S;
        acc[e] = 0.0;
        cs[e] = j < ns ? centers[(int64_t)g * W + w0 + j] : 0.0;
    }
    __syncthreads();
    if (t < ns) {
        for (int64_t r = lo; r < hi; ++r) {
            const int g = ids ? ids[r] : 0;
            if (g < 0 || g >= G) continue;
            const double d = x[r * ld + w] - cs[g * S + t];
            acc[g * S + t] = acc[g * S + t] + d * d;
        }
        double* part = partials + (int64_t)blockIdx.x * G * W;
        for (int g = 0; g < G; ++g) part[(int64_t)g * W + w] = acc[g * S + t];
    }
}

}  // namespace

}  // namespace b200flow

using namespace b200flow;

extern "C" int b200flow_distinct_values(const double* x, int64_t n_rows, int32_t W, int64_t ld, uint64_t* tables, int32_t* counts,
                                        int32_t* overflow, void* stream) {
    B2F_REQUIRE(W >= 1 && W <= kSelMaxW, "distinct_values: 1 <= W <= %d", kSelMaxW);
    B2F_REQUIRE(n_rows >= 0 && ld >= W, "distinct_values: n >= 0, ld >= W");
    if (n_rows == 0) return B200FLOW_OK;
    B2F_REQUIRE(x && tables && counts && overflow, "distinct_values: null pointer");
    const int blocks = grid_for((n_rows + 31) / 32, kDvWarps, kNumSMs * 8);
    distinct_values_kernel<<<blocks, kDvWarps * 32, 0, (cudaStream_t)stream>>>(x, n_rows, W, ld, (unsigned long long*)tables,
                                                                               counts, overflow);
    return check_launch("distinct_values");
}

extern "C" int b200flow_dictionary_ids(const double* values, int64_t n_rows, int64_t ld, const double* dict, int32_t L, int32_t* ids,
                                       void* stream) {
    B2F_REQUIRE(L >= 1 && L <= kDvMaxKeys, "dictionary_ids: 1 <= L <= %d", kDvMaxKeys);
    B2F_REQUIRE(n_rows >= 0 && ld >= 1, "dictionary_ids: n >= 0, ld >= 1");
    if (n_rows == 0) return B200FLOW_OK;
    B2F_REQUIRE(values && dict && ids, "dictionary_ids: null pointer");
    dictionary_ids_kernel<<<grid_for(n_rows, 256, kNumSMs * 8), 256, 0, (cudaStream_t)stream>>>(values, n_rows, ld, dict, L, ids);
    return check_launch("dictionary_ids");
}

extern "C" int b200flow_contingency_counts(const double* x, int64_t n_rows, int32_t W, int64_t ld, const int32_t* label_ids,
                                           int32_t L, const double* dicts, const int32_t* dict_off, int64_t n_values,
                                           int64_t* counts, void* stream) {
    B2F_REQUIRE(W >= 1 && W <= kSelMaxW && L >= 1 && L <= kSelMaxGroups, "contingency_counts: 1 <= W <= %d, 1 <= L <= %d",
                kSelMaxW, kSelMaxGroups);
    B2F_REQUIRE(n_values >= W && n_values * L <= kCtMaxCells, "contingency_counts: W <= n_values <= 2^26 / L");
    B2F_REQUIRE(n_rows >= 0 && ld >= W, "contingency_counts: n >= 0, ld >= W");
    if (n_rows == 0) return B200FLOW_OK;
    B2F_REQUIRE(x && label_ids && dicts && dict_off && counts, "contingency_counts: null pointer");
    const int64_t cells = n_values * L;
    const bool priv = cells * 4 <= kCtPrivBytes;
    const size_t priv_bytes = priv ? (size_t)(cells + 1) / 2 * sizeof(double) : 0;
    const size_t dict_bytes = (size_t)n_values * sizeof(double) + (size_t)(W + 1) * sizeof(int);
    const bool shared = priv_bytes + dict_bytes <= (size_t)(160 << 10);
    const size_t smem = priv_bytes + (shared ? dict_bytes : 0);
    // a privatised counter takes at most total / blocks + 1 values: keep that below 2^32
    const int64_t total = n_rows * W;
    int blocks = grid_for(total, kCtThreads, kNumSMs * 4);
    if (priv && total / blocks >= 0xFFFFFFFFll) blocks = (int)(total / 0xFFFFFFFFll + 1);
    cudaFuncSetAttribute(contingency_counts_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    contingency_counts_kernel<<<blocks, kCtThreads, smem, (cudaStream_t)stream>>>(x, n_rows, W, ld, label_ids, L, dicts, dict_off,
                                                                                 (int)n_values, shared, priv,
                                                                                 (unsigned long long*)counts);
    return check_launch("contingency_counts");
}

extern "C" int b200flow_group_centered_moments(const double* x, int64_t n_rows, int32_t W, int64_t ld, const int32_t* ids,
                                               int32_t G, const double* centers, const double* y, double y_center,
                                               int64_t row_offset, double* partials, void* stream) {
    B2F_REQUIRE(W >= 1 && W <= kSelMaxW && G >= 1 && G <= kSelMaxGroups, "group_centered_moments: 1 <= W <= %d, 1 <= G <= %d",
                kSelMaxW, kSelMaxGroups);
    B2F_REQUIRE(!y || G == 1, "group_centered_moments: G == 1 with y");
    B2F_REQUIRE(ids || y || G == 1, "group_centered_moments: G == 1 without ids");
    B2F_REQUIRE(n_rows >= 0 && row_offset >= 0 && ld >= W, "group_centered_moments: n >= 0, row_offset >= 0, ld >= W");
    if (n_rows == 0) return B200FLOW_OK;
    const int64_t nc = (row_offset + n_rows - 1) / kChunkRows - row_offset / kChunkRows + 1;
    B2F_REQUIRE(nc <= 0x7fffffffll, "group_centered_moments: too many rows");
    B2F_REQUIRE(x && centers && partials, "group_centered_moments: null pointer");
    int S = y ? W : kGmSmemBytes / (2 * G * (int)sizeof(double));
    if (S > W) S = W;
    const int threads = (S + (y ? 1 : 0) + 31) / 32 * 32;
    const size_t smem = y ? 0 : (size_t)2 * G * S * sizeof(double);
    cudaFuncSetAttribute(group_centered_moments_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    const dim3 grid((unsigned)nc, (unsigned)((W + S - 1) / S));
    group_centered_moments_kernel<<<grid, threads, smem, (cudaStream_t)stream>>>(x, n_rows, W, ld, ids, G, centers, y, y_center,
                                                                                row_offset, S, partials);
    return check_launch("group_centered_moments");
}
