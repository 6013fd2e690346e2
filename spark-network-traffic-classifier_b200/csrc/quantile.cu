// quantile.cu — per-column statistics, exact rank select and the column transforms of the preprocessing stages
// (Imputer, RobustScaler, MinMaxScaler, MaxAbsScaler, QuantileDiscretizer, Bucketizer; DESIGN.md §5s).
//
// Every kernel reads D columns of an [n] row set through column descriptors (byte offset in the row, dtype f32 / f64 /
// i32) and one row stride in bytes, so a contiguous or strided matrix and the fields of raw AoS records are read in place.
// The grid-stride loop steps over a whole number of rows of D elements, so a thread keeps one column for its whole loop:
// per-column totals stay in registers and are flushed once per thread.
//
// Statistics (b200flow_column_stats, b200flow_column_sums) are order-independent integers: counts, min / max / max |x|
// as ordered 64-bit keys (Java's Double.compare: -0.0 < 0.0), and the exact 128-bit fixed-point sum of regression.cu's
// grid.  Integer all-reduces of them give the same bits for any world size.
//
// Rank select (b200flow_quantile_hist, b200flow_quantile_step) is an MSB radix select over the ordered keys, 8 passes of
// 8-bit digits.  Each target (column, rank) carries the key prefix found so far; the targets of a column with equal
// prefixes share one group and one 256-bin digit histogram.  A pass counts, for every non-missing value whose key prefix
// is a group's, its next digit in that group's histogram (warp-aggregated with __match_any_sync, so a heavily tied
// column does not serialise a warp on one counter); the caller all-reduces the int64 histograms; one single-block step
// then picks every target's digit, updates its rank within the new prefix and regroups the targets.  The host never
// waits between passes.  The histograms live in shared memory while the pass's group bound fits kQselSmemGroups, else
// in global memory.
#include "radix_sort.cuh"

namespace b200flow {

constexpr int kQThreads = 256;
constexpr int kQselSmemGroups = 48;                          // 48 groups x 256 bins x 4 B = 48 KB of shared histograms
constexpr int kQStepThreads = 1024;
constexpr unsigned long long kQNone = ~0ull;                 // a key no non-missing value has (it decodes to a NaN)

// value of column descriptor cd = (byte offset, dtype) in row i; an f64 field needs only 4-byte alignment
__device__ __forceinline__ double q_load(const unsigned char* __restrict__ base, int64_t i, int64_t row_bytes, int2 cd) {
    const unsigned char* p = base + i * row_bytes + cd.x;
    if (cd.y == B200FLOW_F32) return (double)__ldg((const float*)p);
    if (cd.y == B200FLOW_I32) return (double)__ldg((const int*)p);
    return __hiloint2double(__ldg((const int*)p + 1), __ldg((const int*)p));
}

__device__ __forceinline__ bool q_missing(double x, int has_missing, double missing) {
    return x != x || (has_missing && x == missing);
}

__device__ __forceinline__ double key_value(unsigned long long k) {
    return __longlong_as_double((long long)((k >> 63) ? (k & ~(1ull << 63)) : ~k));
}

// the thread's column and first row, and the row step, of the column-stable grid-stride loop (rows n0 ... past n when the
// thread has no column)
struct QLoop { int c; int64_t i, step; };
__device__ __forceinline__ QLoop q_loop(int64_t n, int D) {
    const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, total = (int64_t)gridDim.x * blockDim.x;
    const int64_t step = total / D;
    QLoop L;
    L.step = step;
    L.c = (int)(tid % D);
    L.i = tid < step * D ? tid / D : n;
    return L;
}

static int q_grid(int64_t n, int D) {
    const int64_t need = (n * D + kQThreads * 8 - 1) / (kQThreads * 8);
    int64_t g = need < (int64_t)kNumSMs * 8 ? need : (int64_t)kNumSMs * 8;
    const int64_t least = (D + kQThreads - 1) / kQThreads;   // every column needs a thread
    if (g < least) g = least;
    return (int)(g < 1 ? 1 : g);
}

// stats [6][D] int64: count of non-missing values, of +inf, of -inf; min and max ordered key (as key ^ 2^63, so signed
// int64 order is key order); the bits of the largest finite |x|
__global__ void __launch_bounds__(kQThreads) q_stats_kernel(const unsigned char* __restrict__ base, int64_t row_bytes, int64_t n,
                                                            int D, const int2* __restrict__ cols, int has_missing, double missing,
                                                            long long* stats) {
    const QLoop L = q_loop(n, D);
    if (L.i >= n) return;
    const int2 cd = cols[L.c];
    unsigned long long cnt = 0, pinf = 0, ninf = 0;
    long long mn = LLONG_MAX, mx = LLONG_MIN, mabs = 0;
    for (int64_t i = L.i; i < n; i += L.step) {
        const double x = q_load(base, i, row_bytes, cd);
        if (q_missing(x, has_missing, missing)) continue;
        ++cnt;
        const long long k = (long long)(asc_key(x) ^ (1ull << 63));
        mn = k < mn ? k : mn;
        mx = k > mx ? k : mx;
        if (isinf(x)) { pinf += x > 0.0; ninf += x < 0.0; continue; }
        const long long a = __double_as_longlong(fabs(x));
        mabs = a > mabs ? a : mabs;
    }
    if (!cnt) return;
    atomicAdd((unsigned long long*)stats + L.c, cnt);
    if (pinf) atomicAdd((unsigned long long*)stats + D + L.c, pinf);
    if (ninf) atomicAdd((unsigned long long*)stats + 2 * D + L.c, ninf);
    atomicMin(stats + 3 * D + L.c, mn);
    atomicMax(stats + 4 * D + L.c, mx);
    if (mabs) atomicMax(stats + 5 * D + L.c, mabs);
}

__global__ void q_stats_init_kernel(int D, long long* stats) {
    for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < 6 * D; j += gridDim.x * blockDim.x)
        stats[j] = j / D == 3 ? LLONG_MAX : (j / D == 4 ? LLONG_MIN : 0);
}

// limbs [D][4] += the 32-bit limbs of rint(x 2^shift[c]) over column c's finite non-missing values
__global__ void __launch_bounds__(kQThreads) q_sums_kernel(const unsigned char* __restrict__ base, int64_t row_bytes, int64_t n,
                                                           int D, const int2* __restrict__ cols, int has_missing, double missing,
                                                           const int* __restrict__ shift, long long* limbs) {
    const QLoop L = q_loop(n, D);
    if (L.i >= n) return;
    const int2 cd = cols[L.c];
    const int sh = shift[L.c];
    long long acc[4] = {0, 0, 0, 0};
    for (int64_t i = L.i; i < n; i += L.step) {
        const double x = q_load(base, i, row_bytes, cd);
        if (q_missing(x, has_missing, missing) || isinf(x)) continue;
        long long l[4];
        fixed_limbs(x, sh, l);
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[j] += l[j];
    }
#pragma unroll
    for (int j = 0; j < 4; ++j)
        if (acc[j]) atomicAdd((unsigned long long*)limbs + 4 * L.c + j, (unsigned long long)acc[j]);
}

// ---------------------------------------------------------------------------------------------------- rank select
// state int64 [6 T + 2 D + 1] (T targets ordered by column, then rank):
//   rank [T]   the target's rank among the values with its prefix (1-based)
//   pref [T]   the key prefix found so far (the whole key after the last pass)
//   gpref [T]  the prefix of group g
//   value [T]  the selected value (after the last pass)
//   col [T]    the target's column
//   group [T]  the target's group
//   gbeg [D], gend [D]: column c's groups are [gbeg[c], gend[c]) (empty for a column without targets)
//   G [1]      the number of groups
struct QState {
    long long *rank, *col, *group, *gbeg, *gend, *G;
    unsigned long long *pref, *gpref;
    double* value;
};
__host__ __device__ inline QState q_state(long long* s, int64_t T, int D) {
    QState q;
    q.rank = s; q.pref = (unsigned long long*)(s + T); q.gpref = (unsigned long long*)(s + 2 * T);
    q.value = (double*)(s + 3 * T); q.col = s + 4 * T; q.group = s + 5 * T;
    q.gbeg = s + 6 * T; q.gend = s + 6 * T + D; q.G = s + 6 * T + 2 * D;
    return q;
}

// one pass: digit histograms hist [group][256] of the values whose key prefix (the top 8 pass bits) is the group's
template <bool kShared>
__global__ void __launch_bounds__(kQThreads) q_hist_kernel(const unsigned char* __restrict__ base, int64_t row_bytes, int64_t n,
                                                           int D, const int2* __restrict__ cols, int has_missing, double missing,
                                                           const long long* __restrict__ gbeg, const long long* __restrict__ gend,
                                                           const unsigned long long* __restrict__ gpref,
                                                           const long long* __restrict__ G_ptr, int pass,
                                                           unsigned long long* hist) {
    extern __shared__ unsigned int sh_hist[];
    const int G = (int)*G_ptr;
    if (kShared) {
        for (int b = threadIdx.x; b < G * 256; b += blockDim.x) sh_hist[b] = 0;
        __syncthreads();
    }
    const QLoop L = q_loop(n, D);
    const int2 cd = cols[L.c];
    const int g0 = (int)gbeg[L.c], g1 = (int)gend[L.c];
    const int shift = 56 - 8 * pass;
    int64_t i = g0 < g1 ? L.i : n;                              // a column without targets is not read
    for (;; i += L.step) {
        const bool live = i < n;
        if (!__any_sync(0xffffffffu, live)) break;
        int bin = -1;
        if (live) {
            const double x = q_load(base, i, row_bytes, cd);
            if (!q_missing(x, has_missing, missing)) {
                const unsigned long long k = asc_key(x);
                int g = g0;
                if (pass > 0) {                                 // the group whose prefix is k's, if any
                    const unsigned long long pre = k >> (64 - 8 * pass);
                    int lo = g0, hi = g1;
                    while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (gpref[mid] <= pre) lo = mid; else hi = mid; }
                    g = gpref[lo] == pre ? lo : -1;
                }
                if (g >= 0) bin = g * 256 + (int)((k >> shift) & 255);
            }
        }
        const unsigned peers = __match_any_sync(0xffffffffu, bin);
        if (bin >= 0 && lane_id() == __ffs(peers) - 1) {
            if (kShared) atomicAdd(sh_hist + bin, (unsigned)__popc(peers));
            else atomicAdd(hist + bin, (unsigned long long)__popc(peers));
        }
    }
    if (kShared) {
        __syncthreads();
        for (int b = threadIdx.x; b < G * 256; b += blockDim.x)
            if (sh_hist[b]) atomicAdd(hist + b, (unsigned long long)sh_hist[b]);
    }
}

// select == 1: every target takes the digit where its group's cumulative count reaches its rank.  Then (always) the
// targets are regrouped by (column, prefix): targets are ordered by column and rank, so equal prefixes of a column are
// adjacent and group ids are a scan over the run heads.  One block.
__global__ void __launch_bounds__(kQStepThreads) q_step_kernel(int64_t T, const unsigned long long* __restrict__ hist,
                                                               int select, long long* state, int D) {
    const QState q = q_state(state, T, D);
    __shared__ int scan_sh[33];
    if (select) {
        for (int64_t t = threadIdx.x; t < T; t += blockDim.x) {
            const unsigned long long* h = hist + 256 * q.group[t];
            long long r = q.rank[t], below = 0;
            int d = 0;
            for (; d < 255; ++d) {
                const long long c = (long long)h[d];
                if (below + c >= r) break;
                below += c;
            }
            q.rank[t] = r - below;
            q.pref[t] = (q.pref[t] << 8) | (unsigned long long)d;
            q.value[t] = key_value(q.pref[t]);
        }
        __syncthreads();
    }
    long long carry = 0;
    for (int64_t b0 = 0; b0 < T; b0 += blockDim.x) {
        const int64_t t = b0 + threadIdx.x;
        const bool in = t < T;
        const bool first = in && (t == 0 || q.col[t] != q.col[t - 1]);
        const bool head = in && (first || q.pref[t] != q.pref[t - 1]);
        int total;
        const int ex = block_exclusive_scan(head ? 1 : 0, scan_sh, &total);
        if (in) {
            const long long g = carry + ex + (head ? 1 : 0) - 1;
            q.group[t] = g;
            if (head) q.gpref[g] = q.pref[t];
            if (first) q.gbeg[q.col[t]] = g;
            if (t == T - 1 || q.col[t + 1] != q.col[t]) q.gend[q.col[t]] = g + 1;
        }
        carry += total;
        __syncthreads();
    }
    if (threadIdx.x == 0) *q.G = carry;
}

// ---------------------------------------------------------------------------------------------------- transforms
// Spark's Bucketizer.binarySearchForBuckets on column c's splits [split_off[c], split_off[c + 1]): NaN -> the last index
// (the caller refuses or drops NaN rows unless handleInvalid is keep, and flags[i] = 0 marks them), x == the last split ->
// the last bucket, else Arrays.binarySearch's hit, or its insertion point - 1.  A value outside the splits is counted in
// checks[1] (the caller raises); NaN values in checks[0].
__global__ void __launch_bounds__(kQThreads) q_bucketize_kernel(const unsigned char* __restrict__ base, int64_t row_bytes, int64_t n,
                                                                int D, const int2* __restrict__ cols, const double* __restrict__ splits,
                                                                const int* __restrict__ split_off, double* out, unsigned char* flags,
                                                                unsigned long long* checks) {
    const QLoop L = q_loop(n, D);
    const int2 cd = cols[L.c];
    const double* s = splits + (L.i < n ? split_off[L.c] : 0);
    const int64_t K = L.i < n ? split_off[L.c + 1] - split_off[L.c] : 0;
    unsigned long long nan = 0, oob = 0;
    for (int64_t i = L.i; i < n; i += L.step) {
        const double x = q_load(base, i, row_bytes, cd);
        double b;
        if (x != x) {
            b = (double)(K - 1);
            ++nan;
            flags[i] = 0;
        } else if (x == s[K - 1]) {
            b = (double)(K - 2);
        } else {
            const int64_t f = java_binary_search(s, K, x);
            const int64_t ins = -f - 1;
            if (f < 0 && (ins == 0 || ins == K)) { ++oob; b = 0.0; }
            else b = (double)(f >= 0 ? f : ins - 1);
        }
        out[i * D + L.c] = b;
    }
    nan = warp_sum(nan); oob = warp_sum(oob);
    if (lane_id() == 0) {
        if (nan) atomicAdd(checks, nan);
        if (oob) atomicAdd(checks + 1, oob);
    }
}

// Imputer: out[c] (column c's own dtype, contiguous) = the value, or fill_bits[c] (the surrogate already cast to that
// dtype) where the value is missing
__global__ void __launch_bounds__(kQThreads) q_fill_kernel(const unsigned char* __restrict__ base, int64_t row_bytes, int64_t n,
                                                           int D, const int2* __restrict__ cols, int has_missing, double missing,
                                                           const unsigned long long* __restrict__ fill_bits,
                                                           const unsigned long long* __restrict__ outs) {
    const QLoop L = q_loop(n, D);
    if (L.i >= n) return;
    const int2 cd = cols[L.c];
    const unsigned long long fb = fill_bits[L.c];
    unsigned char* o = (unsigned char*)outs[L.c];
    for (int64_t i = L.i; i < n; i += L.step) {
        const bool miss = q_missing(q_load(base, i, row_bytes, cd), has_missing, missing);
        const unsigned char* p = base + i * row_bytes + cd.x;
        if (cd.y == B200FLOW_F64) {
            const unsigned long long v = ((unsigned long long)(unsigned)__ldg((const int*)p + 1) << 32) |
                                         (unsigned)__ldg((const int*)p);
            ((unsigned long long*)o)[i] = miss ? fb : v;
        } else {
            ((unsigned*)o)[i] = miss ? (unsigned)fb : (unsigned)__ldg((const int*)p);
        }
    }
}

// MinMaxScalerModel: out [n][D] f64 = (x - emin[c]) * scale[c] + lo when scale[c] != 0, else constant; NaN stays NaN
__global__ void __launch_bounds__(kQThreads) q_min_max_kernel(const unsigned char* __restrict__ base, int64_t row_bytes, int64_t n,
                                                              int D, const int2* __restrict__ cols, const double* __restrict__ emin,
                                                              const double* __restrict__ scale, double lo, double constant,
                                                              double* out) {
    const QLoop L = q_loop(n, D);
    if (L.i >= n) return;
    const int2 cd = cols[L.c];
    const double e = emin[L.c], s = scale[L.c];
    for (int64_t i = L.i; i < n; i += L.step) {
        const double x = q_load(base, i, row_bytes, cd);
        out[i * D + L.c] = x != x ? x : (s != 0.0 ? (x - e) * s + lo : constant);
    }
}

// ---------------------------------------------------------------------------------------------------- mode
// keys of the non-missing values of one column, -0.0 folded into 0.0 (a value's identity for counting), compacted in
// any order; *count += their number
__global__ void __launch_bounds__(kQThreads) q_mode_keys_kernel(const unsigned char* __restrict__ base, int64_t row_bytes, int64_t n,
                                                                int2 cd, int has_missing, double missing,
                                                                unsigned long long* keys, unsigned long long* count) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;; i += (int64_t)gridDim.x * blockDim.x) {
        const bool live = i < n;
        if (!__any_sync(0xffffffffu, live)) break;
        bool keep = false;
        double x = 0.0;
        if (live) {
            x = q_load(base, i, row_bytes, cd);
            keep = !q_missing(x, has_missing, missing);
        }
        const unsigned ballot = __ballot_sync(0xffffffffu, keep);
        unsigned long long at = 0;
        if (lane_id() == 0 && ballot) at = atomicAdd(count, (unsigned long long)__popc(ballot));
        at = __shfl_sync(0xffffffffu, at, 0);
        if (keep) keys[at + __popc(ballot & ((1u << lane_id()) - 1u))] = asc_key(x == 0.0 ? 0.0 : x);
    }
}

// run heads of the sorted keys (kQNone, the padding, sorts last and starts a run of its own)
__global__ void __launch_bounds__(kQThreads) q_mode_heads_kernel(const unsigned long long* __restrict__ k, int64_t M, int32_t* head) {
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < M; p += (int64_t)gridDim.x * blockDim.x)
        head[p] = p == 0 || k[p - 1] != k[p] ? 1 : 0;
}

__global__ void __launch_bounds__(kQThreads) q_mode_pos_kernel(const int32_t* __restrict__ head, const int64_t* __restrict__ rid,
                                                               int64_t M, int64_t* pos) {
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < M; p += (int64_t)gridDim.x * blockDim.x)
        if (head[p]) pos[rid[p]] = p;
}

// best = max over the runs of (length << 32 | ~run index): the longest run, the first (smallest key) among equals
__global__ void __launch_bounds__(kQThreads) q_mode_runs_kernel(const unsigned long long* __restrict__ k, const int64_t* __restrict__ pos,
                                                                const int64_t* __restrict__ U_ptr, int64_t M, unsigned long long* best) {
    const int64_t U = *U_ptr;
    unsigned long long b = 0;
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < U; r += (int64_t)gridDim.x * blockDim.x) {
        if (k[pos[r]] == kQNone) continue;
        const unsigned long long len = (unsigned long long)((r + 1 < U ? pos[r + 1] : M) - pos[r]);
        const unsigned long long v = (len << 32) | (0xFFFFFFFFull - (unsigned long long)r);
        b = v > b ? v : b;
    }
    if (b) atomicMax(best, b);
}

__global__ void q_mode_result_kernel(const unsigned long long* __restrict__ k, const int64_t* __restrict__ pos,
                                     const unsigned long long* __restrict__ best, double* out) {
    const unsigned long long b = *best;
    out[0] = b ? key_value(k[pos[0xFFFFFFFFull - (b & 0xFFFFFFFFull)]]) : __longlong_as_double(0x7ff8000000000000ll);
    out[1] = (double)(b >> 32);
}

struct QModeScratch { int64_t nb; size_t key1, idx0, idx1, hist, offs, head, rid, pos, best, total; };

static size_t q_align(size_t x) { return (x + 255) & ~(size_t)255; }

static QModeScratch q_mode_layout(int64_t M) {
    QModeScratch L;
    L.nb = radix_blocks(M);
    size_t o = 0;
    auto take = [&](size_t bytes) { const size_t at = o; o += q_align(bytes); return at; };
    L.key1 = take(8 * M); L.idx0 = take(4 * M); L.idx1 = take(4 * M);
    L.hist = take(4 * 256 * L.nb); L.offs = take(8 * 256 * L.nb);
    L.head = take(4 * M); L.rid = take(8 * M); L.pos = take(8 * M); L.best = take(16);
    L.total = o;
    return L;
}

}  // namespace b200flow

using namespace b200flow;

#define Q_COLUMNS_OK(base, row_bytes, n, D, cols)                                                                   \
    B2F_REQUIRE((n) >= 0 && (D) >= 1 && (row_bytes) >= 4 && (row_bytes) % 4 == 0 && (cols) && ((base) || (n) == 0), \
                "quantile: n >= 0 rows of D >= 1 columns, a row stride that is a positive multiple of 4 bytes")

extern "C" int b200flow_column_stats(const void* base, int64_t row_bytes, int64_t n, int32_t D, const int32_t* cols,
                                     int32_t has_missing, double missing, int64_t* stats, void* stream) {
    Q_COLUMNS_OK(base, row_bytes, n, D, cols);
    B2F_REQUIRE(stats, "column_stats: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    q_stats_init_kernel<<<(6 * D + 255) / 256, 256, 0, st>>>(D, (long long*)stats);
    if (n) q_stats_kernel<<<q_grid(n, D), kQThreads, 0, st>>>((const unsigned char*)base, row_bytes, n, D, (const int2*)cols,
                                                               has_missing, missing, (long long*)stats);
    return check_launch("column_stats");
}

extern "C" int b200flow_column_sums(const void* base, int64_t row_bytes, int64_t n, int32_t D, const int32_t* cols,
                                    int32_t has_missing, double missing, const int32_t* shift, int64_t* limbs, void* stream) {
    Q_COLUMNS_OK(base, row_bytes, n, D, cols);
    B2F_REQUIRE(shift && limbs && n < ((int64_t)1 << 31), "column_sums: bad arguments, or 2^31 rows or more");
    if (n) q_sums_kernel<<<q_grid(n, D), kQThreads, 0, (cudaStream_t)stream>>>((const unsigned char*)base, row_bytes, n, D,
                                                                                (const int2*)cols, has_missing, missing, shift,
                                                                                (long long*)limbs);
    return check_launch("column_sums");
}

extern "C" int b200flow_quantile_hist(const void* base, int64_t row_bytes, int64_t n, int32_t D, const int32_t* cols,
                                      int32_t has_missing, double missing, int64_t T, int64_t* state, int32_t pass,
                                      int64_t group_bound, int64_t* hist, void* stream) {
    Q_COLUMNS_OK(base, row_bytes, n, D, cols);
    B2F_REQUIRE(T >= 1 && state && hist && pass >= 0 && pass < 8 && group_bound >= 1 && group_bound <= T,
                "quantile_hist: T >= 1 targets, 0 <= pass < 8, 1 <= group_bound <= T");
    cudaStream_t st = (cudaStream_t)stream;
    cudaMemsetAsync(hist, 0, (size_t)group_bound * 256 * 8, st);
    if (n == 0) return check_launch("quantile_hist");
    const QState q = q_state((long long*)state, T, D);
    const unsigned char* b = (const unsigned char*)base;
    const int grid = q_grid(n, D);
    if (group_bound <= kQselSmemGroups)
        q_hist_kernel<true><<<grid, kQThreads, (size_t)group_bound * 256 * 4, st>>>(
            b, row_bytes, n, D, (const int2*)cols, has_missing, missing, q.gbeg, q.gend, q.gpref, q.G, pass,
            (unsigned long long*)hist);
    else
        q_hist_kernel<false><<<grid, kQThreads, 0, st>>>(b, row_bytes, n, D, (const int2*)cols, has_missing, missing, q.gbeg,
                                                         q.gend, q.gpref, q.G, pass, (unsigned long long*)hist);
    return check_launch("quantile_hist");
}

extern "C" int b200flow_quantile_step(int64_t T, int32_t D, int64_t* state, const int64_t* hist, int32_t select, void* stream) {
    B2F_REQUIRE(T >= 1 && D >= 1 && state && (hist || !select), "quantile_step: bad arguments");
    q_step_kernel<<<1, kQStepThreads, 0, (cudaStream_t)stream>>>(T, (const unsigned long long*)hist, select, (long long*)state, D);
    return check_launch("quantile_step");
}

extern "C" int b200flow_bucketize(const void* base, int64_t row_bytes, int64_t n, int32_t D, const int32_t* cols,
                                  const double* splits, const int32_t* split_off, double* out, uint8_t* flags, int64_t* checks,
                                  void* stream) {
    Q_COLUMNS_OK(base, row_bytes, n, D, cols);
    B2F_REQUIRE(splits && split_off && checks && (n == 0 || (out && flags)), "bucketize: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    cudaMemsetAsync(checks, 0, 16, st);
    if (n == 0) return check_launch("bucketize");
    cudaMemsetAsync(flags, 1, (size_t)n, st);
    q_bucketize_kernel<<<q_grid(n, D), kQThreads, 0, st>>>((const unsigned char*)base, row_bytes, n, D, (const int2*)cols, splits,
                                                           split_off, out, flags, (unsigned long long*)checks);
    return check_launch("bucketize");
}

extern "C" int b200flow_impute_fill(const void* base, int64_t row_bytes, int64_t n, int32_t D, const int32_t* cols,
                                    int32_t has_missing, double missing, const uint64_t* fill_bits, const uint64_t* outs,
                                    void* stream) {
    Q_COLUMNS_OK(base, row_bytes, n, D, cols);
    B2F_REQUIRE(fill_bits && outs, "impute_fill: bad arguments");
    if (n) q_fill_kernel<<<q_grid(n, D), kQThreads, 0, (cudaStream_t)stream>>>((const unsigned char*)base, row_bytes, n, D,
                                                                                (const int2*)cols, has_missing, missing,
                                                                                (const unsigned long long*)fill_bits,
                                                                                (const unsigned long long*)outs);
    return check_launch("impute_fill");
}

extern "C" int b200flow_min_max(const void* base, int64_t row_bytes, int64_t n, int32_t D, const int32_t* cols,
                                const double* emin, const double* scale, double lo, double constant, double* out, void* stream) {
    Q_COLUMNS_OK(base, row_bytes, n, D, cols);
    B2F_REQUIRE(emin && scale && (out || n == 0), "min_max: bad arguments");
    if (n) q_min_max_kernel<<<q_grid(n, D), kQThreads, 0, (cudaStream_t)stream>>>((const unsigned char*)base, row_bytes, n, D,
                                                                                   (const int2*)cols, emin, scale, lo,
                                                                                   constant, out);
    return check_launch("min_max");
}

extern "C" int b200flow_mode_keys(const void* base, int64_t row_bytes, int64_t n, const int32_t* col, int32_t has_missing,
                                  double missing, uint64_t* keys, int64_t* count, void* stream) {
    B2F_REQUIRE(n >= 0 && row_bytes >= 4 && row_bytes % 4 == 0 && col && count && ((base && keys) || n == 0),
                "mode_keys: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    cudaMemsetAsync(count, 0, 8, st);
    if (n) q_mode_keys_kernel<<<grid_for(n, kQThreads * 8, kNumSMs * 8), kQThreads, 0, st>>>(
        (const unsigned char*)base, row_bytes, n, make_int2(col[0], col[1]), has_missing, missing,
        (unsigned long long*)keys, (unsigned long long*)count);
    return check_launch("mode_keys");
}

extern "C" int b200flow_mode_scratch(int64_t M, int64_t* scratch_bytes) {
    B2F_REQUIRE(scratch_bytes && M >= 0 && M <= 0xFFFFFFFFll, "mode_scratch: 0 <= M < 2^32 keys");
    *scratch_bytes = (int64_t)q_mode_layout(M).total;
    return B200FLOW_OK;
}

extern "C" int b200flow_mode(uint64_t* keys, int64_t M, void* scratch, int64_t scratch_bytes, double* out, void* stream) {
    B2F_REQUIRE(keys && out && M >= 1 && M <= 0xFFFFFFFFll, "mode: 1 <= M < 2^32 keys");
    const QModeScratch L = q_mode_layout(M);
    B2F_REQUIRE(scratch && ((uintptr_t)scratch & 255) == 0 && scratch_bytes >= (int64_t)L.total,
                "mode: scratch must be 256-byte aligned and hold mode_scratch() bytes");
    cudaStream_t st = (cudaStream_t)stream;
    char* s = (char*)scratch;
    unsigned long long* key[2] = {(unsigned long long*)keys, (unsigned long long*)(s + L.key1)};
    uint32_t* idx[2] = {(uint32_t*)(s + L.idx0), (uint32_t*)(s + L.idx1)};
    int32_t* head = (int32_t*)(s + L.head);
    int64_t* rid = (int64_t*)(s + L.rid);
    int64_t* pos = (int64_t*)(s + L.pos);
    unsigned long long* best = (unsigned long long*)(s + L.best);
    int64_t* U = (int64_t*)(s + L.best + 8);
    cudaMemsetAsync(idx[0], 0, 4 * (size_t)M, st);
    cudaMemsetAsync(best, 0, 16, st);
    int cur = 0;
    for (int pass = 0; pass < 8; ++pass, cur ^= 1) {
        const int rc = radix_pass<false>(key[cur], idx[cur], M, 1, 8 * pass, (int32_t*)(s + L.hist), (int64_t*)(s + L.offs),
                                         key[cur ^ 1], idx[cur ^ 1], stream);
        if (rc) return rc;
    }
    const int grid = grid_for(M, kQThreads * 8, kNumSMs * 16);
    q_mode_heads_kernel<<<grid, kQThreads, 0, st>>>(key[cur], M, head);
    const int rc = b200flow_exclusive_scan_i32_to_i64(head, M, rid, U, stream);
    if (rc) return rc;
    q_mode_pos_kernel<<<grid, kQThreads, 0, st>>>(head, rid, M, pos);
    q_mode_runs_kernel<<<grid, kQThreads, 0, st>>>(key[cur], pos, U, M, best);
    q_mode_result_kernel<<<1, 1, 0, st>>>(key[cur], pos, best, out);
    return check_launch("mode");
}
