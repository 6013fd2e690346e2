// isotonic.cu — IsotonicRegression (DESIGN.md §5p): Spark's one-partition fit, "makeUnique, PAV, compress, PAV again",
// and its binary-search predict.
//
// b200flow_isotonic_fit: one pass builds order-preserving keys of the features (Java's Double.compare order: -0.0 before
// 0.0) and checks the rows; the shared stable LSD radix sort (radix_sort.cuh) orders them with the row index as payload, so
// equal features keep row order.  Then, twice (the second time over the first pass's output points):
//   - tie pooling: run heads from == on the doubles, one thread per run summing y w and w in sorted order;
//   - chunked pool-adjacent-violators over the U unique points, in place on Spark's blockBounds / weights arrays: level 0
//     runs Spark's loop on each chunk of C points, level L resumes it at the junction of two adjacent 2^(L-1) C ranges
//     (each already monotone) and stops at the first junction block that does not violate its successor;
//   - compression: a scan over the block-head flags that merge clears, one or two output points per block.
// Every sum has one order fixed by (data, C), so the model is bit-reproducible; it equals Spark's sequential PAV to rounding.
//
// b200flow_isotonic_predict: one thread per row, java.util.Arrays.binarySearch (bit-pattern tie-break) and Spark's
// interpolation y1 + (y2 - y1) * (x - x1) / (x2 - x1).
#include "radix_sort.cuh"

namespace b200flow {

// Level-0 chunk of the PAV.  Level 0 costs O(C) per thread and the merge levels add log2(U / C) launches; at 4.9 M unique
// points the fit time was flat from C = 16 to C = 256 on the H100 (DESIGN.md §8 "Isotonic regression"), and 64 sits in
// the middle of that range.
constexpr int kIsoChunk = 64;
constexpr int kIsoThreads = 256;
constexpr unsigned long long kIsoDropped = ~0ull;       // zero-weight or refused rows: sorted last (no finite key equals it)

template <typename T>
__global__ void __launch_bounds__(kIsoThreads) iso_keys_kernel(const void* __restrict__ feat, int64_t fstride,
                                                               const double* __restrict__ label, int64_t lstride,
                                                               const double* __restrict__ weight, int64_t wstride,
                                                               int64_t n, unsigned long long* key, uint32_t* idx,
                                                               unsigned long long* counts) {
    unsigned long long bad = 0, neg = 0, valid = 0;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const double x = load_as_double<T>(feat, i * fstride);
        const double y = __ldg(label + i * lstride);
        const double w = weight ? __ldg(weight + i * wstride) : 1.0;
        const bool finite = isfinite(x) && isfinite(y) && isfinite(w);
        bad += !finite;
        neg += w < 0.0;
        const bool keep = finite && w > 0.0;
        valid += keep;
        key[i] = keep ? asc_key(x) : kIsoDropped;
        idx[i] = (uint32_t)i;
    }
    bad = warp_sum(bad); neg = warp_sum(neg); valid = warp_sum(valid);
    if (lane_id() == 0) {
        if (bad) atomicAdd(counts + 0, bad);
        if (neg) atomicAdd(counts + 1, neg);
        if (valid) atomicAdd(counts + 2, valid);
    }
}

// the kept rows in sorted order: (xs, ys, ws) [V], the label negated for an antitonic fit
template <typename T>
__global__ void __launch_bounds__(kIsoThreads) iso_gather_kernel(const uint32_t* __restrict__ idx, const void* __restrict__ feat,
                                                                 int64_t fstride, const double* __restrict__ label,
                                                                 int64_t lstride, const double* __restrict__ weight,
                                                                 int64_t wstride, bool negate, const int64_t* __restrict__ V_ptr,
                                                                 double* xs, double* ys, double* ws) {
    const int64_t V = *V_ptr;
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < V; p += (int64_t)gridDim.x * blockDim.x) {
        const int64_t i = idx[p];
        const double y = __ldg(label + i * lstride);
        xs[p] = load_as_double<T>(feat, i * fstride);
        ys[p] = negate ? -y : y;
        ws[p] = weight ? __ldg(weight + i * wstride) : 1.0;
    }
}

// run heads of the V sorted points (0 past V): Spark's shouldAccumulate is primitive ==, so -0.0 joins a run of 0.0
__global__ void __launch_bounds__(kIsoThreads) iso_heads_kernel(const double* __restrict__ xs, const int64_t* __restrict__ V_ptr,
                                                                int64_t n, int32_t* head) {
    const int64_t V = *V_ptr;
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (int64_t)gridDim.x * blockDim.x)
        head[p] = p < V && (p == 0 || xs[p - 1] != xs[p]) ? 1 : 0;
}

__global__ void __launch_bounds__(kIsoThreads) iso_head_pos_kernel(const int32_t* __restrict__ head, const int64_t* __restrict__ rid,
                                                                   int64_t n, int64_t* head_pos) {
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (int64_t)gridDim.x * blockDim.x)
        if (head[p]) head_pos[rid[p]] = p;
}

// makeUnique, one thread per run [head, next head): (sum y w / sum w, first feature, sum w), both sums from the run's first
// product in sorted order; then PAV's initial state: weights (w, w y), every point its own block.  Spark returns an input
// of at most one point as it is, so V == 1 keeps the raw label.
__global__ void __launch_bounds__(kIsoThreads) iso_tie_kernel(const double* __restrict__ xs, const double* __restrict__ ys,
                                                              const double* __restrict__ ws, const int64_t* __restrict__ head_pos,
                                                              const int64_t* __restrict__ U_ptr, const int64_t* __restrict__ V_ptr,
                                                              double* ux, double2* wt, int64_t* bb, int32_t* bhead) {
    const int64_t U = *U_ptr, V = *V_ptr;
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < U; r += (int64_t)gridDim.x * blockDim.x) {
        const int64_t p0 = head_pos[r], p1 = r + 1 < U ? head_pos[r + 1] : V;
        double swy = ys[p0] * ws[p0], sw = ws[p0];
        for (int64_t p = p0 + 1; p < p1; ++p) { swy += ys[p] * ws[p]; sw += ws[p]; }
        const double y = V == 1 ? ys[p0] : swy / sw;
        ux[r] = xs[p0];
        wt[r] = make_double2(sw, sw * y);
        bb[r] = r;
        bhead[r] = 1;
    }
}

__device__ __forceinline__ double block_avg(const double2* wt, int64_t s) {
    const double2 v = wt[s];
    return v.y / v.x;
}

// Spark's merge(block1, block2); returns block1.  The head flag of block2 is cleared.
__device__ __forceinline__ int64_t block_merge(double2* wt, int64_t* bb, int32_t* bhead, int64_t b1, int64_t b2) {
    const int64_t e2 = bb[b2];
    bb[b1] = e2;
    bb[e2] = b1;
    const double2 w1 = wt[b1], w2 = wt[b2];
    wt[b1] = make_double2(w1.x + w2.x, w1.y + w2.y);
    bhead[b2] = 0;
    return b1;
}

// after a merge at block i: pool backwards while the previous block's average is >= i's, never past lo
__device__ __forceinline__ int64_t pool_back(double2* wt, int64_t* bb, int32_t* bhead, int64_t lo, int64_t i) {
    while (i > lo && block_avg(wt, bb[i - 1]) >= block_avg(wt, i)) i = block_merge(wt, bb, bhead, bb[i - 1], i);
    return i;
}

// level 0: Spark's loop over the chunk [t C, min((t + 1) C, U))
__global__ void __launch_bounds__(kIsoThreads) iso_pav_chunk_kernel(double2* wt, int64_t* bb, int32_t* bhead,
                                                                    const int64_t* __restrict__ U_ptr, int64_t C) {
    const int64_t U = *U_ptr;
    const int64_t lo = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * C;
    if (lo >= U) return;
    const int64_t hi = lo + C < U ? lo + C : U;
    int64_t i = lo;
    while (bb[i] + 1 < hi) {
        const int64_t nx = bb[i] + 1;
        if (block_avg(wt, i) >= block_avg(wt, nx)) {
            block_merge(wt, bb, bhead, i, nx);
            i = pool_back(wt, bb, bhead, lo, i);
        } else {
            i = nx;
        }
    }
}

// level L: ranges [lo, mid) and [mid, hi) of R = 2^(L-1) C points are each monotone.  The loop resumes at the block that
// ends at mid - 1; that block always spans the junction, so the first time it does not violate its successor, everything
// to its right is an untouched, monotone part of the right range and the loop is done.
__global__ void __launch_bounds__(kIsoThreads) iso_pav_merge_kernel(double2* wt, int64_t* bb, int32_t* bhead,
                                                                    const int64_t* __restrict__ U_ptr, int64_t R) {
    const int64_t U = *U_ptr;
    const int64_t lo = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 2 * R, mid = lo + R;
    if (mid >= U) return;
    const int64_t hi = mid + R < U ? mid + R : U;
    int64_t i = bb[mid - 1];
    while (bb[i] + 1 < hi && block_avg(wt, i) >= block_avg(wt, bb[i] + 1)) {
        block_merge(wt, bb, bhead, i, bb[i] + 1);
        i = pool_back(wt, bb, bhead, lo, i);
    }
}

// output points per block (0 past U and off block heads): two when its first and last features differ, else one
__global__ void __launch_bounds__(kIsoThreads) iso_count_kernel(const double* __restrict__ ux, const int64_t* __restrict__ bb,
                                                                const int32_t* __restrict__ bhead,
                                                                const int64_t* __restrict__ U_ptr, int64_t n, int32_t* cnt) {
    const int64_t U = *U_ptr;
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (int64_t)gridDim.x * blockDim.x)
        cnt[p] = p < U && bhead[p] ? (ux[bb[p]] > ux[p] ? 2 : 1) : 0;
}

// (avg, first feature, W / 2) and (avg, last feature, W / 2), or (avg, feature, W); out_w may be NULL
__global__ void __launch_bounds__(kIsoThreads) iso_emit_kernel(const double* __restrict__ ux, const double2* __restrict__ wt,
                                                               const int64_t* __restrict__ bb, const int32_t* __restrict__ bhead,
                                                               const int64_t* __restrict__ U_ptr, const int64_t* __restrict__ off,
                                                               bool negate, double* out_x, double* out_y, double* out_w) {
    const int64_t U = *U_ptr;
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < U; p += (int64_t)gridDim.x * blockDim.x) {
        if (!bhead[p]) continue;
        const double2 v = wt[p];
        const double avg = v.y / v.x, y = negate ? -avg : avg;
        const int64_t o = off[p], e = bb[p];
        if (ux[e] > ux[p]) {
            out_x[o] = ux[p]; out_y[o] = y;
            out_x[o + 1] = ux[e]; out_y[o + 1] = y;
            if (out_w) out_w[o] = out_w[o + 1] = v.x / 2;
        } else {
            out_x[o] = ux[p]; out_y[o] = y;
            if (out_w) out_w[o] = v.x;
        }
    }
}

template <typename T>
__global__ void __launch_bounds__(kIsoThreads) iso_predict_kernel(const void* __restrict__ x, int64_t stride, int64_t n,
                                                                  const double* __restrict__ bx, const double* __restrict__ by,
                                                                  int64_t K, double* out) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const double v = load_as_double<T>(x, i * stride);
        const int64_t f = java_binary_search(bx, K, v), ins = -f - 1;
        double r;
        if (ins == 0) r = by[0];
        else if (ins == K) r = by[K - 1];
        else if (f < 0) {
            const double x1 = bx[ins - 1], y1 = by[ins - 1], x2 = bx[ins], y2 = by[ins];
            r = y1 + (y2 - y1) * (v - x1) / (x2 - x1);
        } else r = by[f];
        out[i] = r;
    }
}

// scratch layout of isotonic_fit over n rows (every piece 256-byte aligned)
struct IsoScratch {
    int64_t nb;
    size_t key0, key1, idx0, idx1, hist, offs, xs, ys, ws, head, rid, head_pos, ux, wt, bb, bhead, counts, total;
};

static size_t iso_align(size_t x) { return (x + 255) & ~(size_t)255; }

static IsoScratch iso_layout(int64_t n) {
    IsoScratch L;
    L.nb = radix_blocks(n);
    size_t o = 0;
    auto take = [&](size_t bytes) { const size_t at = o; o += iso_align(bytes); return at; };
    L.key0 = take(8 * n); L.key1 = take(8 * n);
    L.idx0 = take(4 * n); L.idx1 = take(4 * n);
    L.hist = take(4 * 256 * L.nb); L.offs = take(8 * 256 * L.nb);
    L.xs = take(8 * n); L.ys = take(8 * n); L.ws = take(8 * n);
    L.head = take(4 * n); L.rid = take(8 * n); L.head_pos = take(8 * n);
    L.ux = take(8 * n); L.wt = take(16 * n); L.bb = take(8 * n); L.bhead = take(4 * n);
    L.counts = take(8 * 6);
    L.total = o;
    return L;
}

}  // namespace b200flow

using namespace b200flow;

extern "C" int b200flow_isotonic_scratch(int64_t n, int64_t* scratch_bytes) {
    B2F_REQUIRE(scratch_bytes && n >= 0 && n <= 0xFFFFFFFFll, "isotonic_scratch: 0 <= n < 2^32 rows");
    *scratch_bytes = (int64_t)iso_layout(n).total;
    return B200FLOW_OK;
}

extern "C" int b200flow_isotonic_fit(const void* feature, int32_t feature_dtype, int64_t feature_stride, const double* label,
                                     int64_t label_stride, const double* weight, int64_t weight_stride, int64_t n,
                                     int32_t isotonic, int64_t chunk, void* scratch, int64_t scratch_bytes, double* boundaries,
                                     double* predictions, int64_t* n_out, int64_t* checks, void* stream) {
    B2F_REQUIRE(n >= 0 && n <= 0xFFFFFFFFll && n_out && checks && chunk >= 0 && chunk <= (1ll << 30) &&
                (feature_dtype == B200FLOW_F32 || feature_dtype == B200FLOW_F64),
                "isotonic_fit: 0 <= n < 2^32 rows, an f32 or f64 feature, 0 <= chunk <= 2^30");
    cudaStream_t st = (cudaStream_t)stream;
    cudaMemsetAsync(checks, 0, 16, st);
    cudaMemsetAsync(n_out, 0, 8, st);
    if (n == 0) return check_launch("isotonic_fit");
    B2F_REQUIRE(feature && label && scratch && boundaries && predictions && feature_stride >= 1 && label_stride >= 1 &&
                (!weight || weight_stride >= 1), "isotonic_fit: bad arguments");
    const IsoScratch L = iso_layout(n);
    B2F_REQUIRE(((uintptr_t)scratch & 255) == 0 && scratch_bytes >= (int64_t)L.total,
                "isotonic_fit: scratch must be 256-byte aligned and hold isotonic_scratch() bytes");
    const int64_t C = chunk ? chunk : kIsoChunk;
    char* base = (char*)scratch;
    unsigned long long* key[2] = {(unsigned long long*)(base + L.key0), (unsigned long long*)(base + L.key1)};
    uint32_t* idx[2] = {(uint32_t*)(base + L.idx0), (uint32_t*)(base + L.idx1)};
    int32_t* hist = (int32_t*)(base + L.hist); int64_t* offs = (int64_t*)(base + L.offs);
    double* xs = (double*)(base + L.xs); double* ys = (double*)(base + L.ys); double* ws = (double*)(base + L.ws);
    int32_t* head = (int32_t*)(base + L.head); int64_t* rid = (int64_t*)(base + L.rid);
    int64_t* head_pos = (int64_t*)(base + L.head_pos);
    double* ux = (double*)(base + L.ux); double2* wt = (double2*)(base + L.wt);
    int64_t* bb = (int64_t*)(base + L.bb); int32_t* bhead = (int32_t*)(base + L.bhead);
    // counts: [0] bad rows, [1] negative weights, [2] kept rows V, [3] unique points U, [4] first-pass points P
    int64_t* counts = (int64_t*)(base + L.counts);
    cudaMemsetAsync(counts, 0, 8 * 6, st);
    const int grid = grid_for(n, kIsoThreads * 8, kNumSMs * 16);
    const bool f32 = feature_dtype == B200FLOW_F32;
    if (f32) iso_keys_kernel<float><<<grid, kIsoThreads, 0, st>>>(feature, feature_stride, label, label_stride, weight,
                                                                   weight_stride, n, key[0], idx[0], (unsigned long long*)counts);
    else iso_keys_kernel<double><<<grid, kIsoThreads, 0, st>>>(feature, feature_stride, label, label_stride, weight,
                                                                weight_stride, n, key[0], idx[0], (unsigned long long*)counts);
    cudaMemcpyAsync(checks, counts, 16, cudaMemcpyDeviceToDevice, st);
    int cur = 0;
    for (int pass = 0; pass < 8; ++pass, cur ^= 1) {
        const int rc = radix_pass<false>(key[cur], idx[cur], n, 1, 8 * pass, hist, offs, key[cur ^ 1], idx[cur ^ 1], stream);
        if (rc) return rc;
    }
    if (f32) iso_gather_kernel<float><<<grid, kIsoThreads, 0, st>>>(idx[cur], feature, feature_stride, label, label_stride,
                                                                     weight, weight_stride, !isotonic, counts + 2, xs, ys, ws);
    else iso_gather_kernel<double><<<grid, kIsoThreads, 0, st>>>(idx[cur], feature, feature_stride, label, label_stride,
                                                                  weight, weight_stride, !isotonic, counts + 2, xs, ys, ws);
    // pass 0 over the V sorted rows, pass 1 over pass 0's P output points (already sorted, distinct features)
    for (int pass = 0; pass < 2; ++pass) {
        const int64_t* V = counts + 2 + 2 * pass;
        int64_t* U = counts + 3 + 2 * pass;
        iso_heads_kernel<<<grid, kIsoThreads, 0, st>>>(xs, V, n, head);
        int rc = b200flow_exclusive_scan_i32_to_i64(head, n, rid, U, stream);
        if (rc) return rc;
        iso_head_pos_kernel<<<grid, kIsoThreads, 0, st>>>(head, rid, n, head_pos);
        iso_tie_kernel<<<grid, kIsoThreads, 0, st>>>(xs, ys, ws, head_pos, U, V, ux, wt, bb, bhead);
        iso_pav_chunk_kernel<<<(unsigned)((n + C * kIsoThreads - 1) / (C * kIsoThreads)), kIsoThreads, 0, st>>>(wt, bb, bhead, U, C);
        for (int64_t R = C; R < n; R *= 2) {
            const int64_t pairs = (n + 2 * R - 1) / (2 * R);
            iso_pav_merge_kernel<<<(unsigned)((pairs + kIsoThreads - 1) / kIsoThreads), kIsoThreads, 0, st>>>(wt, bb, bhead, U, R);
        }
        // compression: head reused for the per-block point counts, rid for their exclusive scan
        iso_count_kernel<<<grid, kIsoThreads, 0, st>>>(ux, bb, bhead, U, n, head);
        rc = b200flow_exclusive_scan_i32_to_i64(head, n, rid, pass ? n_out : counts + 4, stream);
        if (rc) return rc;
        if (pass == 0) iso_emit_kernel<<<grid, kIsoThreads, 0, st>>>(ux, wt, bb, bhead, U, rid, false, xs, ys, ws);
        else iso_emit_kernel<<<grid, kIsoThreads, 0, st>>>(ux, wt, bb, bhead, U, rid, !isotonic, boundaries, predictions, nullptr);
    }
    return check_launch("isotonic_fit");
}

extern "C" int b200flow_isotonic_predict(const void* x, int32_t x_dtype, int64_t stride, int64_t n, const double* boundaries,
                                         const double* predictions, int64_t K, double* out, void* stream) {
    B2F_REQUIRE(n >= 0 && K >= 1 && stride >= 1 && (x_dtype == B200FLOW_F32 || x_dtype == B200FLOW_F64),
                "isotonic_predict: n >= 0 rows of an f32 or f64 feature, a model of K >= 1 boundaries");
    if (n == 0) return B200FLOW_OK;
    B2F_REQUIRE(x && boundaries && predictions && out, "isotonic_predict: bad arguments");
    const int grid = grid_for(n, kIsoThreads * 8, kNumSMs * 16);
    cudaStream_t st = (cudaStream_t)stream;
    if (x_dtype == B200FLOW_F32) iso_predict_kernel<float><<<grid, kIsoThreads, 0, st>>>(x, stride, n, boundaries, predictions, K, out);
    else iso_predict_kernel<double><<<grid, kIsoThreads, 0, st>>>(x, stride, n, boundaries, predictions, K, out);
    return check_launch("isotonic_predict");
}
