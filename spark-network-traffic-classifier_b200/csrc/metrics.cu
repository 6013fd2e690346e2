// metrics.cu — BinaryClassificationMetrics (BinaryClassificationEvaluator: areaUnderROC / areaUnderPR), DESIGN.md §5b.
//
// b200flow_binary_counts: S segments of scores -> the distinct scores of every segment in descending order, each with its
// integer positive / negative counts.  A stable LSD radix sort (8-bit digits) of order-preserving 64-bit keys, then of the
// segment id, puts every segment's items in descending score order; run heads, a scan and a difference of two prefix sums
// give each distinct score its counts.  Everything is integer, so the result does not depend on the order of the input
// (or on how rows were spread over ranks).
//
// b200flow_binary_curve: the distinct triples -> the binned curve points (Spark's numBins rule) and the two trapezoid
// areas, each summed sequentially from 0.0 in curve order (Spark's AreaUnderCurve on one partition).
#include "radix_sort.cuh"

namespace b200flow {

constexpr unsigned long long kInvalidKey = ~0ull;                // NaN scores and zero-count items: sorted last, never a run

// descending order of x as an ascending uint64: -0.0 is +0.0; the only key equal to kInvalidKey is a NaN's
__device__ __forceinline__ unsigned long long desc_key(double x) {
    if (x == 0.0) x = 0.0;
    const unsigned long long b = (unsigned long long)__double_as_longlong(x);
    const unsigned long long asc = (b >> 63) ? ~b : (b | (1ull << 63));
    return ~asc;
}

__device__ __forceinline__ double key_score(unsigned long long k) {
    const unsigned long long asc = ~k;
    return __longlong_as_double((long long)((asc >> 63) ? (asc ^ (1ull << 63)) : ~asc));
}

__global__ void __launch_bounds__(256) bc_keys_kernel(const double* __restrict__ scores, int64_t score_stride,
                                                      const int32_t* __restrict__ pos, const int32_t* __restrict__ neg,
                                                      int64_t count_stride, int64_t n, int64_t M,
                                                      unsigned long long* key, uint32_t* idx, unsigned long long* n_nan) {
    unsigned long long nan_local = 0;
    for (int64_t m = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; m < M; m += (int64_t)gridDim.x * blockDim.x) {
        const int64_t s = m / n, i = m - s * n;
        const double x = scores[s * score_stride + i];
        const int64_t c = (int64_t)pos[s * count_stride + i] + neg[s * count_stride + i];
        const bool nan = x != x;
        if (nan && c != 0) ++nan_local;
        key[m] = (nan || c == 0) ? kInvalidKey : desc_key(x);
        idx[m] = (uint32_t)m;
    }
    nan_local = warp_sum(nan_local);
    if (lane_id() == 0 && nan_local) atomicAdd(n_nan, nan_local);
}

// after the sort: run heads, and each item's counts in sorted order (0 for NaN / zero-count items)
__global__ void __launch_bounds__(256) bc_heads_kernel(const unsigned long long* __restrict__ key, const uint32_t* __restrict__ idx,
                                                       const int32_t* __restrict__ pos, const int32_t* __restrict__ neg,
                                                       int64_t count_stride, int64_t n, int64_t M,
                                                       int32_t* head, int32_t* pos_s, int32_t* neg_s) {
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < M; p += (int64_t)gridDim.x * blockDim.x) {
        const unsigned long long k = key[p];
        const bool valid = k != kInvalidKey;
        head[p] = valid && (p % n == 0 || key[p - 1] != k) ? 1 : 0;
        const int64_t m = idx[p], s = m / n, i = m - s * n;
        pos_s[p] = valid ? pos[s * count_stride + i] : 0;
        neg_s[p] = valid ? neg[s * count_stride + i] : 0;
    }
}

__global__ void __launch_bounds__(256) bc_head_pos_kernel(const int32_t* __restrict__ head, const int64_t* __restrict__ rid,
                                                          int64_t M, int64_t* head_pos) {
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < M; p += (int64_t)gridDim.x * blockDim.x)
        if (head[p]) head_pos[rid[p]] = p;
}

// one thread per run: the run spans [head, next head) in sorted order; trailing invalid items add 0 to its sums
__global__ void __launch_bounds__(256) bc_emit_kernel(const unsigned long long* __restrict__ key, const int64_t* __restrict__ rid,
                                                      const int64_t* __restrict__ head_pos, const int64_t* __restrict__ n_runs,
                                                      const int64_t* __restrict__ cpos, const int64_t* __restrict__ cneg,
                                                      int64_t n, int64_t M, double* d_score, int64_t* d_pos, int64_t* d_neg,
                                                      int64_t cap) {
    const int64_t R = *n_runs;
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < R; r += (int64_t)gridDim.x * blockDim.x) {
        const int64_t p = head_pos[r];
        const int64_t e = r + 1 < R ? head_pos[r + 1] : M;
        const int64_t s = p / n;
        const int64_t o = s * cap + (r - rid[s * n]);
        d_score[o] = key_score(key[p]);
        d_pos[o] = cpos[e] - cpos[p];
        d_neg[o] = cneg[e] - cneg[p];
    }
}

__global__ void bc_ndistinct_kernel(const int64_t* __restrict__ rid, const int64_t* __restrict__ n_runs, int64_t n, int S,
                                    int64_t* n_distinct) {
    for (int s = blockIdx.x * blockDim.x + threadIdx.x; s < S; s += gridDim.x * blockDim.x) {
        const int64_t hi = s + 1 < S ? rid[(int64_t)(s + 1) * n] : *n_runs;
        n_distinct[s] = hi - rid[(int64_t)s * n];
    }
}

// ------------------------------------------------------------------ curve + areas
constexpr int kCurveThreads = 1024;

__device__ __forceinline__ int64_t block_exclusive_scan_i64(int64_t v, int64_t* sh, int64_t* total) {
    int64_t inc = warp_inclusive_scan(v);
    if (lane_id() == 31) sh[warp_id()] = inc;
    __syncthreads();
    if (warp_id() == 0) {
        const int nw = (blockDim.x + 31) >> 5;
        const int64_t x = lane_id() < nw ? sh[lane_id()] : 0;
        const int64_t xi = warp_inclusive_scan(x);
        sh[lane_id()] = xi - x;
        if (lane_id() == 31) sh[32] = xi;
    }
    __syncthreads();
    const int64_t res = inc - v + sh[warp_id()];
    *total = sh[32];
    __syncthreads();
    return res;
}

__device__ __forceinline__ double rate(int64_t a, int64_t b) { return b == 0 ? 0.0 : (double)a / (double)b; }
__device__ __forceinline__ double precision(int64_t tp, int64_t fp) { return tp + fp == 0 ? 1.0 : (double)tp / (double)(tp + fp); }
__device__ __forceinline__ double trapezoid(double x1, double y1, double x2, double y2) { return (x2 - x1) * (y2 + y1) / 2.0; }

// One block per segment.  Curve point j (0 <= j < K) is distinct rank min((j + 1) g - 1, nd - 1), g = max(nd / numBins, 1)
// when numBins > 0 and nd / numBins >= 2, else 1; it carries that rank's score and the cumulative counts through it.
__global__ void __launch_bounds__(kCurveThreads) bc_curve_kernel(const double* __restrict__ d_score, const int64_t* __restrict__ d_pos,
                                                                 const int64_t* __restrict__ d_neg, int64_t cap,
                                                                 const int64_t* __restrict__ n_distinct, int num_bins, double* auc,
                                                                 double* c_score, int64_t* c_tp, int64_t* c_fp, int64_t* c_n,
                                                                 double* work) {
    __shared__ int64_t sh[33];
    const int64_t s = blockIdx.x;
    const int64_t nd = n_distinct[s];
    if (nd <= 0) {
        if (threadIdx.x == 0) { auc[2 * s] = auc[2 * s + 1] = __longlong_as_double(0x7ff8000000000000ll); c_n[s] = 0; }
        return;
    }
    int64_t g = num_bins > 0 ? nd / num_bins : 1;
    if (g < 2) g = 1;
    const int64_t K = (nd + g - 1) / g;
    const double* sc = d_score + s * cap; const int64_t* ps = d_pos + s * cap; const int64_t* ng = d_neg + s * cap;
    double* cs = c_score + s * cap; int64_t* ct = c_tp + s * cap; int64_t* cf = c_fp + s * cap;
    double* roc = work + 2 * s * cap; double* pr = roc + cap;
    // cumulative counts: thread t owns the contiguous ranks [a, b)
    const int64_t per = (nd + blockDim.x - 1) / blockDim.x;
    const int64_t a = per * threadIdx.x < nd ? per * threadIdx.x : nd, b = a + per < nd ? a + per : nd;
    int64_t lp = 0, ln = 0;
    for (int64_t r = a; r < b; ++r) { lp += ps[r]; ln += ng[r]; }
    int64_t P, N;
    int64_t tp = block_exclusive_scan_i64(lp, sh, &P);
    int64_t fp = block_exclusive_scan_i64(ln, sh, &N);
    for (int64_t r = a; r < b; ++r) {
        tp += ps[r]; fp += ng[r];
        if ((r + 1) % g == 0 || r == nd - 1) {
            const int64_t j = r / g;
            cs[j] = sc[r]; ct[j] = tp; cf[j] = fp;
        }
    }
    __syncthreads();
    // trapezoid terms in parallel: ROC (0,0), (FPR_j, TPR_j)..., (1,1); PR (0, precision_0), (TPR_j, precision_j)...
    for (int64_t j = threadIdx.x; j < K; j += blockDim.x) {
        const double x = rate(cf[j], N), y = rate(ct[j], P), pj = precision(ct[j], cf[j]);
        const double x0 = j ? rate(cf[j - 1], N) : 0.0, y0 = j ? rate(ct[j - 1], P) : 0.0;
        const double p0 = j ? precision(ct[j - 1], cf[j - 1]) : precision(ct[0], cf[0]);
        roc[j] = trapezoid(x0, y0, x, y);
        pr[j] = trapezoid(y0, p0, y, pj);
    }
    __syncthreads();
    // the sums run in curve order from 0.0, one lane per curve
    if (threadIdx.x == 0) {
        double acc = 0.0;
        for (int64_t j = 0; j < K; ++j) acc += roc[j];
        acc += trapezoid(rate(cf[K - 1], N), rate(ct[K - 1], P), 1.0, 1.0);
        auc[2 * s] = acc;
        c_n[s] = K;
    } else if (threadIdx.x == 32) {
        double acc = 0.0;
        for (int64_t j = 0; j < K; ++j) acc += pr[j];
        auc[2 * s + 1] = acc;
    }
}

// scratch layout of binary_counts (every piece 256-byte aligned)
struct CountsScratch {
    int64_t M, nb;
    size_t key0, key1, idx0, idx1, hist, offs, head, pos_s, neg_s, rid, cpos, cneg, head_pos, n_runs, total;
};

static size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

static CountsScratch counts_layout(int32_t S, int64_t n) {
    CountsScratch L;
    L.M = (int64_t)S * n;
    L.nb = radix_blocks(L.M);
    size_t o = 0;
    auto take = [&](size_t bytes) { const size_t at = o; o += align256(bytes); return at; };
    L.key0 = take(8 * L.M); L.key1 = take(8 * L.M);
    L.idx0 = take(4 * L.M); L.idx1 = take(4 * L.M);
    L.hist = take(4 * 256 * L.nb); L.offs = take(8 * 256 * L.nb);
    L.head = take(4 * L.M); L.pos_s = take(4 * L.M); L.neg_s = take(4 * L.M);
    L.rid = take(8 * L.M); L.cpos = take(8 * (L.M + 1)); L.cneg = take(8 * (L.M + 1));
    L.head_pos = take(8 * L.M); L.n_runs = take(8);
    L.total = o;
    return L;
}

}  // namespace b200flow

using namespace b200flow;

extern "C" int b200flow_binary_counts_scratch(int32_t S, int64_t n, int64_t* scratch_bytes) {
    B2F_REQUIRE(scratch_bytes && S >= 1 && S <= 65536 && n >= 0 && (int64_t)S * n <= 0xFFFFFFFFll,
                "binary_counts_scratch: 1..65536 segments of n >= 0 scores, S * n < 2^32");
    *scratch_bytes = (int64_t)counts_layout(S, n).total;
    return B200FLOW_OK;
}

extern "C" int b200flow_binary_counts(const double* scores, int64_t score_stride, const int32_t* pos, const int32_t* neg,
                                      int64_t count_stride, int32_t S, int64_t n, void* scratch, int64_t scratch_bytes,
                                      double* d_score, int64_t* d_pos, int64_t* d_neg, int64_t cap, int64_t* n_distinct,
                                      int64_t* n_nan, void* stream) {
    B2F_REQUIRE(S >= 1 && S <= 65536 && n >= 0 && (int64_t)S * n <= 0xFFFFFFFFll && n_distinct && n_nan,
                "binary_counts: 1..65536 segments of n >= 0 scores, S * n < 2^32");
    cudaStream_t st = (cudaStream_t)stream;
    cudaMemsetAsync(n_nan, 0, 8, st);
    if (n == 0) { cudaMemsetAsync(n_distinct, 0, 8 * (size_t)S, st); return check_launch("binary_counts"); }
    B2F_REQUIRE(scores && pos && neg && scratch && d_score && d_pos && d_neg && cap >= n && score_stride >= n &&
                (count_stride == 0 || count_stride >= n), "binary_counts: bad arguments");
    const CountsScratch L = counts_layout(S, n);
    B2F_REQUIRE(((uintptr_t)scratch & 255) == 0 && scratch_bytes >= (int64_t)L.total,
                "binary_counts: scratch must be 256-byte aligned and hold binary_counts_scratch() bytes");
    char* base = (char*)scratch;
    unsigned long long* key[2] = {(unsigned long long*)(base + L.key0), (unsigned long long*)(base + L.key1)};
    uint32_t* idx[2] = {(uint32_t*)(base + L.idx0), (uint32_t*)(base + L.idx1)};
    int32_t* hist = (int32_t*)(base + L.hist); int64_t* offs = (int64_t*)(base + L.offs);
    int32_t* head = (int32_t*)(base + L.head); int32_t* pos_s = (int32_t*)(base + L.pos_s); int32_t* neg_s = (int32_t*)(base + L.neg_s);
    int64_t* rid = (int64_t*)(base + L.rid); int64_t* cpos = (int64_t*)(base + L.cpos); int64_t* cneg = (int64_t*)(base + L.cneg);
    int64_t* head_pos = (int64_t*)(base + L.head_pos); int64_t* n_runs = (int64_t*)(base + L.n_runs);
    const int64_t M = L.M;
    const int grid = grid_for(M, 256 * 8, kNumSMs * 16);
    bc_keys_kernel<<<grid, 256, 0, st>>>(scores, score_stride, pos, neg, count_stride, n, M, key[0], idx[0],
                                         (unsigned long long*)n_nan);
    // LSD: the 8 key digits, then the segment id's digits (segment is the primary order)
    const int seg_passes = S <= 1 ? 0 : (S <= 256 ? 1 : 2);
    int cur = 0;
    for (int pass = 0; pass < 8 + seg_passes; ++pass) {
        const bool seg = pass >= 8;
        const int shift = seg ? 8 * (pass - 8) : 8 * pass;
        const int rc = seg ? radix_pass<true>(key[cur], idx[cur], M, n, shift, hist, offs, key[cur ^ 1], idx[cur ^ 1], stream)
                           : radix_pass<false>(key[cur], idx[cur], M, n, shift, hist, offs, key[cur ^ 1], idx[cur ^ 1], stream);
        if (rc) return rc;
        cur ^= 1;
    }
    bc_heads_kernel<<<grid, 256, 0, st>>>(key[cur], idx[cur], pos, neg, count_stride, n, M, head, pos_s, neg_s);
    int rc = b200flow_exclusive_scan_i32_to_i64(head, M, rid, n_runs, stream);
    if (!rc) rc = b200flow_exclusive_scan_i32_to_i64(pos_s, M, cpos, cpos + M, stream);
    if (!rc) rc = b200flow_exclusive_scan_i32_to_i64(neg_s, M, cneg, cneg + M, stream);
    if (rc) return rc;
    bc_head_pos_kernel<<<grid, 256, 0, st>>>(head, rid, M, head_pos);
    bc_emit_kernel<<<grid, 256, 0, st>>>(key[cur], rid, head_pos, n_runs, cpos, cneg, n, M, d_score, d_pos, d_neg, cap);
    bc_ndistinct_kernel<<<(S + 255) / 256, 256, 0, st>>>(rid, n_runs, n, S, n_distinct);
    return check_launch("binary_counts");
}

extern "C" int b200flow_binary_curve(const double* d_score, const int64_t* d_pos, const int64_t* d_neg, int64_t cap,
                                     const int64_t* n_distinct, int32_t S, int32_t num_bins, double* auc, double* c_score,
                                     int64_t* c_tp, int64_t* c_fp, int64_t* c_n, double* work, void* stream) {
    B2F_REQUIRE(S >= 1 && S <= 65536 && cap >= 1 && num_bins >= 0 && d_score && d_pos && d_neg && n_distinct && auc &&
                c_score && c_tp && c_fp && c_n && work, "binary_curve: bad arguments");
    bc_curve_kernel<<<S, kCurveThreads, 0, (cudaStream_t)stream>>>(d_score, d_pos, d_neg, cap, n_distinct, num_bins, auc,
                                                                   c_score, c_tp, c_fp, c_n, work);
    return check_launch("binary_curve");
}
