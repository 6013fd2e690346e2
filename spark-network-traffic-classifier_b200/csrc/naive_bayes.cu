// naive_bayes.cu — NaiveBayes (multinomial, complement, bernoulli, gaussian) fit statistics and scores, DESIGN.md §5u.
//
// b200flow_nb_moments: the one fit reduction.  One CTA per (4096-row global chunk, slab of columns); a thread owns a column
// and walks the chunk's rows in order, so every sum is sequential in row order; the class accumulators (and the centres of
// the second pass) of the slab sit in shared memory, as in b200flow_group_centered_moments.  The first pass also counts the
// inputs a fit must refuse, so the host can raise from all-reduced counts on every rank.
// b200flow_nb_raw: one CTA per 64 rows, staged transposed in shared memory once; the class coefficients stream through in
// tiles, as in b200flow_kmeans_assign.  Each (row, class) value is one sum over the features in feature order from 0.0, so
// it depends on that row and the model alone, never on the batch or the shard.
#include <math.h>

#include "common.cuh"

namespace b200flow {

namespace {

constexpr int kNbChunkRows = 4096;
constexpr int kNbMaxD = 256, kNbMaxC = 256;
constexpr int kNbSmemBytes = 96 << 10;            // moments: accumulators (+ centres) of one slab
enum { kBadNonFinite = 0, kBadNegative, kBadNotBinary, kBadWeight, kBadLabel };

template <typename T>
__global__ void nb_moments_kernel(const T* __restrict__ x, int64_t n, int D, int64_t ld, const int32_t* __restrict__ labels,
                                  const double* __restrict__ weights, int C, const double* __restrict__ centers,
                                  int64_t row_offset, int S, double* __restrict__ partials, unsigned long long* __restrict__ bad) {
    extern __shared__ double nb_sm[];
    const bool second = centers != nullptr;
    const int G = second ? C + 1 : C, Wd = second ? D : D + 1;
    const int w0 = blockIdx.y * S, ns = Wd - w0 < S ? Wd - w0 : S;
    const int t = threadIdx.x, j = w0 + t;
    const int64_t c0 = (row_offset / kNbChunkRows + blockIdx.x) * kNbChunkRows - row_offset;   // local index of the chunk's row 0
    const int64_t lo = c0 > 0 ? c0 : 0, hi = c0 + kNbChunkRows < n ? c0 + kNbChunkRows : n;
    double* acc = nb_sm;                          // [G][S]
    double* cs = nb_sm + G * S;                   // [G][S], second pass only
    for (int e = t; e < G * S; e += blockDim.x) {
        acc[e] = 0.0;
        if (second) {
            const int g = e / S, k = e - g * S;
            cs[e] = k < ns ? centers[(int64_t)g * D + w0 + k] : 0.0;
        }
    }
    __syncthreads();
    if (t >= ns) return;
    double* part = partials + (int64_t)blockIdx.x * G * Wd;
    if (second) {                                 // [c] = sum w (x - theta_c)^2 over class c, [C] = over every row around mu
        for (int64_t r = lo; r < hi; ++r) {
            const int g = labels[r];
            if (g < 0 || g >= C) continue;
            const double w = weights ? weights[r] : 1.0;
            const double v = (double)x[r * ld + j];
            const double d = v - cs[g * S + t], e = v - cs[C * S + t];
            acc[g * S + t] = acc[g * S + t] + w * (d * d);
            acc[C * S + t] = acc[C * S + t] + w * (e * e);
        }
    } else if (j < D) {                           // [c][j] = sum w x_j over class c
        unsigned long long nonfinite = 0, negative = 0, not_binary = 0;
        for (int64_t r = lo; r < hi; ++r) {
            const int g = labels[r];
            const double v = (double)x[r * ld + j];
            nonfinite += !isfinite(v);
            negative += v < 0.0;
            not_binary += v != 0.0 && v != 1.0;
            if (g < 0 || g >= C) continue;
            const double w = weights ? weights[r] : 1.0;
            acc[g * S + t] = acc[g * S + t] + w * v;
        }
        if (bad) {
            if (nonfinite) atomicAdd(bad + kBadNonFinite, nonfinite);
            if (negative) atomicAdd(bad + kBadNegative, negative);
            if (not_binary) atomicAdd(bad + kBadNotBinary, not_binary);
        }
    } else {                                      // [c][D] = sum w over class c
        unsigned long long bad_w = 0, bad_l = 0;
        for (int64_t r = lo; r < hi; ++r) {
            const int g = labels[r];
            const double w = weights ? weights[r] : 1.0;
            bad_w += !(w >= 0.0) || isinf(w);
            if (g < 0 || g >= C) { ++bad_l; continue; }
            acc[g * S + t] = acc[g * S + t] + w;
        }
        if (bad) {
            if (bad_w) atomicAdd(bad + kBadWeight, bad_w);
            if (bad_l) atomicAdd(bad + kBadLabel, bad_l);
        }
    }
    for (int g = 0; g < G; ++g) part[(int64_t)g * Wd + j] = acc[g * S + t];
}

// ------------------------------------------------------------------ scores
constexpr int kRawRows = 64, kRawThreads = 128, kRawRowPitch = kRawRows + 1;

// Thread (ty, tx) owns rows ty + 16i (i < 4) and the tile's classes tx + 8q (q < Q): Q = 4 for the linear forms (a tile of
// 32 classes), Q = 2 for the gaussian form, whose second table (sigma) must fit beside the first at D = 256.
template <typename T, bool kGauss>
__global__ void __launch_bounds__(kRawThreads) nb_raw_kernel(const T* __restrict__ x, int64_t n, int D, int64_t ld,
                                                             const double* __restrict__ a, const double* __restrict__ b,
                                                             const double* __restrict__ c0, const double* __restrict__ c1,
                                                             const uint8_t* __restrict__ present, int C, double* __restrict__ raw,
                                                             unsigned long long* __restrict__ bad) {
    constexpr int Q = kGauss ? 2 : 4, kCls = 8 * Q, kClsPitch = kCls + 1;
    extern __shared__ double raw_sm[];
    double* xs = raw_sm;                                   // [D][kRawRowPitch]
    double* as = xs + (size_t)D * kRawRowPitch;            // [D][kClsPitch]
    double* bs = as + (size_t)D * kClsPitch;               // [D][kClsPitch], gaussian only
    const int tid = threadIdx.x, tx = tid & 7, ty = tid >> 3;
    const int64_t row0 = (int64_t)blockIdx.x * kRawRows;
    unsigned long long not_binary = 0;
    for (int e = tid; e < kRawRows * D; e += kRawThreads) {
        const int r = e / D, j = e - r * D;
        const int64_t gr = row0 + r;
        const double v = gr < n ? (double)x[gr * ld + j] : 0.0;
        not_binary += v != 0.0 && v != 1.0;
        xs[j * kRawRowPitch + r] = v;
    }
    if (bad && not_binary) atomicAdd(bad, not_binary);
    for (int k0 = 0; k0 < C; k0 += kCls) {
        __syncthreads();                                   // the previous class tile is consumed (first pass: nothing)
        for (int e = tid; e < kCls * D; e += kRawThreads) {
            const int c = e / D, j = e - c * D;
            const bool in = k0 + c < C;
            as[j * kClsPitch + c] = in ? a[(int64_t)(k0 + c) * D + j] : 0.0;
            if (kGauss) bs[j * kClsPitch + c] = in ? b[(int64_t)(k0 + c) * D + j] : 1.0;
        }
        __syncthreads();
        double acc[4][Q];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int q = 0; q < Q; ++q) acc[i][q] = 0.0;
#pragma unroll 2
        for (int j = 0; j < D; ++j) {
            double xv[4], av[Q], bv[Q];
#pragma unroll
            for (int i = 0; i < 4; ++i) xv[i] = xs[j * kRawRowPitch + ty + 16 * i];
#pragma unroll
            for (int q = 0; q < Q; ++q) {
                av[q] = as[j * kClsPitch + tx + 8 * q];
                if (kGauss) bv[q] = bs[j * kClsPitch + tx + 8 * q];
            }
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int q = 0; q < Q; ++q) {
                    if (kGauss) {
                        const double d = xv[i] - av[q];
                        acc[i][q] = acc[i][q] + (d * d) / bv[q];
                    } else {
                        acc[i][q] = acc[i][q] + xv[i] * av[q];
                    }
                }
        }
#pragma unroll
        for (int q = 0; q < Q; ++q) {
            const int c = k0 + tx + 8 * q;
            if (c >= C) continue;
            const bool on = present[c] != 0;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int64_t gr = row0 + ty + 16 * i;
                if (gr >= n) continue;
                double v = -INFINITY;
                if (on) v = kGauss ? c0[c] - (acc[i][q] + c1[c]) / 2.0 : acc[i][q] + c0[c];
                raw[gr * C + c] = v;
            }
        }
    }
}

// raw[i][c] -= max + log(sum over the present classes, in class order from 0.0, of exp(raw[i][c] - max))
__global__ void __launch_bounds__(256) nb_normalize_kernel(int64_t n, int C, const uint8_t* __restrict__ present,
                                                           double* __restrict__ raw) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        double* z = raw + i * C;
        double m = -INFINITY;
        for (int c = 0; c < C; ++c)
            if (present[c] && z[c] > m) m = z[c];
        double s = 0.0;
        for (int c = 0; c < C; ++c)
            if (present[c]) s = s + exp(z[c] - m);
        const double lse = m + log(s);
        for (int c = 0; c < C; ++c) z[c] = present[c] ? z[c] - lse : -INFINITY;
    }
}

template <typename T>
int launch_nb_raw(const T* x, int64_t n_rows, int32_t D, int64_t ld, int32_t model, const double* a, const double* b,
                  const double* c0, const double* c1, const uint8_t* present, int32_t C, double* raw, int64_t* bad,
                  cudaStream_t stream) {
    const int64_t blocks = (n_rows + kRawRows - 1) / kRawRows;
    B2F_REQUIRE(blocks <= 0x7fffffffll, "nb_raw: too many rows");
    unsigned long long* bad_u = (unsigned long long*)bad;
    if (model == 0) {
        const size_t smem = (size_t)D * (kRawRowPitch + 2 * 17) * sizeof(double);
        cudaFuncSetAttribute(nb_raw_kernel<T, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        nb_raw_kernel<T, true><<<(unsigned)blocks, kRawThreads, smem, stream>>>(x, n_rows, D, ld, a, b, c0, c1, present, C, raw,
                                                                                bad_u);
    } else {
        const size_t smem = (size_t)D * (kRawRowPitch + 33) * sizeof(double);
        cudaFuncSetAttribute(nb_raw_kernel<T, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        nb_raw_kernel<T, false><<<(unsigned)blocks, kRawThreads, smem, stream>>>(x, n_rows, D, ld, a, b, c0, c1, present, C, raw,
                                                                                 bad_u);
        if (model == 2)
            nb_normalize_kernel<<<grid_for(n_rows, 256, kNumSMs * 8), 256, 0, stream>>>(n_rows, C, present, raw);
    }
    return check_launch("nb_raw");
}

template <typename T>
int launch_nb_moments(const T* x, int64_t n_rows, int32_t D, int64_t ld, const int32_t* labels, const double* weights, int32_t C,
                      const double* centers, int64_t row_offset, double* partials, int64_t* bad, cudaStream_t stream) {
    const int64_t nc = (row_offset + n_rows - 1) / kNbChunkRows - row_offset / kNbChunkRows + 1;
    B2F_REQUIRE(nc <= 0x7fffffffll, "nb_moments: too many rows");
    const int G = centers ? C + 1 : C, Wd = centers ? D : D + 1;
    int S = kNbSmemBytes / ((centers ? 2 : 1) * G * (int)sizeof(double));
    if (S > Wd) S = Wd;
    const size_t smem = (size_t)(centers ? 2 : 1) * G * S * sizeof(double);
    cudaFuncSetAttribute(nb_moments_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    const dim3 grid((unsigned)nc, (unsigned)((Wd + S - 1) / S));
    nb_moments_kernel<T><<<grid, (S + 31) / 32 * 32, smem, stream>>>(x, n_rows, D, ld, labels, weights, C, centers, row_offset, S,
                                                                     partials, (unsigned long long*)bad);
    return check_launch("nb_moments");
}

}  // namespace

}  // namespace b200flow

using namespace b200flow;

extern "C" int b200flow_nb_moments(const void* x, int32_t x_dtype, int64_t n_rows, int32_t D, int64_t ld, const int32_t* labels,
                                   const double* weights, int32_t C, const double* centers, int64_t row_offset, double* partials,
                                   int64_t* bad, void* stream) {
    B2F_REQUIRE(D >= 1 && D <= kNbMaxD && C >= 1 && C <= kNbMaxC, "nb_moments: 1 <= D <= %d, 1 <= C <= %d", kNbMaxD, kNbMaxC);
    B2F_REQUIRE(x_dtype == 0 || x_dtype == 1, "nb_moments: x_dtype 0 (f32) or 1 (f64)");
    B2F_REQUIRE(n_rows >= 0 && row_offset >= 0 && ld >= D, "nb_moments: n >= 0, row_offset >= 0, ld >= D");
    if (n_rows == 0) return B200FLOW_OK;
    B2F_REQUIRE(x && labels && partials, "nb_moments: null pointer");
    cudaStream_t s = (cudaStream_t)stream;
    return x_dtype == 0 ? launch_nb_moments((const float*)x, n_rows, D, ld, labels, weights, C, centers, row_offset, partials, bad, s)
                        : launch_nb_moments((const double*)x, n_rows, D, ld, labels, weights, C, centers, row_offset, partials, bad, s);
}

extern "C" int b200flow_nb_raw(const void* x, int32_t x_dtype, int64_t n_rows, int32_t D, int64_t ld, int32_t model, const double* a,
                               const double* b, const double* c0, const double* c1, const uint8_t* present, int32_t C, double* raw,
                               int64_t* bad, void* stream) {
    B2F_REQUIRE(D >= 1 && D <= kNbMaxD && C >= 1 && C <= kNbMaxC, "nb_raw: 1 <= D <= %d, 1 <= C <= %d", kNbMaxD, kNbMaxC);
    B2F_REQUIRE(x_dtype == 0 || x_dtype == 1, "nb_raw: x_dtype 0 (f32) or 1 (f64)");
    B2F_REQUIRE(model >= 0 && model <= 2, "nb_raw: model 0 (gaussian), 1 (linear) or 2 (linear, normalised)");
    B2F_REQUIRE(n_rows >= 0 && ld >= D, "nb_raw: n >= 0, ld >= D");
    if (n_rows == 0) return B200FLOW_OK;
    B2F_REQUIRE(x && a && c0 && present && raw && (model != 0 || (b && c1)), "nb_raw: null pointer");
    cudaStream_t s = (cudaStream_t)stream;
    return x_dtype == 0 ? launch_nb_raw((const float*)x, n_rows, D, ld, model, a, b, c0, c1, present, C, raw, bad, s)
                        : launch_nb_raw((const double*)x, n_rows, D, ld, model, a, b, c0, c1, present, C, raw, bad, s);
}
