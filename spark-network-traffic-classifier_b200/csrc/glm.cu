// glm.cu — GeneralizedLinearRegression: the per-row IRLS / summary / prediction pass, DESIGN.md §5o.
//
// One pass over the rows per IRLS iteration, bound by HBM like linreg.cu, so plain fp64 FMA-free arithmetic.  The
// family and link functions are glm_family.cuh's.
//
// b200flow_glm_rows: one CTA per 4096-row global chunk walks the chunk's 32-row tiles, which sit at fixed global
// positions, in row order.  A tile of x is staged once in shared memory (as f64; rows outside the chunk or outside [0, n)
// as 0 and masked).  Its 32 rows are split four per warp, eight lanes per row:
//   margin: lane s of a row sums p_s = sum of x_j coef_j over j = s, s + 8, s + 16, ... < D in ascending order from +0.0;
//     the eight partial sums combine by butterfly shuffles (xor 4, then 2, then 1), so every lane ends with
//       m = ((p0 + p4) + (p2 + p6)) + ((p1 + p5) + (p3 + p7))
//     (each addition is commutative in IEEE arithmetic, so all eight lanes hold the same bits); eta = (m + b) + offset.
//   lane 0 of the row then evaluates the row's outputs and its terms of the chunk sums.
//   column phase (INIT / REWEIGHT): thread j < D adds w_r x_rj over the tile's rows in order; the last thread adds the
//     scalar terms over the tile's rows in order.
// Every sum runs over the chunk's rows in row order from +0.0, so a chunk's partial depends only on its rows and the
// inputs.  No atomics.
#include "common.cuh"
#include "glm_family.cuh"

namespace b200flow {

namespace {

constexpr int kChunkRows = 4096;
constexpr int kGlmTile = 32;                      // rows per tile: four per warp
constexpr int kGlmThreads = 256;                  // one column thread per feature; the last thread sums the scalars
constexpr int kGlmLanes = 8;                      // lanes per row in the margin
constexpr int kGlmMaxD = 255;
constexpr int kGlmTerms = 8;                      // summary partial width

__host__ __device__ inline int glm_pitch(int D) { return D | 1; }

inline size_t glm_smem(int D) { return ((size_t)kGlmTile * glm_pitch(D) + D) * sizeof(double); }

// one row's outputs and its terms t[k * kGlmTile] of the chunk sums (the caller zeroes them).  Not inlined: the math
// library's slow paths are calls, and the tile loop's state would be saved around each of them.
__device__ __noinline__ void glm_row(GlmSpec s, int mode, double m, bool has_coef, double intercept, double mu_const,
                                     double yv, double w, double off, double* __restrict__ rows_out, int64_t gr,
                                     double* t) {
    if (mode == B200FLOW_GLM_INIT) {
        const double z = glm_link(s, glm_initialize(s, yv, w)) - off;
        rows_out[2 * gr] = z;
        rows_out[2 * gr + 1] = w;
        t[0 * kGlmTile] = w;
        t[1 * kGlmTile] = w * z;
        return;
    }
    double eta, mu;
    if (has_coef) {
        eta = (m + intercept) + off;
        mu = glm_project(s, glm_unlink(s, eta));
    } else {                                      // the null model's constant mean
        mu = mu_const;
        eta = glm_link(s, mu);
    }
    if (mode == B200FLOW_GLM_PREDICT) {
        rows_out[2 * gr] = mu;
        rows_out[2 * gr + 1] = eta;
    } else if (mode == B200FLOW_GLM_REWEIGHT) {
        const double d = glm_deriv(s, mu);
        const double z = (eta - off) + (yv - mu) * d;
        const double ww = w / (d * d * glm_variance(s, mu));
        rows_out[2 * gr] = z;
        rows_out[2 * gr + 1] = ww;
        t[0 * kGlmTile] = ww;
        t[1 * kGlmTile] = ww * z;
    } else {                                      // SUMMARY
        const double r = yv - mu, dev = glm_deviance(s, yv, mu, w);
        const double pr = r * sqrt(w) / sqrt(glm_variance(s, mu));
        if (rows_out) {
            const double dr = sqrt(dev > 0.0 ? dev : 0.0);
            rows_out[4 * gr] = r > 0.0 ? dr : (r < 0.0 ? -dr : 0.0);
            rows_out[4 * gr + 1] = pr;
            rows_out[4 * gr + 2] = r * glm_deriv(s, mu);
            rows_out[4 * gr + 3] = r;
        }
        t[0 * kGlmTile] = w;
        t[1 * kGlmTile] = w * yv;
        t[2 * kGlmTile] = dev;
        t[3 * kGlmTile] = pr * pr;
        t[4 * kGlmTile] = glm_aic_term(s, yv, mu, w);
        if (s.family == B200FLOW_GLM_GAMMA) {
            t[5 * kGlmTile] = w * log(yv);
            t[6 * kGlmTile] = w * (yv / mu);
            t[7 * kGlmTile] = w * log(mu);
        }
    }
}

template <typename T>
__global__ void __launch_bounds__(kGlmThreads) glm_rows_kernel(const T* __restrict__ x, int64_t n, int64_t ld, int D,
                                                               const double* __restrict__ y,
                                                               const double* __restrict__ weight,
                                                               const double* __restrict__ offset,
                                                               const double* __restrict__ coef, double intercept,
                                                               double mu_const, GlmSpec s, int mode, int64_t row_offset,
                                                               double* __restrict__ rows_out, double* __restrict__ partials) {
    extern __shared__ double sm[];
    __shared__ double tv[kGlmTerms][kGlmTile];    // the tile's per-row terms of the chunk sums
    const int pitch = glm_pitch(D);
    double* X = sm;                               // [kGlmTile][pitch]
    double* cs = X + kGlmTile * pitch;            // [D]: coef
    const bool margin = coef != nullptr && mode != B200FLOW_GLM_INIT;
    const bool columns = mode == B200FLOW_GLM_INIT || mode == B200FLOW_GLM_REWEIGHT;
    for (int j = threadIdx.x; j < D; j += kGlmThreads) cs[j] = margin ? coef[j] : 0.0;
    const int64_t c0 = (row_offset / kChunkRows + blockIdx.x) * kChunkRows - row_offset;   // local index of the chunk's row 0
    const int64_t lo = c0 > 0 ? c0 : 0, hi = c0 + kChunkRows < n ? c0 + kChunkRows : n;
    const int tid = threadIdx.x, lane = lane_id(), sub = lane & (kGlmLanes - 1);
    const int row = warp_id() * (32 / kGlmLanes) + lane / kGlmLanes;
    // the scalar sums: the last thread holds both of INIT / REWEIGHT's, thread kGlmThreads - kGlmTerms + k term k of SUMMARY's
    const int term = columns ? 0 : tid - (kGlmThreads - kGlmTerms);
    const bool sums = columns ? tid == kGlmThreads - 1 : term >= 0;
    double g = 0.0, a0 = 0.0, a1 = 0.0;
    for (int64_t base = c0 + (lo - c0) / kGlmTile * kGlmTile; base < hi; base += kGlmTile) {
        __syncthreads();                          // cs is staged; the previous tile is done with X and tv
        if (margin || columns) {
#pragma unroll 4
            for (int e = tid; e < kGlmTile * D; e += kGlmThreads) {
                const int r = e / D, j = e - r * D;
                const int64_t gr = base + r;
                X[r * pitch + j] = gr >= lo && gr < hi ? (double)x[gr * ld + j] : 0.0;
            }
            __syncthreads();
        }
        double m = 0.0;
        if (margin) {
            const double* xr = X + row * pitch;
            double p = 0.0;
            for (int j = sub; j < D; j += kGlmLanes) p = p + xr[j] * cs[j];
            p = p + __shfl_xor_sync(0xffffffffu, p, 4);
            p = p + __shfl_xor_sync(0xffffffffu, p, 2);
            m = p + __shfl_xor_sync(0xffffffffu, p, 1);
        }
        if (sub == 0) {
            const int64_t gr = base + row;
            double* t = &tv[0][row];              // t[k * kGlmTile]: term k of the row
#pragma unroll
            for (int k = 0; k < kGlmTerms; ++k) t[k * kGlmTile] = 0.0;
            if (gr >= lo && gr < hi)
                glm_row(s, mode, m, coef != nullptr, intercept, mu_const, mode == B200FLOW_GLM_PREDICT ? 0.0 : y[gr],
                        weight ? weight[gr] : 1.0, offset ? offset[gr] : 0.0, rows_out, gr, t);
        }
        if (mode == B200FLOW_GLM_PREDICT) continue;
        __syncthreads();
        if (columns && tid < D) {
#pragma unroll 8
            for (int r = 0; r < kGlmTile; ++r) g = g + tv[0][r] * X[r * pitch + tid];
        } else if (sums) {
            for (int r = 0; r < kGlmTile; ++r) {
                a0 = a0 + tv[term][r];
                if (columns) a1 = a1 + tv[1][r];
            }
        }
    }
    if (mode == B200FLOW_GLM_PREDICT) return;
    if (columns) {
        double* part = partials + (int64_t)blockIdx.x * (D + 2);
        if (tid < D) part[1 + tid] = g;
        if (sums) {
            part[0] = a0;
            part[D + 1] = a1;
        }
    } else if (sums) {
        partials[(int64_t)blockIdx.x * kGlmTerms + term] = a0;
    }
}

}  // namespace

}  // namespace b200flow

using namespace b200flow;

extern "C" int b200flow_glm_rows(const void* x, int32_t x_dtype, int64_t n_rows, int64_t ld, int32_t D, const double* y,
                                 const double* weight, const double* offset, const double* coef, double intercept,
                                 double mu_const, int32_t family, int32_t link, double variance_power, double link_power,
                                 int32_t mode, int64_t row_offset, double* rows_out, double* partials, void* stream) {
    B2F_REQUIRE(D >= 1 && D <= kGlmMaxD, "glm_rows: 1 <= D <= %d features, got %d", kGlmMaxD, D);
    B2F_REQUIRE(n_rows >= 0 && row_offset >= 0 && ld >= D && (x_dtype == B200FLOW_F32 || x_dtype == B200FLOW_F64),
                "glm_rows: n >= 0, row_offset >= 0, ld >= D, f32 or f64 features");
    B2F_REQUIRE(mode >= B200FLOW_GLM_INIT && mode <= B200FLOW_GLM_PREDICT, "glm_rows: unknown mode %d", mode);
    B2F_REQUIRE(family >= B200FLOW_GLM_GAUSSIAN && family <= B200FLOW_GLM_TWEEDIE, "glm_rows: unknown family %d", family);
    B2F_REQUIRE(link >= B200FLOW_GLM_IDENTITY && link <= B200FLOW_GLM_POWER, "glm_rows: unknown link %d", link);
    if (n_rows == 0) return B200FLOW_OK;
    const bool needs_coef = mode == B200FLOW_GLM_REWEIGHT || mode == B200FLOW_GLM_PREDICT;
    B2F_REQUIRE(x && (y || mode == B200FLOW_GLM_PREDICT) && (coef || !needs_coef) &&
                    (rows_out || mode == B200FLOW_GLM_SUMMARY) && (partials || mode == B200FLOW_GLM_PREDICT),
                "glm_rows: null pointer");
    const int64_t nc = (row_offset + n_rows - 1) / kChunkRows - row_offset / kChunkRows + 1;
    B2F_REQUIRE(nc <= 0x7fffffffll, "glm_rows: too many rows");
    const GlmSpec s{family, link, variance_power, link_power};
    const size_t smem = glm_smem(D);
    cudaStream_t st = (cudaStream_t)stream;
    if (x_dtype == B200FLOW_F64) {
        cudaFuncSetAttribute(glm_rows_kernel<double>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        glm_rows_kernel<double><<<(unsigned)nc, kGlmThreads, smem, st>>>((const double*)x, n_rows, ld, D, y, weight, offset,
                                                                         coef, intercept, mu_const, s, mode, row_offset,
                                                                         rows_out, partials);
    } else {
        cudaFuncSetAttribute(glm_rows_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        glm_rows_kernel<float><<<(unsigned)nc, kGlmThreads, smem, st>>>((const float*)x, n_rows, ld, D, y, weight, offset,
                                                                        coef, intercept, mu_const, s, mode, row_offset,
                                                                        rows_out, partials);
    }
    return check_launch("glm_rows");
}
