// linreg.cu — LinearRegression and AFTSurvivalRegression: the per-row least-squares / Huber / Weibull AFT loss and gradient
// sums, DESIGN.md §5n, §5q.
//
// One pass over the rows per optimiser evaluation.  At one weight column the pass is bound by HBM (about 0.5 FLOP per
// byte at f64), so it uses plain fp64 FMA-free arithmetic, not tensor cores; what matters is that every element of x is read
// once: a tile is staged in shared memory, scaled, and read from there by both the margin and the gradient phase.
//
// b200flow_linreg_loss_grad: one CTA per 4096-row global chunk walks the chunk's 32-row tiles, which sit at fixed global
// positions, in row order.  A tile is staged as xs = (x − shift)·inv (one fixed rounding order: the subtraction, then the
// product; no shift: the product alone); rows outside the chunk or outside [0, n) are staged as 0 and masked.
//   margin phase: thread r of warp 0 sums m = Σ_j xs[r][j]·w[j] over the features in ascending order from +0.0 and turns
//     it into the row's loss term l, gradient coefficient a and σ-derivative s (all 0 for a masked row):
//       squared: d = m − (y − c)·t, l = d², a = d, s = 0;
//       huber:   z = (y − m − b)/σ; |z| <= ε: l = σ + z²σ, a = −2z, s = 1 − z²;  else l = σ + (2ε|z| − ε²)σ, a = −2ε·sign(z),
//                s = 1 − ε².
//     aft (a separate instantiation, kAft): y = log t, δ the censor (1 observed, 0 censored), z = (y − m − b)/σ;
//                l = δ·log σ − δ·z + e^z, a = (δ − e^z)/σ, s = δ + (δ − e^z)·z.
//   gradient phase: thread j < D adds a[r]·xs[r][j] over the tile's rows in order; the last thread adds l, a and s.
// Each sum runs over the chunk's rows in row order from +0.0, so a chunk's partial depends only on its rows and the
// inputs.  No atomics.
#include "common.cuh"

namespace b200flow {

namespace {

constexpr int kChunkRows = 4096;
constexpr int kLrTile = 32;                       // rows per tile: one margin thread per row (warp 0)
constexpr int kLrThreads = 256;                   // one gradient thread per feature; the last thread sums the scalars
constexpr int kLrMaxD = 255;

__host__ __device__ inline int lr_pitch(int D) { return D | 1; }    // odd: the margin threads' row reads are conflict-free

inline size_t lr_smem(int D) { return ((size_t)kLrTile * lr_pitch(D) + 3 * (size_t)D) * sizeof(double); }

template <typename T, bool kAft>
__global__ void __launch_bounds__(kLrThreads) linreg_loss_grad_kernel(const T* __restrict__ x, int64_t n, int64_t ld, int D,
                                                                      const double* __restrict__ y,
                                                                      const double* __restrict__ shift,
                                                                      const double* __restrict__ inv, double y_shift,
                                                                      double y_scale, const double* __restrict__ w,
                                                                      const double* __restrict__ b_sigma, double eps,
                                                                      int mode, int64_t row_offset,
                                                                      double* __restrict__ partials,
                                                                      const int32_t* __restrict__ censor) {
    extern __shared__ double sm[];
    __shared__ double av[kLrTile], lv[kLrTile], sv[kLrTile];
    const int pitch = lr_pitch(D);
    double* X = sm;                               // [kLrTile][pitch]
    double* ws = X + kLrTile * pitch;             // [D]
    double* ss = ws + D;                          // [D]: shift (0 without one)
    double* is = ss + D;                          // [D]
    for (int j = threadIdx.x; j < D; j += kLrThreads) {
        ws[j] = w[j];
        ss[j] = shift ? shift[j] : 0.0;
        is[j] = inv[j];
    }
    const bool huber = mode == B200FLOW_LINREG_HUBER, shifted = shift != nullptr;
    const double b = huber || kAft ? b_sigma[0] : 0.0, sigma = huber || kAft ? b_sigma[1] : 1.0;
    const double log_sigma = kAft ? b_sigma[2] : 0.0;
    const int64_t c0 = (row_offset / kChunkRows + blockIdx.x) * kChunkRows - row_offset;   // local index of the chunk's row 0
    const int64_t lo = c0 > 0 ? c0 : 0, hi = c0 + kChunkRows < n ? c0 + kChunkRows : n;
    const int tid = threadIdx.x;
    double g = 0.0, loss = 0.0, gb = 0.0, gs = 0.0;
    for (int64_t base = c0 + (lo - c0) / kLrTile * kLrTile; base < hi; base += kLrTile) {
        __syncthreads();                          // ws / ss / is are staged; the previous tile's gradient is done with X
#pragma unroll 4
        for (int e = tid; e < kLrTile * D; e += kLrThreads) {
            const int r = e / D, j = e - r * D;
            const int64_t gr = base + r;
            double v = 0.0;
            if (gr >= lo && gr < hi) {
                v = (double)x[gr * ld + j];
                if (shifted) v = v - ss[j];
                v = v * is[j];
            }
            X[r * pitch + j] = v;
        }
        __syncthreads();
        if (tid < kLrTile) {
            const int64_t gr = base + tid;
            double l = 0.0, a = 0.0, s = 0.0;
            if (gr >= lo && gr < hi) {
                const double* xr = X + tid * pitch;
                double m = 0.0;
                for (int j = 0; j < D; ++j) m = m + xr[j] * ws[j];
                const double yv = y[gr];
                if (kAft) {
                    const double z = (yv - m - b) / sigma, ez = exp(z), dl = censor[gr] ? 1.0 : 0.0;
                    l = dl * log_sigma - dl * z + ez;
                    a = (dl - ez) / sigma;
                    s = dl + (dl - ez) * z;
                } else if (!huber) {
                    const double d = m - (yv - y_shift) * y_scale;
                    l = d * d;
                    a = d;
                } else {
                    const double z = (yv - m - b) / sigma, az = fabs(z);
                    if (az <= eps) {
                        l = sigma + z * z * sigma;
                        a = -2.0 * z;
                        s = 1.0 - z * z;
                    } else {
                        l = sigma + (2.0 * eps * az - eps * eps) * sigma;
                        a = z > 0.0 ? -2.0 * eps : 2.0 * eps;
                        s = 1.0 - eps * eps;
                    }
                }
            }
            av[tid] = a;
            lv[tid] = l;
            sv[tid] = s;
        }
        __syncthreads();
        if (tid < D) {
#pragma unroll 8
            for (int r = 0; r < kLrTile; ++r) g = g + av[r] * X[r * pitch + tid];
        } else if (tid == kLrThreads - 1) {
            for (int r = 0; r < kLrTile; ++r) {
                loss = loss + lv[r];
                gb = gb + av[r];
                gs = gs + sv[r];
            }
        }
    }
    double* part = partials + (int64_t)blockIdx.x * (D + 3);
    if (tid < D) part[1 + tid] = g;
    if (tid == kLrThreads - 1) {
        part[0] = loss;
        part[D + 1] = gb;
        part[D + 2] = gs;
    }
}

}  // namespace

}  // namespace b200flow

using namespace b200flow;

extern "C" int b200flow_linreg_loss_grad(const void* x, int32_t x_dtype, int64_t n_rows, int64_t ld, int32_t D, const double* y,
                                         const double* shift, const double* inv, double y_shift, double y_scale,
                                         const double* w, const double* b_sigma, double epsilon, int32_t mode,
                                         int64_t row_offset, double* partials, void* stream) {
    B2F_REQUIRE(D >= 1 && D <= kLrMaxD, "linreg_loss_grad: 1 <= D <= %d features, got %d", kLrMaxD, D);
    B2F_REQUIRE(n_rows >= 0 && row_offset >= 0 && ld >= D && (x_dtype == B200FLOW_F32 || x_dtype == B200FLOW_F64),
                "linreg_loss_grad: n >= 0, row_offset >= 0, ld >= D, f32 or f64 features");
    B2F_REQUIRE(mode == B200FLOW_LINREG_SQUARED || mode == B200FLOW_LINREG_HUBER, "linreg_loss_grad: unknown mode %d", mode);
    if (n_rows == 0) return B200FLOW_OK;
    B2F_REQUIRE(x && y && inv && w && partials && (mode == B200FLOW_LINREG_SQUARED || b_sigma), "linreg_loss_grad: null pointer");
    const int64_t nc = (row_offset + n_rows - 1) / kChunkRows - row_offset / kChunkRows + 1;
    B2F_REQUIRE(nc <= 0x7fffffffll, "linreg_loss_grad: too many rows");
    const size_t smem = lr_smem(D);
    cudaStream_t st = (cudaStream_t)stream;
    if (x_dtype == B200FLOW_F64) {
        cudaFuncSetAttribute(linreg_loss_grad_kernel<double, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        linreg_loss_grad_kernel<double, false><<<(unsigned)nc, kLrThreads, smem, st>>>((const double*)x, n_rows, ld, D, y,
                                                                                      shift, inv, y_shift, y_scale, w, b_sigma,
                                                                                      epsilon, mode, row_offset, partials,
                                                                                      nullptr);
    } else {
        cudaFuncSetAttribute(linreg_loss_grad_kernel<float, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        linreg_loss_grad_kernel<float, false><<<(unsigned)nc, kLrThreads, smem, st>>>((const float*)x, n_rows, ld, D, y,
                                                                                     shift, inv, y_shift, y_scale, w, b_sigma,
                                                                                     epsilon, mode, row_offset, partials,
                                                                                     nullptr);
    }
    return check_launch("linreg_loss_grad");
}

extern "C" int b200flow_aft_loss_grad(const void* x, int32_t x_dtype, int64_t n_rows, int64_t ld, int32_t D, const double* log_t,
                                      const int32_t* censor, const double* shift, const double* inv, const double* w,
                                      const double* b_sigma, int64_t row_offset, double* partials, void* stream) {
    B2F_REQUIRE(D >= 1 && D <= kLrMaxD, "aft_loss_grad: 1 <= D <= %d features, got %d", kLrMaxD, D);
    B2F_REQUIRE(n_rows >= 0 && row_offset >= 0 && ld >= D && (x_dtype == B200FLOW_F32 || x_dtype == B200FLOW_F64),
                "aft_loss_grad: n >= 0, row_offset >= 0, ld >= D, f32 or f64 features");
    if (n_rows == 0) return B200FLOW_OK;
    B2F_REQUIRE(x && log_t && censor && inv && w && b_sigma && partials, "aft_loss_grad: null pointer");
    const int64_t nc = (row_offset + n_rows - 1) / kChunkRows - row_offset / kChunkRows + 1;
    B2F_REQUIRE(nc <= 0x7fffffffll, "aft_loss_grad: too many rows");
    const size_t smem = lr_smem(D);
    cudaStream_t st = (cudaStream_t)stream;
    if (x_dtype == B200FLOW_F64) {
        cudaFuncSetAttribute(linreg_loss_grad_kernel<double, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        linreg_loss_grad_kernel<double, true><<<(unsigned)nc, kLrThreads, smem, st>>>((const double*)x, n_rows, ld, D, log_t,
                                                                                     shift, inv, 0.0, 1.0, w, b_sigma, 0.0,
                                                                                     B200FLOW_LINREG_SQUARED, row_offset,
                                                                                     partials, censor);
    } else {
        cudaFuncSetAttribute(linreg_loss_grad_kernel<float, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        linreg_loss_grad_kernel<float, true><<<(unsigned)nc, kLrThreads, smem, st>>>((const float*)x, n_rows, ld, D, log_t,
                                                                                    shift, inv, 0.0, 1.0, w, b_sigma, 0.0,
                                                                                    B200FLOW_LINREG_SQUARED, row_offset,
                                                                                    partials, censor);
    }
    return check_launch("aft_loss_grad");
}
