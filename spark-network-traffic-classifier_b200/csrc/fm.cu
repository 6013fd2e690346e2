// fm.cu — FMClassifier and FMRegressor: the logistic / squared-error factorization-machine loss + gradient and the raw
// values, DESIGN.md §5k, §5r.
//
// K binary problems over the same rows at once: column k treats label == positives[k] as y = 1 and every other label as
// y = 0, with weights [V_k (D x F, row-major), w_k (D), b_k].  Per row and column, with s_f = sum_i v_if x_i and
// q_f = sum_i x_i^2 v_if^2,
//     r = (b + x . w) + 1/2 (s_0^2 - q_0) + 1/2 (s_1^2 - q_1) + ...,   g = sigmoid(r) - y,
//     loss = log1pExp(-r) if y = 1 else log1pExp(r),
// and the row adds g [x_i s_f] (the factor gradient before its - v_if x_i^2 term), g x_i, g and g x_i^2 to column k's
// sums.  The host applies the - V (x^2 . g) term once, to the totals.
//
// Each class owns F + 1 consecutive columns of U = [V | w] (factor f of class c is column c (F + 1) + f, its linear
// weights column c (F + 1) + F).  The products S = X U, Q = X^2 U^2 (the squares taken as the fragments are loaded),
// [X, 1]^T [g S | g] and X^2^T g are fp64 tensor-core MMAs (mma.sync m8n8k4 f64), fragments as in svc.cu.  An MMA output
// element depends only on its own row of one operand and column of the other, the contractions run in one fixed order,
// and every class reads only its own columns, intercept and label test.  So column k's partial depends on column k's
// weights and positive label alone: not on K, on the other columns, or on the class block where k lands.
//
// b200flow_fm_loss_grad: one CTA per (4096-row global chunk, class block).  It stages its block's U in shared memory
// once, then walks the chunk's 32-row tiles in row order (tiles sit at fixed global positions): load x as f64 beside a
// ones column, S and Q, then per (row, class) r, g and the loss, a sequential row-order loss sum per class, and the
// gradient products.  The gradient accumulates in registers for the whole chunk: tile t belongs to warp t % 8, slot t / 8.
// Rows outside the launch, and rows the mini-batch draw leaves out, are masked (g = 0, no loss), never padded in.
//
// b200flow_fm_regression_loss_grad: the same kernel with the squared-error policy (kReg): one column, f64 labels read as
// they are, g = 2 (r - y), loss (r - y)^2; no class labels or positives are read.
//
// b200flow_fm_raw: the same tile load, products and per-row arithmetic, r written out per row.
#include "common.cuh"

namespace b200flow {

namespace {

constexpr int kChunkRows = 4096;
constexpr int kFmTile = 32;                       // rows per tile: 4 MMA row blocks
constexpr int kFmWarps = 8, kFmThreads = kFmWarps * 32;
constexpr int kFmSlots = 32;                      // gradient tiles per warp: at most 256 8x8 tiles per class block
constexpr int kFmMaxD = 255;                      // D + 1 (the ones column) padded to at most 256
constexpr int kFmMaxBlockClasses = kFmThreads;    // one thread per class sums its loss
constexpr int kFmMaxSmem = 227 * 1024 - 4096;     // dynamic shared memory; the static label / intercept buffers take the rest
constexpr uint32_t PURPOSE_FMMB = 0x464D4D42u;    // mini-batch draw, ctr = (row_lo,row_hi,0,0), key seed 42 + iteration

struct FmShape {
    int D, Dp, F, F1;                             // features; D + 1 padded to 8; factors; F + 1 columns per class
    int64_t K;                                    // classes
    int kb, blocks;                               // classes per block, class blocks
    int nc, ngt, nst;                             // U columns (kb F1 padded to 8); [X, 1]^T [gS | g] tiles; X^2^T g tiles
    int px, pu, pm, pg;                           // pitches of X [32][px], U [nc][pu], S / Q [32][pm], G [32][pg]
    int xoff, soff, qoff, goff, loff, smem_doubles;   // U at 0, L [32][kb] at loff
};

// the layout for kb classes per block; returns its gradient tiles
int64_t fm_layout(FmShape* s, int kb) {
    const int64_t ndt = s->Dp / 8;
    const int64_t nc = ((int64_t)kb * s->F1 + 7) / 8 * 8;
    const int64_t tiles = (nc / 8 + (kb + 7) / 8) * ndt;
    if (nc > (1 << 20)) return tiles;             // far beyond any fit; keep the int fields below from overflowing
    s->kb = kb;
    s->nc = (int)nc;
    s->ngt = (int)(nc / 8 * ndt);
    s->nst = (int)((kb + 7) / 8 * ndt);
    s->px = s->Dp + 4;                            // 4 mod 8 doubles, as mlp.cu's pitches
    s->pu = s->Dp + 4;
    s->pm = s->nc + 4;
    s->pg = pad8(kb) + 4;
    s->xoff = s->nc * s->pu;
    s->soff = s->xoff + kFmTile * s->px;
    s->qoff = s->soff + kFmTile * s->pm;
    s->goff = s->qoff + kFmTile * s->pm;
    s->loff = s->goff + kFmTile * s->pg;
    s->smem_doubles = s->loff + kFmTile * kb;
    return tiles;
}

bool fm_fits(FmShape* s, int kb) {
    const int64_t tiles = fm_layout(s, kb);
    return tiles <= (int64_t)kFmWarps * kFmSlots && s->kb == kb && (int64_t)s->smem_doubles * 8 <= kFmMaxSmem;
}

int fm_shape(int D, int F, int64_t K, FmShape* s) {
    B2F_REQUIRE(D >= 1 && D <= kFmMaxD, "fm: 1 <= D <= %d features, got %d", kFmMaxD, D);
    B2F_REQUIRE(F >= 1, "fm: factorSize >= 1, got %d", F);
    B2F_REQUIRE(K >= 1, "fm: at least one class column, got %lld", (long long)K);
    s->D = D;
    s->Dp = pad8(D + 1);
    s->F = F;
    s->F1 = F + 1;
    s->K = K;
    s->kb = 0;
    int per = K < kFmMaxBlockClasses ? (int)K : kFmMaxBlockClasses;
    while (per >= 1 && !fm_fits(s, per)) --per;
    B2F_REQUIRE(per >= 1, "fm: D = %d features with factorSize %d exceed one class block (256 gradient tiles of 8x8, %d bytes "
                "of shared memory)", D, F, kFmMaxSmem);
    const int64_t blocks = (K + per - 1) / per;
    B2F_REQUIRE(blocks <= 65535, "fm: at most %lld class columns", (long long)per * 65535);
    s->blocks = (int)blocks;
    fm_layout(s, (int)((K + blocks - 1) / blocks));
    return B200FLOW_OK;
}

// per class: weights [V (D x F) | w (D) | b]
__host__ __device__ inline int64_t fm_params(const FmShape& s) { return (int64_t)s.D * s.F1 + 1; }

// the block's U into shared memory (zeros elsewhere, the ones column's row of U included), intercepts into bsh, the
// rest zeroed, the ones column of X set
__device__ void fm_stage(const FmShape& s, const double* __restrict__ w, int nk, double* sm, double* bsh) {
    const int64_t P = fm_params(s);
    for (int e = threadIdx.x; e < s.nc * s.pu; e += kFmThreads) {
        const int col = e / s.pu, j = e - col * s.pu;
        const int c = col / s.F1, f = col - c * s.F1;
        double v = 0.0;
        if (c < nk && j < s.D) v = w[c * P + (f < s.F ? (int64_t)j * s.F + f : (int64_t)s.D * s.F + j)];
        sm[e] = v;
    }
    for (int e = s.xoff + threadIdx.x; e < s.smem_doubles; e += kFmThreads) sm[e] = 0.0;
    if (threadIdx.x < nk) bsh[threadIdx.x] = w[threadIdx.x * P + P - 1];
    __syncthreads();
    for (int r = threadIdx.x; r < kFmTile; r += kFmThreads) sm[s.xoff + r * s.px + s.D] = 1.0;
}

// rows [base, base + 32) of x into X as f64 (rows outside [0, n) -> 0)
template <typename T>
__device__ void fm_load_tile(const FmShape& s, const T* __restrict__ x, int64_t n, int64_t ld, int64_t base, double* X) {
    const int D = s.D;
    for (int e = threadIdx.x; e < kFmTile * D; e += kFmThreads) {
        const int r = e / D, j = e - r * D;
        const int64_t gr = base + r;
        X[r * s.px + j] = (gr >= 0 && gr < n) ? load_as_double<T>(x, gr * ld + j) : 0.0;
    }
}

// S = X U and Q = X^2 U^2 over all nc columns.  The 8x8 output tiles (column tile, row block) are shared out over the
// warps; every output element accumulates over the features in ascending order whichever warp computes it.
__device__ void fm_products_tile(const FmShape& s, const double* X, const double* U, double* S, double* Q) {
    const int lane = lane_id(), warp = warp_id(), qr = lane >> 2, qc = lane & 3;
    const int nk4 = s.Dp / 4;
    for (int item = warp; item < (s.nc / 8) * 4; item += kFmWarps) {
        const int nt = item >> 2, m = item & 3;
        double c[2] = {0.0, 0.0}, c2[2] = {0.0, 0.0};
        for (int k = 0; k < nk4; ++k) {
            const double a = X[(m * 8 + qr) * s.px + k * 4 + qc], b = U[(nt * 8 + qr) * s.pu + k * 4 + qc];
            dmma(c, a, b);
            dmma(c2, a * a, b * b);
        }
#pragma unroll
        for (int q = 0; q < 2; ++q) {
            const int o = (m * 8 + qr) * s.pm + nt * 8 + 2 * qc + q;
            S[o] = c[q];
            Q[o] = c2[q];
        }
    }
}

// r of one row and class from its S / Q row and first column, in Spark's order: intercept, linear term, then each factor
__device__ __forceinline__ double fm_raw_value(const double* Srow, const double* Qrow, int col0, int F, double b) {
    double r = b + Srow[col0 + F];
    for (int f = 0; f < F; ++f) {
        const double sv = Srow[col0 + f];
        r = r + 0.5 * (sv * sv - Qrow[col0 + f]);
    }
    return r;
}

__device__ __forceinline__ double log1p_exp(double v) { return v > 0.0 ? v + log1p(exp(-v)) : log1p(exp(v)); }

template <typename T, bool kReg>
__global__ void __launch_bounds__(kFmThreads, 1) fm_loss_grad_kernel(const T* __restrict__ x, int64_t n, int64_t ld,
                                                                     const int32_t* __restrict__ y,
                                                                     const int32_t* __restrict__ positives, const FmShape s,
                                                                     const double* __restrict__ w, double fraction,
                                                                     uint64_t batch_seed, int64_t row_offset,
                                                                     double* __restrict__ partials,
                                                                     const double* __restrict__ yreg) {
    extern __shared__ double sm[];
    __shared__ double bsh[kFmMaxBlockClasses];
    __shared__ int ylab[kFmTile], yval[kFmTile], posb[kFmMaxBlockClasses];
    const int lane = lane_id(), warp = warp_id(), qr = lane >> 2, qc = lane & 3;
    const int64_t k0 = (int64_t)blockIdx.y * s.kb;
    const int nk = (int)(s.K - k0 < s.kb ? s.K - k0 : s.kb);
    const int D = s.D, F = s.F, F1 = s.F1, ndt = s.Dp / 8;
    double* X = sm + s.xoff;
    double* S = sm + s.soff;
    double* Q = sm + s.qoff;
    double* G = sm + s.goff;
    double* L = sm + s.loff;
    fm_stage(s, w + k0 * fm_params(s), nk, sm, bsh);
    const int64_t c0 = (row_offset / kChunkRows + blockIdx.x) * kChunkRows - row_offset;   // local index of the chunk's row 0
    const int64_t lo = c0 > 0 ? c0 : 0, hi = c0 + kChunkRows < n ? c0 + kChunkRows : n;
    const bool sampled = fraction < 1.0;
    const uint64_t keep_below = (uint64_t)floor(fraction * 4294967296.0);
    if (!kReg && threadIdx.x < nk) posb[threadIdx.x] = positives[k0 + threadIdx.x];
    double acc[kFmSlots][2];
#pragma unroll
    for (int q = 0; q < kFmSlots; ++q) acc[q][0] = acc[q][1] = 0.0;
    double loss = 0.0, count = 0.0;
    for (int64_t base = c0 + (lo - c0) / kFmTile * kFmTile; base < hi; base += kFmTile) {
        __syncthreads();                                   // the previous tile's gradient has read X, S and G
        fm_load_tile(s, x, n, ld, base, X);
        if (threadIdx.x < kFmTile) {
            const int64_t gr = base + threadIdx.x;
            bool valid = gr >= lo && gr < hi;
            if (valid && sampled) {
                const uint64_t row = (uint64_t)(row_offset + gr);
                valid = philox_keyed(batch_seed, PURPOSE_FMMB, (uint32_t)row, (uint32_t)(row >> 32), 0u, 0u).x < keep_below;
            }
            yval[threadIdx.x] = valid;
            if (!kReg) ylab[threadIdx.x] = valid ? y[gr] : 0;
        }
        __syncthreads();
        fm_products_tile(s, X, sm, S, Q);
        __syncthreads();
        for (int e = threadIdx.x; e < kFmTile * nk; e += kFmThreads) {   // S becomes [g S | g], G = g, L = the loss
            const int r = e / nk, c = e - r * nk, col0 = c * F1;
            double* Sr = S + r * s.pm;
            double g = 0.0, l = 0.0;
            if (yval[r]) {
                const double rv = fm_raw_value(Sr, Q + r * s.pm, col0, F, bsh[c]);
                if (kReg) {
                    const double d = rv - yreg[base + r];
                    g = 2.0 * d;
                    l = d * d;
                } else {
                    const bool pos = ylab[r] == posb[c];
                    g = 1.0 / (1.0 + exp(-rv)) - (pos ? 1.0 : 0.0);
                    l = pos ? log1p_exp(-rv) : log1p_exp(rv);
                }
            }
            for (int f = 0; f < F; ++f) Sr[col0 + f] = yval[r] ? g * Sr[col0 + f] : 0.0;
            Sr[col0 + F] = g;
            G[r * s.pg + c] = g;
            L[r * s.kb + c] = l;
        }
        __syncthreads();
        if (threadIdx.x < nk) {                            // class threadIdx.x sums its loss over the rows in order
            for (int r = 0; r < kFmTile; ++r)
                if (yval[r]) {
                    loss = loss + L[r * s.kb + threadIdx.x];
                    count = count + 1.0;
                }
        }
#pragma unroll
        for (int q = 0; q < kFmSlots; ++q) {               // gradient: [X, 1]^T [g S | g] and X^2^T g over the tile's rows
            const int t = warp + kFmWarps * q;
            if (t < s.ngt) {
                const int ct = t / ndt, dt = t - ct * ndt;
#pragma unroll
                for (int k = 0; k < kFmTile / 4; ++k)
                    dmma(acc[q], S[(k * 4 + qc) * s.pm + ct * 8 + qr], X[(k * 4 + qc) * s.px + dt * 8 + qr]);
            } else if (t < s.ngt + s.nst) {
                const int u = t - s.ngt, ct = u / ndt, dt = u - ct * ndt;
#pragma unroll
                for (int k = 0; k < kFmTile / 4; ++k) {
                    const double xv = X[(k * 4 + qc) * s.px + dt * 8 + qr];
                    dmma(acc[q], G[(k * 4 + qc) * s.pg + ct * 8 + qr], xv * xv);
                }
            }
        }
    }
    // per class: [loss, count, gV (D x F), gw (D), gb, x^2 g (D)]
    const int64_t W = fm_params(s) + 2 + D;
    double* part = partials + ((int64_t)blockIdx.x * s.K + k0) * W;
    if (threadIdx.x < nk) {
        part[(int64_t)threadIdx.x * W] = loss;
        part[(int64_t)threadIdx.x * W + 1] = count;
    }
#pragma unroll
    for (int q = 0; q < kFmSlots; ++q) {
        const int t = warp + kFmWarps * q;
        if (t < s.ngt) {
            const int ct = t / ndt, dt = t - ct * ndt, col = ct * 8 + qr, c = col / F1, f = col - c * F1;
            if (c < nk) {
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int j = dt * 8 + 2 * qc + h;
                    double* pc = part + (int64_t)c * W + 2;
                    if (f < F && j < D) pc[(int64_t)j * F + f] = acc[q][h];
                    else if (f == F && j <= D) pc[(int64_t)D * F + j] = acc[q][h];
                }
            }
        } else if (t < s.ngt + s.nst) {
            const int u = t - s.ngt, ct = u / ndt, dt = u - ct * ndt, c = ct * 8 + qr;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int j = dt * 8 + 2 * qc + h;
                if (c < nk && j < D) part[(int64_t)c * W + 3 + (int64_t)D * F1 + j] = acc[q][h];
            }
        }
    }
}

template <typename T>
__global__ void __launch_bounds__(kFmThreads) fm_raw_kernel(const T* __restrict__ x, int64_t n, int64_t ld, const FmShape s,
                                                            const double* __restrict__ w, double* __restrict__ raw) {
    extern __shared__ double sm[];
    __shared__ double bsh[kFmMaxBlockClasses];
    const int64_t k0 = (int64_t)blockIdx.y * s.kb;
    const int nk = (int)(s.K - k0 < s.kb ? s.K - k0 : s.kb);
    double* X = sm + s.xoff;
    double* S = sm + s.soff;
    double* Q = sm + s.qoff;
    fm_stage(s, w + k0 * fm_params(s), nk, sm, bsh);
    for (int64_t base = (int64_t)blockIdx.x * kFmTile; base < n; base += (int64_t)gridDim.x * kFmTile) {
        __syncthreads();                                   // the previous tile's values are written out
        fm_load_tile(s, x, n, ld, base, X);
        __syncthreads();
        fm_products_tile(s, X, sm, S, Q);
        __syncthreads();
        for (int e = threadIdx.x; e < kFmTile * nk; e += kFmThreads) {
            const int r = e / nk, c = e - r * nk;
            if (base + r < n) raw[(base + r) * s.K + k0 + c] = fm_raw_value(S + r * s.pm, Q + r * s.pm, c * s.F1, s.F, bsh[c]);
        }
    }
}

}  // namespace

}  // namespace b200flow

using namespace b200flow;

extern "C" int b200flow_fm_config(int32_t D, int32_t factor_size, int64_t K, int32_t* block_classes, int32_t* class_blocks,
                                  int64_t* smem_bytes) {
    FmShape s;
    const int rc = fm_shape(D, factor_size, K, &s);
    if (rc != B200FLOW_OK) return rc;
    if (block_classes) *block_classes = s.kb;
    if (class_blocks) *class_blocks = s.blocks;
    if (smem_bytes) *smem_bytes = (int64_t)s.smem_doubles * (int64_t)sizeof(double);
    return B200FLOW_OK;
}

extern "C" int b200flow_fm_loss_grad(const void* x, int32_t x_dtype, int64_t n_rows, int64_t ld, int32_t D, int32_t factor_size,
                                     const int32_t* labels, const int32_t* positives, int64_t K, const double* weights,
                                     double mini_batch_fraction, uint64_t batch_seed, int64_t row_offset, double* partials,
                                     void* stream) {
    FmShape s;
    const int rc = fm_shape(D, factor_size, K, &s);
    if (rc != B200FLOW_OK) return rc;
    B2F_REQUIRE(n_rows >= 0 && row_offset >= 0 && ld >= D && (x_dtype == B200FLOW_F32 || x_dtype == B200FLOW_F64),
                "fm_loss_grad: n >= 0, row_offset >= 0, ld >= D, f32 or f64 features");
    B2F_REQUIRE(mini_batch_fraction > 0.0 && mini_batch_fraction <= 1.0, "fm_loss_grad: miniBatchFraction in (0, 1], got %g",
                mini_batch_fraction);
    if (n_rows == 0) return B200FLOW_OK;
    B2F_REQUIRE(x && labels && positives && weights && partials, "fm_loss_grad: null pointer");
    const int64_t nc = (row_offset + n_rows - 1) / kChunkRows - row_offset / kChunkRows + 1;
    B2F_REQUIRE(nc <= 0x7fffffffll, "fm_loss_grad: too many rows");
    const size_t smem = (size_t)s.smem_doubles * sizeof(double);
    const dim3 grid((unsigned)nc, (unsigned)s.blocks);
    cudaStream_t st = (cudaStream_t)stream;
    if (x_dtype == B200FLOW_F64) {
        cudaFuncSetAttribute(fm_loss_grad_kernel<double, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        fm_loss_grad_kernel<double, false><<<grid, kFmThreads, smem, st>>>((const double*)x, n_rows, ld, labels, positives, s,
                                                                           weights, mini_batch_fraction, batch_seed,
                                                                           row_offset, partials, nullptr);
    } else {
        cudaFuncSetAttribute(fm_loss_grad_kernel<float, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        fm_loss_grad_kernel<float, false><<<grid, kFmThreads, smem, st>>>((const float*)x, n_rows, ld, labels, positives, s,
                                                                          weights, mini_batch_fraction, batch_seed,
                                                                          row_offset, partials, nullptr);
    }
    return check_launch("fm_loss_grad");
}

extern "C" int b200flow_fm_regression_loss_grad(const void* x, int32_t x_dtype, int64_t n_rows, int64_t ld, int32_t D,
                                                int32_t factor_size, const double* labels, const double* weights,
                                                double mini_batch_fraction, uint64_t batch_seed, int64_t row_offset,
                                                double* partials, void* stream) {
    FmShape s;
    const int rc = fm_shape(D, factor_size, 1, &s);
    if (rc != B200FLOW_OK) return rc;
    B2F_REQUIRE(n_rows >= 0 && row_offset >= 0 && ld >= D && (x_dtype == B200FLOW_F32 || x_dtype == B200FLOW_F64),
                "fm_regression_loss_grad: n >= 0, row_offset >= 0, ld >= D, f32 or f64 features");
    B2F_REQUIRE(mini_batch_fraction > 0.0 && mini_batch_fraction <= 1.0,
                "fm_regression_loss_grad: miniBatchFraction in (0, 1], got %g", mini_batch_fraction);
    if (n_rows == 0) return B200FLOW_OK;
    B2F_REQUIRE(x && labels && weights && partials, "fm_regression_loss_grad: null pointer");
    const int64_t nc = (row_offset + n_rows - 1) / kChunkRows - row_offset / kChunkRows + 1;
    B2F_REQUIRE(nc <= 0x7fffffffll, "fm_regression_loss_grad: too many rows");
    const size_t smem = (size_t)s.smem_doubles * sizeof(double);
    const dim3 grid((unsigned)nc, (unsigned)s.blocks);
    cudaStream_t st = (cudaStream_t)stream;
    if (x_dtype == B200FLOW_F64) {
        cudaFuncSetAttribute(fm_loss_grad_kernel<double, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        fm_loss_grad_kernel<double, true><<<grid, kFmThreads, smem, st>>>((const double*)x, n_rows, ld, nullptr, nullptr, s,
                                                                          weights, mini_batch_fraction, batch_seed,
                                                                          row_offset, partials, labels);
    } else {
        cudaFuncSetAttribute(fm_loss_grad_kernel<float, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        fm_loss_grad_kernel<float, true><<<grid, kFmThreads, smem, st>>>((const float*)x, n_rows, ld, nullptr, nullptr, s,
                                                                         weights, mini_batch_fraction, batch_seed,
                                                                         row_offset, partials, labels);
    }
    return check_launch("fm_regression_loss_grad");
}

extern "C" int b200flow_fm_raw(const void* x, int32_t x_dtype, int64_t n_rows, int64_t ld, int32_t D, int32_t factor_size, int64_t K,
                               const double* weights, double* raw, void* stream) {
    FmShape s;
    const int rc = fm_shape(D, factor_size, K, &s);
    if (rc != B200FLOW_OK) return rc;
    B2F_REQUIRE(n_rows >= 0 && ld >= D && (x_dtype == B200FLOW_F32 || x_dtype == B200FLOW_F64),
                "fm_raw: n >= 0, ld >= D, f32 or f64 features");
    if (n_rows == 0) return B200FLOW_OK;
    B2F_REQUIRE(x && weights && raw, "fm_raw: null pointer");
    const size_t smem = (size_t)s.smem_doubles * sizeof(double);
    const int64_t tiles = (n_rows + kFmTile - 1) / kFmTile;
    const int64_t per_sm = (228 * 1024) / (int64_t)(smem + 4096);
    const int64_t cap = (int64_t)kNumSMs * (per_sm > 1 ? per_sm : 1);
    const dim3 grid((unsigned)(tiles < cap ? tiles : cap), (unsigned)s.blocks);
    cudaStream_t st = (cudaStream_t)stream;
    if (x_dtype == B200FLOW_F64) {
        cudaFuncSetAttribute(fm_raw_kernel<double>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        fm_raw_kernel<double><<<grid, kFmThreads, smem, st>>>((const double*)x, n_rows, ld, s, weights, raw);
    } else {
        cudaFuncSetAttribute(fm_raw_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        fm_raw_kernel<float><<<grid, kFmThreads, smem, st>>>((const float*)x, n_rows, ld, s, weights, raw);
    }
    return check_launch("fm_raw");
}
