// svc.cu — LinearSVC: hinge loss + subgradient and the margins, DESIGN.md §5j.
//
// K binary problems over the same rows at once: column k treats label == positives[k] as y' = +1 and every other label
// as y' = -1, with weights w_k = [β_k, b_k] over the scaled features [x · inv_std, 1].  Per row and column,
// m = [xs, 1] · w_k; the row adds the hinge 1 - y' m to column k's loss and -y' [xs, 1] to its gradient iff 1 - y' m > 0.
//
// Both products — the margins Xs · Wᵀ and the gradient Aᵀ · Xs (A[r][k] = -y' or 0, contracting over the tile's rows) —
// are fp64 tensor-core MMAs (mma.sync m8n8k4 f64), fragments as in mlp.cu.  An output element of an MMA depends only on
// its own row of one operand and column of the other, the contraction runs in a fixed order, and every class reads only
// its own weight row, margins and A column.  So column k's partial depends on column k's weights and positive label alone:
// not on K, on the other columns, or on the class block or the position within it where k lands.  Padding columns are
// zero weights whose margins are never stored, so their A columns stay zero.
//
// b200flow_svc_loss_grad: one CTA per (4096-row global chunk, class block).  It stages its block's weights in shared
// memory once, then walks the chunk's 32-row tiles in row order (tiles sit at fixed global positions): load x as f64 and
// scale it (one rounding per element) next to a ones column, margins, hinge values, loss (one thread per class, rows in
// order, so the loss is a sequential sum per column) and A, gradient.  The gradient accumulates in registers for the whole
// chunk: 8x8 tile t (class tile t / ndt, feature tile t % ndt) belongs to warp t % 8, slot t / 8.  Rows outside [0, n) are
// masked (A = 0, no loss), never padded into the loss.
//
// b200flow_svc_margins: the same tile load (unscaled) and margin code, written out per row.
#include "common.cuh"

namespace b200flow {

namespace {

constexpr int kChunkRows = 4096;
constexpr int kSvcTile = 32;                      // rows per tile: 4 MMA row blocks
constexpr int kSvcWarps = 8, kSvcThreads = kSvcWarps * 32;
constexpr int kSvcSlots = 32;                     // gradient tiles per warp: at most 256 8x8 tiles per class block
constexpr int kSvcMaxD = 255;                     // D + 1 (the ones column) padded to at most 256
constexpr int kSvcMaxBlockClasses = kSvcThreads;  // one thread per class sums its loss
constexpr int kSvcMaxSmem = 227 * 1024 - 2048;    // dynamic shared memory; the static label / class buffers take the rest

struct SvcShape {
    int D, Dp;                                    // features; D + 1 padded to 8
    int64_t K;                                    // classes
    int kb, blocks;                               // classes per block (a multiple of 8), class blocks
    int px, pw, pm;                               // pitches of Xs [32][px], W [kb][pw], M / A [32][pm]
    int xoff, moff, smem_doubles;                 // W at 0
};

int svc_shape(int D, int64_t K, SvcShape* s) {
    B2F_REQUIRE(D >= 1 && D <= kSvcMaxD, "svc: 1 <= D <= %d features, got %d", kSvcMaxD, D);
    B2F_REQUIRE(K >= 1, "svc: at least one class column, got %lld", (long long)K);
    s->D = D;
    s->Dp = pad8(D + 1);
    s->K = K;
    const int ndt = s->Dp / 8;
    int per = kSvcWarps * kSvcSlots / ndt;                            // class tiles whose gradient fits the registers
    if (per > kSvcMaxBlockClasses / 8) per = kSvcMaxBlockClasses / 8;
    const int64_t groups = (K + 7) / 8;
    const int64_t blocks = (groups + per - 1) / per;
    B2F_REQUIRE(blocks <= 65535, "svc: at most %lld class columns", (long long)per * 8 * 65535);
    s->blocks = (int)blocks;
    s->kb = (int)((groups + blocks - 1) / blocks) * 8;
    s->px = s->Dp + 4;                                                // 4 mod 8 doubles, as mlp.cu's pitches
    s->pw = s->Dp + 4;
    s->pm = s->kb + 4;
    s->xoff = s->kb * s->pw;
    s->moff = s->xoff + kSvcTile * s->px;
    s->smem_doubles = s->moff + kSvcTile * s->pm;
    B2F_REQUIRE((int64_t)s->smem_doubles * 8 <= kSvcMaxSmem, "svc: %lld bytes of shared memory; at most %d fit",
                (long long)s->smem_doubles * 8, kSvcMaxSmem);
    return B200FLOW_OK;
}

// the block's weights [nk][D + 1] into W (zeros elsewhere), Xs and M zeroed, Xs's ones column set
__device__ void svc_stage(const SvcShape& s, const double* __restrict__ w, int nk, double* sm) {
    const int D1 = s.D + 1;
    for (int e = threadIdx.x; e < s.kb * s.pw; e += kSvcThreads) {
        const int c = e / s.pw, j = e - c * s.pw;
        sm[e] = (c < nk && j < D1) ? w[(int64_t)c * D1 + j] : 0.0;
    }
    for (int e = s.xoff + threadIdx.x; e < s.smem_doubles; e += kSvcThreads) sm[e] = 0.0;
    __syncthreads();
    for (int r = threadIdx.x; r < kSvcTile; r += kSvcThreads) sm[s.xoff + r * s.px + s.D] = 1.0;
}

// rows [base, base + 32) of x into Xs as f64, times inv[j] when inv is given (rows outside [0, n) -> 0)
template <typename T>
__device__ void svc_load_tile(const SvcShape& s, const T* __restrict__ x, int64_t n, int64_t ld, const double* __restrict__ inv,
                              int64_t base, double* X) {
    const int D = s.D;
    for (int e = threadIdx.x; e < kSvcTile * D; e += kSvcThreads) {
        const int r = e / D, j = e - r * D;
        const int64_t gr = base + r;
        double v = 0.0;
        if (gr >= 0 && gr < n) {
            v = (double)x[gr * ld + j];
            if (inv) v = v * __ldg(inv + j);
        }
        X[r * s.px + j] = v;
    }
}

// M[r][c] = Xs[r] · W[c] for the block's nk real columns.  The 8x8 output tiles (column tile, row block) are shared out
// over the warps, so that a block of one column tile still keeps 4 warps busy; every output element accumulates over the
// features in ascending order whichever warp computes it.
__device__ void svc_margins_tile(const SvcShape& s, const double* X, const double* W, double* M, int nk) {
    const int lane = lane_id(), warp = warp_id(), qr = lane >> 2, qc = lane & 3;
    const int nk4 = s.Dp / 4;
    for (int item = warp; item < (s.kb / 8) * 4; item += kSvcWarps) {
        const int nt = item >> 2, m = item & 3;
        double c[2] = {0.0, 0.0};
        for (int k = 0; k < nk4; ++k) dmma(c, X[(m * 8 + qr) * s.px + k * 4 + qc], W[(nt * 8 + qr) * s.pw + k * 4 + qc]);
#pragma unroll
        for (int q = 0; q < 2; ++q) {
            const int col = nt * 8 + 2 * qc + q;
            if (col < nk) M[(m * 8 + qr) * s.pm + col] = c[q];
        }
    }
}

template <typename T>
__global__ void __launch_bounds__(kSvcThreads, 1) svc_loss_grad_kernel(const T* __restrict__ x, int64_t n, int64_t ld,
                                                                       const int32_t* __restrict__ y,
                                                                       const int32_t* __restrict__ positives,
                                                                       const double* __restrict__ inv, const SvcShape s,
                                                                       const double* __restrict__ w, int64_t row_offset,
                                                                       double* __restrict__ partials) {
    extern __shared__ double sm[];
    __shared__ int ylab[kSvcTile], yval[kSvcTile], posb[kSvcMaxBlockClasses];
    const int lane = lane_id(), warp = warp_id(), qr = lane >> 2, qc = lane & 3;
    const int64_t k0 = (int64_t)blockIdx.y * s.kb;
    const int nk = (int)(s.K - k0 < s.kb ? s.K - k0 : s.kb);
    const int D1 = s.D + 1, ndt = s.Dp / 8, ntiles = (s.kb / 8) * ndt;
    double* X = sm + s.xoff;
    double* M = sm + s.moff;
    svc_stage(s, w + k0 * D1, nk, sm);
    const int64_t c0 = (row_offset / kChunkRows + blockIdx.x) * kChunkRows - row_offset;   // local index of the chunk's row 0
    const int64_t lo = c0 > 0 ? c0 : 0, hi = c0 + kChunkRows < n ? c0 + kChunkRows : n;
    if (threadIdx.x < nk) posb[threadIdx.x] = positives[k0 + threadIdx.x];
    double acc[kSvcSlots][2];
#pragma unroll
    for (int q = 0; q < kSvcSlots; ++q) acc[q][0] = acc[q][1] = 0.0;
    double loss = 0.0;
    for (int64_t base = c0 + (lo - c0) / kSvcTile * kSvcTile; base < hi; base += kSvcTile) {
        __syncthreads();                                   // the previous tile's gradient has read Xs and A
        svc_load_tile(s, x, n, ld, inv, base, X);
        if (threadIdx.x < kSvcTile) {
            const int64_t gr = base + threadIdx.x;
            const bool valid = gr >= lo && gr < hi;
            yval[threadIdx.x] = valid;
            ylab[threadIdx.x] = valid ? y[gr] : 0;
        }
        __syncthreads();
        svc_margins_tile(s, X, sm, M, nk);
        __syncthreads();
        for (int e = threadIdx.x; e < kSvcTile * nk; e += kSvcThreads) {   // M becomes the hinge 1 - y' m (0 when masked)
            const int r = e / nk, c = e - r * nk;
            const double yp = ylab[r] == posb[c] ? 1.0 : -1.0;
            M[r * s.pm + c] = yval[r] ? 1.0 - yp * M[r * s.pm + c] : 0.0;
        }
        __syncthreads();
        if (threadIdx.x < nk) {                            // column threadIdx.x sums its loss over the rows in order; M becomes A
            const int c = threadIdx.x, pos = posb[c];
            for (int r = 0; r < kSvcTile; ++r) {
                const double h = M[r * s.pm + c];
                double a = 0.0;
                if (h > 0.0) {
                    loss = loss + h;
                    a = ylab[r] == pos ? -1.0 : 1.0;
                }
                M[r * s.pm + c] = a;
            }
        }
        __syncthreads();
#pragma unroll
        for (int q = 0; q < kSvcSlots; ++q) {              // gradient: Aᵀ · [xs, 1] over the tile's rows
            const int t = warp + kSvcWarps * q;
            if (t < ntiles) {
                const int ct = t / ndt, dt = t - ct * ndt;
#pragma unroll
                for (int k = 0; k < kSvcTile / 4; ++k)
                    dmma(acc[q], M[(k * 4 + qc) * s.pm + ct * 8 + qr], X[(k * 4 + qc) * s.px + dt * 8 + qr]);
            }
        }
    }
    double* part = partials + ((int64_t)blockIdx.x * s.K + k0) * (D1 + 1);
    if (threadIdx.x < nk) part[(int64_t)threadIdx.x * (D1 + 1)] = loss;
#pragma unroll
    for (int q = 0; q < kSvcSlots; ++q) {
        const int t = warp + kSvcWarps * q;
        if (t < ntiles) {
            const int ct = t / ndt, dt = t - ct * ndt, c = ct * 8 + qr;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int j = dt * 8 + 2 * qc + h;
                if (c < nk && j < D1) part[(int64_t)c * (D1 + 1) + 1 + j] = acc[q][h];
            }
        }
    }
}

template <typename T>
__global__ void __launch_bounds__(kSvcThreads) svc_margins_kernel(const T* __restrict__ x, int64_t n, int64_t ld, const SvcShape s,
                                                                  const double* __restrict__ w, double* __restrict__ raw) {
    extern __shared__ double sm[];
    const int64_t k0 = (int64_t)blockIdx.y * s.kb;
    const int nk = (int)(s.K - k0 < s.kb ? s.K - k0 : s.kb);
    double* X = sm + s.xoff;
    double* M = sm + s.moff;
    svc_stage(s, w + k0 * (s.D + 1), nk, sm);
    for (int64_t base = (int64_t)blockIdx.x * kSvcTile; base < n; base += (int64_t)gridDim.x * kSvcTile) {
        __syncthreads();                                   // the previous tile's margins are written out
        svc_load_tile(s, x, n, ld, (const double*)nullptr, base, X);
        __syncthreads();
        svc_margins_tile(s, X, sm, M, nk);
        __syncthreads();
        for (int e = threadIdx.x; e < kSvcTile * nk; e += kSvcThreads) {
            const int r = e / nk, c = e - r * nk;
            if (base + r < n) raw[(base + r) * s.K + k0 + c] = M[r * s.pm + c];
        }
    }
}

}  // namespace

}  // namespace b200flow

using namespace b200flow;

extern "C" int b200flow_svc_config(int32_t D, int64_t K, int32_t* block_classes, int32_t* class_blocks, int64_t* smem_bytes) {
    SvcShape s;
    const int rc = svc_shape(D, K, &s);
    if (rc != B200FLOW_OK) return rc;
    if (block_classes) *block_classes = s.kb;
    if (class_blocks) *class_blocks = s.blocks;
    if (smem_bytes) *smem_bytes = (int64_t)s.smem_doubles * (int64_t)sizeof(double);
    return B200FLOW_OK;
}

extern "C" int b200flow_svc_loss_grad(const void* x, int32_t x_dtype, int64_t n_rows, int64_t ld, int32_t D, const int32_t* labels,
                                      const int32_t* positives, int64_t K, const double* inv_std, const double* weights,
                                      int64_t row_offset, double* partials, void* stream) {
    SvcShape s;
    const int rc = svc_shape(D, K, &s);
    if (rc != B200FLOW_OK) return rc;
    B2F_REQUIRE(n_rows >= 0 && row_offset >= 0 && ld >= D && (x_dtype == B200FLOW_F32 || x_dtype == B200FLOW_F64),
                "svc_loss_grad: n >= 0, row_offset >= 0, ld >= D, f32 or f64 features");
    if (n_rows == 0) return B200FLOW_OK;
    B2F_REQUIRE(x && labels && positives && inv_std && weights && partials, "svc_loss_grad: null pointer");
    const int64_t nc = (row_offset + n_rows - 1) / kChunkRows - row_offset / kChunkRows + 1;
    B2F_REQUIRE(nc <= 0x7fffffffll, "svc_loss_grad: too many rows");
    const size_t smem = (size_t)s.smem_doubles * sizeof(double);
    const dim3 grid((unsigned)nc, (unsigned)s.blocks);
    cudaStream_t st = (cudaStream_t)stream;
    if (x_dtype == B200FLOW_F64) {
        cudaFuncSetAttribute(svc_loss_grad_kernel<double>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        svc_loss_grad_kernel<double><<<grid, kSvcThreads, smem, st>>>((const double*)x, n_rows, ld, labels, positives, inv_std, s,
                                                                      weights, row_offset, partials);
    } else {
        cudaFuncSetAttribute(svc_loss_grad_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        svc_loss_grad_kernel<float><<<grid, kSvcThreads, smem, st>>>((const float*)x, n_rows, ld, labels, positives, inv_std, s,
                                                                     weights, row_offset, partials);
    }
    return check_launch("svc_loss_grad");
}

extern "C" int b200flow_svc_margins(const void* x, int32_t x_dtype, int64_t n_rows, int64_t ld, int32_t D, int64_t K,
                                    const double* weights, double* raw, void* stream) {
    SvcShape s;
    const int rc = svc_shape(D, K, &s);
    if (rc != B200FLOW_OK) return rc;
    B2F_REQUIRE(n_rows >= 0 && ld >= D && (x_dtype == B200FLOW_F32 || x_dtype == B200FLOW_F64),
                "svc_margins: n >= 0, ld >= D, f32 or f64 features");
    if (n_rows == 0) return B200FLOW_OK;
    B2F_REQUIRE(x && weights && raw, "svc_margins: null pointer");
    const size_t smem = (size_t)s.smem_doubles * sizeof(double);
    const int64_t tiles = (n_rows + kSvcTile - 1) / kSvcTile;
    const int64_t per_sm = (228 * 1024) / (int64_t)(smem + 2048);
    const int64_t cap = (int64_t)kNumSMs * (per_sm > 1 ? per_sm : 1);
    const dim3 grid((unsigned)(tiles < cap ? tiles : cap), (unsigned)s.blocks);
    cudaStream_t st = (cudaStream_t)stream;
    if (x_dtype == B200FLOW_F64) {
        cudaFuncSetAttribute(svc_margins_kernel<double>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        svc_margins_kernel<double><<<grid, kSvcThreads, smem, st>>>((const double*)x, n_rows, ld, s, weights, raw);
    } else {
        cudaFuncSetAttribute(svc_margins_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        svc_margins_kernel<float><<<grid, kSvcThreads, smem, st>>>((const float*)x, n_rows, ld, s, weights, raw);
    }
    return check_launch("svc_margins");
}
