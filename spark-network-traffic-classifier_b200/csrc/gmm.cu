// gmm.cu — GaussianMixture (full covariance): the E-step and the responsibility-weighted moments, DESIGN.md §5g.
//
// Component i is given by its mean μ_i [D], its root R_i [D][D] (R = diag(1/√d) Uᵀ of the eigendecomposition Σ = U diag(d) Uᵀ,
// zero rows for the eigenvalues the host dropped) and c_i = log w_i + u_i (u_i the density constant).  For a row x:
//   y = R_i (x − μ_i),  q_i = Σ_j y_j² (j in order from +0.0),  s_i = c_i − 0.5 q_i,
//   t_i = logaddexp(log EPSILON, s_i),  lse = logsumexp(t),  r_i = exp(t_i − lse).
//
// Both products are fp64 tensor-core MMAs (mma.sync m8n8k4 f64, SASS DMMA.8x8x4).  Fragments of m8n8k4.f64 (PTX ISA): A holds
// (row lane>>2, k lane&3), B holds (k lane&3, col lane>>2), C/D hold (row lane>>2, col 2(lane&3) + {0,1}).  Widths are
// zero-padded to multiples of 8 and the padding is exact zeros, so it adds nothing to a product.
//
// Both kernels run one CTA per 4096-row global chunk and walk the chunk's 32-row tiles, which sit at fixed global positions,
// in row order.  Rows outside [0, n) are masked: their x is staged as 0, their responsibilities as 0, and they are never
// written nor added to a sum.  So a chunk's partial depends only on that chunk's rows, whichever rank or launch computes it.
// There are no atomics.
//
// b200flow_gmm_estep: the tile's x (Dp = ceil8(D) columns) stays in shared memory.  Per component, R_i streams through shared
// memory in slabs of 64 rows (L2 holds all of R: at most 64 x 512 KB); warp w computes output columns [64s + 8w, 64s + 8w + 8)
// of y for all 32 rows (B fragments of R, A fragments x − μ formed exactly at load) and writes them over the slab rows only
// it reads.  Lane r of warp 0 then adds the slab's y_j² to q of row r in j order.  Lane r of warp 0 finally forms t, lse and
// r of row r; the chunk's log-likelihood partial is the sum of the valid rows' lse in row order from +0.0.
//
// b200flow_gmm_moments: the tile's x is staged with a column of ones after the last feature (Da = ceil8(D + 1) columns), so
// one contraction over the rows gives all three sums: Xaᵀ diag(r_i) Xa holds Q_i (a, b < D), S_i (b = D) and W_i
// (a = b = D).  Only its upper-triangle 8x8 tiles are computed.  Work item j = (component j / T, tile j % T), T = nt(nt+1)/2
// tiles with nt = Da / 8 and tile (at, bt), at <= bt, at index at + bt(bt+1)/2.  A pass holds 8 x 32 items in registers
// (item j of the pass belongs to warp j % 8, slot j / 8) and contracts them over the chunk's tiles in row order, 4 rows per
// MMA; the A fragment r·x is rounded once per element.  Passes repeat until every item is done.
#include <math.h>

#include "common.cuh"

namespace b200flow {

namespace {

constexpr int kChunkRows = 4096;
constexpr int kGmmTile = 32;                      // rows per tile: 4 MMA row blocks
constexpr int kGmmWarps = 8, kGmmThreads = kGmmWarps * 32;
constexpr int kGmmSlab = 64;                      // rows of R per shared-memory slab: 8 output column tiles, one per warp
constexpr int kGmmSlots = 32;                     // moment tiles per warp and pass
constexpr int kGmmMaxD = 256, kGmmMaxK = 64;

// 4 mod 8 doubles: fragment loads take the minimum 2 wavefronts; at least 36, so that 8 rows of a slab hold a warp's
// [kGmmTile][8] block of y
__host__ __device__ inline int estep_pitch(int D) { return (pad8(D) > 32 ? pad8(D) : 32) + 4; }
__host__ __device__ inline int64_t gmm_width(int k, int D) { return 1 + (int64_t)k * (1 + D + (int64_t)D * (D + 1) / 2); }

// x rows [base, base + kGmmTile) into xs [kGmmTile][pitch] as f64; 0 outside [0, n) and in columns [D, width); a column of
// ones at `ones` (< 0: none) for the rows inside
__device__ void gmm_load_tile(const double* __restrict__ x, int64_t n, int64_t ld, int D, int width, int ones, int64_t base,
                              double* xs, int pitch) {
    for (int e = threadIdx.x; e < kGmmTile * width; e += kGmmThreads) {
        const int r = e / width, j = e - r * width;
        const int64_t gr = base + r;
        const bool in = gr >= 0 && gr < n;
        xs[r * pitch + j] = in && j < D ? x[gr * ld + j] : (in && j == ones ? 1.0 : 0.0);
    }
}

__device__ __forceinline__ int64_t chunk_row0(int64_t row_offset) {
    return (row_offset / kChunkRows + blockIdx.x) * kChunkRows - row_offset;   // local index of the chunk's row 0
}

__global__ void __launch_bounds__(kGmmThreads, 1) gmm_estep_kernel(const double* __restrict__ x, int64_t n, int64_t ld, int D,
                                                                  int k, const double* __restrict__ mu,
                                                                  const double* __restrict__ R, const double* __restrict__ c,
                                                                  int64_t row_offset, double* __restrict__ resp,
                                                                  int32_t* __restrict__ pred, double* __restrict__ partials) {
    extern __shared__ double sm[];
    const int Dp = pad8(D), pitch = estep_pitch(D);
    double* xs = sm;                              // [kGmmTile][pitch]
    double* rs = xs + kGmmTile * pitch;           // [kGmmSlab][pitch]; warp w's y block [kGmmTile][8] over rows 8w..
    double* ms = rs + kGmmSlab * pitch;           // [Dp]
    double* sv = ms + Dp;                         // [kGmmTile][k]: s, then t
    __shared__ double lseb[kGmmTile];
    const int lane = lane_id(), warp = warp_id(), qr = lane >> 2, qc = lane & 3;
    const int64_t c0 = chunk_row0(row_offset);
    const int64_t lo = c0 > 0 ? c0 : 0, hi = c0 + kChunkRows < n ? c0 + kChunkRows : n;
    const double log_eps = log(2.220446049250313e-16);
    double ll = 0.0;
    for (int64_t base = c0 + (lo - c0) / kGmmTile * kGmmTile; base < hi; base += kGmmTile) {
        __syncthreads();                          // the previous tile is finished with xs and sv
        gmm_load_tile(x, n, ld, D, Dp, -1, base, xs, pitch);
        for (int i = 0; i < k; ++i) {
            double q = 0.0;                       // warp 0, lane = row
            for (int s0 = 0; s0 < D; s0 += kGmmSlab) {
                __syncthreads();                  // the previous slab's y is summed
                for (int e = threadIdx.x; e < kGmmSlab * Dp; e += kGmmThreads) {
                    const int o = e / Dp, j = e - o * Dp;
                    rs[o * pitch + j] = (s0 + o < D && j < D) ? R[((int64_t)i * D + s0 + o) * D + j] : 0.0;
                }
                if (s0 == 0)
                    for (int j = threadIdx.x; j < Dp; j += kGmmThreads) ms[j] = j < D ? mu[(int64_t)i * D + j] : 0.0;
                __syncthreads();
                if (s0 + warp * 8 < Dp) {
                    const double* B = rs + warp * 8 * pitch;
                    double acc[4][2] = {};
                    for (int kk = 0; kk < Dp / 4; ++kk) {
                        const int col = kk * 4 + qc;
                        const double b = B[qr * pitch + col], m = ms[col];
#pragma unroll
                        for (int mb = 0; mb < 4; ++mb) dmma(acc[mb], xs[(mb * 8 + qr) * pitch + col] - m, b);
                    }
                    __syncwarp();                 // every lane has read its B fragments: the block is this warp's
                    double* Y = rs + warp * 8 * pitch;
#pragma unroll
                    for (int mb = 0; mb < 4; ++mb) {
                        Y[(mb * 8 + qr) * 8 + 2 * qc] = acc[mb][0];
                        Y[(mb * 8 + qr) * 8 + 2 * qc + 1] = acc[mb][1];
                    }
                }
                __syncthreads();
                if (warp == 0) {
                    const int w = D - s0 < kGmmSlab ? D - s0 : kGmmSlab;
                    for (int j = 0; j < w; ++j) {
                        const double y = rs[(j >> 3) * 8 * pitch + lane * 8 + (j & 7)];
                        q = q + y * y;
                    }
                }
            }
            if (warp == 0) sv[lane * k + i] = c[i] - 0.5 * q;
        }
        if (warp == 0) {                          // t, lse, r and the prediction, one row per lane
            const int64_t gr = base + lane;
            double lse = 0.0;
            if (gr >= lo && gr < hi) {
                double* t = sv + lane * k;
                double m = -INFINITY;
                for (int i = 0; i < k; ++i) {
                    const double s = t[i], a = s > log_eps ? s : log_eps, b = s > log_eps ? log_eps : s;
                    const double v = a + log1p(exp(b - a));
                    t[i] = v;
                    m = v > m ? v : m;
                }
                double se = 0.0;
                for (int i = 0; i < k; ++i) se = se + exp(t[i] - m);
                lse = m + log(se);
                int best = 0;
                double bp = -1.0;
                for (int i = 0; i < k; ++i) {
                    const double p = exp(t[i] - lse);
                    if (resp) resp[gr * k + i] = p;
                    if (p > bp) { bp = p; best = i; }
                }
                if (pred) pred[gr] = best;
            }
            lseb[lane] = lse;
            __syncwarp();
            if (lane == 0)
                for (int r = 0; r < kGmmTile; ++r)
                    if (base + r >= lo && base + r < hi) ll = ll + lseb[r];
        }
    }
    if (partials && threadIdx.x == 0) partials[(int64_t)blockIdx.x * gmm_width(k, D)] = ll;
}

__global__ void __launch_bounds__(kGmmThreads, 1) gmm_moments_kernel(const double* __restrict__ x, int64_t n, int64_t ld, int D,
                                                                    int k, const double* __restrict__ resp, int64_t row_offset,
                                                                    double* __restrict__ partials) {
    extern __shared__ double sm[];
    const int Da = pad8(D + 1), pitch = Da + 4, nt = Da / 8, T = nt * (nt + 1) / 2;
    double* xs = sm;                              // [kGmmTile][pitch]
    double* rt = xs + kGmmTile * pitch;           // [kGmmTile][k]
    const int lane = lane_id(), warp = warp_id(), qr = lane >> 2, qc = lane & 3;
    const int64_t c0 = chunk_row0(row_offset);
    const int64_t lo = c0 > 0 ? c0 : 0, hi = c0 + kChunkRows < n ? c0 + kChunkRows : n;
    const int64_t first = c0 + (lo - c0) / kGmmTile * kGmmTile;
    const int items = k * T;
    double* part = partials + (int64_t)blockIdx.x * gmm_width(k, D);
    const int64_t per_comp = 1 + D + (int64_t)D * (D + 1) / 2;
    for (int p0 = 0; p0 < items; p0 += kGmmWarps * kGmmSlots) {
        int item[kGmmSlots];                      // component << 16 | at << 8 | bt, -1: none
        double acc[kGmmSlots][2];
#pragma unroll
        for (int q = 0; q < kGmmSlots; ++q) {
            const int j = p0 + warp + kGmmWarps * q;
            int cc = -1, bt = 0, at = 0;
            if (j < items) {
                cc = j / T;
                const int t = j - cc * T;
                while ((bt + 1) * (bt + 2) / 2 <= t) ++bt;
                at = t - bt * (bt + 1) / 2;
            }
            item[q] = cc < 0 ? -1 : cc << 16 | at << 8 | bt;
            acc[q][0] = acc[q][1] = 0.0;
        }
        for (int64_t base = first; base < hi; base += kGmmTile) {
            __syncthreads();                      // the previous tile's MMAs are done with xs and rt
            gmm_load_tile(x, n, ld, D, Da, D, base, xs, pitch);
            for (int e = threadIdx.x; e < kGmmTile * k; e += kGmmThreads) {
                const int r = e / k, i = e - r * k;
                const int64_t gr = base + r;
                rt[e] = gr >= lo && gr < hi ? resp[gr * k + i] : 0.0;
            }
            __syncthreads();
#pragma unroll
            for (int q = 0; q < kGmmSlots; ++q) {
                if (item[q] >= 0) {
                    const int a0 = (item[q] >> 8 & 0xff) * 8 + qr, b0 = (item[q] & 0xff) * 8 + qr, cc = item[q] >> 16;
#pragma unroll 4                  // fully unrolled, the 32 slots' fragments spill
                    for (int kk = 0; kk < kGmmTile / 4; ++kk) {
                        const int row = kk * 4 + qc;
                        dmma(acc[q], rt[row * k + cc] * xs[row * pitch + a0], xs[row * pitch + b0]);
                    }
                }
            }
        }
#pragma unroll
        for (int q = 0; q < kGmmSlots; ++q) {
            if (item[q] < 0) continue;
            double* pc = part + 1 + (item[q] >> 16) * per_comp;
            const int a = (item[q] >> 8 & 0xff) * 8 + qr;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int b = (item[q] & 0xff) * 8 + 2 * qc + h;
                if (a > b || b > D) continue;
                if (b < D) pc[1 + D + a + (int64_t)b * (b + 1) / 2] = acc[q][h];
                else if (a < D) pc[1 + a] = acc[q][h];
                else pc[0] = acc[q][h];
            }
        }
    }
}

int gmm_check(int64_t n_rows, int64_t ld, int32_t D, int32_t k, int64_t row_offset, const char* what) {
    B2F_REQUIRE(D >= 1 && D <= kGmmMaxD && k >= 1 && k <= kGmmMaxK, "%s: 1 <= D <= %d and 1 <= k <= %d", what, kGmmMaxD,
                kGmmMaxK);
    B2F_REQUIRE(n_rows >= 0 && row_offset >= 0 && ld >= D, "%s: n >= 0, row_offset >= 0, ld >= D", what);
    const int64_t nc = n_rows ? (row_offset + n_rows - 1) / kChunkRows - row_offset / kChunkRows + 1 : 0;
    B2F_REQUIRE(nc <= 0x7fffffffll, "%s: too many rows", what);
    return B200FLOW_OK;
}

int64_t gmm_chunks(int64_t row_offset, int64_t n_rows) {
    return (row_offset + n_rows - 1) / kChunkRows - row_offset / kChunkRows + 1;
}

}  // namespace

}  // namespace b200flow

using namespace b200flow;

extern "C" int b200flow_gmm_estep(const double* x, int64_t n_rows, int32_t D, int64_t ld, int32_t k, const double* means,
                                  const double* roots, const double* log_consts, int64_t row_offset, double* resp, int32_t* pred,
                                  double* partials, void* stream) {
    const int rc = gmm_check(n_rows, ld, D, k, row_offset, "gmm_estep");
    if (rc != B200FLOW_OK) return rc;
    if (n_rows == 0) return B200FLOW_OK;
    B2F_REQUIRE(x && means && roots && log_consts, "gmm_estep: null pointer");
    const int Dp = pad8(D);
    const size_t smem = ((size_t)(kGmmTile + kGmmSlab) * estep_pitch(D) + Dp + (size_t)kGmmTile * k) * sizeof(double);
    cudaFuncSetAttribute(gmm_estep_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    gmm_estep_kernel<<<(unsigned)gmm_chunks(row_offset, n_rows), kGmmThreads, smem, (cudaStream_t)stream>>>(
        x, n_rows, ld, D, k, means, roots, log_consts, row_offset, resp, pred, partials);
    return check_launch("gmm_estep");
}

extern "C" int b200flow_gmm_moments(const double* x, int64_t n_rows, int32_t D, int64_t ld, int32_t k, const double* resp,
                                    int64_t row_offset, double* partials, void* stream) {
    const int rc = gmm_check(n_rows, ld, D, k, row_offset, "gmm_moments");
    if (rc != B200FLOW_OK) return rc;
    if (n_rows == 0) return B200FLOW_OK;
    B2F_REQUIRE(x && resp && partials, "gmm_moments: null pointer");
    const size_t smem = ((size_t)kGmmTile * (pad8(D + 1) + 4) + (size_t)kGmmTile * k) * sizeof(double);
    cudaFuncSetAttribute(gmm_moments_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    gmm_moments_kernel<<<(unsigned)gmm_chunks(row_offset, n_rows), kGmmThreads, smem, (cudaStream_t)stream>>>(
        x, n_rows, ld, D, k, resp, row_offset, partials);
    return check_launch("gmm_moments");
}
