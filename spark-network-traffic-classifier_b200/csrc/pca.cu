// pca.cu — PCA and Pearson correlation: the centred Gram matrix and the projection, DESIGN.md §5h.
//
// Both products are fp64 tensor-core MMAs (common.cuh's dmma).  Widths are zero-padded in shared memory and the padding is
// exact zeros, so it adds nothing to a product.  There are no atomics.
//
// b200flow_centered_gram: one CTA per 4096-row global chunk walks the chunk's 32-row tiles, which sit at fixed global
// positions, in row order.  A tile is staged in shared memory as x − shift (Dq = ceil16(D) columns); rows outside [0, n) and
// the padding columns are staged as 0, so a chunk's partial depends only on which of its rows are present.  The upper
// triangle of (X − shift)ᵀ(X − shift) is cut into 16x16 blocks (ab, bb), ab <= bb, block j at ab + bb(bb+1)/2; a block is
// four 8x8 MMA tiles that share two A and two B fragments per 4 rows.  A pass holds 8 x 8 blocks in registers (block j of
// the pass belongs to warp j % 8, slot j / 8) and contracts them over the chunk's tiles, 4 rows per MMA; passes repeat
// until every block is done (one pass up to D = 176, three at D = 256).
// b200flow_weighted_centered_gram is the Weighted instantiation: the tile's row weights are staged beside it (0 outside
// [0, n)) and every B fragment (x_b − shift_b of one row) is multiplied by its row's weight as it is loaded, so the
// contraction is (X − shift)ᵀ W (X − shift) in the same order.  The unweighted instantiation is the same code as before.
//
// b200flow_pca_project: one CTA per 1024 rows walks 32-row tiles.  The tile's x (Dp = ceil8(D) columns) is staged once; pc
// sits in shared memory in slabs of 64 columns: the only slab stays for the whole CTA when k <= 64, otherwise the slabs
// stream through per tile (L2 holds pc: at most 512 KB).  A work item is one 8x8 output tile (row block, column tile) whose
// accumulator takes the features in ascending order, 4 per MMA, so a row's output depends on that row and pc alone.
#include "common.cuh"

namespace b200flow {

namespace {

constexpr int kChunkRows = 4096;
constexpr int kPcaTile = 32;                      // rows per tile: 8 MMA k-steps of the Gram, 4 MMA row blocks of the projection
constexpr int kPcaWarps = 8, kPcaThreads = kPcaWarps * 32;
constexpr int kPcaSlots = 8;                      // 16x16 Gram blocks per warp and pass
constexpr int kPcaMaxD = 256;
constexpr int kProjRows = 1024;                   // rows per CTA of the projection
constexpr int kProjSlab = 64;                     // columns of pc per shared-memory slab

__host__ __device__ inline int pad16(int v) { return (v + 15) / 16 * 16; }

template <bool Weighted>
__global__ void __launch_bounds__(kPcaThreads, 1) centered_gram_kernel(const double* __restrict__ x, int64_t n, int64_t ld, int D,
                                                                      const double* __restrict__ shift, int64_t row_offset,
                                                                      double* __restrict__ partials,
                                                                      const double* __restrict__ w) {
    extern __shared__ double sm[];
    const int Dq = pad16(D), pitch = Dq + 4, nb = Dq / 16, B = nb * (nb + 1) / 2;    // pitch 4 mod 8: 2-wavefront fragment loads
    double* xs = sm;                              // [kPcaTile][pitch]
    double* ss = xs + kPcaTile * pitch;           // [Dq]
    double* wt = ss + Dq;                         // [kPcaTile]: the tile's row weights (Weighted only)
    const int lane = lane_id(), warp = warp_id(), qr = lane >> 2, qc = lane & 3;
    const int64_t c0 = (row_offset / kChunkRows + blockIdx.x) * kChunkRows - row_offset;   // local index of the chunk's row 0
    const int64_t lo = c0 > 0 ? c0 : 0, hi = c0 + kChunkRows < n ? c0 + kChunkRows : n;
    const int64_t first = c0 + (lo - c0) / kPcaTile * kPcaTile;
    double* part = partials + (int64_t)blockIdx.x * ((int64_t)D * (D + 1) / 2);
    for (int j = threadIdx.x; j < Dq; j += kPcaThreads) ss[j] = shift && j < D ? shift[j] : 0.0;
    for (int p0 = 0; p0 < B; p0 += kPcaWarps * kPcaSlots) {
        int item[kPcaSlots];                      // ab << 8 | bb, -1: none
        double acc[kPcaSlots][4][2];              // tiles (lo, lo), (lo, hi), (hi, lo), (hi, hi) of the block
#pragma unroll
        for (int q = 0; q < kPcaSlots; ++q) {
            const int j = p0 + warp + kPcaWarps * q;
            int bb = 0;
            while ((bb + 1) * (bb + 2) / 2 <= j) ++bb;
            item[q] = j < B ? (j - bb * (bb + 1) / 2) << 8 | bb : -1;
#pragma unroll
            for (int t = 0; t < 4; ++t) acc[q][t][0] = acc[q][t][1] = 0.0;
        }
        for (int64_t base = first; base < hi; base += kPcaTile) {
            __syncthreads();                      // ss is written; the previous tile's MMAs are done with xs
            for (int e = threadIdx.x; e < kPcaTile * Dq; e += kPcaThreads) {
                const int r = e / Dq, j = e - r * Dq;
                const int64_t gr = base + r;
                xs[r * pitch + j] = gr >= 0 && gr < n && j < D ? x[gr * ld + j] - ss[j] : 0.0;
            }
            if constexpr (Weighted) {
                if (threadIdx.x < kPcaTile) {
                    const int64_t gr = base + threadIdx.x;
                    wt[threadIdx.x] = gr >= 0 && gr < n ? w[gr] : 0.0;
                }
            }
            __syncthreads();
#pragma unroll
            for (int q = 0; q < kPcaSlots; ++q) {
                if (item[q] >= 0) {
                    const double* pa = xs + qc * pitch + (item[q] >> 8) * 16 + qr;
                    const double* pb = xs + qc * pitch + (item[q] & 0xff) * 16 + qr;
#pragma unroll 4
                    for (int kk = 0; kk < kPcaTile / 4; ++kk) {
                        const int o = kk * 4 * pitch;
                        const double al = pa[o], ah = pa[o + 8];
                        double bl = pb[o], bh = pb[o + 8];
                        if constexpr (Weighted) {
                            const double wr = wt[kk * 4 + qc];    // the B fragment's row: kk * 4 + qc
                            bl = bl * wr;
                            bh = bh * wr;
                        }
                        dmma(acc[q][0], al, bl);
                        dmma(acc[q][1], al, bh);
                        dmma(acc[q][2], ah, bl);
                        dmma(acc[q][3], ah, bh);
                    }
                }
            }
        }
#pragma unroll
        for (int q = 0; q < kPcaSlots; ++q) {
            if (item[q] < 0) continue;
#pragma unroll
            for (int t = 0; t < 4; ++t) {
                const int a = (item[q] >> 8) * 16 + (t >> 1) * 8 + qr;
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int b = (item[q] & 0xff) * 16 + (t & 1) * 8 + 2 * qc + h;
                    if (a <= b && b < D) part[a + (int64_t)b * (b + 1) / 2] = acc[q][t][h];
                }
            }
        }
    }
}

// columns [s0, s0 + ks) of pc [D][k] into ps [ceil8(D)][ks + 4]; 0 beyond D rows and k columns
__device__ __forceinline__ void proj_load_slab(const double* __restrict__ pc, int D, int k, int s0, int ks, double* ps) {
    for (int e = threadIdx.x; e < pad8(D) * ks; e += kPcaThreads) {
        const int a = e / ks, j = e - a * ks;
        ps[a * (ks + 4) + j] = a < D && s0 + j < k ? pc[(int64_t)a * k + s0 + j] : 0.0;
    }
}

// 4 CTAs per SM (64 registers): small k leaves most warps of a CTA idle, other CTAs' loads and MMAs fill the SM
__global__ void __launch_bounds__(kPcaThreads, 4) pca_project_kernel(const double* __restrict__ x, int64_t n, int64_t ld,
                                                                    int D, const double* __restrict__ pc, int k,
                                                                    double* __restrict__ out) {
    extern __shared__ double sm[];
    const int Dp = pad8(D), kp = pad8(k), ks = kp < kProjSlab ? kp : kProjSlab;
    const int xp = Dp + 4, pp = ks + 4;           // both 4 mod 8: 2-wavefront fragment loads
    double* xs = sm;                              // [kPcaTile][xp]
    double* ps = xs + kPcaTile * xp;              // [Dp][pp]: columns [s0, s0 + ks) of pc
    const int lane = lane_id(), warp = warp_id(), qr = lane >> 2, qc = lane & 3;
    const int64_t row0 = (int64_t)blockIdx.x * kProjRows, end = row0 + kProjRows < n ? row0 + kProjRows : n;
    const bool resident = kp <= kProjSlab;
    if (resident) proj_load_slab(pc, D, k, 0, ks, ps);
    for (int64_t base = row0; base < end; base += kPcaTile) {
        __syncthreads();                          // the previous tile's MMAs are done with xs and ps
        for (int e = threadIdx.x; e < kPcaTile * Dp; e += kPcaThreads) {
            const int r = e / Dp, j = e - r * Dp;
            xs[r * xp + j] = base + r < end && j < D ? x[(base + r) * ld + j] : 0.0;
        }
        for (int s0 = 0; s0 < kp; s0 += kProjSlab) {
            if (!resident) {
                if (s0) __syncthreads();          // the previous slab's MMAs are done with ps
                proj_load_slab(pc, D, k, s0, ks, ps);
            }
            __syncthreads();
            const int nct = (kp - s0 < ks ? kp - s0 : ks) / 8;
            for (int it = warp; it < 4 * nct; it += kPcaWarps) {
                const int mb = it & 3, ct = it >> 2;
                const double* A = xs + (mb * 8 + qr) * xp + qc;
                const double* Bf = ps + qc * pp + ct * 8 + qr;
                double acc[2] = {0.0, 0.0};
                for (int kk = 0; kk < Dp / 4; ++kk) dmma(acc, A[kk * 4], Bf[kk * 4 * pp]);
                const int64_t r = base + mb * 8 + qr;
                const int c = s0 + ct * 8 + 2 * qc;
                if (r < end) {
                    if (c < k) out[r * k + c] = acc[0];
                    if (c + 1 < k) out[r * k + c + 1] = acc[1];
                }
            }
        }
    }
}

}  // namespace

}  // namespace b200flow

using namespace b200flow;

namespace {

template <bool Weighted>
int launch_centered_gram(const char* what, const double* x, int64_t n_rows, int32_t D, int64_t ld, const double* shift,
                         const double* w, int64_t row_offset, double* partials, void* stream) {
    B2F_REQUIRE(D >= 1 && D <= kPcaMaxD, "%s: 1 <= D <= %d", what, kPcaMaxD);
    B2F_REQUIRE(n_rows >= 0 && row_offset >= 0 && ld >= D, "%s: n >= 0, row_offset >= 0, ld >= D", what);
    if (n_rows == 0) return B200FLOW_OK;
    const int64_t nc = (row_offset + n_rows - 1) / kChunkRows - row_offset / kChunkRows + 1;
    B2F_REQUIRE(nc <= 0x7fffffffll, "%s: too many rows", what);
    B2F_REQUIRE(x && partials && (w || !Weighted), "%s: null pointer", what);
    const int Dq = pad16(D);
    const size_t smem = ((size_t)kPcaTile * (Dq + 4) + Dq + (Weighted ? kPcaTile : 0)) * sizeof(double);
    cudaFuncSetAttribute(centered_gram_kernel<Weighted>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    centered_gram_kernel<Weighted><<<(unsigned)nc, kPcaThreads, smem, (cudaStream_t)stream>>>(x, n_rows, ld, D, shift,
                                                                                              row_offset, partials, w);
    return check_launch(what);
}

}  // namespace

extern "C" int b200flow_centered_gram(const double* x, int64_t n_rows, int32_t D, int64_t ld, const double* shift,
                                      int64_t row_offset, double* partials, void* stream) {
    return launch_centered_gram<false>("centered_gram", x, n_rows, D, ld, shift, nullptr, row_offset, partials, stream);
}

extern "C" int b200flow_weighted_centered_gram(const double* x, int64_t n_rows, int32_t D, int64_t ld, const double* shift,
                                               const double* w, int64_t row_offset, double* partials, void* stream) {
    return launch_centered_gram<true>("weighted_centered_gram", x, n_rows, D, ld, shift, w, row_offset, partials, stream);
}

extern "C" int b200flow_pca_project(const double* x, int64_t n_rows, int32_t D, int64_t ld, const double* pc, int32_t k,
                                    double* out, void* stream) {
    B2F_REQUIRE(D >= 1 && D <= kPcaMaxD && k >= 1 && k <= kPcaMaxD, "pca_project: 1 <= D <= %d and 1 <= k <= %d", kPcaMaxD,
                kPcaMaxD);
    B2F_REQUIRE(n_rows >= 0 && ld >= D, "pca_project: n >= 0, ld >= D");
    if (n_rows == 0) return B200FLOW_OK;
    const int64_t blocks = (n_rows + kProjRows - 1) / kProjRows;
    B2F_REQUIRE(blocks <= 0x7fffffffll, "pca_project: too many rows");
    B2F_REQUIRE(x && pc && out, "pca_project: null pointer");
    const int Dp = pad8(D), kp = pad8(k), ks = kp < kProjSlab ? kp : kProjSlab;
    const size_t smem = ((size_t)kPcaTile * (Dp + 4) + (size_t)Dp * (ks + 4)) * sizeof(double);
    cudaFuncSetAttribute(pca_project_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    pca_project_kernel<<<(unsigned)blocks, kPcaThreads, smem, (cudaStream_t)stream>>>(x, n_rows, ld, D, pc, k, out);
    return check_launch("pca_project");
}
