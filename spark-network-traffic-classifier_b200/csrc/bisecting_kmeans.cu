// bisecting_kmeans.cu — BisectingKMeans split assignment and tree-walk predict, DESIGN.md §5t.
//
// Both kernels follow the distance contract of kmeans.cu (§5c): acc = acc + t*t in feature order from 0.0 with
// t = x_j - c_j (-fmad=false: no FMA, no norm trick).  A row's result depends on that row and the centers alone: no
// cross-row reduction, so the bits do not depend on how rows are spread over ranks.  Every sum of the fit goes through
// b200flow_group_sums / _chain.
//
// Layout (both kernels): one 128-thread CTA per 64 rows, staged transposed in shared memory once (odd pitch, as
// kmeans_assign); the two lanes 2r and 2r+1 own row r, lane 2r measures the left child and lane 2r+1 the right one, and
// the pair trades its two distances with one shuffle.  The centers are read through L1.
#include <math.h>

#include "common.cuh"

namespace b200flow {

constexpr int kBkmRows = 64, kBkmThreads = 128, kBkmPitch = kBkmRows + 1, kBkmMaxD = 256, kBkmMaxDepth = 63;

__device__ __forceinline__ void bkm_stage_rows(double* xs, const double* __restrict__ x, int64_t n, int D, int64_t ld,
                                               int64_t row0) {
#pragma unroll 4
    for (int e = threadIdx.x; e < kBkmRows * D; e += kBkmThreads) {
        const int r = e / D, j = e - r * D;
        const int64_t gr = row0 + r;
        xs[j * kBkmPitch + r] = gr < n ? x[gr * ld + j] : 0.0;
    }
}

// the squared distance of staged row r to center c [D], summed in feature order from 0.0
__device__ __forceinline__ double bkm_sqdist(const double* xs, int r, const double* __restrict__ c, int D) {
    double acc = 0.0;
#pragma unroll 4
    for (int j = 0; j < D; ++j) {
        const double t = xs[j * kBkmPitch + r] - __ldg(c + j);
        acc = acc + t * t;
    }
    return acc;
}

__global__ void __launch_bounds__(kBkmThreads) bkm_assign_kernel(const double* __restrict__ x, int64_t n, int D, int64_t ld,
                                                                 const int32_t* __restrict__ node, int num_nodes,
                                                                 const int32_t* __restrict__ slot_of_node,
                                                                 const double* __restrict__ centers, int m,
                                                                 const uint8_t* __restrict__ present,
                                                                 const int32_t* __restrict__ prev, int32_t* __restrict__ child,
                                                                 double* __restrict__ dist_prev) {
    extern __shared__ double bkm_sm[];
    const int64_t row0 = (int64_t)blockIdx.x * kBkmRows;
    bkm_stage_rows(bkm_sm, x, n, D, ld, row0);
    __syncthreads();
    const int r = threadIdx.x >> 1, side = threadIdx.x & 1;
    const int64_t i = row0 + r;
    if (i >= n) return;                                    // both lanes of the pair leave together
    const int u = node[i];
    const int s = (u >= 0 && u < num_nodes) ? slot_of_node[u] : -1;
    if (s < 0 || s >= m) {                                 // the row's node is not dividing
        if (side == 0) {
            child[i] = -1;
            if (dist_prev) dist_prev[i] = 0.0;
        }
        return;
    }
    const unsigned pair = 3u << (lane_id() & ~1);
    const double mine = bkm_sqdist(bkm_sm, r, centers + (int64_t)(2 * s + side) * D, D);
    const double other = __shfl_xor_sync(pair, mine, 1);
    if (side) return;
    const double dl = mine, dr = other;
    const bool pl = present[2 * s] != 0, pr = present[2 * s + 1] != 0;
    child[i] = pl && !(pr && dr < dl) ? 2 * s : (pr ? 2 * s + 1 : -1);   // strict <: a tie goes left
    if (dist_prev) {
        const int p = prev[i];
        double dp = 0.0;
        if (p == 2 * s) dp = dl;
        else if (p == 2 * s + 1) dp = dr;
        else if (p >= 0 && p < 2 * m) dp = bkm_sqdist(bkm_sm, r, centers + (int64_t)p * D, D);
        dist_prev[i] = dp;
    }
}

__global__ void __launch_bounds__(kBkmThreads) bkm_predict_kernel(const double* __restrict__ x, int64_t n, int D, int64_t ld,
                                                                  const int32_t* __restrict__ left, const int32_t* __restrict__ right,
                                                                  const int32_t* __restrict__ leaf, const double* __restrict__ centers,
                                                                  int root, int32_t* __restrict__ out_leaf,
                                                                  double* __restrict__ out_dist) {
    extern __shared__ double bkm_sm[];
    const int64_t row0 = (int64_t)blockIdx.x * kBkmRows;
    bkm_stage_rows(bkm_sm, x, n, D, ld, row0);
    __syncthreads();
    const int r = threadIdx.x >> 1, side = threadIdx.x & 1;
    const int64_t i = row0 + r;
    if (i >= n) return;
    const unsigned pair = 3u << (lane_id() & ~1);
    int u = root;
    double d = 0.0;
    if (leaf[u] >= 0) d = bkm_sqdist(bkm_sm, r, centers + (int64_t)u * D, D);   // the root is the only leaf
    // both lanes walk the same path: each measures one child, and the pair agrees on the choice
    for (int depth = 0; depth < kBkmMaxDepth && leaf[u] < 0; ++depth) {
        const int a = left[u], b = right[u];
        if (a < 0 && b < 0) break;                        // a malformed internal node: stop rather than leave the tree
        const int c = side ? b : a;
        const double mine = c >= 0 ? bkm_sqdist(bkm_sm, r, centers + (int64_t)c * D, D) : INFINITY;
        const double other = __shfl_xor_sync(pair, mine, 1);
        const double da = side ? other : mine, db = side ? mine : other;
        if (a >= 0 && (b < 0 || da <= db)) { u = a; d = da; }   // a tie goes to the first child
        else { u = b; d = db; }
    }
    if (side == 0) {
        out_leaf[i] = leaf[u];
        out_dist[i] = d;
    }
}

}  // namespace b200flow

using namespace b200flow;

extern "C" int b200flow_bkm_assign(const double* x, int64_t n_rows, int32_t D, int64_t ld, const int32_t* node, int32_t num_nodes,
                                   const int32_t* slot_of_node, const double* centers, int32_t m, const uint8_t* present,
                                   const int32_t* prev, int32_t* child, double* dist_prev, void* stream) {
    B2F_REQUIRE(n_rows >= 0 && D >= 1 && D <= kBkmMaxD && ld >= D && num_nodes >= 1 && m >= 1 && (!prev || dist_prev),
                "bkm_assign: n >= 0, 1 <= D <= %d, ld >= D, num_nodes >= 1, m >= 1, dist_prev with prev", kBkmMaxD);
    if (n_rows == 0) return B200FLOW_OK;
    B2F_REQUIRE(x && node && slot_of_node && centers && present && child, "bkm_assign: null pointer");
    const size_t smem = (size_t)D * kBkmPitch * sizeof(double);
    cudaFuncSetAttribute(bkm_assign_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    const int64_t blocks = (n_rows + kBkmRows - 1) / kBkmRows;
    B2F_REQUIRE(blocks <= 0x7fffffffll, "bkm_assign: too many rows");
    bkm_assign_kernel<<<(unsigned)blocks, kBkmThreads, smem, (cudaStream_t)stream>>>(x, n_rows, D, ld, node, num_nodes, slot_of_node,
                                                                                    centers, m, present, prev, child,
                                                                                    prev ? dist_prev : nullptr);
    return check_launch("bkm_assign");
}

extern "C" int b200flow_bkm_predict(const double* x, int64_t n_rows, int32_t D, int64_t ld, const int32_t* left, const int32_t* right,
                                    const int32_t* leaf, const double* centers, int32_t num_nodes, int32_t root, int32_t* out_leaf,
                                    double* out_dist, void* stream) {
    B2F_REQUIRE(n_rows >= 0 && D >= 1 && D <= kBkmMaxD && ld >= D && num_nodes >= 1 && num_nodes <= 4095 && root >= 0 &&
                root < num_nodes, "bkm_predict: n >= 0, 1 <= D <= %d, ld >= D, 1 <= num_nodes <= 4095, 0 <= root < num_nodes",
                kBkmMaxD);
    if (n_rows == 0) return B200FLOW_OK;
    B2F_REQUIRE(x && left && right && leaf && centers && out_leaf && out_dist, "bkm_predict: null pointer");
    const size_t smem = (size_t)D * kBkmPitch * sizeof(double);
    cudaFuncSetAttribute(bkm_predict_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    const int64_t blocks = (n_rows + kBkmRows - 1) / kBkmRows;
    B2F_REQUIRE(blocks <= 0x7fffffffll, "bkm_predict: too many rows");
    bkm_predict_kernel<<<(unsigned)blocks, kBkmThreads, smem, (cudaStream_t)stream>>>(x, n_rows, D, ld, left, right, leaf, centers,
                                                                                     root, out_leaf, out_dist);
    return check_launch("bkm_predict");
}
