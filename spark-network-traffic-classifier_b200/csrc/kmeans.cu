// kmeans.cu — KMeans (k-means||, Lloyd) and the silhouette ClusteringEvaluator, DESIGN.md §5c.
//
// b200flow_kmeans_assign: first argmin center and its squared distance per row, the distance summed in feature order from
// 0.0 as acc = acc + t*t with t = x_j - c_j (-fmad=false: no FMA, no norm trick), so every term rounds as on the host.
// b200flow_group_sums / group_sums_chain: the one reduction of the feature.  Global rows are cut into fixed 4096-row chunks;
// a chunk's partial of (group, column) is the sequential sum of its member rows in row order, and the total is the
// sequential sum of the partials in chunk order.  The grouping is fixed by the global row index alone, so the bits do
// not depend on how rows are spread over ranks.
#include <math.h>

#include "common.cuh"

namespace b200flow {

constexpr uint32_t PURPOSE_KMNS = 0x4B4D4E53u;   // k-means init: ctr = (row_lo, row_hi, step, 0)
constexpr int kChunkRows = 4096;
constexpr int kMaxGroups = 4096;

// ------------------------------------------------------------------ assign
constexpr int kAsgRows = 64, kAsgCenters = 32, kAsgThreads = 128;
constexpr int kAsgRowPitch = kAsgRows + 1, kAsgCenterPitch = kAsgCenters + 1;   // odd pitches: staging stores are conflict-light
constexpr int kAsgMaxD = 256;

// One CTA per 64 rows, staged transposed in shared memory once; the centers stream through in tiles of 32.  Thread
// (ty, tx) owns rows ty + 16i and centers tx + 8q (i, q < 4): 16 independent sub-mul-add chains per feature.
__global__ void __launch_bounds__(kAsgThreads) kmeans_assign_kernel(const double* __restrict__ x, int64_t n, int D, int64_t ld,
                                                                   const double* __restrict__ centers, int k,
                                                                   int32_t* __restrict__ cluster, double* __restrict__ dist) {
    extern __shared__ double sm[];
    double* xs = sm;                                       // [D][kAsgRowPitch]
    double* cs = sm + (size_t)D * kAsgRowPitch;            // [D][kAsgCenterPitch]
    const int tid = threadIdx.x, tx = tid & 7, ty = tid >> 3;
    const int64_t row0 = (int64_t)blockIdx.x * kAsgRows;
    for (int e = tid; e < kAsgRows * D; e += kAsgThreads) {
        const int r = e / D, j = e - r * D;
        const int64_t gr = row0 + r;
        xs[j * kAsgRowPitch + r] = gr < n ? x[gr * ld + j] : 0.0;
    }
    double best[4];
    int bi[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) { best[i] = INFINITY; bi[i] = 0x7fffffff; }
    for (int c0 = 0; c0 < k; c0 += kAsgCenters) {
        __syncthreads();                                   // the previous center tile is consumed (first pass: nothing)
        for (int e = tid; e < kAsgCenters * D; e += kAsgThreads) {
            const int c = e / D, j = e - c * D;
            cs[j * kAsgCenterPitch + c] = c0 + c < k ? centers[(int64_t)(c0 + c) * D + j] : 0.0;
        }
        __syncthreads();
        double acc[4][4];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int q = 0; q < 4; ++q) acc[i][q] = 0.0;
#pragma unroll 2
        for (int j = 0; j < D; ++j) {
            double xv[4], cv[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) xv[i] = xs[j * kAsgRowPitch + ty + 16 * i];
#pragma unroll
            for (int q = 0; q < 4; ++q) cv[q] = cs[j * kAsgCenterPitch + tx + 8 * q];
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const double t = xv[i] - cv[q];
                    acc[i][q] = acc[i][q] + t * t;
                }
        }
#pragma unroll
        for (int q = 0; q < 4; ++q) {                      // a thread meets its centers in increasing order: strict < keeps the first
            const int c = c0 + tx + 8 * q;
            if (c < k) {
#pragma unroll
                for (int i = 0; i < 4; ++i)
                    if (acc[i][q] < best[i]) { best[i] = acc[i][q]; bi[i] = c; }
            }
        }
    }
    // (dist, index) lexicographic min over the 8 threads of a row group (lanes differing in the low 3 bits)
#pragma unroll
    for (int i = 0; i < 4; ++i) {
#pragma unroll
        for (int o = 1; o < 8; o <<= 1) {
            const double od = __shfl_xor_sync(0xffffffffu, best[i], o);
            const int oi = __shfl_xor_sync(0xffffffffu, bi[i], o);
            if (od < best[i] || (od == best[i] && oi < bi[i])) { best[i] = od; bi[i] = oi; }
        }
        const int64_t gr = row0 + ty + 16 * i;
        if (tx == 0 && gr < n) { cluster[gr] = bi[i]; dist[gr] = best[i]; }
    }
}

// ------------------------------------------------------------------ grouped sums
constexpr int kGsThreads = 256;

// One CTA per chunk.  Warp 0 counting-sorts the chunk's rows by group, stably (lanes with equal ids rank by lane through
// __match_any_sync, a per-group cursor carries the rank across rounds), so each (group, column) item then sums its rows
// in row order.
__global__ void __launch_bounds__(kGsThreads) group_sums_kernel(const double* __restrict__ v, int64_t ld, const int32_t* __restrict__ ids,
                                                                int64_t n, int W, int G, int64_t row_offset,
                                                                double* __restrict__ partials, unsigned long long* counts) {
    extern __shared__ int gs_sm[];
    int* cnt = gs_sm;                                      // [G]
    int* cur = gs_sm + G;                                  // [G]: group starts, then ends
    uint16_t* order = (uint16_t*)(gs_sm + 2 * G);          // [kChunkRows]
    __shared__ int scan_sh[33];
    const int64_t chunk = row_offset / kChunkRows + blockIdx.x;
    const int64_t lo = max((int64_t)0, chunk * kChunkRows - row_offset), hi = min(n, (chunk + 1) * kChunkRows - row_offset);
    const int m = (int)(hi - lo);
    const int tid = threadIdx.x;
    if (ids) {
        for (int g = tid; g < G; g += kGsThreads) cnt[g] = 0;
        __syncthreads();
        for (int r = tid; r < m; r += kGsThreads) {
            const int g = ids[lo + r];
            if (g >= 0 && g < G) atomicAdd(&cnt[g], 1);
        }
        __syncthreads();
        const int per = (G + kGsThreads - 1) / kGsThreads;
        const int a = min(G, tid * per), b = min(G, a + per);
        int local = 0;
        for (int g = a; g < b; ++g) local += cnt[g];
        int total;
        int run = block_exclusive_scan(local, scan_sh, &total);
        for (int g = a; g < b; ++g) { cur[g] = run; run += cnt[g]; }
        __syncthreads();
        if (warp_id() == 0) {
            const int lane = lane_id();
            const unsigned lt = (1u << lane) - 1u;
            for (int base = 0; base < m; base += 32) {
                const int r = base + lane;
                int g = r < m ? ids[lo + r] : -1;
                if (g >= G) g = -1;
                const unsigned peers = __match_any_sync(0xffffffffu, g);
                const int before = g >= 0 ? cur[g] : 0;
                __syncwarp();
                if (g >= 0 && (peers & lt) == 0) cur[g] = before + __popc(peers);
                __syncwarp();
                if (g >= 0) order[before + __popc(peers & lt)] = (uint16_t)r;
            }
        }
        __syncthreads();
    } else if (tid == 0) {                                 // one group: every row of the chunk, in order
        cnt[0] = m;
        cur[0] = m;
    }
    __syncthreads();
    double* out = partials + (int64_t)blockIdx.x * G * W;
    for (int it = tid; it < G * W; it += kGsThreads) {
        const int g = it / W, w = it - g * W;
        const int c = cnt[g], s = cur[g] - c;
        double acc = 0.0;
        if (ids) {
            for (int p = s; p < s + c; ++p) acc = acc + v[(lo + order[p]) * ld + w];
        } else {
            for (int r = 0; r < c; ++r) acc = acc + v[(lo + r) * ld + w];
        }
        out[it] = acc;
    }
    if (counts)
        for (int g = tid; g < G; g += kGsThreads)
            if (cnt[g]) atomicAdd(counts + g, (unsigned long long)cnt[g]);
}

__global__ void __launch_bounds__(256) group_sums_chain_kernel(const double* __restrict__ partials, int64_t n_chunks, int64_t GW,
                                                               double* totals) {
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < GW; e += (int64_t)gridDim.x * blockDim.x) {
        double acc = totals[e];
        for (int64_t b = 0; b < n_chunks; ++b) acc = acc + partials[b * GW + e];
        totals[e] = acc;
    }
}

// ------------------------------------------------------------------ init draws
__global__ void __launch_bounds__(256) kmeans_row_keys_kernel(uint64_t seed, int64_t row_offset, int64_t n, long long* keys) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const uint64_t g = (uint64_t)(row_offset + i);
        const uint4 r = philox_keyed(seed, PURPOSE_KMNS, (uint32_t)g, (uint32_t)(g >> 32), 0u, 0u);
        keys[i] = (long long)((((uint64_t)r.x << 32) | r.y) ^ (1ull << 63));
    }
}

__global__ void __launch_bounds__(256) kmeans_select_kernel(uint64_t seed, int64_t row_offset, int64_t n, int32_t step,
                                                            const double* __restrict__ cost, double k, double sum_cost,
                                                            uint8_t* flag) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const uint64_t g = (uint64_t)(row_offset + i);
        const uint4 r = philox_keyed(seed, PURPOSE_KMNS, (uint32_t)g, (uint32_t)(g >> 32), (uint32_t)step, 0u);
        const double u = (double)((((uint64_t)r.x) << 21) | (r.y >> 11)) * 0x1.0p-53;
        flag[i] = u < ((2.0 * cost[i]) * k) / sum_cost ? 1 : 0;
    }
}

// ------------------------------------------------------------------ silhouette
__global__ void __launch_bounds__(256) silhouette_rows_kernel(const double* __restrict__ x, int64_t n, int D, int64_t ld,
                                                              const double* __restrict__ norms, const int32_t* __restrict__ cluster,
                                                              const double* __restrict__ Y, const double* __restrict__ psi,
                                                              const int64_t* __restrict__ N, int G, double* __restrict__ out) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const double* xi = x + i * ld;
        const double nx = norms[i];
        const int own = cluster[i];
        double d_own = 0.0, b = INFINITY;
        for (int g = 0; g < G; ++g) {
            const int64_t ng = N[g];
            if (ng == 0) continue;                         // a cluster absent from the data is not a neighbour
            const double* y = Y + (int64_t)g * D;
            double dot = 0.0;
            for (int j = 0; j < D; ++j) dot = dot + xi[j] * y[j];
            const double nd = (double)ng;
            const double d = (nx + psi[g] / nd) - (2.0 * dot) / nd;
            if (g == own) d_own = d;
            else if (d < b) b = d;
        }
        const int64_t n_own = N[own];
        double s = 0.0;
        if (n_own > 1) {
            const double a = d_own * (double)n_own / (double)(n_own - 1);
            if (a < b) s = 1.0 - a / b;
            else if (a > b) s = b / a - 1.0;
        }
        out[i] = s;
    }
}

}  // namespace b200flow

using namespace b200flow;

extern "C" int b200flow_kmeans_assign(const double* x, int64_t n_rows, int32_t D, int64_t ld, const double* centers, int32_t k,
                                      int32_t* cluster, double* dist, void* stream) {
    B2F_REQUIRE(n_rows >= 0 && D >= 1 && D <= kAsgMaxD && ld >= D && k >= 1, "kmeans_assign: n >= 0, 1 <= D <= %d, ld >= D, k >= 1",
                kAsgMaxD);
    if (n_rows == 0) return B200FLOW_OK;
    B2F_REQUIRE(x && centers && cluster && dist, "kmeans_assign: null pointer");
    const size_t smem = (size_t)D * (kAsgRowPitch + kAsgCenterPitch) * sizeof(double);
    cudaFuncSetAttribute(kmeans_assign_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    const int64_t blocks = (n_rows + kAsgRows - 1) / kAsgRows;
    B2F_REQUIRE(blocks <= 0x7fffffffll, "kmeans_assign: too many rows");
    kmeans_assign_kernel<<<(unsigned)blocks, kAsgThreads, smem, (cudaStream_t)stream>>>(x, n_rows, D, ld, centers, k, cluster, dist);
    return check_launch("kmeans_assign");
}

extern "C" int b200flow_group_sums_chunks(int64_t row_offset, int64_t n_rows, int64_t* n_chunks) {
    B2F_REQUIRE(n_chunks && row_offset >= 0 && n_rows >= 0, "group_sums_chunks: row_offset >= 0, n_rows >= 0");
    *n_chunks = n_rows == 0 ? 0 : (row_offset + n_rows - 1) / kChunkRows - row_offset / kChunkRows + 1;
    return B200FLOW_OK;
}

extern "C" int b200flow_group_sums(const double* values, int64_t ld, const int32_t* ids, int64_t n_rows, int32_t W, int32_t G,
                                   int64_t row_offset, double* partials, int64_t* counts, void* stream) {
    B2F_REQUIRE(n_rows >= 0 && W >= 1 && ld >= W && G >= 1 && G <= kMaxGroups && row_offset >= 0 && (ids || G == 1),
                "group_sums: W >= 1, ld >= W, 1 <= G <= %d (G == 1 without ids), row_offset >= 0", kMaxGroups);
    int64_t nc = 0;
    b200flow_group_sums_chunks(row_offset, n_rows, &nc);
    if (nc == 0) return B200FLOW_OK;
    B2F_REQUIRE(values && partials, "group_sums: null pointer");
    const size_t smem = 2 * (size_t)G * sizeof(int) + kChunkRows * sizeof(uint16_t);
    group_sums_kernel<<<(unsigned)nc, kGsThreads, smem, (cudaStream_t)stream>>>(values, ld, ids, n_rows, W, G, row_offset, partials,
                                                                                (unsigned long long*)counts);
    return check_launch("group_sums");
}

extern "C" int b200flow_group_sums_chain(const double* partials, int64_t n_chunks, int32_t G, int32_t W, double* totals, void* stream) {
    B2F_REQUIRE(n_chunks >= 0 && G >= 1 && W >= 1 && totals && (partials || n_chunks == 0), "group_sums_chain: bad arguments");
    if (n_chunks == 0) return B200FLOW_OK;
    const int64_t GW = (int64_t)G * W;
    group_sums_chain_kernel<<<grid_for(GW, 256, kNumSMs * 8), 256, 0, (cudaStream_t)stream>>>(partials, n_chunks, GW, totals);
    return check_launch("group_sums_chain");
}

extern "C" int b200flow_kmeans_row_keys(uint64_t seed, int64_t row_offset, int64_t n_rows, int64_t* keys, void* stream) {
    B2F_REQUIRE(n_rows >= 0 && row_offset >= 0 && (keys || n_rows == 0), "kmeans_row_keys: bad arguments");
    if (n_rows == 0) return B200FLOW_OK;
    kmeans_row_keys_kernel<<<grid_for(n_rows, 256, kNumSMs * 16), 256, 0, (cudaStream_t)stream>>>(seed, row_offset, n_rows,
                                                                                                   (long long*)keys);
    return check_launch("kmeans_row_keys");
}

extern "C" int b200flow_kmeans_select(uint64_t seed, int64_t row_offset, int64_t n_rows, int32_t step, const double* cost,
                                      int32_t k, double sum_cost, uint8_t* flag, void* stream) {
    B2F_REQUIRE(n_rows >= 0 && row_offset >= 0 && step >= 1 && k >= 1 && ((cost && flag) || n_rows == 0),
                "kmeans_select: bad arguments");
    if (n_rows == 0) return B200FLOW_OK;
    kmeans_select_kernel<<<grid_for(n_rows, 256, kNumSMs * 16), 256, 0, (cudaStream_t)stream>>>(seed, row_offset, n_rows, step, cost,
                                                                                                 (double)k, sum_cost, flag);
    return check_launch("kmeans_select");
}

extern "C" int b200flow_silhouette_rows(const double* x, int64_t n_rows, int32_t D, int64_t ld, const double* norms,
                                        const int32_t* cluster, const double* Y, const double* psi, const int64_t* N, int32_t G,
                                        double* out, void* stream) {
    B2F_REQUIRE(n_rows >= 0 && D >= 1 && ld >= D && G >= 1, "silhouette_rows: bad arguments");
    if (n_rows == 0) return B200FLOW_OK;
    B2F_REQUIRE(x && norms && cluster && Y && psi && N && out, "silhouette_rows: null pointer");
    silhouette_rows_kernel<<<grid_for(n_rows, 256, kNumSMs * 16), 256, 0, (cudaStream_t)stream>>>(x, n_rows, D, ld, norms, cluster, Y,
                                                                                                   psi, N, G, out);
    return check_launch("silhouette_rows");
}
