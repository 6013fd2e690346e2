// radix_sort.cuh — the stable LSD radix sort (8-bit digits) of 64-bit keys with a 32-bit payload, shared by
// metrics.cu (BinaryClassificationMetrics, DESIGN.md §5b) and isotonic.cu (IsotonicRegression, DESIGN.md §5p).
//
// One pass = a per-block digit histogram (digit-major, so an exclusive scan over it gives every (digit, block) its first
// output slot), that scan, and a stable scatter.  Passes over shifts 0, 8, ..., 56 sort by the whole key; ties keep the
// input order of the payload.
#pragma once
#include "common.cuh"

namespace b200flow {

constexpr int kSortThreads = 256;
constexpr int kSortItems = 16;                                   // items per thread and pass
constexpr int kSortTile = kSortThreads * kSortItems;             // 4096 items per block and pass
constexpr int kSortWarps = kSortThreads / 32;

// digit of item p in this pass: key bits, or (seg_pass) bits of the segment id of the item's original index
template <bool kSegPass>
__device__ __forceinline__ int sort_digit(unsigned long long k, uint32_t id, int shift, int64_t n) {
    if (kSegPass) return (int)(((uint64_t)id / (uint64_t)n) >> shift) & 255;
    return (int)(k >> shift) & 255;
}

// per-block digit counts, digit-major: hist[d * nb + b] (a scan over it gives every (digit, block) its first output slot)
template <bool kSegPass>
__global__ void __launch_bounds__(kSortThreads) radix_hist_kernel(const unsigned long long* __restrict__ key,
                                                                  const uint32_t* __restrict__ idx, int64_t M, int64_t n,
                                                                  int shift, int32_t* hist) {
    __shared__ int cnt[256];
    cnt[threadIdx.x] = 0;
    __syncthreads();
    const int64_t base = (int64_t)blockIdx.x * kSortTile;
#pragma unroll 4
    for (int k = 0; k < kSortItems; ++k) {
        const int64_t p = base + (int64_t)k * kSortThreads + threadIdx.x;
        if (p < M) atomicAdd(&cnt[sort_digit<kSegPass>(kSegPass ? 0ull : key[p], kSegPass ? idx[p] : 0u, shift, n)], 1);
    }
    __syncthreads();
    hist[(int64_t)threadIdx.x * gridDim.x + blockIdx.x] = cnt[threadIdx.x];
}

// stable scatter of one pass.  Warp w owns items [w*512, (w+1)*512) of the block's tile, 32 at a time in order; lanes with
// equal digits find each other with __match_any_sync and rank by lane, and a per-warp digit counter in shared memory
// carries the rank across rounds.  Warp bases per digit follow from the counters, block bases from the global scan.
template <bool kSegPass>
__global__ void __launch_bounds__(kSortThreads) radix_scatter_kernel(const unsigned long long* __restrict__ key,
                                                                     const uint32_t* __restrict__ idx, int64_t M, int64_t n,
                                                                     int shift, const int64_t* __restrict__ offs,
                                                                     unsigned long long* key_out, uint32_t* idx_out) {
    __shared__ int cnt[kSortWarps][257];                         // digit 256: items past the end
    __shared__ int64_t wbase[kSortWarps][256];
    const int w = warp_id(), lane = lane_id();
    for (int i = threadIdx.x; i < kSortWarps * 257; i += kSortThreads) (&cnt[0][0])[i] = 0;
    __syncthreads();
    const unsigned lt = (1u << lane) - 1u;
    const int64_t base = (int64_t)blockIdx.x * kSortTile + (int64_t)w * (kSortTile / kSortWarps);
    unsigned long long k[kSortItems]; uint32_t id[kSortItems]; int dg[kSortItems], rk[kSortItems];
#pragma unroll
    for (int r = 0; r < kSortItems; ++r) {
        const int64_t p = base + r * 32 + lane;
        const bool live = p < M;
        k[r] = live ? key[p] : 0ull;
        id[r] = live ? idx[p] : 0u;
        dg[r] = live ? sort_digit<kSegPass>(k[r], id[r], shift, n) : 256;
        const unsigned peers = __match_any_sync(0xffffffffu, dg[r]);
        const int before = cnt[w][dg[r]];
        __syncwarp();
        if ((peers & lt) == 0) cnt[w][dg[r]] = before + __popc(peers);      // the lowest lane of each digit group
        __syncwarp();
        rk[r] = before + __popc(peers & lt);
    }
    __syncthreads();
    {
        const int d = threadIdx.x;                                   // kSortThreads == 256 digits
        int64_t run = offs[(int64_t)d * gridDim.x + blockIdx.x];
        for (int ww = 0; ww < kSortWarps; ++ww) { wbase[ww][d] = run; run += cnt[ww][d]; }
    }
    __syncthreads();
#pragma unroll
    for (int r = 0; r < kSortItems; ++r) {
        if (dg[r] == 256) continue;
        const int64_t q = wbase[w][dg[r]] + rk[r];
        key_out[q] = k[r];
        idx_out[q] = id[r];
    }
}

// blocks of one pass over M items
inline int64_t radix_blocks(int64_t M) { return (M + kSortTile - 1) / kSortTile; }

// one pass (histogram, scan, scatter) from (key, idx) into (key_out, idx_out); hist int32 [256 * nb] and offs int64
// [256 * nb] are scratch, nb = radix_blocks(M)
template <bool kSegPass>
inline int radix_pass(const unsigned long long* key, const uint32_t* idx, int64_t M, int64_t n, int shift, int32_t* hist,
                      int64_t* offs, unsigned long long* key_out, uint32_t* idx_out, void* stream) {
    const int64_t nb = radix_blocks(M);
    cudaStream_t st = (cudaStream_t)stream;
    radix_hist_kernel<kSegPass><<<(unsigned)nb, kSortThreads, 0, st>>>(key, idx, M, n, shift, hist);
    const int rc = b200flow_exclusive_scan_i32_to_i64(hist, 256 * nb, offs, nullptr, stream);
    if (rc) return rc;
    radix_scatter_kernel<kSegPass><<<(unsigned)nb, kSortThreads, 0, st>>>(key, idx, M, n, shift, offs, key_out, idx_out);
    return 0;
}

}  // namespace b200flow
