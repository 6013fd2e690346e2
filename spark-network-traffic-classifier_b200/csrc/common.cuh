// common.cuh — shared device helpers for libb200flow (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/b200flow.h"

namespace b200flow {

void set_error(const char* fmt, ...);
int check_launch(const char* what);

#define B2F_REQUIRE(cond, ...)                                   \
    do {                                                         \
        if (!(cond)) { b200flow::set_error(__VA_ARGS__); return B200FLOW_ERR_ARG; } \
    } while (0)

constexpr int kNumSMs = 132;   // H100 SXM; grids are sized in multiples of this

// ------------------------------------------------------------------ Philox4x32-10
// Counter-based RNG (DESIGN.md §RNG): key = (lo32(seed) ^ purpose, hi32(seed)).
constexpr uint32_t PURPOSE_SAMPLE = 0x53414D50u;  // findSplits row sample      ctr = (row_lo,row_hi,0,0)
constexpr uint32_t PURPOSE_BAG    = 0x42414747u;  // Poisson bagging            ctr = (row_lo,row_hi,tree/4,0), word tree%4
constexpr uint32_t PURPOSE_FEAT   = 0x46454154u;  // per-node feature subset    ctr = (tree,nid,draw/4,0)
constexpr uint32_t PURPOSE_RSPLIT = 0x5253504Cu;  // DataFrame.randomSplit      ctr = (row_lo,row_hi,0,0)

__device__ __forceinline__ uint4 philox4x32_10(uint32_t k0, uint32_t k1, uint4 c) {
    const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        uint32_t hi0 = __umulhi(M0, c.x), lo0 = M0 * c.x;
        uint32_t hi1 = __umulhi(M1, c.z), lo1 = M1 * c.z;
        c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
        k0 += W0; k1 += W1;
    }
    return c;
}
__device__ __forceinline__ uint4 philox_keyed(uint64_t seed, uint32_t purpose, uint32_t c0, uint32_t c1,
                                              uint32_t c2, uint32_t c3) {
    return philox4x32_10((uint32_t)seed ^ purpose, (uint32_t)(seed >> 32), make_uint4(c0, c1, c2, c3));
}

// Poisson weights by inverse CDF over 32 increasing integer thresholds: w = #{k : cdf[k] != 2^32-1 and r >= cdf[k]}.
// One Philox call serves FOUR trees: counter = (row_lo, row_hi, tree >> 2, 0), word = tree & 3.
__device__ __forceinline__ uint32_t poisson_weight(uint32_t r, const uint32_t* cdf_sh) {
    uint32_t k = 0;
    while (k < 32 && cdf_sh[k] != 0xFFFFFFFFu && r >= cdf_sh[k]) ++k;      // thresholds increase: first failure ends the count
    return k;
}
__device__ __forceinline__ uint4 bag_draw4(uint64_t seed, int tree_quad, uint64_t grow) {
    return philox_keyed(seed, PURPOSE_BAG, (uint32_t)grow, (uint32_t)(grow >> 32), (uint32_t)tree_quad, 0u);
}

// bagged entry = (index of a UNIQUE TreePoint record, summed bag weight of the rows that share it): 8 bytes
typedef uint2 b2f_entry;      // .x = record index, .y = weight

// ------------------------------------------------------------------ warp / block helpers
__device__ __forceinline__ int lane_id() { return threadIdx.x & 31; }
__device__ __forceinline__ int warp_id() { return threadIdx.x >> 5; }

template <typename T>
__device__ __forceinline__ T warp_sum(T v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
template <typename T>
__device__ __forceinline__ T warp_inclusive_scan(T v) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { T u = __shfl_up_sync(0xffffffffu, v, o); if (lane_id() >= o) v += u; }
    return v;
}

// block-wide exclusive scan of one int per thread (blockDim <= 1024); returns exclusive prefix,
// *total = block sum.  sh must hold 33 ints.  Contains two __syncthreads.
__device__ __forceinline__ int block_exclusive_scan(int v, int* sh, int* total) {
    int inc = warp_inclusive_scan(v);
    if (lane_id() == 31) sh[warp_id()] = inc;
    __syncthreads();
    if (warp_id() == 0) {
        int nw = (blockDim.x + 31) >> 5;
        int w = lane_id() < nw ? sh[lane_id()] : 0;
        int winc = warp_inclusive_scan(w);
        sh[lane_id()] = winc - w;
        if (lane_id() == 31) sh[32] = winc;
    }
    __syncthreads();
    int res = inc - v + sh[warp_id()];
    *total = sh[32];
    return res;
}

// ------------------------------------------------------------------ TMA bulk copy (1-D) + mbarrier
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
// global -> shared bulk copy (UBLKCP), completion signalled on an mbarrier; 16-byte aligned, size % 16 == 0
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
// shared -> global bulk copy, tracked by bulk async-groups
__device__ __forceinline__ void bulk_s2g(void* dst_gmem, const void* src_smem, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst_gmem), "r"(smem_u32(src_smem)),
                 "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory"); }
// make generic-proxy smem writes visible to the async proxy (before a bulk store reads them)
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// Ampere-style asynchronous global->shared copies (LDGSTS): no register staging, tracked by commit groups
__device__ __forceinline__ void cp_async4(void* dst_smem, const void* src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(dst_smem)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async8(void* dst_smem, const void* src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(smem_u32(dst_smem)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async16(void* dst_smem, const void* src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst_smem)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

// read-once / write-once 64-bit accesses marked evict-first in the L2: the bagged-entry stream (1 GB per level) passes through
// once per level and must not push the re-used TreePoint records (61 MB on KDD99-full, gathered at random) out of the 50 MB L2
__device__ __forceinline__ uint2 ld_evict_first_u2(const void* p) {
    uint2 r;
    asm volatile("ld.global.cs.v2.u32 {%0,%1}, [%2];" : "=r"(r.x), "=r"(r.y) : "l"(p));      // .cs = cache-streaming: evict-first
    return r;
}
__device__ __forceinline__ void st_evict_first_u2(void* p, uint2 v) {      // .cs = cache-streaming: evict-first
    asm volatile("st.global.cs.v2.u32 [%0], {%1,%2};" ::"l"(p), "r"(v.x), "r"(v.y) : "memory");
}

// streaming (read-once) 128-bit load / store that do not pollute L1
__device__ __forceinline__ uint4 ld_stream_u4(const void* p) {
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}
__device__ __forceinline__ void st_stream_u4(void* p, uint4 v) {
    asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

// ------------------------------------------------------------------ fp64 tensor-core MMA (mma.sync m8n8k4 f64, SASS DMMA.8x8x4)
// Fragments (PTX ISA): A holds (row lane>>2, k lane&3), B holds (k lane&3, col lane>>2), C/D hold (row lane>>2,
// col 2(lane&3) + {0,1}).  c += a b, the four products of a (row, col) rounded once.
__device__ __forceinline__ void dmma(double (&c)[2], double a, double b) {
    asm("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
        : "+d"(c[0]), "+d"(c[1])
        : "d"(a), "d"(b));
}
// widths are zero-padded to multiples of the 8-wide fragments; the padding is exact zeros and adds nothing to a product
__host__ __device__ inline int pad8(int v) { return (v + 7) / 8 * 8; }

template <typename T> __device__ __forceinline__ double load_as_double(const void* base, int64_t idx);
template <> __device__ __forceinline__ double load_as_double<float>(const void* base, int64_t idx) {
    return (double)__ldg((const float*)base + idx);
}
template <> __device__ __forceinline__ double load_as_double<double>(const void* base, int64_t idx) {
    return __ldg((const double*)base + idx);
}

// ------------------------------------------------------------------ Java double order, exact fixed-point sums
// (shared by isotonic.cu, quantile.cu and regression.cu)
// ascending order of x as a uint64, Java's Double.compare: -0.0 sorts before 0.0
__device__ __forceinline__ unsigned long long asc_key(double x) {
    const unsigned long long b = (unsigned long long)__double_as_longlong(x);
    return (b >> 63) ? ~b : (b | (1ull << 63));
}

// java.util.Arrays.binarySearch(double[], double) on b [K]: the index of a hit, else -(insertion point) - 1.  Equal values
// order by Double.doubleToLongBits (NaN canonical) as signed longs, so -0.0 < 0.0 and NaN is above everything.
__device__ __forceinline__ int64_t java_binary_search(const double* __restrict__ b, int64_t K, double key) {
    const long long kb = key != key ? 0x7ff8000000000000ll : __double_as_longlong(key);
    int64_t low = 0, high = K - 1;
    while (low <= high) {
        const int64_t mid = (low + high) >> 1;
        const double m = b[mid];
        if (m < key) low = mid + 1;
        else if (m > key) high = mid - 1;
        else {
            const long long mb = m != m ? 0x7ff8000000000000ll : __double_as_longlong(m);
            if (mb == kb) return mid;
            if (mb < kb) low = mid + 1;
            else high = mid - 1;
        }
    }
    return -(low + 1);
}

// rint(t 2^sh) (|.| < 2^126) as a two's-complement 128-bit integer: 32-bit limbs, the top one signed
__device__ __forceinline__ void fixed_limbs(double t, int sh, long long* limb) {
    const double v = rint(ldexp(t, sh));
    const double a = fabs(v);
    unsigned __int128 u;
    if (a < 9223372036854775808.0) {
        u = (unsigned __int128)(unsigned long long)a;
    } else {
        int e;
        const double mnt = frexp(a, &e);                               // a = mnt 2^e, 2^63 <= a < 2^126: e - 53 >= 11
        u = (unsigned __int128)(unsigned long long)ldexp(mnt, 53) << (e - 53);
    }
    if (v < 0.0) u = ~u + 1;
    limb[0] = (long long)(u & 0xffffffffull);
    limb[1] = (long long)((u >> 32) & 0xffffffffull);
    limb[2] = (long long)((u >> 64) & 0xffffffffull);
    limb[3] = (long long)(int)(unsigned)(u >> 96);
}

// chunk id -> (slot, chunk-in-slot) by binary search over the exclusive scan chunk_off[n_slots+1]
__device__ __forceinline__ int find_slot(const int64_t* __restrict__ chunk_off, int n_slots, int64_t c) {
    int lo = 0, hi = n_slots;                          // last s with chunk_off[s] <= c
    while (hi - lo > 1) { int mid = (lo + hi) >> 1; if (__ldg(chunk_off + mid) <= c) lo = mid; else hi = mid; }
    return lo;
}

inline int grid_for(int64_t work_items, int per_block, int max_blocks) {
    int64_t b = (work_items + per_block - 1) / per_block;
    if (b < 1) b = 1;
    if (b > max_blocks) b = max_blocks;
    return (int)b;
}

}  // namespace b200flow
