// encode.cu — the fused row-parallel encode path (SURVEY.md §8a R1, R2, R3, R3b, R3c).
//
// Replaces, for the reference call sites kdd99.py:34-37,45-46 and cicids17.py:41-46, MLlib's
// StringIndexer.fit (category counts), StringIndexerModel.transform (code -> rank lookup),
// OneHotEncoder (expand), StandardScaler (fit moments + scale) and VectorAssembler (concat)
// with ONE pass over the raw AoS flow records.
//
// encode kernel, data movement (HBM-bound; algorithmic bytes/row = row_bytes + n_out*sizeof(out) + 4):
//   HBM --cp.async.bulk (TMA, UBLKCP) + mbarrier--> smem record tile [R x row_bytes], NS-deep ring
//   threads: one fixed OUTPUT slot per thread, rows strided -> smem out tile [R x n_out] (bank-conflict free)
//   smem out tile --cp.async.bulk store (bulk_group)--> HBM, triple buffered; ONE __syncthreads per tile
// Arithmetic is fp64 ((v - mean) * scale, no FMA contraction) and rounded once to the output type.
#include <stdlib.h>

#include "common.cuh"

namespace b200flow {

// ------------------------------------------------------------------ R1 category counts
__global__ void __launch_bounds__(256) category_counts_kernel(const uint8_t* __restrict__ rec, int64_t n, int row_bytes,
                                                              int src_off, int K, unsigned long long* counts,
                                                              int use_smem) {
    extern __shared__ uint32_t sh_cnt[];
    if (use_smem) {
        for (int i = threadIdx.x; i < K; i += blockDim.x) sh_cnt[i] = 0;
        __syncthreads();
    }
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        int code = __ldg((const int*)(rec + i * row_bytes + src_off));
        if (code >= 0 && code < K) {
            if (use_smem) atomicAdd(&sh_cnt[code], 1u);
            else atomicAdd(&counts[code], 1ull);
        }
    }
    if (use_smem) {
        __syncthreads();
        for (int i = threadIdx.x; i < K; i += blockDim.x)
            if (sh_cnt[i]) atomicAdd(&counts[i], (unsigned long long)sh_cnt[i]);
    }
}

// several columns in ONE pass over the records: the code fields of a flow record sit in the same one or two 32-byte sectors,
// so four StringIndexer fits cost one read of the batch instead of four (kdd99.py:34-37 fits four indexers back to back)
struct CountCols { int n; int off[8]; int K[8]; int base[8]; };

__global__ void __launch_bounds__(256) category_counts_multi_kernel(const uint8_t* __restrict__ rec, int64_t n, int row_bytes,
                                                                    const CountCols cc, int total, unsigned long long* counts) {
    extern __shared__ uint32_t sh_cnt[];
    for (int i = threadIdx.x; i < total; i += blockDim.x) sh_cnt[i] = 0;
    __syncthreads();
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const uint8_t* r = rec + i * row_bytes;
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            if (c < cc.n) {
                const int code = __ldg((const int*)(r + cc.off[c]));
                if (code >= 0 && code < cc.K[c]) atomicAdd(&sh_cnt[cc.base[c] + code], 1u);
            }
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < total; i += blockDim.x)
        if (sh_cnt[i]) atomicAdd(&counts[i], (unsigned long long)sh_cnt[i]);
}

// ------------------------------------------------------------------ fused encode
struct EncodeArgs {
    const uint8_t* records; int64_t n_rows; int row_bytes;
    const b200flow_slot* plan; int n_out;
    const int32_t* lut; int lut_total; int lut_in_smem;
    int label_off, label_lut_off, label_lut_len, check_nan;
    void* out; int32_t* label_out; uint8_t* valid_out;
    int R;            // rows per tile (multiple of 4)
    int stages;       // depth of the TMA load ring (2 or 3)
    int in_stride;    // bytes per input stage (128-aligned)
    int out_stride;   // bytes per output stage (128-aligned)
};

constexpr int kEncStages = 3;     // TMA load ring depth
constexpr int kEncOutBufs = 3;    // output tiles: two bulk stores may be in flight while the third tile is computed
constexpr int kEncThreads = 256;
constexpr int kEncMaxCat = 8;     // distinct categorical sources whose rank is shared through shared memory

template <typename OUT>
__global__ void __launch_bounds__(kEncThreads, 4) encode_kernel(const EncodeArgs a) {
    extern __shared__ __align__(128) uint8_t smem[];
    // layout: [in ring][out x3][mbar][badtag 2*R][plan][lut]
    uint8_t* in_base = smem;
    uint8_t* out_base = in_base + (size_t)a.stages * a.in_stride;
    uint64_t* mbar = (uint64_t*)(out_base + kEncOutBufs * (size_t)a.out_stride);
    int32_t* badtag = (int32_t*)(mbar + kEncStages);
    b200flow_slot* plan_sh = (b200flow_slot*)(badtag + 2 * a.R + ((2 * a.R) & 1));   // keep 8-byte alignment
    int32_t* cat_tab = (int32_t*)(plan_sh + a.n_out);          // [3][kEncMaxCat + 1]: field offset, LUT offset, LUT length
    int32_t* rank_sh = cat_tab + 3 * (kEncMaxCat + 1);         // [R][kEncMaxCat]: StringIndexer rank per (row, categorical source)
    int16_t* slot_cat = (int16_t*)(rank_sh + a.R * kEncMaxCat);   // [n_out]: categorical source of a slot, -1 numeric, -2 inline
    int16_t* slot_rep = slot_cat + a.n_out + (a.n_out & 1);
    int32_t* lut_sh = (int32_t*)(slot_rep + a.n_out + (a.n_out & 1));
    __shared__ int sh_ncat;

    const int tid = threadIdx.x, bd = blockDim.x;
    const int R = a.R, n_out = a.n_out, row_bytes = a.row_bytes;
    const int64_t n_tiles = (a.n_rows + R - 1) / R;
    const uint32_t tile_in_bytes = (uint32_t)R * row_bytes;
    const uint32_t tile_out_bytes = (uint32_t)R * n_out * sizeof(OUT);

    if (tid == 0) {
        for (int s = 0; s < a.stages; ++s) mbar_init(&mbar[s], 1);
        fence_mbar_init();
    }
    for (int i = tid; i < n_out * (int)(sizeof(b200flow_slot) / 4); i += bd) ((uint32_t*)plan_sh)[i] = ((const uint32_t*)a.plan)[i];
    if (a.lut_in_smem) for (int i = tid; i < a.lut_total; i += bd) lut_sh[i] = a.lut[i];
    for (int i = tid; i < 2 * R; i += bd) badtag[i] = 0;
    __syncthreads();
    const int32_t* lut = a.lut_in_smem ? lut_sh : a.lut;
    // distinct categorical sources (field, LUT): the code -> rank lookup is done ONCE per (row, source) in a pre-pass, not
    // once per one-hot slot (70 slots share KDD's `service` lookup)
    for (int d = tid; d < n_out; d += bd) {
        int rep = -1;
        if (plan_sh[d].kind >= B200FLOW_SRC_INDEX) {
            rep = d;
            if (n_out <= 1024)
                for (int e = 0; e < d; ++e)
                    if (plan_sh[e].kind >= B200FLOW_SRC_INDEX && plan_sh[e].src_off == plan_sh[d].src_off &&
                        plan_sh[e].lut_off == plan_sh[d].lut_off && plan_sh[e].lut_len == plan_sh[d].lut_len) { rep = e; break; }
        }
        slot_rep[d] = (int16_t)rep;
    }
    __syncthreads();
    if (tid == 0) {
        int nc = 0;
        for (int d = 0; d < n_out; ++d) {
            int id = -1;
            if (slot_rep[d] == d) {
                if (nc < kEncMaxCat && n_out <= 1024) {
                    id = nc; cat_tab[nc] = plan_sh[d].src_off; cat_tab[(kEncMaxCat + 1) + nc] = plan_sh[d].lut_off;
                    cat_tab[2 * (kEncMaxCat + 1) + nc] = plan_sh[d].lut_len; ++nc;
                } else id = -2;
            }
            slot_cat[d] = (int16_t)id;
        }
        int n_cat_slots = 0;
        for (int d = 0; d < n_out; ++d) n_cat_slots += slot_rep[d] >= 0 ? 1 : 0;
        if (n_cat_slots < 3 * nc) {                          // few slots per source (plain StringIndexer columns): the shared
            nc = 0;                                          // pre-pass and its barrier cost more than the inline lookups
            for (int d = 0; d < n_out; ++d) if (slot_rep[d] >= 0) slot_cat[d] = -2;
        }
        if (a.label_off >= 0) {                              // the label column is one more source (index nc)
            cat_tab[nc] = a.label_off; cat_tab[(kEncMaxCat + 1) + nc] = a.label_lut_off; cat_tab[2 * (kEncMaxCat + 1) + nc] = a.label_lut_len;
        }
        sh_ncat = nc;
    }
    __syncthreads();
    for (int d = tid; d < n_out; d += bd) { const int rep = slot_rep[d]; if (rep >= 0 && rep != d) slot_cat[d] = slot_cat[rep]; }
    __syncthreads();
    const int ncat = sh_ncat, nsrc = ncat + (a.label_off >= 0 ? 1 : 0);

    auto issue_load = [&](int64_t tile, int s) {
        int64_t rows = a.n_rows - tile * R;
        if (rows >= R) {
            mbar_arrive_expect_tx(&mbar[s], tile_in_bytes);
            bulk_g2s(in_base + (size_t)s * a.in_stride, a.records + tile * (int64_t)tile_in_bytes, tile_in_bytes, &mbar[s]);
        } else {
            mbar_arrive(&mbar[s]);      // ragged last tile: loaded cooperatively below
        }
    };
    if (tid == 0)
        for (int s = 0; s < a.stages; ++s) {
            int64_t t = (int64_t)blockIdx.x + (int64_t)s * gridDim.x;
            if (t < n_tiles) issue_load(t, s);
        }

    // thread -> output slot mapping: one fixed slot per thread when n_out <= blockDim, rows fastest, so that the lanes of
    // a warp share their slot's source kind (no divergence between the numeric and the lookup loops)
    const bool fixed = n_out <= bd;
    const int rp = fixed ? bd / n_out : 1;
    const int d0 = fixed ? tid / rp : tid;
    const int r0 = fixed ? tid % rp : 0;
    const int dstep = fixed ? n_out : bd;
    const bool active = fixed ? (tid < rp * n_out) : true;

    b200flow_slot my_sl = plan_sh[0]; int my_cat = -2;
    if (fixed && active) { my_sl = plan_sh[d0]; my_cat = slot_cat[d0]; }

    int it = 0;
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, ++it) {
        const int s = it % a.stages, o = it % kEncOutBufs, ob = it & 1;
        const uint32_t ph = (uint32_t)(it / a.stages) & 1u;
        const int64_t row_base = tile * R;
        const int rows = (int)min((int64_t)R, a.n_rows - row_base);
        const bool full = rows == R;
        uint8_t* in_t = in_base + (size_t)s * a.in_stride;
        OUT* out_t = (OUT*)(out_base + (size_t)o * a.out_stride);
        int32_t* bad = badtag + ob * R;
        const int tag = it + 1;

        mbar_wait(&mbar[s], ph);
        if (!full) {
            const uint32_t* src = (const uint32_t*)(a.records + row_base * row_bytes);
            for (int i = tid; i < rows * row_bytes / 4; i += bd) ((uint32_t*)in_t)[i] = __ldg(src + i);
            __syncthreads();
        }

        if (nsrc > 0) {
            for (int idx = tid; idx < rows * nsrc; idx += bd) {
                const int r = idx / nsrc, c = idx - r * nsrc;
                const int code = *(const int32_t*)(in_t + r * row_bytes + cat_tab[c]);
                const int rank = (code >= 0 && code < cat_tab[2 * (kEncMaxCat + 1) + c]) ? lut[cat_tab[(kEncMaxCat + 1) + c] + code] : -1;
                if (rank < 0) bad[r] = tag;
                if (c < ncat) rank_sh[r * kEncMaxCat + c] = rank;
                else if (a.label_out) a.label_out[row_base + r] = rank;
            }
            if (ncat > 0) __syncthreads();          // ranks visible to the slot loops (label-only: nothing to wait for)
        }
        if (active) {
            // one tight loop per source kind: the slot (and so the kind) is fixed per thread, rows are strided by rp; with one slot
            // per thread (n_out <= blockDim) its descriptor lives in registers, loaded once before the tile loop
            for (int d = d0; d < n_out; d += dstep) {
                b200flow_slot sl = my_sl; int cat = my_cat;
                if (!fixed) { sl = plan_sh[d]; cat = slot_cat[d]; }
                const uint8_t* p = in_t + r0 * row_bytes + sl.src_off;
                OUT* op = out_t + r0 * n_out + d;
                const int pstep = rp * row_bytes, ostep = rp * n_out;
                const bool ident = sl.mean == 0.0 && sl.scale == 1.0;
                const double mean = sl.mean, scale = sl.scale;
                if (sl.kind == B200FLOW_SRC_F32) {
                    if (ident && sizeof(OUT) == 4 && !a.check_nan) {
#pragma unroll 4
                        for (int r = r0; r < rows; r += rp, p += pstep, op += ostep) *(uint32_t*)op = *(const uint32_t*)p;   // assemble = move
                    } else {
#pragma unroll 4
                        for (int r = r0; r < rows; r += rp, p += pstep, op += ostep) {
                            const double v = (double)(*(const float*)p);
                            if (a.check_nan && v != v) bad[r] = tag;
                            *op = ident ? (OUT)v : (OUT)((v - mean) * scale);
                        }
                    }
                } else if (sl.kind == B200FLOW_SRC_F64) {
#pragma unroll 4
                    for (int r = r0; r < rows; r += rp, p += pstep, op += ostep) {
                        const uint32_t* q = (const uint32_t*)p;              // 4-byte aligned reads: fields need not be 8-aligned
                        const double v = __hiloint2double((int)q[1], (int)q[0]);
                        if (a.check_nan && v != v) bad[r] = tag;
                        *op = ident ? (OUT)v : (OUT)((v - mean) * scale);
                    }
                } else if (sl.kind == B200FLOW_SRC_I32) {
#pragma unroll 4
                    for (int r = r0; r < rows; r += rp, p += pstep, op += ostep) {
                        const double v = (double)(*(const int32_t*)p);
                        *op = ident ? (OUT)v : (OUT)((v - mean) * scale);
                    }
                } else {
                    const bool index = sl.kind == B200FLOW_SRC_INDEX;
                    const OUT hot = (OUT)((1.0 - mean) * scale), cold = (OUT)((0.0 - mean) * scale);
                    if (cat >= 0) {                  // rank looked up once per (row, source) by the pre-pass
                        const int32_t* rk = rank_sh + r0 * kEncMaxCat + cat;
                        const int rstep = rp * kEncMaxCat;
                        if (index) {
#pragma unroll 4
                            for (int r = r0; r < rows; r += rp, rk += rstep, op += ostep) *op = (OUT)(((double)*rk - mean) * scale);
                        } else {
                            const int hotrank = sl.hot;
#pragma unroll 4
                            for (int r = r0; r < rows; r += rp, rk += rstep, op += ostep) *op = (*rk == hotrank) ? hot : cold;
                        }
                    } else {                         // more than kEncMaxCat distinct sources: inline lookup
                        const int32_t* lt = lut + sl.lut_off;
                        for (int r = r0; r < rows; r += rp, p += pstep, op += ostep) {
                            const int code = *(const int32_t*)p;
                            const int rank = (code >= 0 && code < sl.lut_len) ? lt[code] : -1;
                            if (rank < 0) bad[r] = tag;
                            *op = index ? (OUT)(((double)rank - mean) * scale) : (rank == sl.hot ? hot : cold);
                        }
                    }
                }
            }
        }
        if (tid == 0) bulk_wait_read<1>();           // all but the latest store have drained: the next tile's out buffer is free
        fence_proxy_async();
        __syncthreads();                            // the only barrier per tile: tile computed, input stage s consumed
        if (tid == 0) {
            if (full) { bulk_s2g((OUT*)a.out + row_base * n_out, out_t, tile_out_bytes); bulk_commit(); }
            int64_t next = tile + (int64_t)a.stages * gridDim.x;
            if (next < n_tiles) issue_load(next, s);
        }
        if (!full) {
            OUT* dst = (OUT*)a.out + row_base * n_out;
            for (int i = tid; i < rows * n_out; i += bd) dst[i] = out_t[i];
        }
        if (a.valid_out) for (int r = tid; r < rows; r += bd) a.valid_out[row_base + r] = (bad[r] != tag) ? 1 : 0;
    }
    if (tid == 0) bulk_wait_all<0>();
}

// ------------------------------------------------------------------ fused encode -> TreePoint bins (R2+R3 feeding R5)
// The tree trainer never needs the dense feature matrix: it needs TreePoint bins.  These two kernels go from the raw AoS
// records straight to (a) the findSplits row sample and (b) the binned uint8 records, evaluating every slot of the encode
// plan in fp64 exactly like encode_kernel does (SURVEY.md 8d "Encode -> bins": KDD 168 + 41 + 1 = 210 B/row instead of
// writing, compacting and re-reading a 164 B/row f32 matrix).
__device__ __forceinline__ double slot_value(const uint8_t* row, const b200flow_slot& sl, const int32_t* __restrict__ lut,
                                             int round_f32, bool* invalid, bool* is_nan) {
    double v;
    if (sl.kind == B200FLOW_SRC_F32) { v = (double)(*(const float*)(row + sl.src_off)); *is_nan = v != v; }
    else if (sl.kind == B200FLOW_SRC_F64) { const uint32_t* q = (const uint32_t*)(row + sl.src_off); v = __hiloint2double((int)q[1], (int)q[0]); *is_nan = v != v; }
    else if (sl.kind == B200FLOW_SRC_I32) v = (double)(*(const int32_t*)(row + sl.src_off));
    else {
        const int code = *(const int32_t*)(row + sl.src_off);
        const int rank = (code >= 0 && code < sl.lut_len) ? lut[sl.lut_off + code] : -1;
        if (rank < 0) *invalid = true;
        v = sl.kind == B200FLOW_SRC_INDEX ? (double)rank : (rank == sl.hot ? 1.0 : 0.0);
    }
    if (!(sl.mean == 0.0 && sl.scale == 1.0)) v = (v - sl.mean) * sl.scale;
    if (round_f32) v = (double)(float)v;                   // the value an f32 feature matrix would have held
    return v;
}

// R4 on raw records: Bernoulli row sample keyed by the GLOBAL row, every sampled row encoded through the plan
__global__ void __launch_bounds__(256) sample_records_kernel(const uint8_t* __restrict__ rec, int64_t n, int row_bytes,
                                                             const b200flow_slot* __restrict__ plan, int F,
                                                             const int32_t* __restrict__ lut, int round_f32, uint64_t seed,
                                                             uint64_t keep_thr, int64_t row_offset, double* sample, int64_t cap,
                                                             int32_t* n_sampled) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const uint64_t g = (uint64_t)(row_offset + i);
        const uint4 r = philox_keyed(seed, PURPOSE_SAMPLE, (uint32_t)g, (uint32_t)(g >> 32), 0u, 0u);
        if ((uint64_t)r.x < keep_thr) {
            const int slot = atomicAdd(n_sampled, 1);
            if (slot < cap) {
                const uint8_t* row = rec + i * row_bytes;
                for (int f = 0; f < F; ++f) {
                    bool inv = false, nan = false;
                    const b200flow_slot sl = plan[f];
                    sample[(int64_t)f * cap + slot] = slot_value(row, sl, lut, round_f32, &inv, &nan);
                }
            }
        }
    }
}

struct EncodeBinsArgs {
    const uint8_t* records; int64_t n_rows; int row_bytes;
    const b200flow_slot* plan; int F;
    const int32_t* lut; int lut_total; int lut_in_smem;
    int label_off, label_lut_off, label_lut_len, check_nan, round_f32;
    const double* thresholds; const int32_t* n_thr; const int32_t* arity; int max_bins; int thr_in_smem;
    uint8_t* tp; int stride; int32_t* label_out; int32_t* bad;    // bad[0]: categorical cells outside [0, arity); bad[1]: NaN cells + unseen codes
    int R; int in_stride;
};

constexpr int kBinMaxThreads = 512;

// Persistent CTAs; per tile of R = 32 * RPL records (one TMA bulk load, 3-deep ring): a WARP owns a feature for the whole
// tile, so the slot descriptor, the arity and the threshold array are warp-uniform — the first steps of the search hit one
// or two shared-memory words per step (broadcast) instead of 32 different arrays — and trip counts do not diverge; every lane
// runs RPL independent searches side by side (ILP hides the dependent shared-memory loads).
// lower_bound (first b with v <= thr[b]) is the branch-free power-of-two descent  pos += st  while  !(v <= thr[pos + st - 1]):
// four instructions per step.  TT = float when every continuous value is exactly a float (f32 fields, identity scaling, or
// an f32 feature matrix being emulated): thresholds are rounded DOWN to float once, and  v <= thr  <=>  v <= rd(thr)  for
// every float v — the same bins as the fp64 compare, at half the shared-memory bytes; TT = double otherwise.
// Bins land in a padded byte tile (row pitch = stride + 4 bytes: conflict-free byte stores across rows), which the whole CTA
// then streams out as 16-byte words; the tile is double-buffered, so there is ONE barrier per tile.
template <int RPL, typename TT>
__global__ void __launch_bounds__(kBinMaxThreads) encode_bins_kernel(const EncodeBinsArgs a) {
    extern __shared__ __align__(128) uint8_t smem[];
    constexpr int R = 32 * RPL;
    const int tid = threadIdx.x, bd = blockDim.x, lane = lane_id(), wid = warp_id(), nw = bd / 32;
    const int F = a.F, row_bytes = a.row_bytes, ns = a.max_bins - 1, stride = a.stride, pitch = stride + 4;
    uint8_t* in_base = smem;
    uint8_t* out_base = in_base + (size_t)kEncStages * a.in_stride;                 // [2][R][pitch]
    uint64_t* mbar = (uint64_t*)(out_base + (((size_t)2 * R * pitch + 7) & ~(size_t)7));
    b200flow_slot* plan_sh = (b200flow_slot*)(mbar + kEncStages);
    int32_t* nthr_sh = (int32_t*)(plan_sh + F);
    int32_t* arity_sh = nthr_sh + F;
    int32_t* lut_sh = arity_sh + F;
    // (offset arithmetic on the shared window keeps the address space: a pointer rebuilt from a uintptr_t makes every search load generic)
    TT* thr_sh = (TT*)(smem + (((size_t)((const uint8_t*)(lut_sh + (a.lut_in_smem ? a.lut_total : 0)) - smem) + 7) & ~(size_t)7));
    const int64_t n_tiles = (a.n_rows + R - 1) / R;
    const uint32_t tile_in_bytes = (uint32_t)R * row_bytes;

    if (tid == 0) {
        for (int s = 0; s < kEncStages; ++s) mbar_init(&mbar[s], 1);
        fence_mbar_init();
    }
    for (int i = tid; i < F * (int)(sizeof(b200flow_slot) / 4); i += bd) ((uint32_t*)plan_sh)[i] = ((const uint32_t*)a.plan)[i];
    for (int i = tid; i < F; i += bd) { nthr_sh[i] = a.n_thr[i]; arity_sh[i] = a.arity[i]; }
    if (a.lut_in_smem) for (int i = tid; i < a.lut_total; i += bd) lut_sh[i] = a.lut[i];
    if (a.thr_in_smem)
        for (int i = tid; i < F * ns; i += bd) {
            if (sizeof(TT) == 4) ((float*)thr_sh)[i] = __double2float_rd(a.thresholds[i]);
            else ((double*)thr_sh)[i] = a.thresholds[i];
        }
    for (int i = tid; i < 2 * R * pitch / 4; i += bd) ((uint32_t*)out_base)[i] = 0;      // pad bytes stay zero for ever
    __syncthreads();
    const int32_t* lut = a.lut_in_smem ? lut_sh : a.lut;

    auto issue_load = [&](int64_t tile, int s) {
        if (a.n_rows - tile * R >= R) {
            mbar_arrive_expect_tx(&mbar[s], tile_in_bytes);
            bulk_g2s(in_base + (size_t)s * a.in_stride, a.records + tile * (int64_t)tile_in_bytes, tile_in_bytes, &mbar[s]);
        } else mbar_arrive(&mbar[s]);                       // ragged last tile: loaded cooperatively below
    };
    if (tid == 0)
        for (int s = 0; s < kEncStages; ++s) {
            const int64_t t = (int64_t)blockIdx.x + (int64_t)s * gridDim.x;
            if (t < n_tiles) issue_load(t, s);
        }
    int n_bad = 0, n_inv = 0;
    int it = 0;
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, ++it) {
        const int s = it % kEncStages;
        const uint32_t ph = (uint32_t)(it / kEncStages) & 1u;
        const int64_t row_base = tile * R;
        const int rows = (int)min((int64_t)R, a.n_rows - row_base);
        uint8_t* in_t = in_base + (size_t)s * a.in_stride;
        uint8_t* out_t = out_base + (size_t)(it & 1) * R * pitch;
        mbar_wait(&mbar[s], ph);
        if (rows < R) {
            const uint32_t* src = (const uint32_t*)(a.records + row_base * row_bytes);
            for (int i = tid; i < rows * row_bytes / 4; i += bd) ((uint32_t*)in_t)[i] = __ldg(src + i);
            for (int i = rows * row_bytes / 4 + tid; i < R * row_bytes / 4; i += bd) ((uint32_t*)in_t)[i] = 0;   // rows past the end: defined, never stored
            __syncthreads();
        }
        for (int f = wid; f <= F; f += nw) {                // task F = the label column
            if (f == F) {
                if (a.label_off < 0) continue;
#pragma unroll
                for (int q = 0; q < RPL; ++q) {
                    const int r = lane + 32 * q;
                    if (r >= rows) continue;
                    const int code = *(const int32_t*)(in_t + r * row_bytes + a.label_off);
                    const int rank = (code >= 0 && code < a.label_lut_len) ? lut[a.label_lut_off + code] : -1;
                    if (rank < 0) ++n_inv;
                    out_t[r * pitch + F] = (uint8_t)rank;
                    if (a.label_out) a.label_out[row_base + r] = rank;
                }
                continue;
            }
            const b200flow_slot sl = plan_sh[f];
            const int ar = arity_sh[f], nt = nthr_sh[f];
            int b[RPL];
            if (ar > 0 || sizeof(TT) == 8 || sl.kind != B200FLOW_SRC_F32) {
                double v[RPL];
#pragma unroll
                for (int q = 0; q < RPL; ++q) {
                    bool inv = false, nan = false;
                    const int r = lane + 32 * q;
                    v[q] = slot_value(in_t + r * row_bytes, sl, lut, a.round_f32, &inv, &nan);
                    if (r < rows && (inv || (a.check_nan && nan))) ++n_inv;
                }
                if (ar > 0) {
#pragma unroll
                    for (int q = 0; q < RPL; ++q) {
                        b[q] = (int)v[q];
                        if (!((double)b[q] == v[q]) || b[q] < 0 || b[q] >= ar) { b[q] = ar < 255 ? ar : 255; if (lane + 32 * q < rows) ++n_bad; }   // bin `arity` is no category (arity <= 255, build_metadata): never inside a left-set mask
                    }
                } else {
#pragma unroll
                    for (int q = 0; q < RPL; ++q) b[q] = 0;
                    if (sizeof(TT) == 8) {
                        if (a.thr_in_smem) {                // table (+ padding) in shared memory: unconditional load, predicated add
                            const double* thr = (const double*)thr_sh + f * ns;
                            for (int st = nt > 0 ? 1 << (31 - __clz(nt)) : 0; st > 0; st >>= 1) {
#pragma unroll
                                for (int q = 0; q < RPL; ++q) { const int i = b[q] + st - 1; const double t = thr[i]; b[q] += (i < nt && !(v[q] <= t)) ? st : 0; }
                            }
                        } else {
                            const double* thr = a.thresholds + (int64_t)f * ns;
                            for (int st = nt > 0 ? 1 << (31 - __clz(nt)) : 0; st > 0; st >>= 1) {
#pragma unroll
                                for (int q = 0; q < RPL; ++q) { const int i = b[q] + st - 1; if (i < nt && !(v[q] <= thr[i])) b[q] += st; }
                            }
                        }
                    } else {                                // float table, non-f32 source whose value an f32 matrix would have held
                        const float* thr = (const float*)thr_sh + f * ns;
                        for (int st = nt > 0 ? 1 << (31 - __clz(nt)) : 0; st > 0; st >>= 1) {
#pragma unroll
                            for (int q = 0; q < RPL; ++q) { const int i = b[q] + st - 1; const float t = thr[i]; b[q] += (i < nt && !((float)v[q] <= t)) ? st : 0; }
                        }
                    }
                }
            } else {                                        // f32 field, float thresholds: no fp64 at all
                const float* thr = (const float*)thr_sh + f * ns;
                const bool ident = sl.mean == 0.0 && sl.scale == 1.0;
                float v[RPL];
#pragma unroll
                for (int q = 0; q < RPL; ++q) {
                    const int r = lane + 32 * q;
                    v[q] = *(const float*)(in_t + r * row_bytes + sl.src_off);
                    if (a.check_nan && r < rows && v[q] != v[q]) ++n_inv;
                    if (!ident) v[q] = (float)(((double)v[q] - sl.mean) * sl.scale);      // round_f32 mode: the f32 matrix value
                    b[q] = 0;
                }
                for (int st = nt > 0 ? 1 << (31 - __clz(nt)) : 0; st > 0; st >>= 1) {     // the padded table makes the load unconditional
#pragma unroll
                    for (int q = 0; q < RPL; ++q) { const int i = b[q] + st - 1; const float t = thr[i]; b[q] += (i < nt && !(v[q] <= t)) ? st : 0; }
                }
            }
#pragma unroll
            for (int q = 0; q < RPL; ++q) out_t[(lane + 32 * q) * pitch + f] = (uint8_t)b[q];
        }
        __syncthreads();                                    // tile binned; input stage s consumed
        if (tid == 0) { const int64_t next = tile + (int64_t)kEncStages * gridDim.x; if (next < n_tiles) issue_load(next, s); }
        const int q16 = stride / 16;
        uint4* dst = (uint4*)(a.tp + row_base * stride);
        for (int i = tid; i < rows * q16; i += bd) {
            const int r = i / q16, q = i - r * q16;
            const uint32_t* w = (const uint32_t*)(out_t + r * pitch + q * 16);
            st_stream_u4(dst + i, make_uint4(w[0], w[1], w[2], w[3]));
        }
    }
    n_bad = warp_sum(n_bad); n_inv = warp_sum(n_inv);
    if (lane == 0) { if (n_bad) atomicAdd(&a.bad[0], n_bad); if (n_inv) atomicAdd(&a.bad[1], n_inv); }
}

// ------------------------------------------------------------------ R3c column moments
template <typename T>
__global__ void __launch_bounds__(256) column_moments_kernel(const T* __restrict__ x, int64_t n, int D, int64_t ld,
                                                             const double* __restrict__ shift, double* sum, double* sumsq) {
    extern __shared__ double sh_m[];     // [2][blockDim]
    const int tid = threadIdx.x, bd = blockDim.x;
    const int64_t rows_per_block = (n + gridDim.x - 1) / gridDim.x;
    const int64_t rb = (int64_t)blockIdx.x * rows_per_block, re = min(n, rb + rows_per_block);
    for (int dbase = 0; dbase < D; dbase += bd) {
        const int dn = min(bd, D - dbase);
        const int rp = bd / dn;
        double s = 0.0, q = 0.0;
        if (tid < rp * dn) {
            const int d = dbase + tid % dn;
            const double sft = shift ? shift[d] : 0.0;
            for (int64_t r = rb + tid / dn; r < re; r += rp) {
                double v = (double)x[r * ld + d] - sft;
                s += v; q += v * v;
            }
        }
        sh_m[tid] = s; sh_m[bd + tid] = q;
        __syncthreads();
        if (tid < dn) {
            for (int k = 1; k < rp; ++k) { s += sh_m[tid + k * dn]; q += sh_m[bd + tid + k * dn]; }
            atomicAdd(&sum[dbase + tid], s);
            atomicAdd(&sumsq[dbase + tid], q);
        }
        __syncthreads();
    }
}

}  // namespace b200flow

using namespace b200flow;

extern "C" int b200flow_category_counts(const void* records, int64_t n_rows, int32_t row_bytes, int32_t src_off,
                                        int32_t K, int64_t* counts, void* stream) {
    if (n_rows <= 0) return B200FLOW_OK;            // empty batch: nothing to do (pointers may be NULL)
    B2F_REQUIRE(records && counts && K > 0 && row_bytes >= 4 && src_off >= 0 && src_off + 4 <= row_bytes && (src_off & 3) == 0 &&
                    (row_bytes & 3) == 0, "category_counts: bad arguments");
    int use_smem = K <= 8192;
    int grid = grid_for(n_rows, 256 * 8, kNumSMs * 8);
    category_counts_kernel<<<grid, 256, use_smem ? K * 4 : 0, (cudaStream_t)stream>>>(
        (const uint8_t*)records, n_rows, row_bytes, src_off, K, (unsigned long long*)counts, use_smem);
    return check_launch("category_counts");
}

extern "C" int b200flow_category_counts_multi(const void* records, int64_t n_rows, int32_t row_bytes, int32_t n_cols,
                                              const int32_t* src_offs_host, const int32_t* Ks_host, int64_t* counts, void* stream) {
    if (n_rows <= 0) return B200FLOW_OK;
    B2F_REQUIRE(records && counts && src_offs_host && Ks_host && n_cols >= 1 && n_cols <= 8 && row_bytes >= 4 && (row_bytes & 3) == 0,
                "category_counts_multi: bad arguments");
    CountCols cc; cc.n = n_cols;
    int total = 0;
    for (int c = 0; c < 8; ++c) {
        cc.off[c] = c < n_cols ? src_offs_host[c] : 0; cc.K[c] = c < n_cols ? Ks_host[c] : 0; cc.base[c] = total;
        if (c < n_cols) {
            B2F_REQUIRE(cc.K[c] > 0 && cc.off[c] >= 0 && cc.off[c] + 4 <= row_bytes && (cc.off[c] & 3) == 0, "category_counts_multi: bad column %d", c);
            total += cc.K[c];
        }
    }
    B2F_REQUIRE(total <= 8192, "category_counts_multi: more than 8192 categories in total (count the columns one by one)");
    int grid = grid_for(n_rows, 256 * 8, kNumSMs * 8);
    category_counts_multi_kernel<<<grid, 256, total * 4, (cudaStream_t)stream>>>((const uint8_t*)records, n_rows, row_bytes, cc, total,
                                                                                (unsigned long long*)counts);
    return check_launch("category_counts_multi");
}

extern "C" int b200flow_encode(const void* records, int64_t n_rows, int32_t row_bytes, const b200flow_slot* plan,
                               int32_t n_out, const int32_t* lut, int32_t lut_total, int32_t label_off,
                               int32_t label_lut_off, int32_t label_lut_len, int32_t check_nan, void* out,
                               int32_t out_dtype, int32_t* label_out, uint8_t* valid_out, void* stream) {
    if (n_rows <= 0) return B200FLOW_OK;            // empty batch: nothing to do (pointers may be NULL)
    B2F_REQUIRE(records && plan && out, "encode: null pointer");
    B2F_REQUIRE(n_out > 0 && n_out <= 4096 && row_bytes >= 4 && (row_bytes & 3) == 0, "encode: bad n_out/row_bytes");
    B2F_REQUIRE(out_dtype == B200FLOW_F32 || out_dtype == B200FLOW_F64, "encode: bad out_dtype");
    B2F_REQUIRE(((uintptr_t)records & 15) == 0 && ((uintptr_t)out & 15) == 0, "encode: records/out must be 16-byte aligned");
    B2F_REQUIRE(label_off < 0 || (label_off + 4 <= row_bytes && (label_off & 3) == 0 && lut), "encode: bad label_off");
    const int osz = out_dtype == B200FLOW_F32 ? 4 : 8;
    EncodeArgs a;
    a.records = (const uint8_t*)records; a.n_rows = n_rows; a.row_bytes = row_bytes; a.plan = plan; a.n_out = n_out;
    a.lut = lut; a.lut_total = lut ? lut_total : 0; a.lut_in_smem = (lut && lut_total > 0 && lut_total <= 4096) ? 1 : 0;
    a.label_off = label_off; a.label_lut_off = label_lut_off; a.label_lut_len = label_lut_len; a.check_nan = check_nan;
    a.out = out; a.label_out = label_out; a.valid_out = valid_out;
    // tile rows: keep one CTA near 52 KB of smem so four CTAs share an SM (>= 64 KB of loads in flight per SM)
    const int fixed_bytes = kEncStages * 8 + n_out * (int)sizeof(b200flow_slot) + (a.lut_in_smem ? a.lut_total * 4 : 0) + 1024 +
                            3 * (kEncMaxCat + 1) * 4 + 4 * (n_out + 1);
    static int stages = -1;                                // tuning knob: depth of the TMA load ring
    if (stages < 0) { const char* e = getenv("B200FLOW_ENC_STAGES"); stages = (e && atoi(e) == 2) ? 2 : 3; }
    a.stages = stages;
    const int per_row = row_bytes * stages + n_out * osz * kEncOutBufs + 8 + kEncMaxCat * 4;
    static int budget_kb = -1;                             // tuning knob: per-CTA shared memory target
    if (budget_kb < 0) { const char* e = getenv("B200FLOW_ENC_SMEM_KB"); budget_kb = e ? atoi(e) : 52; }
    int budget = budget_kb * 1024 - fixed_bytes;
    int R = budget > 0 ? budget / per_row : 0;
    if (R < 4) R = 4;                    // very wide rows: fewer CTAs per SM
    if (R > 512) R = 512;
    R &= ~3;
    if ((int64_t)R > ((n_rows + 3) & ~(int64_t)3)) R = (int)((n_rows + 3) & ~(int64_t)3);
    a.R = R;
    a.in_stride = (R * row_bytes + 127) & ~127;
    a.out_stride = (R * n_out * osz + 127) & ~127;
    size_t smem = (size_t)stages * a.in_stride + kEncOutBufs * (size_t)a.out_stride + kEncStages * 8 + (2 * R + 2) * 4 +
                  (size_t)n_out * sizeof(b200flow_slot) + (a.lut_in_smem ? (size_t)a.lut_total * 4 : 0) + 16 +
                  3 * (kEncMaxCat + 1) * 4 + (size_t)R * kEncMaxCat * 4 + 4 * ((size_t)n_out + 1);
    // the kernel's static shared memory (sh_ncat, padded to the 128-byte alignment of the dynamic window) counts against the
    // same 227 KB per block: without it the widest plans passed this check and failed in cudaFuncSetAttribute instead
    cudaFuncAttributes fa;
    cudaError_t e = cudaFuncGetAttributes(&fa, out_dtype == B200FLOW_F32 ? (const void*)encode_kernel<float> : (const void*)encode_kernel<double>);
    if (e != cudaSuccess) { cudaGetLastError(); set_error("encode: cudaFuncGetAttributes: %s", cudaGetErrorString(e)); return B200FLOW_ERR_CUDA; }
    B2F_REQUIRE(smem + fa.sharedSizeBytes <= 227 * 1024, "encode: record too wide for shared memory (row_bytes=%d n_out=%d)", row_bytes, n_out);
    const int64_t n_tiles = (n_rows + R - 1) / R;
    int ctas_per_sm = (int)((220 * 1024) / (smem + 1024));
    if (ctas_per_sm < 1) ctas_per_sm = 1;
    if (ctas_per_sm > 8) ctas_per_sm = 8;
    int grid = (int)(n_tiles < (int64_t)kNumSMs * ctas_per_sm ? n_tiles : (int64_t)kNumSMs * ctas_per_sm);
    if (out_dtype == B200FLOW_F32) {
        e = cudaFuncSetAttribute(encode_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e == cudaSuccess) encode_kernel<float><<<grid, kEncThreads, smem, (cudaStream_t)stream>>>(a);
    } else {
        e = cudaFuncSetAttribute(encode_kernel<double>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e == cudaSuccess) encode_kernel<double><<<grid, kEncThreads, smem, (cudaStream_t)stream>>>(a);
    }
    if (e != cudaSuccess) {               // clear the error too: left pending, the next unrelated CUDA call would report it
        cudaGetLastError(); set_error("encode: cudaFuncSetAttribute: %s", cudaGetErrorString(e)); return B200FLOW_ERR_CUDA;
    }
    return check_launch("encode");
}

extern "C" int b200flow_column_moments(const void* x, int32_t dtype, int64_t n_rows, int32_t D, int64_t ld,
                                       const double* shift, double* sum, double* sumsq, void* stream) {
    if (n_rows <= 0) return B200FLOW_OK;            // empty batch: nothing to do (pointers may be NULL)
    B2F_REQUIRE(x && sum && sumsq && D > 0 && ld >= D, "column_moments: bad arguments");
    B2F_REQUIRE(dtype == B200FLOW_F32 || dtype == B200FLOW_F64, "column_moments: bad dtype");
    int grid = grid_for(n_rows, 256, kNumSMs * 4);
    size_t smem = 2 * 256 * sizeof(double);
    if (dtype == B200FLOW_F32)
        column_moments_kernel<float><<<grid, 256, smem, (cudaStream_t)stream>>>((const float*)x, n_rows, D, ld, shift, sum, sumsq);
    else
        column_moments_kernel<double><<<grid, 256, smem, (cudaStream_t)stream>>>((const double*)x, n_rows, D, ld, shift, sum, sumsq);
    return check_launch("column_moments");
}

extern "C" int b200flow_sample_records(const void* records, int64_t n_rows, int32_t row_bytes, const b200flow_slot* plan, int32_t F,
                                       const int32_t* lut, int32_t round_f32, uint64_t seed, uint64_t keep_threshold,
                                       int64_t row_offset, double* sample, int64_t cap, int32_t* n_sampled, void* stream) {
    if (n_rows <= 0) return B200FLOW_OK;
    B2F_REQUIRE(records && plan && sample && n_sampled && F > 0 && cap > 0 && row_bytes >= 4 && (row_bytes & 3) == 0, "sample_records: bad arguments");
    const int grid = grid_for(n_rows, 256 * 4, kNumSMs * 8);
    sample_records_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>((const uint8_t*)records, n_rows, row_bytes, plan, F, lut, round_f32, seed,
                                                                 keep_threshold, row_offset, sample, cap, n_sampled);
    return check_launch("sample_records");
}

extern "C" int b200flow_encode_bins(const void* records, int64_t n_rows, int32_t row_bytes, const b200flow_slot* plan, int32_t F,
                                    const int32_t* lut, int32_t lut_total, int32_t label_off, int32_t label_lut_off,
                                    int32_t label_lut_len, int32_t check_nan, int32_t round_f32, int32_t thr_f32, const double* thresholds,
                                    const int32_t* n_thr, const int32_t* arity, int32_t max_bins, uint8_t* tp, int32_t tp_stride,
                                    int32_t* label_out, int32_t* bad, void* stream) {
    if (n_rows <= 0) return B200FLOW_OK;
    B2F_REQUIRE(records && plan && thresholds && n_thr && arity && tp && bad, "encode_bins: null pointer");
    B2F_REQUIRE(F > 0 && F < 4096 && row_bytes >= 4 && (row_bytes & 3) == 0 && max_bins >= 2 && max_bins <= 256, "encode_bins: bad shape");
    B2F_REQUIRE(tp_stride >= F + 1 && (tp_stride & 15) == 0 && ((uintptr_t)tp & 15) == 0 && ((uintptr_t)records & 15) == 0,
                "encode_bins: records/tp must be 16-byte aligned, tp_stride a multiple of 16 >= F + 1");
    B2F_REQUIRE(label_off < 0 || (label_off + 4 <= row_bytes && (label_off & 3) == 0 && lut), "encode_bins: bad label_off");
    EncodeBinsArgs a;
    a.records = (const uint8_t*)records; a.n_rows = n_rows; a.row_bytes = row_bytes; a.plan = plan; a.F = F;
    a.lut = lut; a.lut_total = lut ? lut_total : 0; a.lut_in_smem = (lut && lut_total > 0 && lut_total <= 4096) ? 1 : 0;
    a.label_off = label_off; a.label_lut_off = label_lut_off; a.label_lut_len = label_lut_len; a.check_nan = check_nan; a.round_f32 = round_f32;
    a.thresholds = thresholds; a.n_thr = n_thr; a.arity = arity; a.max_bins = max_bins;
    const size_t thr_bytes = (size_t)F * (max_bins - 1) * 8;
    a.tp = tp; a.stride = tp_stride; a.label_out = label_out; a.bad = bad;
    // float thresholds when every continuous value is exactly a float: f32 fields with identity scaling, or the f32 feature
    // matrix being emulated (round_f32); the plan is a HOST-side fact of the caller, passed as thr_f32
    const bool f32_table = thr_f32 != 0;
    const size_t thr_smem = ((size_t)F * (max_bins - 1) + 256) * (f32_table ? 4 : 8);   // + 256 entries: the branch-free descent may read (never use) past a row
    a.thr_in_smem = (f32_table || thr_smem <= 56 * 1024) ? 1 : 0;   // a double table beyond that stays in global memory (L1 keeps the top levels)
    B2F_REQUIRE(!f32_table || thr_smem <= 100 * 1024, "encode_bins: float threshold table exceeds shared memory");
    const size_t fixed_bytes = kEncStages * 8 + (size_t)F * sizeof(b200flow_slot) + 8 * (size_t)F + (a.lut_in_smem ? (size_t)a.lut_total * 4 : 0) + 16 +
                               (a.thr_in_smem ? thr_smem : 0) + 256;
    const size_t per_row = (size_t)row_bytes * kEncStages + 2 * (size_t)(tp_stride + 4);
    static int budget_kb = -1;                             // tuning knob: per-CTA shared memory target (2 CTAs per SM at ~110 KB)
    if (budget_kb < 0) { const char* e = getenv("B200FLOW_BINS_SMEM_KB"); budget_kb = e ? atoi(e) : 110; }
    B2F_REQUIRE(fixed_bytes + 32 * per_row <= 224 * 1024, "encode_bins: record too wide for shared memory (row_bytes=%d F=%d)", row_bytes, F);
    int rpl = 4;                                            // rows per lane: the most that fits the budget
    while (rpl > 1 && fixed_bytes + (size_t)32 * rpl * per_row > (size_t)budget_kb * 1024) rpl >>= 1;
    const int R = 32 * rpl;
    a.R = R;
    a.in_stride = (R * row_bytes + 127) & ~127;
    const size_t smem = (size_t)kEncStages * a.in_stride + (((size_t)2 * R * (tp_stride + 4) + 7) & ~(size_t)7) + fixed_bytes;
    B2F_REQUIRE(smem <= 227 * 1024, "encode_bins: shared memory budget exceeded");
    // warps per CTA: F + 1 warp tasks per tile (one per feature + the label); take the count in 12..16 that leaves the fewest idle
    int nw = 16, best_idle = 1 << 30;
    for (int w = 16; w >= 12; --w) { const int idle = (F + 1 + w - 1) / w * w - (F + 1); if (idle < best_idle) { best_idle = idle; nw = w; } }
    const int64_t n_tiles = (n_rows + R - 1) / R;
    int ctas_per_sm = (int)((227 * 1024) / (smem + 1024));
    if (ctas_per_sm < 1) ctas_per_sm = 1;
    if (ctas_per_sm > 4) ctas_per_sm = 4;                   // 2048 threads per SM
    const int grid = (int)(n_tiles < (int64_t)kNumSMs * ctas_per_sm ? n_tiles : (int64_t)kNumSMs * ctas_per_sm);
    cudaError_t e;
#define B2F_BINS_LAUNCH(RPL, TT)                                                                                          \
    e = cudaFuncSetAttribute(encode_bins_kernel<RPL, TT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);        \
    if (e == cudaSuccess) encode_bins_kernel<RPL, TT><<<grid, nw * 32, smem, (cudaStream_t)stream>>>(a);
    if (f32_table) { if (rpl == 4) { B2F_BINS_LAUNCH(4, float) } else if (rpl == 2) { B2F_BINS_LAUNCH(2, float) } else { B2F_BINS_LAUNCH(1, float) } }
    else { if (rpl == 4) { B2F_BINS_LAUNCH(4, double) } else if (rpl == 2) { B2F_BINS_LAUNCH(2, double) } else { B2F_BINS_LAUNCH(1, double) } }
#undef B2F_BINS_LAUNCH
    if (e != cudaSuccess) { set_error("encode_bins: cudaFuncSetAttribute: %s", cudaGetErrorString(e)); return B200FLOW_ERR_CUDA; }
    return check_launch("encode_bins");
}
