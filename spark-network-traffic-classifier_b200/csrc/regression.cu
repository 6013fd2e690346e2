// regression.cu — DecisionTreeRegressor / RandomForestRegressor and RegressionEvaluator on the device, DESIGN.md §5l: what
// the variance-tree kernels of gbt.cu do not do.
//
// Trainer.  Real labels go on the fixed-point grid of gbt.cu with a scale taken from the data: y' = y 2^-E (|y'| <= 1, an
// exact scaling), q = rint(y' 2^S), q2 = rint((q 2^-S)^2 2^S2).  b200flow_reg_labels checks the labels, finds max |y| and
// writes each row's label bits into the spare bytes of its TreePoint record, so that de-duplication keys on (bins, label);
// b200flow_reg_tree_weights gives each tree's total bag weight (the bound behind S and S2); b200flow_reg_grid puts every
// unique record on the grid; b200flow_reg_leaf_table turns the node stats into leaf values (and the leaf variances).
//
// GBTRegressor (DESIGN.md §5m).  The boosting residual has no a-priori bound, so each iteration's grid exponent comes from
// the all-reduced max |r|: b200flow_gbr_update walks the newest tree, adds its payload to F, writes r = -loss.gradient and
// folds max |r|; b200flow_reg_grid then puts r on that iteration's grid, and b200flow_gbr_leaf_values computes one tree's
// payloads with that tree's own scale.
//
// Evaluator.  Every sum is exact in 128-bit fixed point: a term t becomes rint(t 2^sh) (sh from the all-reduced max |t|,
// leaving ceil(log2 n) bits of headroom below 2^126), cut into four 32-bit limbs, and each limb is summed in int64 with
// integer atomics, so that neither the order of the rows nor the number of ranks can change a bit.
// Compiled with -fmad=false: every fp64 expression below is restated operation for operation by tests/regression_oracle.py.
#include <float.h>
#include <math.h>
#include <string.h>

#include "common.cuh"
#include "portable_exp.h"
#include "tree_walk.cuh"

namespace b200flow {

constexpr int kRegThreads = 256;

__device__ __forceinline__ unsigned long long abs_bits(double v) {
    return (unsigned long long)__double_as_longlong(fabs(v));       // ordered like the values for |v| (non-negative, not NaN)
}

// ------------------------------------------------------------------ trainer
// out[0] += rows whose label is NaN or ±inf, out[1] = max over the finite labels of |y| (as bits); with tp, the 8 bytes of
// y go to bytes [offset, offset + 8) of the row's record
__global__ void reg_labels_kernel(const double* __restrict__ y, int64_t n, uint8_t* tp, int stride, int offset,
                                  unsigned long long* out) {
    unsigned long long bad = 0ull, mx = 0ull;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const double v = y[i];
        if (isfinite(v)) mx = max(mx, abs_bits(v)); else ++bad;
        if (tp) {
            uint8_t b[8];
            memcpy(b, &v, 8);
            uint8_t* dst = tp + i * stride + offset;
#pragma unroll
            for (int k = 0; k < 8; ++k) dst[k] = b[k];
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        bad += __shfl_xor_sync(0xffffffffu, bad, o);
        mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    }
    if (lane_id() == 0) {
        if (bad) atomicAdd(out, bad);
        if (mx) atomicMax(out + 1, mx);
    }
}

// totals[t] += Σ_u W[t][u]: one grid row of CTAs per tree
__global__ void reg_tree_weights_kernel(const int32_t* __restrict__ W, int64_t U, unsigned long long* totals) {
    const int t = blockIdx.y;
    long long s = 0;
    for (int64_t u = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; u < U; u += (int64_t)gridDim.x * blockDim.x)
        s += W[(int64_t)t * U + u];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane_id() == 0 && s) atomicAdd(totals + t, (unsigned long long)s);
}

// record u's label (from its record bytes, or y[u]) -> {q, q2}
__global__ void reg_grid_kernel(const uint8_t* __restrict__ tp, int stride, int offset, const double* __restrict__ y, int64_t n,
                                int E, int S, int S2, longlong2* rq) {
    const int64_t u = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= n) return;
    double v;
    if (tp) {
        uint8_t b[8];
        const uint8_t* src = tp + u * stride + offset;
#pragma unroll
        for (int k = 0; k < 8; ++k) b[k] = src[k];
        memcpy(&v, b, 8);
    } else {
        v = y[u];
    }
    const double ys = v * pexp_pow2(-E);
    const long long q = __double2ll_rn(ys * pexp_pow2(S));
    const double yh = (double)q * pexp_pow2(-S);
    rq[u] = make_longlong2(q, __double2ll_rn(yh * yh * pexp_pow2(S2)));
}

// table[i][0] = (Σw·q s1) / Σw (LeafNode prediction); width 2 adds table[i][1] = Variance.calculate of the node's stats
__global__ void reg_leaf_table_kernel(int64_t n_nodes, const long long* __restrict__ stats, double s1, double s2, double* table,
                                      int width) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_nodes) return;
    const long long w = stats[3 * i], wq = stats[3 * i + 1], wq2 = stats[3 * i + 2];
    table[i * width] = ((double)wq * s1) / (double)w;
    if (width == 2) {
        const double cnt = (double)w;
        double var = 0.0;
        if (cnt != 0.0) {
            const double sum = (double)wq * s1, sq = (double)wq2 * s2;
            var = (sq - sum * sum / cnt) / cnt;
        }
        table[i * width + 1] = var;
    }
}

// out[i] = in[i] / d, IEEE-rounded (the forest's mean over its trees; torch's division by a scalar multiplies by 1 / d)
__global__ void reg_divide_kernel(const double* in, int64_t n, double d, double* out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = in[i] / d;
}

// ------------------------------------------------------------------ GBTRegressor (DESIGN.md §5m)
// payload[i] = weight * ((Σw·q s1) / Σw) for the nodes of tree `tree` only: every tree keeps the scale of its own grid
__global__ void gbr_leaf_values_kernel(int64_t n_nodes, const long long* __restrict__ stats, const int32_t* __restrict__ node_tree,
                                       int tree, double weight, double s1, double* payload) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_nodes || node_tree[i] != tree) return;
    payload[i] = weight * (((double)stats[3 * i + 1] * s1) / (double)stats[3 * i]);
}

// root < 0: F = +0.0 and r = y.  root >= 0: walk the tree rooted at pool node `root`, F += its leaf's payload, then
// r = -loss.gradient(F, y): squared 2 (y - F), absolute -1 if y - F < 0 else +1.  A NaN r (an empty tree's leaf is 0/0)
// becomes 0.  out = max |r| over the records, as ordered bits.
__global__ void gbr_update_kernel(const uint8_t* __restrict__ tp, int stride, int offset, const double* __restrict__ y, int64_t n,
                                  const int4* __restrict__ nodes, const unsigned long long* __restrict__ node_mask,
                                  const double* __restrict__ payload, int root, int loss, double* margin, double* resid,
                                  unsigned long long* out) {
    unsigned long long mx = 0ull;
    for (int64_t u = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; u < n; u += (int64_t)gridDim.x * blockDim.x) {
        const uint8_t* rec = tp + u * stride;
        double v;
        if (y) {
            v = y[u];
        } else {
            uint8_t b[8];
#pragma unroll
            for (int k = 0; k < 8; ++k) b[k] = rec[offset + k];
            memcpy(&v, b, 8);
        }
        double Fm = 0.0, r = v;
        if (root >= 0) {
            Fm = margin[u] + payload[variance_tree_leaf(rec, nodes, node_mask, root)];
            const double d = v - Fm;
            r = loss == 0 ? 2.0 * d : (d < 0.0 ? -1.0 : 1.0);
        }
        if (r != r) r = 0.0;
        margin[u] = Fm;
        resid[u] = r;
        mx = max(mx, abs_bits(r));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if (lane_id() == 0 && mx) atomicMax(out, mx);
}

// ------------------------------------------------------------------ evaluator
// mode 0: {y, y², (y - ŷ)², |y - ŷ|}; mode 1: {(y - m)², (ŷ - m)²} with m the label mean
__device__ __forceinline__ int reg_terms(double y, double p, int mode, double m, double* t) {
    if (mode == 0) {
        const double d = y - p;
        t[0] = y; t[1] = y * y; t[2] = d * d; t[3] = fabs(d);
        return 4;
    }
    const double a = y - m, b = p - m;
    t[0] = a * a; t[1] = b * b;
    return 2;
}

// out[0] += rows with a non-finite label, prediction or term; out[1 + k] = max |term k| (as bits) over the other rows
__global__ void reg_eval_max_kernel(const double* __restrict__ y, const double* __restrict__ p, int64_t n, int mode, double m,
                                    unsigned long long* out) {
    unsigned long long bad = 0ull, mx[4] = {0ull, 0ull, 0ull, 0ull};
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        double t[4];
        const double yi = y[i], pi = p[i];
        const int K = reg_terms(yi, pi, mode, m, t);
        bool ok = isfinite(yi) && isfinite(pi);
        for (int k = 0; k < K; ++k) ok = ok && isfinite(t[k]);
        if (!ok) { ++bad; continue; }
        for (int k = 0; k < K; ++k) mx[k] = max(mx[k], abs_bits(t[k]));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        bad += __shfl_xor_sync(0xffffffffu, bad, o);
#pragma unroll
        for (int k = 0; k < 4; ++k) mx[k] = max(mx[k], __shfl_xor_sync(0xffffffffu, mx[k], o));
    }
    if (lane_id() == 0) {
        if (bad) atomicAdd(out, bad);
#pragma unroll
        for (int k = 0; k < 4; ++k) if (mx[k]) atomicMax(out + 1 + k, mx[k]);
    }
}

// limbs[k][j] += Σ over the rows of limb j of term k on its grid 2^sh[k]; rows with a non-finite input or term are skipped
// (the caller has already counted them and returns NaN)
__global__ void __launch_bounds__(kRegThreads) reg_eval_sums_kernel(const double* __restrict__ y, const double* __restrict__ p,
                                                                    int64_t n, int mode, double m, int4 sh,
                                                                    unsigned long long* limbs) {
    long long acc[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) acc[j] = 0;
    const int shs[4] = {sh.x, sh.y, sh.z, sh.w};
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        double t[4];
        const double yi = y[i], pi = p[i];
        const int K = reg_terms(yi, pi, mode, m, t);
        bool ok = isfinite(yi) && isfinite(pi);
        for (int k = 0; k < K; ++k) ok = ok && isfinite(t[k]);
        if (!ok) continue;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            if (k >= K) break;
            long long l[4];
            fixed_limbs(t[k], shs[k], l);
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[k * 4 + j] += l[j];
        }
    }
#pragma unroll
    for (int j = 0; j < 16; ++j) {
        long long v = acc[j];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (lane_id() == 0 && v) atomicAdd(limbs + j, (unsigned long long)v);
    }
}

static int reg_grid_size(int64_t n) {
    const int64_t b = (n + kRegThreads - 1) / kRegThreads;
    return (int)(b < (int64_t)kNumSMs * 8 ? (b > 0 ? b : 1) : (int64_t)kNumSMs * 8);
}

}  // namespace b200flow

using namespace b200flow;

extern "C" int b200flow_reg_labels(const double* y, int64_t n_rows, uint8_t* tp, int32_t tp_stride, int32_t offset, int64_t* out,
                                   void* stream) {
    B2F_REQUIRE(out, "reg_labels: null pointer");
    if (n_rows <= 0) return B200FLOW_OK;
    B2F_REQUIRE(y, "reg_labels: null pointer");
    B2F_REQUIRE(!tp || (offset >= 0 && offset + 8 <= tp_stride), "reg_labels: the label bytes do not fit in the record");
    reg_labels_kernel<<<reg_grid_size(n_rows), kRegThreads, 0, (cudaStream_t)stream>>>(y, n_rows, tp, tp_stride, offset,
                                                                                       (unsigned long long*)out);
    return check_launch("reg_labels");
}

extern "C" int b200flow_reg_tree_weights(const int32_t* W, int32_t n_trees, int64_t n_unique, int64_t* totals, void* stream) {
    B2F_REQUIRE(totals && n_trees >= 0 && n_trees < 65536, "reg_tree_weights: bad arguments");
    if (n_unique <= 0 || n_trees == 0) return B200FLOW_OK;
    B2F_REQUIRE(W, "reg_tree_weights: null pointer");
    const int64_t b = (n_unique + kRegThreads - 1) / kRegThreads;
    const dim3 grid((unsigned)(b < 64 ? b : 64), (unsigned)n_trees);
    reg_tree_weights_kernel<<<grid, kRegThreads, 0, (cudaStream_t)stream>>>(W, n_unique, (unsigned long long*)totals);
    return check_launch("reg_tree_weights");
}

extern "C" int b200flow_reg_grid(const uint8_t* tp, int32_t tp_stride, int32_t offset, const double* y, int64_t n_rows, int32_t E,
                                 int32_t S, int32_t S2, int64_t* rq, void* stream) {
    B2F_REQUIRE(rq && (tp || y || n_rows <= 0), "reg_grid: null pointer");
    B2F_REQUIRE(((uintptr_t)rq & 15) == 0, "reg_grid: rq must be 16-byte aligned");
    B2F_REQUIRE(!tp || (offset >= 0 && offset + 8 <= tp_stride), "reg_grid: the label bytes do not fit in the record");
    B2F_REQUIRE(E >= -1000 && E <= 1000 && S > 0 && S <= 62 && S2 > 0 && S2 <= 62, "reg_grid: bad grid (E=%d S=%d S2=%d)", E, S, S2);
    if (n_rows <= 0) return B200FLOW_OK;
    reg_grid_kernel<<<(unsigned)((n_rows + kRegThreads - 1) / kRegThreads), kRegThreads, 0, (cudaStream_t)stream>>>(
        tp, tp_stride, offset, y, n_rows, E, S, S2, (longlong2*)rq);
    return check_launch("reg_grid");
}

extern "C" int b200flow_reg_leaf_table(int64_t n_nodes, const int64_t* stats, int32_t S, int32_t S2, double* table, int32_t width,
                                       void* stream) {
    B2F_REQUIRE(stats && table && (width == 1 || width == 2), "reg_leaf_table: bad arguments");
    B2F_REQUIRE(S > -1022 && S < 1022 && S2 > -1022 && S2 < 1022, "reg_leaf_table: bad scale");
    if (n_nodes <= 0) return B200FLOW_OK;
    reg_leaf_table_kernel<<<(unsigned)((n_nodes + kRegThreads - 1) / kRegThreads), kRegThreads, 0, (cudaStream_t)stream>>>(
        n_nodes, (const long long*)stats, ldexp(1.0, -S), ldexp(1.0, -S2), table, width);
    return check_launch("reg_leaf_table");
}

extern "C" int b200flow_reg_divide(const double* in, int64_t n_rows, double d, double* out, void* stream) {
    if (n_rows <= 0) return B200FLOW_OK;
    B2F_REQUIRE(in && out, "reg_divide: null pointer");
    reg_divide_kernel<<<(unsigned)((n_rows + kRegThreads - 1) / kRegThreads), kRegThreads, 0, (cudaStream_t)stream>>>(in, n_rows, d,
                                                                                                                     out);
    return check_launch("reg_divide");
}

extern "C" int b200flow_gbr_leaf_values(int64_t n_nodes, const int64_t* stats, const int32_t* node_tree, int32_t tree,
                                        double weight, int32_t S, double* payload, void* stream) {
    B2F_REQUIRE(stats && node_tree && payload && tree >= 0, "gbr_leaf_values: bad arguments");
    B2F_REQUIRE(S > -1022 && S < 1022, "gbr_leaf_values: bad scale %d", S);
    if (n_nodes <= 0) return B200FLOW_OK;
    gbr_leaf_values_kernel<<<(unsigned)((n_nodes + kRegThreads - 1) / kRegThreads), kRegThreads, 0, (cudaStream_t)stream>>>(
        n_nodes, (const long long*)stats, node_tree, tree, weight, ldexp(1.0, -S), payload);
    return check_launch("gbr_leaf_values");
}

extern "C" int b200flow_gbr_update(const uint8_t* tp, int32_t tp_stride, int32_t offset, const double* y, int64_t n_rows,
                                   const b200flow_node* nodes, const uint64_t* node_mask, const double* payload, int32_t tree,
                                   int32_t loss, double* margin, double* resid, int64_t* max_out, void* stream) {
    B2F_REQUIRE(max_out && (loss == 0 || loss == 1), "gbr_update: bad arguments");
    if (n_rows <= 0) return B200FLOW_OK;
    B2F_REQUIRE(tp && margin && resid && (tree < 0 || (nodes && payload)), "gbr_update: null pointer");
    B2F_REQUIRE(y || (offset >= 0 && offset + 8 <= tp_stride), "gbr_update: the label bytes do not fit in the record");
    gbr_update_kernel<<<reg_grid_size(n_rows), kRegThreads, 0, (cudaStream_t)stream>>>(
        tp, tp_stride, offset, y, n_rows, (const int4*)nodes, (const unsigned long long*)node_mask, payload, tree, loss, margin,
        resid, (unsigned long long*)max_out);
    return check_launch("gbr_update");
}

extern "C" int b200flow_reg_eval_max(const double* label, const double* pred, int64_t n_rows, int32_t mode, double mean,
                                     int64_t* out, void* stream) {
    B2F_REQUIRE(out && (mode == 0 || mode == 1), "reg_eval_max: bad arguments");
    if (n_rows <= 0) return B200FLOW_OK;
    B2F_REQUIRE(label && pred, "reg_eval_max: null pointer");
    reg_eval_max_kernel<<<reg_grid_size(n_rows), kRegThreads, 0, (cudaStream_t)stream>>>(label, pred, n_rows, mode, mean,
                                                                                         (unsigned long long*)out);
    return check_launch("reg_eval_max");
}

extern "C" int b200flow_reg_eval_sums(const double* label, const double* pred, int64_t n_rows, int32_t mode, double mean,
                                      int32_t sh0, int32_t sh1, int32_t sh2, int32_t sh3, int64_t* limbs, void* stream) {
    B2F_REQUIRE(limbs && (mode == 0 || mode == 1), "reg_eval_sums: bad arguments");
    B2F_REQUIRE(n_rows < ((int64_t)1 << 31), "reg_eval_sums: more than 2^31 - 1 rows (the limb sums would overflow)");
    if (n_rows <= 0) return B200FLOW_OK;
    B2F_REQUIRE(label && pred, "reg_eval_sums: null pointer");
    reg_eval_sums_kernel<<<reg_grid_size(n_rows), kRegThreads, 0, (cudaStream_t)stream>>>(
        label, pred, n_rows, mode, mean, make_int4(sh0, sh1, sh2, sh3), (unsigned long long*)limbs);
    return check_launch("reg_eval_sums");
}
