// mlp.cu — MultilayerPerceptronClassifier: loss + gradient and the forward pass, DESIGN.md §5d.
//
// The network is layers = [D, h_1, ..., h_k, K]: affine + sigmoid per hidden layer, affine + softmax on top.  The flat
// weight vector is Spark's: layer after layer, W (out x in, column-major) then b (out).  Read as one column-major
// out x (in + 1) matrix whose last column is b, a layer's block is the matrix that multiplies [a, 1]; the kernels keep a
// column of ones after every activation so that the bias rides along in the three products.
//
// All three products — A·Wᵀ (forward), δ·W (back-propagation) and δᵀ·A (weight gradient, contracting over the tile's
// rows) — are fp64 tensor-core MMAs (mma.sync m8n8k4 f64, SASS DMMA.8x8x4).  Widths are zero-padded to multiples of 8
// and contractions to multiples of 4.  Fragments of m8n8k4.f64 (PTX ISA): A holds (row lane>>2, k lane&3), B holds
// (k lane&3, col lane>>2), C/D hold (row lane>>2, col 2(lane&3) + {0,1}).
//
// b200flow_mlp_loss_grad: one CTA per 4096-row global chunk.  It stages the padded weights in shared memory once, then
// walks the chunk's 32-row tiles in row order (tiles sit at fixed global positions): forward, softmax / loss / δ_L,
// back-propagation, weight gradient.  Activations live in shared memory; δ_l overwrites a_l once a_l has served the
// gradient of the layer above.  The gradient accumulates in registers: 8x8 gradient tile t belongs to warp t % 8, slot
// t / 8, for the whole chunk.  Rows outside [0, n) are masked (their δ is zero, their loss is skipped), never padded
// into the loss.  So a chunk's partial depends only on that chunk's rows, whichever rank or launch computes it.
#include <math.h>

#include "common.cuh"

namespace b200flow {

namespace {

constexpr int kChunkRows = 4096;
constexpr int kMlpMaxLayers = 8;                  // affine layers
constexpr int kMlpTile = 32;                      // rows per tile: 4 MMA row blocks
constexpr int kMlpWarps = 8, kMlpThreads = kMlpWarps * 32;
constexpr int kMlpSlots = 32;                     // gradient tiles per warp: at most 256 8x8 tiles in all
constexpr int kMlpMaxSmem = 227 * 1024 - 1024;    // dynamic shared memory; the static label / loss buffers take the rest

struct MlpShape {
    int L;                                        // affine layers
    int in[kMlpMaxLayers], out[kMlpMaxLayers];
    int inp[kMlpMaxLayers], outp[kMlpMaxLayers];  // in + 1 (the ones column) and out, padded to 8
    int wpitch[kMlpMaxLayers], woff[kMlpMaxLayers];          // staged W: element (o, i) at woff + o + i * wpitch
    int goff[kMlpMaxLayers];                      // the layer's offset in the flat Spark vector
    int apitch[kMlpMaxLayers + 1], aoff[kMlpMaxLayers + 1];  // activation buffers a_0 (x) .. a_L (logits), [kMlpTile][apitch]
    int toff[kMlpMaxLayers + 1];                  // first 8x8 gradient tile of each layer
    int smem_doubles;
    int64_t P;
};

__device__ __forceinline__ void dmma(double (&c)[2], double a, double b) {
    asm("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
        : "+d"(c[0]), "+d"(c[1])
        : "d"(a), "d"(b));
}

// padded W blocks from the flat vector, zeros outside (o < out, i <= in); activation buffers zeroed, ones columns set
__device__ void mlp_stage(const MlpShape& s, const double* __restrict__ w, double* sm) {
    for (int l = 0; l < s.L; ++l) {
        const int pw = s.wpitch[l], out = s.out[l], in = s.in[l];
        for (int e = threadIdx.x; e < s.inp[l] * pw; e += kMlpThreads) {
            const int i = e / pw, o = e - i * pw;
            sm[s.woff[l] + e] = (o < out && i <= in) ? w[s.goff[l] + o + (int64_t)i * out] : 0.0;
        }
    }
    for (int e = s.aoff[0] + threadIdx.x; e < s.smem_doubles; e += kMlpThreads) sm[e] = 0.0;
    __syncthreads();
    for (int l = 0; l < s.L; ++l)
        for (int r = threadIdx.x; r < kMlpTile; r += kMlpThreads) sm[s.aoff[l] + r * s.apitch[l] + s.in[l]] = 1.0;
}

// rows [base, base + kMlpTile) of x into a_0 as f64 (rows outside [0, n) -> 0), their labels into ylab (-1 outside)
template <typename T>
__device__ void mlp_load_tile(const MlpShape& s, const T* __restrict__ x, int64_t n, int64_t ld, const int32_t* __restrict__ y,
                              int64_t base, double* sm, int* ylab) {
    const int D = s.in[0], pa = s.apitch[0];
    double* a0 = sm + s.aoff[0];
    for (int e = threadIdx.x; e < kMlpTile * D; e += kMlpThreads) {
        const int r = e / D, j = e - r * D;
        const int64_t gr = base + r;
        a0[r * pa + j] = (gr >= 0 && gr < n) ? (double)x[gr * ld + j] : 0.0;
    }
    if (y && threadIdx.x < kMlpTile) {
        const int64_t gr = base + threadIdx.x;
        ylab[threadIdx.x] = (gr >= 0 && gr < n) ? y[gr] : -1;
    }
}

// a_{l+1} = sigmoid(a_l · W_lᵀ) for hidden layers, the logits for the last.  Warp w takes output column tiles w, w+8, ...
// over all 4 row blocks, so each B fragment serves 4 MMAs.
__device__ void mlp_forward_tile(const MlpShape& s, double* sm) {
    const int lane = lane_id(), warp = warp_id(), qr = lane >> 2, qc = lane & 3;
    for (int l = 0; l < s.L; ++l) {
        const double* A = sm + s.aoff[l];
        double* Z = sm + s.aoff[l + 1];
        const double* W = sm + s.woff[l];
        const int pa = s.apitch[l], pz = s.apitch[l + 1], pw = s.wpitch[l];
        const int nk = s.inp[l] / 4, nn = s.outp[l] / 8, out = s.out[l];
        const bool last = l == s.L - 1;
        for (int nt = warp; nt < nn; nt += kMlpWarps) {
            double c[4][2] = {};
            for (int k = 0; k < nk; ++k) {
                const double b = W[nt * 8 + qr + (k * 4 + qc) * pw];
#pragma unroll
                for (int m = 0; m < 4; ++m) dmma(c[m], A[(m * 8 + qr) * pa + k * 4 + qc], b);
            }
#pragma unroll
            for (int m = 0; m < 4; ++m)
#pragma unroll
                for (int q = 0; q < 2; ++q) {
                    const int col = nt * 8 + 2 * qc + q;
                    if (col < out) {
                        double v = c[m][q];
                        if (!last) v = 1.0 / (1.0 + exp(-v));
                        Z[(m * 8 + qr) * pz + col] = v;
                    }
                }
        }
        __syncthreads();
    }
}

template <typename T>
__global__ void __launch_bounds__(kMlpThreads, 1) mlp_loss_grad_kernel(const T* __restrict__ x, int64_t n, int64_t ld,
                                                                       const int32_t* __restrict__ y, const MlpShape s,
                                                                       const double* __restrict__ w, int64_t row_offset,
                                                                       double* __restrict__ partials) {
    extern __shared__ double sm[];
    __shared__ int ylab[kMlpTile];
    __shared__ double lossb[kMlpTile];
    const int lane = lane_id(), warp = warp_id(), qr = lane >> 2, qc = lane & 3;
    mlp_stage(s, w, sm);
    const int64_t c0 = (row_offset / kChunkRows + blockIdx.x) * kChunkRows - row_offset;   // local index of the chunk's row 0
    const int64_t lo = c0 > 0 ? c0 : 0, hi = c0 + kChunkRows < n ? c0 + kChunkRows : n;
    const int L = s.L, K = s.out[L - 1];
    double acc[kMlpSlots][2];
#pragma unroll
    for (int q = 0; q < kMlpSlots; ++q) acc[q][0] = acc[q][1] = 0.0;
    double loss = 0.0;
    for (int64_t base = c0 + (lo - c0) / kMlpTile * kMlpTile; base < hi; base += kMlpTile) {
        __syncthreads();                                   // the previous tile's gradient has read a_0
        mlp_load_tile(s, x, n, ld, y, base, sm, ylab);
        __syncthreads();
        mlp_forward_tile(s, sm);
        if (warp == 0) {                                   // softmax, loss and δ_L = softmax - onehot, one row per lane
            double* z = sm + s.aoff[L] + lane * s.apitch[L];
            const int yl = ylab[lane];
            double lr = 0.0;
            if (yl >= 0) {
                double m = z[0];
                for (int k = 1; k < K; ++k) m = z[k] > m ? z[k] : m;
                double se = 0.0;
                for (int k = 0; k < K; ++k) se = se + exp(z[k] - m);
                lr = (m + log(se)) - z[yl];
                for (int k = 0; k < K; ++k) {
                    const double p = exp(z[k] - m) / se;
                    z[k] = k == yl ? p - 1.0 : p;
                }
            } else {
                for (int k = 0; k < K; ++k) z[k] = 0.0;
            }
            lossb[lane] = lr;
            __syncwarp();
            if (lane == 0)
                for (int r = 0; r < kMlpTile; ++r)
                    if (ylab[r] >= 0) loss = loss + lossb[r];
        }
        __syncthreads();
        for (int l = L - 1; l >= 0; --l) {
            const double* Dl = sm + s.aoff[l + 1];         // δ_{l+1}
            double* A = sm + s.aoff[l];                    // a_l, then δ_l
            const int pd = s.apitch[l + 1], pa = s.apitch[l];
            const int t0 = s.toff[l], t1 = s.toff[l + 1], ni = s.inp[l] / 8;
#pragma unroll
            for (int q = 0; q < kMlpSlots; ++q) {          // gradient of layer l: δ_{l+1}ᵀ · [a_l, 1] over the tile's rows
                const int t = warp + kMlpWarps * q;
                if (t >= t0 && t < t1) {
                    const int lt = t - t0, ot = lt / ni, it = lt - ot * ni;
#pragma unroll
                    for (int k = 0; k < kMlpTile / 4; ++k)
                        dmma(acc[q], Dl[(k * 4 + qc) * pd + ot * 8 + qr], A[(k * 4 + qc) * pa + it * 8 + qr]);
                }
            }
            if (l == 0) break;
            __syncthreads();                               // a_l has served the gradient: δ_l may overwrite it
            const double* W = sm + s.woff[l];
            const int pw = s.wpitch[l], nk = s.outp[l] / 4, in = s.in[l];
            for (int nt = warp; nt < (in + 7) / 8; nt += kMlpWarps) {
                double c[4][2] = {};
                for (int k = 0; k < nk; ++k) {
                    const double b = W[k * 4 + qc + (nt * 8 + qr) * pw];
#pragma unroll
                    for (int m = 0; m < 4; ++m) dmma(c[m], Dl[(m * 8 + qr) * pd + k * 4 + qc], b);
                }
#pragma unroll
                for (int m = 0; m < 4; ++m)
#pragma unroll
                    for (int q = 0; q < 2; ++q) {
                        const int col = nt * 8 + 2 * qc + q;
                        if (col < in) {
                            double* p = A + (m * 8 + qr) * pa + col;
                            const double a = *p;
                            *p = c[m][q] * (a * (1.0 - a));
                        }
                    }
            }
            __syncthreads();
        }
    }
    double* part = partials + (int64_t)blockIdx.x * (s.P + 1);
    if (threadIdx.x == 0) part[0] = loss;
#pragma unroll
    for (int q = 0; q < kMlpSlots; ++q) {
        const int t = warp + kMlpWarps * q;
        if (t < s.toff[L]) {
            int l = 0;
            while (t >= s.toff[l + 1]) ++l;
            const int ni = s.inp[l] / 8, lt = t - s.toff[l], ot = lt / ni, it = lt - ot * ni;
            const int o = ot * 8 + qr;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int i = it * 8 + 2 * qc + h;
                if (o < s.out[l] && i <= s.in[l]) part[1 + s.goff[l] + o + (int64_t)i * s.out[l]] = acc[q][h];
            }
        }
    }
}

template <typename T>
__global__ void __launch_bounds__(kMlpThreads) mlp_forward_kernel(const T* __restrict__ x, int64_t n, int64_t ld, const MlpShape s,
                                                                  const double* __restrict__ w, double* __restrict__ raw) {
    extern __shared__ double sm[];
    mlp_stage(s, w, sm);
    const int L = s.L, K = s.out[L - 1], pz = s.apitch[L];
    for (int64_t base = (int64_t)blockIdx.x * kMlpTile; base < n; base += (int64_t)gridDim.x * kMlpTile) {
        __syncthreads();                                   // the previous tile's logits are written out
        mlp_load_tile(s, x, n, ld, (const int32_t*)nullptr, base, sm, nullptr);
        __syncthreads();
        mlp_forward_tile(s, sm);
        const double* z = sm + s.aoff[L];
        for (int e = threadIdx.x; e < kMlpTile * K; e += kMlpThreads) {
            const int r = e / K, k = e - r * K;
            if (base + r < n) raw[(base + r) * K + k] = z[r * pz + k];
        }
    }
}

int mlp_shape(const int32_t* layers, int32_t n_layers, MlpShape* s) {
    B2F_REQUIRE(layers && n_layers >= 2 && n_layers - 1 <= kMlpMaxLayers, "mlp: 2 to %d layer sizes", kMlpMaxLayers + 1);
    for (int l = 0; l < n_layers; ++l) B2F_REQUIRE(layers[l] >= 1 && layers[l] <= 65536, "mlp: layer sizes must be in [1, 65536]");
    s->L = n_layers - 1;
    int64_t P = 0, woff = 0, tiles = 0;
    s->toff[0] = 0;
    for (int l = 0; l < s->L; ++l) {
        const int in = layers[l], out = layers[l + 1];
        s->in[l] = in;
        s->out[l] = out;
        s->inp[l] = (in + 1 + 7) / 8 * 8;
        s->outp[l] = (out + 7) / 8 * 8;
        s->wpitch[l] = s->outp[l] + 4;                 // 4 mod 8 doubles: fragment loads take the minimum 2 wavefronts
        s->goff[l] = (int)P;
        P += (int64_t)(in + 1) * out;
        s->woff[l] = (int)woff;
        woff += (int64_t)s->inp[l] * s->wpitch[l];
        tiles += (int64_t)(s->outp[l] / 8) * (s->inp[l] / 8);
        s->toff[l + 1] = (int)(tiles < (1 << 30) ? tiles : (1 << 30));
        B2F_REQUIRE(woff < (1 << 24), "mlp: layers too wide");
    }
    int64_t a = woff;
    for (int l = 0; l <= s->L; ++l) {
        s->apitch[l] = (l < s->L ? s->inp[l] : s->outp[l - 1]) + 4;
        s->aoff[l] = (int)a;
        a += (int64_t)kMlpTile * s->apitch[l];
    }
    s->smem_doubles = (int)a;
    s->P = P;
    B2F_REQUIRE(tiles <= kMlpWarps * kMlpSlots,
                "mlp: the gradient needs %lld 8x8 tiles (sum over layers of ceil(out/8) * ceil((in+1)/8)); at most %d fit in "
                "registers", (long long)tiles, kMlpWarps * kMlpSlots);
    B2F_REQUIRE(a * (int64_t)sizeof(double) <= kMlpMaxSmem,
                "mlp: weights and activation tiles need %lld bytes of shared memory; at most %d fit",
                (long long)(a * sizeof(double)), kMlpMaxSmem);
    return B200FLOW_OK;
}

}  // namespace

}  // namespace b200flow

using namespace b200flow;

extern "C" int b200flow_mlp_config(const int32_t* layers, int32_t n_layers, int64_t* n_params, int64_t* smem_bytes) {
    MlpShape s;
    const int rc = mlp_shape(layers, n_layers, &s);
    if (rc != B200FLOW_OK) return rc;
    if (n_params) *n_params = s.P;
    if (smem_bytes) *smem_bytes = (int64_t)s.smem_doubles * (int64_t)sizeof(double);
    return B200FLOW_OK;
}

extern "C" int b200flow_mlp_loss_grad(const void* x, int32_t x_dtype, int64_t n_rows, int64_t ld, const int32_t* labels,
                                      const int32_t* layers, int32_t n_layers, const double* weights, int64_t row_offset,
                                      double* partials, void* stream) {
    MlpShape s;
    const int rc = mlp_shape(layers, n_layers, &s);
    if (rc != B200FLOW_OK) return rc;
    B2F_REQUIRE(n_rows >= 0 && row_offset >= 0 && ld >= s.in[0] && (x_dtype == B200FLOW_F32 || x_dtype == B200FLOW_F64),
                "mlp_loss_grad: n >= 0, row_offset >= 0, ld >= layers[0], f32 or f64 features");
    if (n_rows == 0) return B200FLOW_OK;
    B2F_REQUIRE(x && labels && weights && partials, "mlp_loss_grad: null pointer");
    const int64_t nc = (row_offset + n_rows - 1) / kChunkRows - row_offset / kChunkRows + 1;
    B2F_REQUIRE(nc <= 0x7fffffffll, "mlp_loss_grad: too many rows");
    const size_t smem = (size_t)s.smem_doubles * sizeof(double);
    cudaStream_t st = (cudaStream_t)stream;
    if (x_dtype == B200FLOW_F64) {
        cudaFuncSetAttribute(mlp_loss_grad_kernel<double>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        mlp_loss_grad_kernel<double><<<(unsigned)nc, kMlpThreads, smem, st>>>((const double*)x, n_rows, ld, labels, s, weights,
                                                                              row_offset, partials);
    } else {
        cudaFuncSetAttribute(mlp_loss_grad_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        mlp_loss_grad_kernel<float><<<(unsigned)nc, kMlpThreads, smem, st>>>((const float*)x, n_rows, ld, labels, s, weights,
                                                                            row_offset, partials);
    }
    return check_launch("mlp_loss_grad");
}

extern "C" int b200flow_mlp_forward(const void* x, int32_t x_dtype, int64_t n_rows, int64_t ld, const int32_t* layers,
                                    int32_t n_layers, const double* weights, double* raw, void* stream) {
    MlpShape s;
    const int rc = mlp_shape(layers, n_layers, &s);
    if (rc != B200FLOW_OK) return rc;
    B2F_REQUIRE(n_rows >= 0 && ld >= s.in[0] && (x_dtype == B200FLOW_F32 || x_dtype == B200FLOW_F64),
                "mlp_forward: n >= 0, ld >= layers[0], f32 or f64 features");
    if (n_rows == 0) return B200FLOW_OK;
    B2F_REQUIRE(x && weights && raw, "mlp_forward: null pointer");
    const size_t smem = (size_t)s.smem_doubles * sizeof(double);
    const int64_t tiles = (n_rows + kMlpTile - 1) / kMlpTile;
    const int64_t per_sm = (228 * 1024) / (int64_t)(smem + 2048);
    const int64_t cap = (int64_t)kNumSMs * (per_sm > 1 ? per_sm : 1);
    const unsigned grid = (unsigned)(tiles < cap ? tiles : cap);
    cudaStream_t st = (cudaStream_t)stream;
    if (x_dtype == B200FLOW_F64) {
        cudaFuncSetAttribute(mlp_forward_kernel<double>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        mlp_forward_kernel<double><<<grid, kMlpThreads, smem, st>>>((const double*)x, n_rows, ld, s, weights, raw);
    } else {
        cudaFuncSetAttribute(mlp_forward_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        mlp_forward_kernel<float><<<grid, kMlpThreads, smem, st>>>((const float*)x, n_rows, ld, s, weights, raw);
    }
    return check_launch("mlp_forward");
}
