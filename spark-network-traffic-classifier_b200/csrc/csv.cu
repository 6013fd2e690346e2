// csv.cu — CSV text in HBM -> typed AoS flow records (SURVEY.md 8f-3: the data format in front of the path).
// Replaces `spark.read.csv(path, inferSchema=True, header=...)` at network_traffic_classifier_kdd99.py:25 and
// network_traffic_classifier_cicids17.py:19-20: the file's bytes are copied to the device once and everything else happens here.
//
//   csv_count_lines / csv_line_starts   line index: byte offset of every non-empty line (LF or CRLF), 16 bytes per thread
//   csv_rows_kernel<MODE_INFER>         Spark's type inference per column: max over rows of {null < int < long < double < string}
//   csv_rows_kernel<MODE_DICT>          string columns: 64-bit hash -> open-addressing table, first occurrence kept (atomicMin)
//   csv_rows_kernel<MODE_PARSE>         fields -> int32 / float64 / dictionary code, written into the AoS record of the row
//
// One WARP per row: the row's bytes are staged in shared memory with coalesced loads while ballots find the delimiters, then
// lane f converts field f (f + 32, ...).  Decimal -> double is exact (csv_number.h); a literal outside its exact range, a
// ragged row, a quoted field or a hash collision is COUNTED and the host raises — nothing is approximated silently.
#include "common.cuh"
#include "csv_number.h"

namespace b200flow {

constexpr int kCsvWarps = 8;
constexpr int kCsvRowCap = 4096;          // longest row (bytes before its '\n', a CRLF's '\r' included) the tokenizer stages
constexpr int kCsvMaxCols = 1024;
constexpr int kIdxThreads = 256;          // 256 threads x 16 bytes = one 4 KB block of text per CTA

enum { MODE_INFER = 0, MODE_DICT = 1, MODE_PARSE = 2 };
enum { BAD_RAGGED = 0, BAD_RAGGED_FIRST = 1, BAD_LONG = 2, BAD_NUMBER = 3, BAD_UNSUPPORTED = 4, BAD_NUMBER_FIRST = 5, BAD_DICT_FULL = 6, BAD_DICT_MISS = 7 };

// ---------------------------------------------------------------------------------------------- line index
// bit i of the result: a non-empty line starts at byte o + i (o = 16 * global thread index)
__device__ __forceinline__ uint32_t line_start_mask(const uint8_t* __restrict__ text, int64_t n, int64_t o, bool* quote) {
    if (o >= n) return 0u;
    uint8_t c[19];                                             // c[0] = byte before, c[1..16] = mine, c[17..18] = look-ahead
    if (o + 16 <= n) {
        const uint4 v = __ldg((const uint4*)(text + o));
        const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int i = 0; i < 16; ++i) c[1 + i] = (uint8_t)(w[i >> 2] >> (8 * (i & 3)));
    } else {
#pragma unroll
        for (int i = 0; i < 16; ++i) c[1 + i] = o + i < n ? text[o + i] : (uint8_t)'\n';
    }
    c[0] = o > 0 ? text[o - 1] : (uint8_t)'\n';
    c[17] = o + 16 < n ? text[o + 16] : (uint8_t)'\n';
    c[18] = o + 17 < n ? text[o + 17] : (uint8_t)'\n';
    uint32_t m = 0;
    bool q = false;
#pragma unroll
    for (int i = 0; i < 16; ++i) {
        const uint8_t cur = c[1 + i];
        q |= cur == '"';
        const bool empty = cur == '\n' || (cur == '\r' && c[2 + i] == '\n');
        if (c[i] == '\n' && !empty && o + i < n) m |= 1u << i;
    }
    *quote = q;
    return m;
}

__global__ void __launch_bounds__(kIdxThreads) csv_count_lines_kernel(const uint8_t* __restrict__ text, int64_t n, int32_t* __restrict__ counts,
                                                                      unsigned long long* __restrict__ flags) {
    __shared__ int sh[33];
    const int64_t o = ((int64_t)blockIdx.x * kIdxThreads + threadIdx.x) * 16;
    bool q = false;
    const int c = __popc(line_start_mask(text, n, o, &q));
    int total;
    block_exclusive_scan(c, sh, &total);
    if (threadIdx.x == 0) counts[blockIdx.x] = total;
    if (__syncthreads_or(q) && threadIdx.x == 0) atomicOr(flags, 1ull);
}

__global__ void __launch_bounds__(kIdxThreads) csv_line_starts_kernel(const uint8_t* __restrict__ text, int64_t n, const int64_t* __restrict__ bases,
                                                                      int64_t* __restrict__ row_starts) {
    __shared__ int sh[33];
    const int64_t o = ((int64_t)blockIdx.x * kIdxThreads + threadIdx.x) * 16;
    bool q;
    uint32_t m = line_start_mask(text, n, o, &q);
    int total;
    const int ex = block_exclusive_scan(__popc(m), sh, &total);
    int64_t at = bases[blockIdx.x] + ex;
    while (m) { const int i = __ffs(m) - 1; m &= m - 1; row_starts[at++] = o + i; }
}

// ---------------------------------------------------------------------------------------------- rows
struct CsvArgs {
    const uint8_t* text; int64_t n_bytes;
    const int64_t* row_starts; int64_t n_rows;
    int n_cols; int flags;                                    // bit 0: ignoreLeadingWhiteSpace, bit 1: ignoreTrailingWhiteSpace
    int32_t* col_class; int32_t* col_null;                    // INFER
    const b200flow_csv_col* cols;                             // DICT, PARSE
    unsigned long long* keys; long long* pos_len; const int32_t* slot_code; int cap_log2;
    uint8_t* records; int row_bytes;
    unsigned long long* bad;
};

__device__ __forceinline__ void dict_insert(unsigned long long* keys, long long* pos_len, uint32_t mask, uint64_t h, long long pl,
                                            unsigned long long* bad) {
    uint32_t s = (uint32_t)(h ^ (h >> 32)) & mask;
    for (int probe = 0; probe < 4096; ++probe) {
        unsigned long long k = __ldcg(keys + s);
        if (k == 0ull) { k = atomicCAS(keys + s, 0ull, (unsigned long long)h); if (k == 0ull) k = h; }
        if (k == h) { if (__ldcg(pos_len + s) > pl) atomicMin(pos_len + s, pl); return; }   // plain read first: the minimum settles fast
        s = (s + 1) & mask;
    }
    atomicAdd(bad + BAD_DICT_FULL, 1ull);
}

__device__ __forceinline__ int dict_lookup(const CsvArgs& a, int str_index, const uint8_t* f, int len, uint64_t h) {
    const uint32_t mask = (1u << a.cap_log2) - 1u;
    const unsigned long long* keys = a.keys + ((size_t)str_index << a.cap_log2);
    const long long* pl = a.pos_len + ((size_t)str_index << a.cap_log2);
    uint32_t s = (uint32_t)(h ^ (h >> 32)) & mask;
    for (int probe = 0; probe < 4096; ++probe) {
        const unsigned long long k = __ldg(keys + s);
        if (k == h) {                                          // same hash: the bytes must equal the slot's first occurrence
            const long long v = __ldg(pl + s);
            const int rl = (int)(v & 0xFFFF);
            const uint8_t* rep = a.text + (v >> 16);
            bool same = rl == len;
            for (int i = 0; same && i < len; ++i) same = rep[i] == f[i];
            return same ? __ldg(a.slot_code + ((size_t)str_index << a.cap_log2) + s) : -2;
        }
        if (k == 0ull) return -2;
        s = (s + 1) & mask;
    }
    return -2;
}

template <int MODE>
__global__ void __launch_bounds__(kCsvWarps * 32) csv_rows_kernel(const CsvArgs a) {
    extern __shared__ __align__(16) uint8_t sm[];
    const int lane = lane_id(), wid = warp_id();
    const int fs_bytes = ((a.n_cols + 2) * 2 + 15) & ~15;
    int32_t* sh_class = (int32_t*)sm;                          // [n_cols] (INFER)
    int32_t* sh_null = sh_class + (MODE == MODE_INFER ? a.n_cols : 0);
    uint8_t* warp_base = sm + (MODE == MODE_INFER ? (((size_t)a.n_cols * 8 + 15) & ~(size_t)15) : 0) + (size_t)wid * (kCsvRowCap + fs_bytes);
    uint8_t* buf = warp_base;
    uint16_t* fs = (uint16_t*)(warp_base + kCsvRowCap);
    if (MODE == MODE_INFER) {
        for (int i = threadIdx.x; i < 2 * a.n_cols; i += blockDim.x) sh_class[i] = 0;
        __syncthreads();
    }
    const uint32_t lt = (1u << lane) - 1u;
    const int64_t warp0 = (int64_t)blockIdx.x * kCsvWarps + wid, nwarps = (int64_t)gridDim.x * kCsvWarps;
    for (int64_t r = warp0; r < a.n_rows; r += nwarps) {
        const int64_t s = __ldg(a.row_starts + r);
        int nf = 0, len = 0;
        bool done = false;
        if (lane == 0) fs[0] = 0;
        for (int base = 0; base <= kCsvRowCap && !done; base += 32) {
            const int64_t p = s + base + lane;
            const uint8_t c = p < a.n_bytes ? __ldg(a.text + p) : (uint8_t)'\n';
            const uint32_t nl = __ballot_sync(0xffffffffu, c == '\n');
            if (base == kCsvRowCap && !(nl & 1u)) break;         // a row of exactly kCsvRowCap bytes: only its '\n' is read here
            const int upto = nl ? __ffs(nl) - 1 : 32;
            const bool valid = lane < upto;
            if (valid) buf[base + lane] = c;
            const bool comma = valid && c == ',';
            const uint32_t cm = __ballot_sync(0xffffffffu, comma);
            if (comma) { const int idx = nf + __popc(cm & lt) + 1; if (idx <= a.n_cols) fs[idx] = (uint16_t)(base + lane + 1); }
            nf += __popc(cm);
            len = base + upto;
            done = nl != 0u;
        }
        __syncwarp();
        if (!done) { if (lane == 0) atomicAdd(a.bad + BAD_LONG, 1ull); continue; }
        if (len > 0 && buf[len - 1] == '\r') --len;              // CRLF
        if (nf + 1 != a.n_cols) {
            if (lane == 0) { atomicAdd(a.bad + BAD_RAGGED, 1ull); atomicMin(a.bad + BAD_RAGGED_FIRST, (unsigned long long)r); }
            __syncwarp();
            continue;
        }
        if (lane == 0) fs[a.n_cols] = (uint16_t)(len + 1);
        __syncwarp();
        for (int f = lane; f < a.n_cols; f += 32) {
            int b = fs[f], e = (int)fs[f + 1] - 1;
            if (a.flags & 1) while (b < e && csv_is_space(buf[b])) ++b;
            if (a.flags & 2) while (e > b && csv_is_space(buf[e - 1])) --e;
            const uint8_t* fp = buf + b;
            const int fl = e - b;
            if (MODE == MODE_INFER) {
                const int cls = csv_classify(fp, fl);
                if (cls == CSV_NULL) { if (sh_null[f] == 0) sh_null[f] = 1; }
                else if (sh_class[f] < cls) atomicMax(sh_class + f, cls);
            } else {
                const b200flow_csv_col col = a.cols[f];
                if (MODE == MODE_DICT) {
                    if (col.type == B200FLOW_CSV_STRING && fl > 0)
                        dict_insert(a.keys + ((size_t)col.str_index << a.cap_log2), a.pos_len + ((size_t)col.str_index << a.cap_log2),
                                    (1u << a.cap_log2) - 1u, csv_hash(fp, fl), (long long)(((s + b) << 16) | fl), a.bad);
                } else {
                    uint8_t* out = a.records + r * a.row_bytes + col.rec_off;
                    int st = CSVNUM_OK;
                    if (col.type == B200FLOW_CSV_INT32) {
                        int32_t v = 0;
                        st = csv_parse_int32(fp, fl, &v);
                        *(int32_t*)out = v;
                    } else if (col.type == B200FLOW_CSV_DOUBLE) {
                        double v = 0.0;
                        st = csv_parse_double(fp, fl, &v);
                        const long long bits = __double_as_longlong(v);
                        ((int32_t*)out)[0] = (int32_t)bits; ((int32_t*)out)[1] = (int32_t)(bits >> 32);   // fields are 4-byte aligned
                    } else if (col.type == B200FLOW_CSV_STRING) {
                        int code = -1;                                  // empty field: null
                        if (fl > 0) { code = dict_lookup(a, col.str_index, fp, fl, csv_hash(fp, fl)); if (code == -2) atomicAdd(a.bad + BAD_DICT_MISS, 1ull); }
                        *(int32_t*)out = code;
                    }
                    if (st != CSVNUM_OK) {
                        atomicAdd(a.bad + (st == CSVNUM_UNSUPPORTED ? BAD_UNSUPPORTED : BAD_NUMBER), 1ull);
                        atomicMin(a.bad + BAD_NUMBER_FIRST, ((unsigned long long)r << 16) | (unsigned long long)f);
                    }
                }
            }
        }
        __syncwarp();
    }
    if (MODE == MODE_INFER) {
        __syncthreads();
        for (int i = threadIdx.x; i < a.n_cols; i += blockDim.x) {
            if (sh_class[i]) atomicMax(a.col_class + i, sh_class[i]);
            if (sh_null[i]) atomicOr(a.col_null + i, 1);
        }
    }
}

static size_t csv_rows_smem(int mode, int n_cols) {
    const size_t fs_bytes = (((size_t)n_cols + 2) * 2 + 15) & ~(size_t)15;
    return (mode == MODE_INFER ? (((size_t)n_cols * 8 + 15) & ~(size_t)15) : 0) + (size_t)kCsvWarps * (kCsvRowCap + fs_bytes);
}

template <int MODE>
static int csv_rows_launch(const CsvArgs& a, cudaStream_t stream, const char* what) {
    const size_t smem = csv_rows_smem(MODE, a.n_cols);
    // the limit belongs to the current device: set it on every launch, or a second GPU of the process could not run wide files
    const cudaError_t e = cudaFuncSetAttribute(csv_rows_kernel<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) { cudaGetLastError(); set_error("%s: cudaFuncSetAttribute: %s", what, cudaGetErrorString(e)); return B200FLOW_ERR_CUDA; }
    const int64_t want = (a.n_rows + kCsvWarps - 1) / kCsvWarps;
    const int grid = (int)(want < (int64_t)kNumSMs * 4 ? want : (int64_t)kNumSMs * 4);
    csv_rows_kernel<MODE><<<grid, kCsvWarps * 32, smem, stream>>>(a);
    return check_launch(what);
}

}  // namespace b200flow

using namespace b200flow;

extern "C" int b200flow_csv_count_lines(const uint8_t* text, int64_t n_bytes, int32_t* counts, unsigned long long* flags, void* stream) {
    if (n_bytes <= 0) return B200FLOW_OK;
    B2F_REQUIRE(text && counts && flags && ((uintptr_t)text & 15) == 0, "csv_count_lines: null or unaligned pointer");
    const int64_t blocks = (n_bytes + kIdxThreads * 16 - 1) / (kIdxThreads * 16);
    B2F_REQUIRE(blocks <= 0x7fffffff, "csv_count_lines: text too large for one call");
    csv_count_lines_kernel<<<(int)blocks, kIdxThreads, 0, (cudaStream_t)stream>>>(text, n_bytes, counts, flags);
    return check_launch("csv_count_lines");
}

extern "C" int b200flow_csv_line_starts(const uint8_t* text, int64_t n_bytes, const int64_t* bases, int64_t* row_starts, void* stream) {
    if (n_bytes <= 0) return B200FLOW_OK;
    B2F_REQUIRE(text && bases && row_starts && ((uintptr_t)text & 15) == 0, "csv_line_starts: null or unaligned pointer");
    const int64_t blocks = (n_bytes + kIdxThreads * 16 - 1) / (kIdxThreads * 16);
    csv_line_starts_kernel<<<(int)blocks, kIdxThreads, 0, (cudaStream_t)stream>>>(text, n_bytes, bases, row_starts);
    return check_launch("csv_line_starts");
}

extern "C" int b200flow_csv_infer(const uint8_t* text, int64_t n_bytes, const int64_t* row_starts, int64_t n_rows, int32_t n_cols, int32_t flags,
                                  int32_t* col_class, int32_t* col_null, unsigned long long* bad, void* stream) {
    if (n_rows <= 0) return B200FLOW_OK;
    B2F_REQUIRE(text && row_starts && col_class && col_null && bad && n_cols >= 1 && n_cols <= kCsvMaxCols, "csv_infer: bad arguments");
    CsvArgs a{};
    a.text = text; a.n_bytes = n_bytes; a.row_starts = row_starts; a.n_rows = n_rows; a.n_cols = n_cols; a.flags = flags;
    a.col_class = col_class; a.col_null = col_null; a.bad = bad;
    return csv_rows_launch<MODE_INFER>(a, (cudaStream_t)stream, "csv_infer");
}

extern "C" int b200flow_csv_dictionary(const uint8_t* text, int64_t n_bytes, const int64_t* row_starts, int64_t n_rows, int32_t n_cols,
                                       int32_t flags, const b200flow_csv_col* cols, unsigned long long* keys, long long* pos_len,
                                       int32_t cap_log2, unsigned long long* bad, void* stream) {
    if (n_rows <= 0) return B200FLOW_OK;
    B2F_REQUIRE(text && row_starts && cols && keys && pos_len && bad && n_cols >= 1 && n_cols <= kCsvMaxCols && cap_log2 >= 4 && cap_log2 <= 28,
                "csv_dictionary: bad arguments");
    CsvArgs a{};
    a.text = text; a.n_bytes = n_bytes; a.row_starts = row_starts; a.n_rows = n_rows; a.n_cols = n_cols; a.flags = flags;
    a.cols = cols; a.keys = keys; a.pos_len = pos_len; a.cap_log2 = cap_log2; a.bad = bad;
    return csv_rows_launch<MODE_DICT>(a, (cudaStream_t)stream, "csv_dictionary");
}

extern "C" int b200flow_csv_parse(const uint8_t* text, int64_t n_bytes, const int64_t* row_starts, int64_t n_rows, int32_t n_cols, int32_t flags,
                                  const b200flow_csv_col* cols, const unsigned long long* keys, const long long* pos_len,
                                  const int32_t* slot_code, int32_t cap_log2, void* records, int32_t row_bytes, unsigned long long* bad,
                                  void* stream) {
    if (n_rows <= 0) return B200FLOW_OK;
    B2F_REQUIRE(text && row_starts && cols && records && bad && n_cols >= 1 && n_cols <= kCsvMaxCols && row_bytes >= 4 && (row_bytes & 3) == 0,
                "csv_parse: bad arguments");
    B2F_REQUIRE((keys && pos_len && slot_code && cap_log2 >= 4 && cap_log2 <= 28) || (!keys && !pos_len && !slot_code), "csv_parse: bad dictionary tables");
    CsvArgs a{};
    a.text = text; a.n_bytes = n_bytes; a.row_starts = row_starts; a.n_rows = n_rows; a.n_cols = n_cols; a.flags = flags;
    a.cols = cols; a.keys = (unsigned long long*)keys; a.pos_len = (long long*)pos_len; a.slot_code = slot_code; a.cap_log2 = keys ? cap_log2 : 4;
    a.records = (uint8_t*)records; a.row_bytes = row_bytes; a.bad = bad;
    return csv_rows_launch<MODE_PARSE>(a, (cudaStream_t)stream, "csv_parse");
}
