// windowStats.py on the device: per-window mean, median, min, max, sd, sum and quantiles of numeric columns (windowStats.py
// 147-186, genomics.py GenoFileReader / parseGenoLine 1884-1945).
//
// The text is streamed in chunks of complete lines (pg_ws_chunk).  Per chunk:
//   ingest.cu's pg_text_load uploads the text and indexes its data lines ('#' and blank lines are skipped);
//   k_ws_lines : ONE WARP PER DATA LINE (pg_warp_fields): field 0 -> scaffold hash, field 1 -> position as int64, field 2 + c
//                -> the value of column c when an output slot reads it, parsed by wstats_parse.h into the resident values
//                [slot x line] (float64, column-major), with a token record (offset, length, status) for the tokens the
//                parser rejects or leaves to the host;
//   pg_scaffold_flags and a CUB select give the first line of every scaffold run, and a second select the flagged tokens.
// The chunk's text is then free; only values and positions stay.  pg_ws_stats, on the first call, compacts every slot's
// non-NaN values in file order (CUB select) with an exclusive count of them (CUB scan), so that window w's values of slot c
// are the contiguous range [cnt_c[lo_w], cnt_c[hi_w]) of the compacted slot: overlapping windows copy nothing.  Then
//   k_ws_moments : ONE WARP PER (window, slot): count, min and max (order-preserving keys), numpy's pairwise sum (the lanes
//                  sum the <= 128-value leaves, lane 0 combines them in the tree's association), the mean and a second
//                  pairwise pass over (x - mean)^2 for sd;
//   order statistics, only when median or a quantile is asked: the windows' ranges are gathered as uint64 keys into scratch,
//   in batches bounded by a byte budget, sorted by CUB DeviceSegmentedSort, and k_ws_pick reads the median and the quantiles.
#include <algorithm>
#include <cmath>
#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>
#include <thrust/iterator/transform_iterator.h>

#include "pgwin_internal.h"
#include "wstats_parse.h"

namespace {

enum { WE_POS = 1, WE_NO_POS = 2, WE_POS_RANGE = 3, WE_FIELDS = 4, WE_BYTE = 5, WE_CR = 6, WE_MISSING = 7 };
enum { ST_MEAN = 0, ST_MEDIAN = 1, ST_MIN = 2, ST_MAX = 3, ST_SD = 4, ST_SUM = 5, ST_QUANTILE = 6 };
constexpr int MAX_STATS = 64;

__device__ uint64_t d_pow5[PG_POW5_QMAX - PG_POW5_QMIN + 1][2];

struct LineParams {
    const uint8_t* buf;
    size_t len;
    const long long* starts;
    int64_t S;                  // data lines of the chunk
    int64_t S0, cap;            // lines before the chunk, the resident arrays' line capacity
    int n_cols, n_slots, n_fields;   // n_fields >= 0: every line has exactly that many value fields
    const int32_t* col_slot;    // [n_cols] the slot that reads value column c, or -1
    const int32_t* slot_col;    // [n_slots]
    double* vals;               // [n_slots x cap]
    long long* pos;             // [cap]
    unsigned long long* hash;   // [S]
    unsigned long long* tok;    // [n_slots x S]: chunk offset << 32 | length << 2 | status
    unsigned long long* err;    // (line + 1) << 28 | slot << 4 | code, first line then first slot wins
};

__device__ __forceinline__ void report(const LineParams& p, int code, int64_t line, int slot) {
    atomicMin(p.err, ((unsigned long long)(line + 1) << 28) | ((unsigned long long)min(slot, (1 << 24) - 1) << 4) |
                         (unsigned long long)code);
}

__global__ void __launch_bounds__(256) k_ws_lines(const __grid_constant__ LineParams p) {
    const int lane = threadIdx.x & 31;
    const int64_t line = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (line >= p.S) return;
    const size_t l0 = (size_t)p.starts[line];
    bool hi = false, lone_cr = false;
    const unsigned n_fields = pg_warp_fields(p.buf, p.len, l0, &hi, &lone_cr, [&](unsigned fidx, size_t q) {
        if (fidx == 0) {
            unsigned long long h = 1469598103934665603ull;
            for (size_t j = q;; ++j) {
                const unsigned c = pg_byte_at(p.buf, p.len, j);
                if (c == '\n' || pg_sblank(c)) break;
                h = (h ^ c) * 1099511628211ull;
            }
            p.hash[line] = h;
        } else if (fidx == 1) {                                     // [+-]?[0-9]+ within int64
            size_t j = q;
            unsigned c = pg_byte_at(p.buf, p.len, j);
            bool neg = false;
            if (c == '-' || c == '+') {
                neg = c == '-';
                c = pg_byte_at(p.buf, p.len, ++j);
            }
            const bool ok = c >= '0' && c <= '9';
            unsigned long long v = 0;
            bool over = false;
            while (c >= '0' && c <= '9') {
                if (v > (~0ull - 9) / 10) over = true;
                else v = v * 10 + (c - '0');
                c = pg_byte_at(p.buf, p.len, ++j);
            }
            if (!ok || !(c == '\n' || pg_sblank(c))) {
                report(p, WE_POS, line, 0);
            } else if (over || v > (1ull << 63) - (neg ? 0 : 1)) {
                report(p, WE_POS_RANGE, line, 0);
            }
            p.pos[p.S0 + line] = neg ? (long long)(0ull - v) : (long long)v;
        } else {
            const int col = (int)fidx - 2;
            if (col >= p.n_cols) return;
            const int slot = p.col_slot[col];
            if (slot < 0) return;
            size_t j = q;
            while (j - q < (1u << 29)) {
                const unsigned c = pg_byte_at(p.buf, p.len, j);
                if (c == '\n' || pg_sblank(c)) break;
                ++j;
            }
            double v = 0.0;
            const int st = pgws::parse_double(p.buf + q, (int)(j - q), d_pow5, &v);
            p.vals[(size_t)slot * p.cap + p.S0 + line] = st == PG_WS_OK ? v : __longlong_as_double(0x7ff8000000000000ll);
            p.tok[(size_t)slot * p.S + line] = ((unsigned long long)q << 32) | ((unsigned long long)(j - q) << 2) | st;
        }
    });
    if (lane == 0) {
        if (hi) report(p, WE_BYTE, line, 0);
        if (lone_cr) report(p, WE_CR, line, 0);
        if (n_fields < 2) report(p, WE_NO_POS, line, 0);
        if (n_fields == 0) p.hash[line] = 0;
        const int nv = n_fields >= 2 ? (int)n_fields - 2 : 0;
        if (p.n_fields >= 0 && nv != p.n_fields && n_fields >= 2) report(p, WE_FIELDS, line, 0);
    }
    for (int k = lane; k < p.n_slots; k += 32)
        if (p.slot_col[k] >= (int)n_fields - 2 && p.n_fields < 0) report(p, WE_MISSING, line, k);
}

__global__ void k_ws_gather_u64(const unsigned long long* __restrict__ src, const long long* __restrict__ idx, int64_t n,
                                unsigned long long* __restrict__ dst) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        dst[i] = src[idx[i]];
}

__global__ void k_ws_scatter(const long long* __restrict__ at, const double* __restrict__ v, int64_t n, double* __restrict__ dst) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        dst[at[i]] = v[i];
}

__global__ void k_ws_run_off(const long long* __restrict__ starts, const long long* __restrict__ run_line, int64_t n,
                             long long* __restrict__ run_off) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        run_off[i] = starts[run_line[i]];
}

// order-preserving keys of float64: unsigned order of the keys = numeric order, -0.0 before +0.0
__device__ __forceinline__ unsigned long long dkey(double x) {
    const unsigned long long u = (unsigned long long)__double_as_longlong(x);
    return (u >> 63) ? ~u : (u | (1ull << 63));
}
__device__ __forceinline__ double dval(unsigned long long k) {
    return __longlong_as_double((long long)((k >> 63) ? (k & ~(1ull << 63)) : ~k));
}

struct NotNan {
    const double* v;
    int64_t n;
    __device__ __forceinline__ int64_t operator()(int64_t i) const { return i < n && !isnan(v[i]) ? 1 : 0; }
};
struct IsNotNan {
    __device__ __forceinline__ bool operator()(double x) const { return !isnan(x); }
};
struct Flagged {
    const unsigned long long* tok;
    __device__ __forceinline__ bool operator()(long long i) const { return (tok[i] & 3ull) != 0; }
};

// numpy's pairwise_sum over a leaf of n <= 128 values f(x[i])
template <class F>
__device__ __forceinline__ double leaf_sum(const double* x, int64_t n, F f) {
    if (n < 8) {
        double res = -0.0;
        for (int64_t i = 0; i < n; ++i) res += f(x[i]);
        return res;
    }
    double r[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) r[j] = f(x[j]);
    int64_t i = 8;
    for (; i < n - (n % 8); i += 8)
#pragma unroll
        for (int j = 0; j < 8; ++j) r[j] += f(x[i + j]);
    double res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]));
    for (; i < n; ++i) res += f(x[i]);
    return res;
}

struct Leaf {
    long long off, len;
    int tag;                    // the tree nodes that end with this leaf (each adds its two children after it)
};

// ONE WARP: numpy's pairwise_sum of f(x[0 .. n)): a node of more than 128 values splits at n2 = n / 2 - (n / 2) % 8 into
// pairwise(left) + pairwise(right).  Lane 0 walks the tree depth-first and hands out 32 leaves at a time; the lanes sum them;
// lane 0 folds the leaf sums on a stack in the tree's association.  The result is returned to every lane.
template <class F>
__device__ double warp_pairwise(const double* x, int64_t n, F f, Leaf* sl, double* sv) {
    const int lane = threadIdx.x & 31;
    Leaf st[48];                // pending right children: one per level of the tree
    double vs[50];
    int sp = 0, vp = 0;
    if (lane == 0) st[sp++] = Leaf{0, n, 0};
    while (true) {
        int cnt = 0;
        if (lane == 0) {
            while (cnt < 32 && sp > 0) {
                Leaf nd = st[--sp];
                while (nd.len > 128) {
                    long long n2 = nd.len / 2;
                    n2 -= n2 % 8;
                    st[sp++] = Leaf{nd.off + n2, nd.len - n2, nd.tag + 1};
                    nd = Leaf{nd.off, n2, 0};
                }
                sl[cnt++] = nd;
            }
        }
        cnt = __shfl_sync(0xffffffffu, cnt, 0);
        if (cnt == 0) break;
        __syncwarp();
        double v = 0.0;
        if (lane < cnt) v = leaf_sum(x + sl[lane].off, sl[lane].len, f);
        sv[lane] = v;
        __syncwarp();
        if (lane == 0)
            for (int j = 0; j < cnt; ++j) {
                vs[vp++] = sv[j];
                for (int t = sl[j].tag; t > 0; --t) {
                    const double b = vs[--vp], a = vs[--vp];
                    vs[vp++] = a + b;
                }
            }
        __syncwarp();
    }
    const double r = lane == 0 ? vs[0] : 0.0;
    return __shfl_sync(0xffffffffu, r, 0);
}

struct StatParams {
    const double* comp;         // [n_slots x S] compacted values
    const long long* cnt;       // [n_slots x (S + 1)] exclusive counts of non-NaN values
    int64_t S;
    int n_slots;
    int64_t W;
    const long long* lo;        // [W]
    const long long* hi;
    int K;
    int code[MAX_STATS];
    double q[MAX_STATS];
    double* out;                // [W x n_slots x K]
    long long* n_out;           // [W x n_slots]
};

__global__ void __launch_bounds__(128) k_ws_moments(const __grid_constant__ StatParams p) {
    __shared__ Leaf sl[4][32];
    __shared__ double sv[4][32];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const int64_t pair = (int64_t)blockIdx.x * 4 + wib;
    if (pair >= p.W * p.n_slots) return;
    const int64_t w = pair / p.n_slots;
    const int c = (int)(pair % p.n_slots);
    const long long* cc = p.cnt + (size_t)c * (p.S + 1);
    const long long a = cc[p.lo[w]], b = cc[p.hi[w]];
    const int64_t n = b - a;
    const double* x = p.comp + (size_t)c * p.S + a;
    bool want_mm = false, want_sum = false, want_sd = false;
    for (int k = 0; k < p.K; ++k) {
        want_mm |= p.code[k] == ST_MIN || p.code[k] == ST_MAX;
        want_sum |= p.code[k] == ST_MEAN || p.code[k] == ST_SUM || p.code[k] == ST_SD;
        want_sd |= p.code[k] == ST_SD;
    }
    unsigned long long kmin = ~0ull, kmax = 0ull;
    if (want_mm) {
        for (int64_t i = lane; i < n; i += 32) {
            const unsigned long long k = dkey(x[i]);
            kmin = min(kmin, k);
            kmax = max(kmax, k);
        }
#pragma unroll
        for (int d = 16; d >= 1; d >>= 1) {
            kmin = min(kmin, __shfl_xor_sync(0xffffffffu, kmin, d));
            kmax = max(kmax, __shfl_xor_sync(0xffffffffu, kmax, d));
        }
    }
    double sum = 0.0, mean = 0.0, sd = 0.0;
    if (want_sum) {
        sum = 0.0 + warp_pairwise(x, n, [](double v) { return v; }, sl[wib], sv[wib]);
        mean = sum / (double)n;
        if (want_sd) {
            const double m = mean;
            const double ss = 0.0 + warp_pairwise(x, n, [m](double v) { const double d = v - m; return d * d; }, sl[wib], sv[wib]);
            sd = rint(sqrt(ss / (double)n) * 1e6) / 1e6;
        }
    }
    if (lane != 0) return;
    double* o = p.out + (size_t)pair * p.K;
    p.n_out[pair] = n;
    for (int k = 0; k < p.K; ++k) {
        switch (p.code[k]) {
            case ST_MEAN: o[k] = mean; break;
            case ST_SUM: o[k] = sum; break;
            case ST_SD: o[k] = sd; break;
            case ST_MIN: o[k] = n ? dval(kmin) : __longlong_as_double(0x7ff8000000000000ll); break;
            case ST_MAX: o[k] = n ? dval(kmax) : __longlong_as_double(0x7ff8000000000000ll); break;
            default: break;
        }
    }
}

// ONE WARP PER (window, slot) of the batch: its values as keys into the batch's segment
__global__ void __launch_bounds__(256) k_ws_gather(const __grid_constant__ StatParams p, int64_t p0, int64_t p1,
                                                   const long long* __restrict__ seg, unsigned long long* __restrict__ keys) {
    const int lane = threadIdx.x & 31;
    const int64_t pair = p0 + (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (pair >= p1) return;
    const int64_t w = pair / p.n_slots;
    const int c = (int)(pair % p.n_slots);
    const long long* cc = p.cnt + (size_t)c * (p.S + 1);
    const long long a = cc[p.lo[w]], b = cc[p.hi[w]];
    const double* x = p.comp + (size_t)c * p.S + a;
    unsigned long long* d = keys + seg[pair - p0];
    for (long long i = lane; i < b - a; i += 32) d[i] = dkey(x[i]);
}

// ONE THREAD PER (window, slot) of the batch: median (the mean of the middle one or two, as np.median) and the linear
// quantiles (numpy's lerp: b - (b - a)(1 - g) for g >= 0.5 or at the last value, else a + (b - a) g)
__global__ void k_ws_pick(const __grid_constant__ StatParams p, int64_t p0, int64_t p1, const long long* __restrict__ seg,
                          const unsigned long long* __restrict__ keys) {
    const int64_t pair = p0 + (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (pair >= p1) return;
    const long long s0 = seg[pair - p0], n = seg[pair - p0 + 1] - s0;
    const unsigned long long* s = keys + s0;
    double* o = p.out + (size_t)pair * p.K;
    const double qnan = __longlong_as_double(0x7ff8000000000000ll);
    for (int k = 0; k < p.K; ++k) {
        if (p.code[k] == ST_MEDIAN) {
            if (n == 0) o[k] = qnan;
            else if (n & 1) o[k] = 0.0 + (-0.0 + dval(s[n / 2]));
            else o[k] = (0.0 + ((-0.0 + dval(s[n / 2 - 1])) + dval(s[n / 2]))) / 2.0;
        } else if (p.code[k] == ST_QUANTILE) {
            if (n == 0) {
                o[k] = qnan;
                continue;
            }
            const double v = (double)(n - 1) * p.q[k];
            const double fl = floor(v);
            const double g = v - fl;
            const long long i = min((long long)fl, n - 1);         // at or past the last value: both neighbours are it
            const double A = dval(s[i]), B = dval(s[min(i + 1, n - 1)]);
            const double diff = B - A;
            o[k] = (g >= 0.5 || i == n - 1) ? B - diff * (1.0 - g) : A + diff * g;
        }
    }
}

struct WsState {
    int n_cols = 0, n_slots = 0, n_fields = -1;
    bool spec = false, final = false;
    PgBuf spec_tab;                     // col_slot [n_cols], slot_col [n_slots]
    double* vals = nullptr;             // [n_slots x cap]
    long long* pos = nullptr;           // [cap]
    int64_t S = 0, cap = 0;
    // the current chunk
    PgBuf hash, tok, err, cub, runs, flagged;
    int64_t chunk_S = 0, n_runs = 0, n_flag = 0;
    uint64_t text_gen = 0;
    // after the compaction
    PgBuf comp, cnt, win, keys, seg, out;
    void free_vals() {
        if (vals) cudaFree(vals);
        if (pos) cudaFree(pos);
        vals = nullptr;
        pos = nullptr;
    }
};

WsState* wstate(pg_ctx* ctx) {
    if (!ctx->ws_state) ctx->ws_state = new WsState();
    return (WsState*)ctx->ws_state;
}

// grow the resident values and positions to hold `need` lines, keeping the first ws->S
int ws_grow(pg_ctx* ctx, WsState* ws, int64_t need) {
    if (need <= ws->cap) return PG_OK;
    const int64_t cap = std::max<int64_t>(need, ws->cap + ws->cap / 2);
    const size_t bytes = (size_t)cap * 8 * (ws->n_slots + 1);
    size_t free_b = 0, total_b = 0;
    PG_CUDA(cudaMemGetInfo(&free_b, &total_b));
    PG_CHECK(bytes + (256u << 20) <= free_b, "windowStats: the values of %lld lines x %d columns (%.1f GiB) do not fit in the "
             "%.1f GiB of free device memory", (long long)cap, ws->n_slots, bytes / 1073741824.0, free_b / 1073741824.0);
    double* v = nullptr;
    long long* p = nullptr;
    PG_CUDA(cudaMalloc(&v, (size_t)cap * 8 * std::max(ws->n_slots, 1)));
    PG_CUDA(cudaMalloc(&p, (size_t)cap * 8));
    if (ws->S > 0) {
        if (ws->n_slots)
            PG_CUDA(cudaMemcpy2DAsync(v, (size_t)cap * 8, ws->vals, (size_t)ws->cap * 8, (size_t)ws->S * 8, ws->n_slots,
                                      cudaMemcpyDeviceToDevice, ctx->stream));
        PG_CUDA(cudaMemcpyAsync(p, ws->pos, (size_t)ws->S * 8, cudaMemcpyDeviceToDevice, ctx->stream));
        PG_CUDA(cudaStreamSynchronize(ctx->stream));
    }
    ws->free_vals();
    ws->vals = v;
    ws->pos = p;
    ws->cap = cap;
    return PG_OK;
}

}  // namespace

void pg_ws_free(pg_ctx* ctx) {
    WsState* ws = (WsState*)ctx->ws_state;
    if (!ws) return;
    ws->free_vals();
    PgBuf* bufs[] = {&ws->spec_tab, &ws->hash, &ws->tok, &ws->err, &ws->cub, &ws->runs, &ws->flagged, &ws->comp, &ws->cnt,
                     &ws->win, &ws->keys, &ws->seg, &ws->out};
    for (PgBuf* b : bufs) b->release();
    delete ws;
    ctx->ws_state = nullptr;
}

extern "C" int pg_ws_spec(pg_ctx* ctx, int32_t n_cols, const int32_t* col_slot, int32_t n_slots, int32_t n_fields) {
    PG_CHECK(ctx && (n_cols == 0 || col_slot), "pg_ws_spec: null argument");
    PG_CHECK(n_cols >= 0 && n_slots >= 0 && n_fields >= -1, "pg_ws_spec: %d columns, %d slots, %d fields", n_cols, n_slots,
             n_fields);
    std::vector<int32_t> slot_col((size_t)n_slots, -1);
    for (int c = 0; c < n_cols; ++c) {
        PG_CHECK(col_slot[c] >= -1 && col_slot[c] < n_slots, "pg_ws_spec: column %d has slot %d of %d", c, col_slot[c], n_slots);
        if (col_slot[c] >= 0) {
            PG_CHECK(slot_col[col_slot[c]] < 0, "pg_ws_spec: slot %d is read by two columns", col_slot[c]);
            slot_col[col_slot[c]] = c;
        }
    }
    for (int k = 0; k < n_slots; ++k) PG_CHECK(slot_col[k] >= 0, "pg_ws_spec: slot %d is read by no column", k);
    PG_CUDA(cudaSetDevice(ctx->device));
    pg_ws_free(ctx);
    WsState* ws = wstate(ctx);
    std::vector<int32_t> tab(col_slot, col_slot + n_cols);
    tab.insert(tab.end(), slot_col.begin(), slot_col.end());
    PG_TRY(ws->spec_tab.ensure(tab.size() * 4 + 64));
    PG_CUDA(cudaMemcpyAsync(ws->spec_tab.p, tab.data(), tab.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
    static bool pow5_up[64] = {};
    if (!pow5_up[ctx->device & 63]) {
        PG_CUDA(cudaMemcpyToSymbol(d_pow5, pg_pow5_128, sizeof(pg_pow5_128)));
        pow5_up[ctx->device & 63] = true;
    }
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    ws->n_cols = n_cols;
    ws->n_slots = n_slots;
    ws->n_fields = n_fields;
    ws->spec = true;
    return PG_OK;
}

extern "C" int pg_ws_chunk(pg_ctx* ctx, const char* text, size_t len, int64_t* n_lines, int64_t* n_runs, int64_t* n_flag,
                           int64_t* error) {
    PG_CHECK(ctx && (text || len == 0) && n_lines && n_runs && n_flag && error, "pg_ws_chunk: null argument");
    WsState* ws = wstate(ctx);
    PG_CHECK(ws->spec, "pg_ws_chunk: no pg_ws_spec");
    PG_CHECK(!ws->final, "pg_ws_chunk: the values are already compacted (pg_ws_stats); start again with pg_ws_spec");
    PG_CHECK(len < ((size_t)1 << 32), "pg_ws_chunk: a chunk of %zu bytes (a line of 4 GiB or more; token offsets are 32-bit)",
             len);
    *n_lines = *n_runs = *n_flag = 0;
    for (int k = 0; k < 3; ++k) error[k] = 0;
    PG_CUDA(cudaSetDevice(ctx->device));
    pg_timings_reset(ctx);
    int64_t S = 0;
    PG_TRY(pg_text_load(ctx, text ? text : "", -1, 0, len, &S));
    ctx->ingest_sites = -1;                             // the text no longer belongs to the resident matrix
    PG_TRY(ws_grow(ctx, ws, ws->S + S));
    const size_t nt = (size_t)S * ws->n_slots;
    PG_TRY(ws->hash.ensure((size_t)S * 8 + 64));
    PG_TRY(ws->tok.ensure(nt * 8 + 64));
    PG_TRY(ws->runs.ensure((size_t)(S + 1) * 16 + 64));
    PG_TRY(ws->flagged.ensure(nt * 16 + 64));
    PG_TRY(ws->err.ensure((size_t)S + 128));            // the error word, the selected count, the scaffold flags
    unsigned long long* d_err = (unsigned long long*)ws->err.p;
    int64_t* d_n = (int64_t*)(d_err + 1);
    int8_t* d_flags = (int8_t*)(d_n + 1);
    PG_CUDA(cudaMemsetAsync(d_err, 0xff, 8, ctx->stream));
    PG_CUDA(cudaMemsetAsync(ws->tok.p, 0, nt * 8 + 8, ctx->stream));
    ws->chunk_S = S;
    ws->n_runs = ws->n_flag = 0;
    ws->text_gen = ctx->text_gen;
    if (S > 0) {
        LineParams p;
        p.buf = (const uint8_t*)ctx->text.p;
        p.len = len;
        p.starts = (const long long*)ctx->starts.p;
        p.S = S;
        p.S0 = ws->S;
        p.cap = ws->cap;
        p.n_cols = ws->n_cols;
        p.n_slots = ws->n_slots;
        p.n_fields = ws->n_fields;
        p.col_slot = (const int32_t*)ws->spec_tab.p;
        p.slot_col = p.col_slot + ws->n_cols;
        p.vals = ws->vals;
        p.pos = ws->pos;
        p.hash = (unsigned long long*)ws->hash.p;
        p.tok = (unsigned long long*)ws->tok.p;
        p.err = d_err;
        const unsigned grid = (unsigned)((S + 7) / 8);                 // one warp per line
        PG_TRY(pg_timed(ctx, "ws_lines", [&] { k_ws_lines<<<grid, 256, 0, ctx->stream>>>(p); }));
        PG_TRY(pg_scaffold_flags(ctx, p.hash, S, d_flags));
        long long* d_run_line = (long long*)ws->runs.p;
        thrust::counting_iterator<long long> idx(0);
        size_t tmp = 0, tmp2 = 0;
        long long* d_fidx = (long long*)ws->flagged.p;
        PG_CUDA(cub::DeviceSelect::Flagged(nullptr, tmp, idx, d_flags, d_run_line, d_n, S, ctx->stream));
        PG_CUDA(cub::DeviceSelect::If(nullptr, tmp2, idx, d_fidx, d_n + 1, (int64_t)nt, Flagged{p.tok}, ctx->stream));
        PG_TRY(ws->cub.ensure(std::max(tmp, tmp2) + 64));
        PG_TRY(pg_timed(ctx, "ws_runs", [&] {
            cub::DeviceSelect::Flagged(ws->cub.p, tmp, idx, d_flags, d_run_line, d_n, S, ctx->stream);
        }));
        if (nt > 0)
            PG_TRY(pg_timed(ctx, "ws_flagged", [&] {
                cub::DeviceSelect::If(ws->cub.p, tmp2, idx, d_fidx, d_n + 1, (int64_t)nt, Flagged{p.tok}, ctx->stream);
            }));
        else
            PG_CUDA(cudaMemsetAsync(d_n + 1, 0, 8, ctx->stream));
        int64_t h[2] = {0, 0};
        unsigned long long w = ~0ull;
        PG_CUDA(cudaMemcpyAsync(h, d_n, 16, cudaMemcpyDeviceToHost, ctx->stream));
        PG_CUDA(cudaMemcpyAsync(&w, d_err, 8, cudaMemcpyDeviceToHost, ctx->stream));
        PG_CUDA(cudaStreamSynchronize(ctx->stream));
        ws->n_runs = h[0];
        ws->n_flag = h[1];
        PG_TRY(pg_timed(ctx, "ws_runs", [&] {
            k_ws_run_off<<<(unsigned)std::min<int64_t>((h[0] + 255) / 256, 1024), 256, 0, ctx->stream>>>(
                p.starts, d_run_line, h[0], d_run_line + (S + 1));
        }));
        if (h[1] > 0)
            PG_TRY(pg_timed(ctx, "ws_flagged", [&] {
                k_ws_gather_u64<<<(unsigned)std::min<int64_t>((h[1] + 255) / 256, 1024), 256, 0, ctx->stream>>>(
                    p.tok, d_fidx, h[1], (unsigned long long*)(d_fidx + nt));
            }));
        ctx->launches += 6;
        if (w != ~0ull) {
            error[0] = (int64_t)(w & 15ull);
            error[1] = (int64_t)(w >> 28) - 1;
            error[2] = (int64_t)((w >> 4) & 0xffffffull);
        }
    }
    ws->S += S;
    *n_lines = S;
    *n_runs = ws->n_runs;
    *n_flag = ws->n_flag;
    return PG_OK;
}

extern "C" int pg_ws_chunk_info(pg_ctx* ctx, int64_t* run_line, int64_t* run_off, int64_t* flag_idx, uint64_t* flag_tok) {
    PG_CHECK(ctx, "pg_ws_chunk_info: null argument");
    WsState* ws = wstate(ctx);
    PG_CHECK(ws->spec && ws->text_gen == ctx->text_gen && !ws->final, "pg_ws_chunk_info: no pg_ws_chunk on the current text");
    PG_CUDA(cudaSetDevice(ctx->device));
    const long long* d = (const long long*)ws->runs.p;
    const size_t nt = (size_t)ws->chunk_S * ws->n_slots;
    if (ws->n_runs && run_line && run_off) {
        PG_CUDA(cudaMemcpyAsync(run_line, d, (size_t)ws->n_runs * 8, cudaMemcpyDeviceToHost, ctx->stream));
        PG_CUDA(cudaMemcpyAsync(run_off, d + (ws->chunk_S + 1), (size_t)ws->n_runs * 8, cudaMemcpyDeviceToHost, ctx->stream));
    }
    if (ws->n_flag && flag_idx && flag_tok) {
        const long long* f = (const long long*)ws->flagged.p;
        PG_CUDA(cudaMemcpyAsync(flag_idx, f, (size_t)ws->n_flag * 8, cudaMemcpyDeviceToHost, ctx->stream));
        PG_CUDA(cudaMemcpyAsync(flag_tok, f + nt, (size_t)ws->n_flag * 8, cudaMemcpyDeviceToHost, ctx->stream));
    }
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    return PG_OK;
}

extern "C" int pg_ws_set_values(pg_ctx* ctx, int64_t n, const int64_t* line, const int32_t* slot, const double* v) {
    PG_CHECK(ctx && (n == 0 || (line && slot && v)), "pg_ws_set_values: null argument");
    WsState* ws = wstate(ctx);
    PG_CHECK(ws->spec && !ws->final, "pg_ws_set_values: no values to set");
    if (n == 0) return PG_OK;
    std::vector<long long> at((size_t)n);
    for (int64_t i = 0; i < n; ++i) {
        PG_CHECK(line[i] >= 0 && line[i] < ws->S && slot[i] >= 0 && slot[i] < ws->n_slots,
                 "pg_ws_set_values: line %lld, slot %d of %lld x %d", (long long)line[i], slot[i], (long long)ws->S, ws->n_slots);
        at[(size_t)i] = (long long)slot[i] * ws->cap + line[i];
    }
    PG_CUDA(cudaSetDevice(ctx->device));
    PG_TRY(ws->win.ensure((size_t)n * 16 + 64));
    long long* d_at = (long long*)ws->win.p;
    double* d_v = (double*)(d_at + n);
    PG_CUDA(cudaMemcpyAsync(d_at, at.data(), (size_t)n * 8, cudaMemcpyHostToDevice, ctx->stream));
    PG_CUDA(cudaMemcpyAsync(d_v, v, (size_t)n * 8, cudaMemcpyHostToDevice, ctx->stream));
    PG_TRY(pg_timed(ctx, "ws_set", [&] {
        k_ws_scatter<<<(unsigned)std::min<int64_t>((n + 255) / 256, 1024), 256, 0, ctx->stream>>>(d_at, d_v, n, ws->vals);
    }));
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    return PG_OK;
}

extern "C" int pg_ws_meta(pg_ctx* ctx, int64_t* n_lines, int64_t* pos) {
    PG_CHECK(ctx && n_lines, "pg_ws_meta: null argument");
    WsState* ws = wstate(ctx);
    PG_CHECK(ws->spec && !ws->final, "pg_ws_meta: no pg_ws_spec, or the positions are gone after pg_ws_stats");
    *n_lines = ws->S;
    if (!pos || ws->S == 0) return PG_OK;
    PG_CUDA(cudaSetDevice(ctx->device));
    return pg_d2h_staged(ctx, pos, ws->pos, (size_t)ws->S * 8);
}

extern "C" int pg_ws_stats(pg_ctx* ctx, int64_t W, const int64_t* lo, const int64_t* hi, int32_t K, const int32_t* code,
                           const double* q, int64_t sort_budget, double* out, int64_t* n_out) {
    PG_CHECK(ctx && (W == 0 || (lo && hi && out && n_out)) && (K == 0 || (code && q)), "pg_ws_stats: null argument");
    WsState* ws = wstate(ctx);
    PG_CHECK(ws->spec, "pg_ws_stats: no pg_ws_spec");
    PG_CHECK(K >= 0 && K <= MAX_STATS, "pg_ws_stats: %d statistics (at most %d)", K, MAX_STATS);
    bool order = false;
    for (int k = 0; k < K; ++k) {
        PG_CHECK(code[k] >= 0 && code[k] <= ST_QUANTILE, "pg_ws_stats: statistic code %d", code[k]);
        PG_CHECK(code[k] != ST_QUANTILE || (q[k] >= 0.0 && q[k] <= 1.0), "pg_ws_stats: quantile %g", q[k]);
        order |= code[k] == ST_MEDIAN || code[k] == ST_QUANTILE;
    }
    const int64_t S = ws->S;
    for (int64_t w = 0; w < W; ++w)
        PG_CHECK(lo[w] >= 0 && lo[w] <= hi[w] && hi[w] <= S, "pg_ws_stats: window %lld spans lines [%lld, %lld) of %lld",
                 (long long)w, (long long)lo[w], (long long)hi[w], (long long)S);
    PG_CUDA(cudaSetDevice(ctx->device));
    pg_timings_reset(ctx);
    const int C = ws->n_slots;
    if (!ws->final) {                                   // compact every slot's non-NaN values, count them, free the rest
        PG_TRY(ws->comp.ensure((size_t)std::max<int64_t>(S, 1) * std::max(C, 1) * 8 + 64));
        PG_TRY(ws->cnt.ensure((size_t)(S + 1) * std::max(C, 1) * 8 + 64));
        PG_TRY(ws->err.ensure(128));
        int64_t* d_n = (int64_t*)ws->err.p;
        size_t t1 = 0, t2 = 0;
        for (int c = 0; c < C; ++c) {
            const double* v = ws->vals + (size_t)c * ws->cap;
            auto flags = thrust::make_transform_iterator(thrust::counting_iterator<int64_t>(0), NotNan{v, S});
            PG_CUDA(cub::DeviceSelect::If(nullptr, t1, v, (double*)ws->comp.p, d_n, S, IsNotNan{}, ctx->stream));
            PG_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, t2, flags, (long long*)ws->cnt.p, S + 1, ctx->stream));
            PG_TRY(ws->cub.ensure(std::max(t1, t2) + 64));
            double* dst = (double*)ws->comp.p + (size_t)c * S;
            long long* cnt = (long long*)ws->cnt.p + (size_t)c * (S + 1);
            PG_TRY(pg_timed(ctx, "ws_compact", [&] {
                cub::DeviceSelect::If(ws->cub.p, t1, v, dst, d_n, S, IsNotNan{}, ctx->stream);
            }));
            PG_TRY(pg_timed(ctx, "ws_count", [&] {
                cub::DeviceScan::ExclusiveSum(ws->cub.p, t2, flags, cnt, S + 1, ctx->stream);
            }));
            ctx->launches += 2;
        }
        PG_CUDA(cudaStreamSynchronize(ctx->stream));
        ws->free_vals();
        ws->cap = 0;
        PgBuf* chunk_bufs[] = {&ws->hash, &ws->tok, &ws->runs, &ws->flagged};
        for (PgBuf* b : chunk_bufs) b->release();
        ws->final = true;
    }
    if (W == 0 || C == 0) return PG_OK;
    StatParams p;
    memset(&p, 0, sizeof(p));
    p.comp = (const double*)ws->comp.p;
    p.cnt = (const long long*)ws->cnt.p;
    p.S = S;
    p.n_slots = C;
    p.W = W;
    p.K = K;
    for (int k = 0; k < K; ++k) {
        p.code[k] = code[k];
        p.q[k] = q[k];
    }
    PG_TRY(ws->win.ensure((size_t)W * 16 + 64));
    PG_TRY(ws->out.ensure((size_t)W * C * (K + 1) * 8 + 64));
    long long* d_lo = (long long*)ws->win.p;
    PG_CUDA(cudaMemcpyAsync(d_lo, lo, (size_t)W * 8, cudaMemcpyHostToDevice, ctx->stream));
    PG_CUDA(cudaMemcpyAsync(d_lo + W, hi, (size_t)W * 8, cudaMemcpyHostToDevice, ctx->stream));
    p.lo = d_lo;
    p.hi = d_lo + W;
    p.out = (double*)ws->out.p;
    p.n_out = (long long*)(p.out + (size_t)W * C * K);
    const int64_t pairs = W * C;
    PG_TRY(pg_timed(ctx, "ws_moments", [&] { k_ws_moments<<<(unsigned)((pairs + 3) / 4), 128, 0, ctx->stream>>>(p); }));
    ctx->launches += 1;
    PG_CUDA(cudaMemcpyAsync(n_out, p.n_out, (size_t)pairs * 8, cudaMemcpyDeviceToHost, ctx->stream));
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    if (order) {
        const int64_t budget = std::max<int64_t>(sort_budget, 8) / 8;      // keys per batch (one window at least)
        std::vector<long long> seg;
        for (int64_t p0 = 0; p0 < pairs;) {
            seg.assign(1, 0);
            int64_t p1 = p0;
            while (p1 < pairs && (p1 == p0 || seg.back() + n_out[p1] <= budget)) {
                seg.push_back(seg.back() + n_out[p1]);
                ++p1;
            }
            const int64_t nseg = p1 - p0, nkeys = seg.back();
            PG_TRY(ws->seg.ensure((size_t)(nseg + 1) * 8 + 64));
            PG_TRY(ws->keys.ensure((size_t)std::max<int64_t>(nkeys, 1) * 16 + 64));
            long long* d_seg = (long long*)ws->seg.p;
            unsigned long long* k_in = (unsigned long long*)ws->keys.p;
            unsigned long long* k_out = k_in + std::max<int64_t>(nkeys, 1);
            PG_CUDA(cudaMemcpyAsync(d_seg, seg.data(), (size_t)(nseg + 1) * 8, cudaMemcpyHostToDevice, ctx->stream));
            PG_TRY(pg_timed(ctx, "ws_gather", [&] {
                k_ws_gather<<<(unsigned)((nseg + 7) / 8), 256, 0, ctx->stream>>>(p, p0, p1, d_seg, k_in);
            }));
            size_t tmp = 0;
            PG_CUDA(cub::DeviceSegmentedSort::SortKeys(nullptr, tmp, k_in, k_out, nkeys, nseg, d_seg, d_seg + 1, ctx->stream));
            PG_TRY(ws->cub.ensure(tmp + 64));
            PG_TRY(pg_timed(ctx, "ws_sort", [&] {
                cub::DeviceSegmentedSort::SortKeys(ws->cub.p, tmp, k_in, k_out, nkeys, nseg, d_seg, d_seg + 1, ctx->stream);
            }));
            PG_TRY(pg_timed(ctx, "ws_pick", [&] {
                k_ws_pick<<<(unsigned)((nseg + 127) / 128), 128, 0, ctx->stream>>>(p, p0, p1, d_seg, k_out);
            }));
            ctx->launches += 3;
            PG_CUDA(cudaStreamSynchronize(ctx->stream));
            p0 = p1;
        }
    }
    PG_TRY(pg_d2h_staged(ctx, out, p.out, (size_t)pairs * K * 8));
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    return PG_OK;
}
