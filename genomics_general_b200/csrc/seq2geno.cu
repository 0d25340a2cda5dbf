// seqToGeno.py on the device: FASTA / PHYLIP alignments -> .geno rows (seqToGeno.py:37-98, genomics.parseFasta /
// parsePhylip / haploToPhased, genomics.py:2256-2283, 412-446).
//
// The sequences reach one resident layout (seq bytes, {rec_off, rec_len} per sequence) by one of two loaders:
//   FASTA  : fasta.cu's shared loader (pg_s2g_fasta_load / _starts / _index), as genoToVCF loads its reference.
//   PHYLIP : ingest.cu's pg_text_load uploads the text and indexes its lines; k_s2g_lines gives every line ONE WARP
//            (pg_warp_fields, str.split()'s classification): the spans of fields 0 and 1, the field count, and whether the
//            line is a header (its first two fields pass Python's int(), the count N parsed).  The host reads the line table
//            back, checks the structure and gives every used field-1 span its destination (numpy prefix sums per sequence);
//            k_s2g_gather copies the spans, cut into pieces of at most S2G_PIECE bytes, one CTA per piece.
// The plan (pg_s2g_plan) is a list of blocks, each one contig of the output: a name, a row count and its member sequences in
// output order, each with the byte that follows it in a row ('|' inside a ploidy group, '\t' after a group, '\n' after the
// last).  Row x of block b (position x + 1) is "name\t<x + 1>\t" then two bytes per member, so its length is
// name + digits(x + 1) + 2 + 2M and its offset is closed-form over the decimal-digit ranges: no per-row scan.
// k_s2g_tile is the transpose: a CTA stages a tile of TS sites x TM members in shared memory, reading along each member's
// sequence (consecutive threads, consecutive sites), then writes the tile's rows, consecutive threads on consecutive bytes
// of one row; the CTAs of a site tile's first member tile also write the rows' prefixes.  The output is cut into slabs of a
// byte range; a row may end in the next slab.
#include <algorithm>
#include <cub/cub.cuh>

#include "pgwin_internal.h"

namespace {

constexpr int TS = 64;              // sites per tile
constexpr int TM = 32;              // member sequences per tile
constexpr int TPITCH = TS + 4;      // shared-memory row of one member (conflict-free reads across members)
constexpr int64_t S2G_PIECE = 1 << 16;
constexpr int LINE_WORDS = 7;       // the line table: {f0, f0_len, f1, f1_len, n_fields, flags, head_n} int64 per line
enum { LF_HI = 1, LF_CR = 2, LF_HEAD = 4 };

// digits of v >= 1
__host__ __device__ __forceinline__ int s2g_digits(int64_t v) {
    int n = 1;
    while (v >= 10) v /= 10, ++n;
    return n;
}

// sum of digits(i) for i = 1..x: every power of ten p <= x adds one digit to the x - p + 1 numbers from p on
__host__ __device__ __forceinline__ int64_t s2g_digits_upto(int64_t x) {
    int64_t s = 0;
    for (int64_t p = 1; p <= x; p *= 10) {
        s += x - p + 1;
        if (p > INT64_MAX / 10) break;
    }
    return s;
}

struct Block {
    int64_t byte_off;   // first byte of the block's rows in the output
    int64_t name_off, name_len;
    int64_t rows;
    int64_t mem0, M;    // members [mem0, mem0 + M) of the member tables
    int64_t width;      // row bytes without the position's digits: name + 2 + 2M
    int64_t task0;      // first CTA task of the block: ceil(rows / TS) x ceil(M / TM) tasks
};

// byte offset of row x in its block
__host__ __device__ __forceinline__ int64_t row_off(const Block& b, int64_t x) { return x * b.width + s2g_digits_upto(x); }

// token end: the first blank or '\n' from byte q, one warp scanning 128 bytes per step
__device__ __forceinline__ size_t warp_token_end(const uint8_t* buf, size_t len, size_t q) {
    const int lane = threadIdx.x & 31;
    for (size_t base = q;; base += 128) {
        int first = 4;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const unsigned c = pg_byte_at(buf, len, base + (size_t)lane * 4 + k);
            if (first == 4 && (c == '\n' || pg_sblank(c))) first = k;
        }
        const unsigned hit = __ballot_sync(0xffffffffu, first < 4);
        if (hit) {
            const int l = __ffs(hit) - 1;
            return base + (size_t)l * 4 + (size_t)__shfl_sync(0xffffffffu, first, l);
        }
    }
}

// Python int() of an ASCII token [q, e): [+-]?[0-9](_?[0-9])*; *v = its value, clamped to int64
__device__ __forceinline__ bool py_int(const uint8_t* buf, size_t q, size_t e, int64_t* v) {
    bool neg = false;
    if (q < e && (buf[q] == '+' || buf[q] == '-')) neg = buf[q++] == '-';
    if (q == e) return false;
    unsigned long long u = 0;
    bool over = false, prev_digit = false;
    for (; q < e; ++q) {
        const unsigned c = buf[q];
        if (c >= '0' && c <= '9') {
            if (u > (~0ull - 9) / 10) over = true;
            else u = u * 10 + (c - '0');
            prev_digit = true;
        } else if (c == '_' && prev_digit && q + 1 < e) {
            prev_digit = false;
        } else {
            return false;
        }
    }
    if (!prev_digit) return false;
    if (over || u > (unsigned long long)INT64_MAX) *v = neg ? INT64_MIN : INT64_MAX;
    else *v = neg ? -(int64_t)u : (int64_t)u;
    return true;
}

__global__ void __launch_bounds__(256) k_s2g_lines(const uint8_t* __restrict__ buf, size_t len,
                                                   const long long* __restrict__ starts, int64_t S, int64_t* __restrict__ tab) {
    const int lane = threadIdx.x & 31;
    const int64_t line = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (line >= S) return;
    long long f[2] = {-1, -1};
    bool hi = false, lone_cr = false;
    const unsigned n_fields = pg_warp_fields(buf, len, (size_t)starts[line], &hi, &lone_cr, [&](unsigned fidx, size_t q) {
        if (fidx == 0) f[0] = (long long)q;
        else if (fidx == 1) f[1] = (long long)q;
    });
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1)
#pragma unroll
        for (int k = 0; k < 2; ++k) f[k] = max(f[k], __shfl_xor_sync(0xffffffffu, f[k], d));
    int64_t e[2] = {0, 0};
#pragma unroll
    for (int k = 0; k < 2; ++k)
        if (f[k] >= 0) e[k] = (int64_t)warp_token_end(buf, len, (size_t)f[k]);
    if (lane != 0) return;
    int64_t flags = (hi ? LF_HI : 0) | (lone_cr ? LF_CR : 0), n = 0, l = 0;
    if (f[1] >= 0 && py_int(buf, (size_t)f[0], (size_t)e[0], &n) && py_int(buf, (size_t)f[1], (size_t)e[1], &l))
        flags |= LF_HEAD;
    int64_t* t = tab + line * LINE_WORDS;
    t[0] = f[0];
    t[1] = f[0] >= 0 ? e[0] - f[0] : 0;
    t[2] = f[1];
    t[3] = f[1] >= 0 ? e[1] - f[1] : 0;
    t[4] = n_fields;
    t[5] = flags;
    t[6] = (flags & LF_HEAD) ? n : 0;
}

// the PHYLIP sequences: piece k copies piece[3k + 2] bytes from text byte piece[3k] to sequence byte piece[3k + 1]
__global__ void __launch_bounds__(256) k_s2g_gather(const uint8_t* __restrict__ text, const int64_t* __restrict__ piece,
                                                    int64_t n_piece, uint8_t* __restrict__ seq) {
    for (int64_t k = blockIdx.x; k < n_piece; k += gridDim.x) {
        const int64_t src = piece[3 * k], dst = piece[3 * k + 1], n = piece[3 * k + 2];
        for (int64_t i = threadIdx.x; i < n; i += blockDim.x) seq[dst + i] = text[src + i];
    }
}

struct EmitParams {
    const uint8_t* seq;
    const int64_t* rec_off;     // [n_rec]
    const Block* blk;           // [n_blk]
    const int64_t* task0;       // [n_blk + 1]
    int64_t n_blk;
    const char* names;
    const int64_t* mem_rec;     // [n_mem] the member's sequence
    const uint8_t* mem_sep;     // [n_mem] the byte after it
    int64_t t0;                 // first task of the launch
    int64_t b0, b1;             // the slab: output bytes [b0, b1)
    char* out;
};

__device__ __forceinline__ void put(const EmitParams& p, int64_t at, char c) {
    if (at >= p.b0 && at < p.b1) p.out[at - p.b0] = c;
}

__global__ void __launch_bounds__(256) k_s2g_tile(const __grid_constant__ EmitParams p) {
    __shared__ uint8_t tile[TM * TPITCH];
    __shared__ int64_t m_off[TM];
    __shared__ uint8_t m_sep[TM];
    const int64_t t = p.t0 + blockIdx.x;
    int64_t a = 0, z = p.n_blk - 1;                     // the last block with task0 <= t
    while (a < z) {
        const int64_t mid = (a + z + 1) >> 1;
        if (p.task0[mid] <= t) a = mid;
        else z = mid - 1;
    }
    const Block b = p.blk[a];
    const int64_t mt = (b.M + TM - 1) / TM;
    const int64_t local = t - b.task0;
    const int64_t x0 = (local / mt) * TS, m0 = (local % mt) * TM;
    const int nx = (int)min((int64_t)TS, b.rows - x0), nm = (int)min((int64_t)TM, b.M - m0);
    const int64_t base = b.byte_off + row_off(b, x0);
    if (base >= p.b1 || b.byte_off + row_off(b, x0 + nx) <= p.b0) return;   // the tile's rows miss the slab
    if (threadIdx.x < nm) {
        const int64_t m = b.mem0 + m0 + threadIdx.x;
        m_off[threadIdx.x] = p.rec_off[p.mem_rec[m]] + x0;
        m_sep[threadIdx.x] = p.mem_sep[m];
    }
    __syncthreads();
    for (int i = threadIdx.x; i < nm * TS; i += blockDim.x) {     // along each member's sequence
        const int j = i / TS, x = i % TS;
        if (x < nx) tile[j * TPITCH + x] = p.seq[m_off[j] + x];
    }
    __syncthreads();
    const int rb = 2 * nm;                              // the tile's bytes of one row
    for (int i = threadIdx.x; i < nx * rb; i += blockDim.x) {
        const int x = i / rb, k = i % rb;
        const int64_t row = x0 + x;
        const int64_t at = b.byte_off + row_off(b, row) + b.name_len + 2 + s2g_digits(row + 1) + 2 * m0 + k;
        put(p, at, (k & 1) ? (char)m_sep[k >> 1] : (char)tile[(k >> 1) * TPITCH + x]);
    }
    if (m0 != 0) return;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int x = warp; x < nx; x += blockDim.x >> 5) {  // the prefixes "name\t<x + 1>\t", one warp per row
        const int64_t row = x0 + x;
        const int64_t o = b.byte_off + row_off(b, row);
        for (int64_t i = lane; i < b.name_len; i += 32) put(p, o + i, p.names[b.name_off + i]);
        const int nd = s2g_digits(row + 1);
        if (lane == 0) {
            put(p, o + b.name_len, '\t');
            put(p, o + b.name_len + 1 + nd, '\t');
        }
        if (lane < nd) {
            int64_t v = row + 1;
            for (int i = nd - 1; i > lane; --i) v /= 10;
            put(p, o + b.name_len + 1 + lane, (char)('0' + v % 10));
        }
    }
}

struct S2gState {
    PgFasta fa;                 // the resident sequences (both formats) and, for FASTA, the loader's buffers
    PgBuf lines, pieces, plan, out;
    int fmt = -1;               // 0 FASTA, 1 PHYLIP
    int64_t S = -1;             // PHYLIP lines of the line table
    size_t len = 0;
    uint64_t text_gen = 0;
    std::vector<int64_t> rec_len;
    // the plan: blocks, their tasks, the names and member tables (device copies in `plan`)
    std::vector<Block> blk;
    int64_t n_tasks = 0, total = 0, n_mem = 0, names_len = 0;
    bool planned = false;
};

S2gState* sstate(pg_ctx* ctx) {
    if (!ctx->s2g_state) ctx->s2g_state = new S2gState();
    return (S2gState*)ctx->s2g_state;
}

// the input of len bytes and `extra` more bytes of device buffers must fit in device memory with 1 GiB to spare
int fits(pg_ctx* ctx, const char* who, size_t len, size_t extra) {
    size_t free_b = 0, total_b = 0;
    PG_CUDA(cudaMemGetInfo(&free_b, &total_b));
    const size_t need = len + extra + ((size_t)1 << 30);
    PG_CHECK(need <= free_b, "%s: the input of %zu bytes needs %zu bytes of device memory with 1 GiB to spare (%zu free); "
             "do not fit in device memory", who, len, need, free_b);
    return PG_OK;
}

void reset(S2gState* ss) {
    ss->fa.release();
    ss->lines.release();
    ss->pieces.release();
    ss->plan.release();
    ss->rec_len.clear();
    ss->blk.clear();
    ss->S = -1;
    ss->fmt = -1;
    ss->planned = false;
}

}  // namespace

void pg_s2g_free(pg_ctx* ctx) {
    S2gState* ss = (S2gState*)ctx->s2g_state;
    if (!ss) return;
    reset(ss);
    ss->out.release();
    delete ss;
    ctx->s2g_state = nullptr;
}

extern "C" int pg_s2g_fasta_load(pg_ctx* ctx, const char* text, size_t len, int64_t* n_rec) {
    PG_CHECK(ctx && (text || len == 0) && n_rec, "pg_s2g_fasta_load: null argument");
    *n_rec = 0;
    PG_CUDA(cudaSetDevice(ctx->device));
    pg_timings_reset(ctx);
    S2gState* ss = sstate(ctx);
    reset(ss);
    PG_TRY(fits(ctx, "pg_s2g_fasta_load", len, 2 * len));       // text, flags, sequences
    PG_TRY(pg_fa_load(ctx, ss->fa, text, len, "s2g", n_rec));
    ss->fmt = 0;
    return PG_OK;
}

extern "C" int pg_s2g_fasta_starts(pg_ctx* ctx, int64_t* starts) {
    PG_CHECK(ctx && starts, "pg_s2g_fasta_starts: null argument");
    S2gState* ss = sstate(ctx);
    PG_CHECK(ss->fmt == 0 && !ss->fa.indexed, "pg_s2g_fasta_starts: no pg_s2g_fasta_load before it");
    PG_CUDA(cudaSetDevice(ctx->device));
    return pg_fa_starts(ctx, ss->fa, starts);
}

extern "C" int pg_s2g_fasta_index(pg_ctx* ctx, int64_t n_rec, const int64_t* lo, const int64_t* hi, int64_t* rec_len) {
    PG_CHECK(ctx && (n_rec == 0 || (lo && hi && rec_len)), "pg_s2g_fasta_index: null argument");
    S2gState* ss = sstate(ctx);
    PG_CHECK(ss->fmt == 0 && !ss->fa.indexed && n_rec == ss->fa.n_rec,
             "pg_s2g_fasta_index: %lld records, the last pg_s2g_fasta_load found %lld", (long long)n_rec,
             (long long)ss->fa.n_rec);
    for (int64_t k = 0; k < n_rec; ++k)
        PG_CHECK(lo[k] >= 0 && lo[k] <= hi[k] && hi[k] <= (int64_t)ss->fa.fa_len && (k == 0 || lo[k] >= hi[k - 1]),
                 "pg_s2g_fasta_index: record %lld spans [%lld, %lld) (sorted, disjoint, inside the %zu bytes)", (long long)k,
                 (long long)lo[k], (long long)hi[k], ss->fa.fa_len);
    PG_CUDA(cudaSetDevice(ctx->device));
    pg_timings_reset(ctx);
    if (n_rec == 0) {                                   // no records: an empty layout
        ss->fa.fa.release();
        ss->fa.flags.release();
        ss->fa.indexed = true;
        return PG_OK;
    }
    PG_TRY(pg_fa_index(ctx, ss->fa, n_rec, lo, hi, "s2g", rec_len));
    ss->rec_len.assign(rec_len, rec_len + n_rec);
    return PG_OK;
}

extern "C" int pg_s2g_phylip_load(pg_ctx* ctx, const char* text, size_t len, int64_t* n_lines) {
    PG_CHECK(ctx && (text || len == 0) && n_lines, "pg_s2g_phylip_load: null argument");
    *n_lines = 0;
    PG_CUDA(cudaSetDevice(ctx->device));
    pg_timings_reset(ctx);
    S2gState* ss = sstate(ctx);
    reset(ss);
    const size_t nl = text ? (size_t)std::count(text, text + len, '\n') + 1 : 1;
    PG_TRY(fits(ctx, "pg_s2g_phylip_load", len, len + nl * LINE_WORDS * 8));  // text, sequences, line table
    int64_t S = 0;
    PG_TRY(pg_text_load(ctx, text ? text : "", -1, 0, len, &S));
    ctx->ingest_sites = -1;                             // the text no longer belongs to the resident matrix
    PG_TRY(ss->lines.ensure((size_t)S * LINE_WORDS * 8 + 64));
    if (S > 0) {
        PG_TRY(pg_timed(ctx, "s2g_lines", [&] {
            k_s2g_lines<<<(unsigned)((S + 7) / 8), 256, 0, ctx->stream>>>((const uint8_t*)ctx->text.p, len,
                                                                          (const long long*)ctx->starts.p, S,
                                                                          (int64_t*)ss->lines.p);
        }));
        ctx->launches += 1;
    }
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    ss->fmt = 1;
    ss->S = S;
    ss->len = len;
    ss->text_gen = ctx->text_gen;
    *n_lines = S;
    return PG_OK;
}

extern "C" int pg_s2g_phylip_lines(pg_ctx* ctx, int64_t* lines) {
    PG_CHECK(ctx && lines, "pg_s2g_phylip_lines: null argument");
    S2gState* ss = sstate(ctx);
    PG_CHECK(ss->fmt == 1 && ss->S >= 0 && ss->text_gen == ctx->text_gen, "pg_s2g_phylip_lines: no pg_s2g_phylip_load");
    if (ss->S == 0) return PG_OK;
    PG_CUDA(cudaSetDevice(ctx->device));
    PG_TRY(pg_d2h_staged(ctx, lines, ss->lines.p, (size_t)ss->S * LINE_WORDS * 8));
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    return PG_OK;
}

extern "C" int pg_s2g_phylip_pack(pg_ctx* ctx, int64_t n_seq, const int64_t* seq_len, int64_t n_span, const int64_t* span) {
    PG_CHECK(ctx && (n_seq == 0 || seq_len) && (n_span == 0 || span), "pg_s2g_phylip_pack: null argument");
    S2gState* ss = sstate(ctx);
    PG_CHECK(ss->fmt == 1 && ss->S >= 0 && ss->text_gen == ctx->text_gen, "pg_s2g_phylip_pack: no pg_s2g_phylip_load");
    std::vector<int64_t> tab((size_t)n_seq * 2);        // rec_off [n_seq], rec_len [n_seq]
    int64_t total = 0;
    for (int64_t k = 0; k < n_seq; ++k) {
        PG_CHECK(seq_len[k] >= 0, "pg_s2g_phylip_pack: sequence %lld has length %lld", (long long)k, (long long)seq_len[k]);
        tab[(size_t)k] = total;
        tab[(size_t)(n_seq + k)] = seq_len[k];
        total += seq_len[k];
    }
    std::vector<int64_t> piece;                         // the spans cut into pieces of at most S2G_PIECE bytes
    int64_t copied = 0;
    for (int64_t k = 0; k < n_span; ++k) {
        const int64_t src = span[3 * k], dst = span[3 * k + 1], n = span[3 * k + 2];
        PG_CHECK(src >= 0 && n >= 0 && src + n <= (int64_t)ss->len && dst >= 0 && dst + n <= total,
                 "pg_s2g_phylip_pack: span %lld copies %lld bytes from %lld to %lld (text %zu, sequences %lld bytes)",
                 (long long)k, (long long)n, (long long)src, (long long)dst, ss->len, (long long)total);
        for (int64_t o = 0; o < n; o += S2G_PIECE) {
            piece.push_back(src + o);
            piece.push_back(dst + o);
            piece.push_back(std::min(S2G_PIECE, n - o));
        }
        copied += n;
    }
    PG_CHECK(copied == total, "pg_s2g_phylip_pack: the spans copy %lld bytes, the sequences hold %lld", (long long)copied,
             (long long)total);
    PG_CUDA(cudaSetDevice(ctx->device));
    pg_timings_reset(ctx);
    PG_TRY(ss->fa.seq.ensure((size_t)total + 64));
    PG_TRY(ss->fa.rec.ensure(tab.size() * 8 + 64));
    PG_TRY(ss->pieces.ensure(piece.size() * 8 + 64));
    if (!tab.empty()) PG_CUDA(cudaMemcpyAsync(ss->fa.rec.p, tab.data(), tab.size() * 8, cudaMemcpyHostToDevice, ctx->stream));
    const int64_t n_piece = (int64_t)piece.size() / 3;
    if (n_piece) {
        PG_CUDA(cudaMemcpyAsync(ss->pieces.p, piece.data(), piece.size() * 8, cudaMemcpyHostToDevice, ctx->stream));
        const unsigned grid = (unsigned)std::min<int64_t>(n_piece, (int64_t)ctx->sm_count * 16);
        PG_TRY(pg_timed(ctx, "s2g_gather", [&] {
            k_s2g_gather<<<grid, 256, 0, ctx->stream>>>((const uint8_t*)ctx->text.p, (const int64_t*)ss->pieces.p, n_piece,
                                                        (uint8_t*)ss->fa.seq.p);
        }));
        ctx->launches += 1;
    }
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    ss->pieces.release();
    ss->lines.release();
    ss->fa.n_rec = n_seq;
    ss->fa.indexed = true;
    ss->rec_len.assign(seq_len, seq_len + n_seq);
    return PG_OK;
}

extern "C" int pg_s2g_plan(pg_ctx* ctx, int64_t n_blk, const int64_t* blk, const char* names, int64_t names_len,
                           int64_t n_mem, const int64_t* mem_rec, const uint8_t* mem_sep, int64_t* n_bytes) {
    PG_CHECK(ctx && (n_blk == 0 || blk) && (names_len == 0 || names) && (n_mem == 0 || (mem_rec && mem_sep)) && n_bytes,
             "pg_s2g_plan: null argument");
    S2gState* ss = sstate(ctx);
    PG_CHECK(ss->fa.indexed, "pg_s2g_plan: no sequences (pg_s2g_fasta_index or pg_s2g_phylip_pack)");
    const int64_t n_rec = (int64_t)ss->rec_len.size();
    *n_bytes = 0;
    ss->planned = false;
    ss->blk.assign((size_t)n_blk, Block{});
    int64_t off = 0, tasks = 0;
    for (int64_t b = 0; b < n_blk; ++b) {
        const int64_t* r = blk + 4 * b;                 // {name_off, name_len, rows, mem0}
        const int64_t mem1 = b + 1 < n_blk ? blk[4 * (b + 1) + 3] : n_mem;
        Block& B = ss->blk[(size_t)b];
        B.name_off = r[0];
        B.name_len = r[1];
        B.rows = r[2];
        B.mem0 = r[3];
        B.M = mem1 - r[3];
        PG_CHECK(B.name_off >= 0 && B.name_len >= 0 && B.name_off + B.name_len <= names_len && B.rows >= 0 && B.mem0 >= 0 &&
                     B.M >= 1 && mem1 <= n_mem,
                 "pg_s2g_plan: block %lld: name [%lld, +%lld), %lld rows, members [%lld, %lld)", (long long)b,
                 (long long)B.name_off, (long long)B.name_len, (long long)B.rows, (long long)B.mem0, (long long)mem1);
        for (int64_t m = B.mem0; m < mem1; ++m) {
            PG_CHECK(mem_rec[m] >= 0 && mem_rec[m] < n_rec && ss->rec_len[(size_t)mem_rec[m]] >= B.rows,
                     "pg_s2g_plan: block %lld: member %lld is sequence %lld of %lld, shorter than the %lld rows", (long long)b,
                     (long long)m, (long long)mem_rec[m], (long long)n_rec, (long long)B.rows);
            PG_CHECK(mem_sep[m] == '|' || mem_sep[m] == '\t' || mem_sep[m] == '\n',
                     "pg_s2g_plan: member %lld is followed by byte %d", (long long)m, (int)mem_sep[m]);
        }
        B.width = B.name_len + 2 + 2 * B.M;
        B.byte_off = off;
        B.task0 = tasks;
        off += row_off(B, B.rows);
        tasks += (B.rows + TS - 1) / TS * ((B.M + TM - 1) / TM);
    }
    PG_CUDA(cudaSetDevice(ctx->device));
    // device plan: blocks [n_blk], task0 [n_blk + 1], member records [n_mem], names, member bytes [n_mem]
    const size_t b_bytes = (size_t)n_blk * sizeof(Block), t_bytes = (size_t)(n_blk + 1) * 8, m_bytes = (size_t)n_mem * 8;
    PG_TRY(ss->plan.ensure(b_bytes + t_bytes + m_bytes + (size_t)names_len + (size_t)n_mem + 64));
    char* d = (char*)ss->plan.p;
    std::vector<int64_t> task0((size_t)n_blk + 1);
    for (int64_t b = 0; b < n_blk; ++b) task0[(size_t)b] = ss->blk[(size_t)b].task0;
    task0[(size_t)n_blk] = tasks;
    if (n_blk) PG_CUDA(cudaMemcpyAsync(d, ss->blk.data(), b_bytes, cudaMemcpyHostToDevice, ctx->stream));
    PG_CUDA(cudaMemcpyAsync(d + b_bytes, task0.data(), t_bytes, cudaMemcpyHostToDevice, ctx->stream));
    if (n_mem) PG_CUDA(cudaMemcpyAsync(d + b_bytes + t_bytes, mem_rec, m_bytes, cudaMemcpyHostToDevice, ctx->stream));
    if (names_len)
        PG_CUDA(cudaMemcpyAsync(d + b_bytes + t_bytes + m_bytes, names, (size_t)names_len, cudaMemcpyHostToDevice, ctx->stream));
    if (n_mem)
        PG_CUDA(cudaMemcpyAsync(d + b_bytes + t_bytes + m_bytes + names_len, mem_sep, (size_t)n_mem, cudaMemcpyHostToDevice,
                                ctx->stream));
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    ss->n_tasks = tasks;
    ss->total = off;
    ss->n_mem = n_mem;
    ss->names_len = names_len;
    ss->planned = true;
    *n_bytes = off;
    return PG_OK;
}

extern "C" int pg_s2g_emit(pg_ctx* ctx, int64_t byte0, char* out, size_t cap, size_t* bytes) {
    PG_CHECK(ctx && out && bytes, "pg_s2g_emit: null argument");
    S2gState* ss = sstate(ctx);
    PG_CHECK(ss->planned, "pg_s2g_emit: no pg_s2g_plan");
    PG_CHECK(byte0 >= 0 && byte0 <= ss->total && cap > 0, "pg_s2g_emit: byte %lld of %lld", (long long)byte0,
             (long long)ss->total);
    *bytes = 0;
    if (byte0 == ss->total) return PG_OK;
    const int64_t b1 = std::min<int64_t>(ss->total, byte0 + (int64_t)cap);
    // the task of the tile that holds byte `at` (at < total): its block (the last one starting at or before it), its row
    auto task_of = [&](int64_t at, bool last) {
        const auto it = std::upper_bound(ss->blk.begin(), ss->blk.end(), at,
                                         [](int64_t v, const Block& B) { return v < B.byte_off; });
        const Block& B = *(it - 1);
        int64_t a = 0, z = B.rows - 1;                  // the last row starting at or before `at`
        while (a < z) {
            const int64_t mid = (a + z + 1) >> 1;
            if (B.byte_off + row_off(B, mid) <= at) a = mid;
            else z = mid - 1;
        }
        const int64_t mt = (B.M + TM - 1) / TM;
        return B.task0 + (a / TS) * mt + (last ? mt : 0);
    };
    const int64_t t0 = task_of(byte0, false), t1 = task_of(b1 - 1, true);
    PG_CUDA(cudaSetDevice(ctx->device));
    pg_timings_reset(ctx);
    PG_TRY(ss->out.ensure((size_t)(b1 - byte0) + 64));
    const int64_t n_blk = (int64_t)ss->blk.size();
    const char* d = (const char*)ss->plan.p;
    const size_t b_bytes = (size_t)n_blk * sizeof(Block), t_bytes = (size_t)(n_blk + 1) * 8;
    EmitParams p;
    p.seq = (const uint8_t*)ss->fa.seq.p;
    p.rec_off = (const int64_t*)ss->fa.rec.p;
    p.blk = (const Block*)d;
    p.task0 = (const int64_t*)(d + b_bytes);
    p.n_blk = n_blk;
    p.mem_rec = (const int64_t*)(d + b_bytes + t_bytes);
    p.names = d + b_bytes + t_bytes + (size_t)ss->n_mem * 8;
    p.mem_sep = (const uint8_t*)(p.names + ss->names_len);
    p.t0 = t0;
    p.b0 = byte0;
    p.b1 = b1;
    p.out = (char*)ss->out.p;
    for (int64_t t = t0; t < t1; t += (int64_t)INT32_MAX) {
        p.t0 = t;
        const unsigned grid = (unsigned)std::min<int64_t>(t1 - t, (int64_t)INT32_MAX);
        PG_TRY(pg_timed(ctx, "s2g_tile", [&] { k_s2g_tile<<<grid, 256, 0, ctx->stream>>>(p); }));
        ctx->launches += 1;
    }
    PG_CUDA(cudaMemcpyAsync(out, ss->out.p, (size_t)(b1 - byte0), cudaMemcpyDeviceToHost, ctx->stream));
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    *bytes = (size_t)(b1 - byte0);
    return PG_OK;
}
