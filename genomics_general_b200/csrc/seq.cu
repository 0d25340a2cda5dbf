// genoToSeq.py on the device: the genotype tokens of a .geno body -> FASTA / PHYLIP alignments (genoToSeq.py:56-120:
// parseGenoFile / the window generators, GenoWindow.seqDict and makeAlnString, genomics.py:1949-2108, 1790-1793, 2232-2251).
//
// The text goes to HBM and its data lines are indexed by ingest.cu's pg_text_load.  Then:
//   k_seq_tokens : ONE WARP PER DATA LINE, classifying as k_parse_lines does (4 bytes per lane and step, a warp prefix sum of
//                  the field starts).  Field 0 -> scaffold hash, field 1 -> position, field 2 + c -> the line-relative start
//                  of column c's token in tok[line x n_slots] when the column has a slot; every slot's token must be as wide
//                  as on the first data line.  The first offending line (then column) wins through one atomicMin word.
//   k_seq_len    : one thread per output row (per window: the PHYLIP header row, then one row per sequence): its bytes; a CUB
//                  exclusive scan gives every row's offset.
//   k_seq_frame  : one thread per row of a slab: the name prefix (or the PHYLIP header) and the row's final '\n'.
//   k_seq_tile   : the transpose.  A CTA stages a tile of (TS sites x TQ sequences) in shared memory, reading along the site
//                  rows of the text (consecutive threads take consecutive sequences of one line), with --splitPhased's even
//                  offsets and --NtoGap's translation applied on the way; then one warp per sequence writes the tile's run
//                  of sites as contiguous bytes.  One launch covers every window of a slab.
// A slab is a range of (row, part) cells: part -1 = the prefix, 0..n-1 = the sites, n = the final '\n'; a row longer than the
// slab is cut after a site and resumed in the next one.
#include <fcntl.h>
#include <sys/stat.h>
#include <unistd.h>

#include <algorithm>
#include <cub/cub.cuh>

#include "pgwin_internal.h"

namespace {

constexpr int TQ = 32;              // sequences per tile
constexpr int TILE_ROW = 1024;      // bytes of one sequence's run in a tile (sites x width)
constexpr int TS_MAX = 256;         // sites per tile
constexpr int SEQ_MAX_WIDTH = 1024; // widest token

enum { SE_NONE = 0, SE_POS = 1, SE_NO_POS = 2, SE_POS_RANGE = 3, SE_WIDTH = 4, SE_MISSING = 5, SE_COUNT = 6, SE_BYTE = 7,
       SE_CR = 8 };

// str.split() blanks of ASCII text ('\n' ends the line)
__device__ __forceinline__ bool sblank(unsigned c) {
    return c == ' ' || c == '\t' || c == '\r' || c == '\v' || c == '\f' || (c >= 0x1c && c <= 0x1f);
}

struct TokParams {
    const uint8_t* buf;
    size_t len;
    const long long* starts;
    int64_t S;
    int n_cols;                 // genotype columns of the header
    const int32_t* col_slot;    // [n_cols] slot of the column, or -1
    int n_slots;
    const int32_t* slot_width;  // [n_slots] token width of every slot (first data line)
    int exact;                  // 1: a line holds exactly n_cols genotype columns; 0: at least every slot's column
    uint32_t* tok;              // [S x n_slots]
    int32_t* pos;
    unsigned long long* hash;
    unsigned long long* err;    // all ones = ok, else (data line << 28) | (genotype column << 4) | code, both 1-based
};

__device__ __forceinline__ void report(const TokParams& tp, int code, int64_t line, int col) {
    const unsigned long long c1 = (unsigned long long)min(max(col + 1, 0), (1 << 24) - 1);
    atomicMin(tp.err, ((unsigned long long)(line + 1) << 28) | (c1 << 4) | (unsigned long long)code);
}

__device__ __forceinline__ unsigned byte_at(const TokParams& tp, size_t i) { return i < tp.len ? tp.buf[i] : (unsigned)'\n'; }

__global__ void __launch_bounds__(256) k_seq_tokens(const __grid_constant__ TokParams tp) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
    for (int64_t line = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); line < tp.S; line += warps) {
        const size_t l0 = (size_t)tp.starts[line];
        const size_t a0 = l0 & ~(size_t)3;
        unsigned fields_before = 0;
        bool prev_ws = true;
        unsigned found = 0;
        bool have_pos = false, done = false;
        for (size_t step = 0; !done; ++step) {
            const size_t wbase = a0 + step * 128 + (size_t)lane * 4;
            uint32_t w = 0x0a0a0a0au;
            if (wbase + 4 <= tp.len) w = *reinterpret_cast<const uint32_t*>(tp.buf + wbase);
            else if (wbase < tp.len) {
                for (int k = 0; k < 4; ++k)
                    if (wbase + k < tp.len) w = (w & ~(0xffu << (8 * k))) | ((uint32_t)tp.buf[wbase + k] << (8 * k));
            }
            unsigned ws = 0, nl = 0, hi = 0, cr = 0;
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const unsigned c = (w >> (8 * k)) & 0xffu;
                const bool before = (wbase + k) < l0;
                if (before || sblank(c)) ws |= 1u << k;
                else if (c == '\n') nl |= 1u << k;
                if (!before && c >= 0x80u) hi |= 1u << k;
                if (!before && c == '\r') cr |= 1u << k;
            }
            const unsigned nl_lanes = __ballot_sync(0xffffffffu, nl != 0);
            if (nl_lanes) {
                const int first = __ffs(nl_lanes) - 1;
                if (lane > first) ws = 0xfu, nl = 0, hi = 0, cr = 0;
                else if (lane == first) {
                    const unsigned from = nl & (0u - nl);
                    ws |= ~(from - 1u) & 0xfu;
                    hi &= from - 1u;
                    cr &= from - 1u;
                }
                done = true;
            }
            // text the reference reads differently: a byte of a multi-byte character (str.split() knows more blanks, and a
            // token's width counts characters), a '\r' that ends a line by itself (universal newlines)
            if (hi) report(tp, SE_BYTE, line, -1);
            for (unsigned m = cr; m; m &= m - 1)
                if (byte_at(tp, wbase + __ffs(m)) != '\n') report(tp, SE_CR, line, -1);
            const unsigned last_ws = (ws >> 3) & 1u;
            unsigned pw = __shfl_up_sync(0xffffffffu, last_ws, 1);
            if (lane == 0) pw = prev_ws ? 1u : 0u;
            const unsigned prevbits = ((ws << 1) | pw) & 0xfu;
            const unsigned st = ~ws & prevbits & 0xfu;
            unsigned cnt = __popc(st), incl = cnt;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const unsigned v = __shfl_up_sync(0xffffffffu, incl, d);
                if (lane >= d) incl += v;
            }
            unsigned fidx = fields_before + incl - cnt;
            fields_before += __shfl_sync(0xffffffffu, incl, 31);
            prev_ws = (__shfl_sync(0xffffffffu, last_ws, 31) != 0);
            for (unsigned m = st; m; m &= m - 1, ++fidx) {
                const size_t q = wbase + (__ffs(m) - 1);
                if (fidx == 0) {                                        // scaffold name -> hash
                    unsigned long long h = 1469598103934665603ull;
                    for (size_t j = q;; ++j) {
                        const unsigned c = byte_at(tp, j);
                        if (c == '\n' || sblank(c)) break;
                        h = (h ^ c) * 1099511628211ull;
                    }
                    tp.hash[line] = h;
                } else if (fidx == 1) {                                 // position: int() of the field (genomics.py:1901)
                    size_t j = q;
                    unsigned c = byte_at(tp, j);
                    bool neg = false;
                    if (c == '-' || c == '+') {
                        neg = (c == '-');
                        c = byte_at(tp, ++j);
                    }
                    bool ok = c >= '0' && c <= '9';
                    long long v = 0;
                    while (c >= '0' && c <= '9') {
                        if (v <= (1ll << 31)) v = v * 10 + (long long)(c - '0');
                        c = byte_at(tp, ++j);
                    }
                    if (!ok || !(c == '\n' || sblank(c))) report(tp, SE_POS, line, -1);
                    else if (v > (1ll << 31) - (neg ? 0 : 1)) report(tp, SE_POS_RANGE, line, -1);
                    tp.pos[line] = (int32_t)(neg ? -v : v);
                    have_pos = true;
                } else {
                    const int col = (int)fidx - 2;
                    if (col >= tp.n_cols) continue;
                    const int slot = tp.col_slot[col];
                    if (slot < 0) continue;
                    const int want = tp.slot_width[slot];
                    int tl = 0;
                    while (tl <= want) {
                        const unsigned c = byte_at(tp, q + tl);
                        if (c == '\n' || sblank(c)) break;
                        ++tl;
                    }
                    if (tl != want) {
                        report(tp, SE_WIDTH, line, col);
                        continue;
                    }
                    tp.tok[(size_t)line * tp.n_slots + slot] = (uint32_t)(q - l0);
                    ++found;
                }
            }
        }
#pragma unroll
        for (int d = 16; d >= 1; d >>= 1) found += __shfl_xor_sync(0xffffffffu, found, d);
        const bool any_pos = __any_sync(0xffffffffu, have_pos);
        if (lane == 0) {
            const int n_geno = (int)fields_before - 2;
            if (!any_pos) report(tp, SE_NO_POS, line, -1);
            else if (tp.exact && n_geno != tp.n_cols) report(tp, SE_COUNT, line, n_geno);
            else if ((int)found != tp.n_slots && !(tp.exact && n_geno == tp.n_cols)) report(tp, SE_MISSING, line, n_geno);
        }
    }
}

struct RowParams {
    int fmt;                    // 0 FASTA, 1 PHYLIP (one header row first in every window)
    int nto_gap;
    int n_seq, rpw, maxw;       // sequences, rows per window, widest sequence step
    const int64_t* name_off;    // [n_seq + 1] into names
    const char* names;
    const int32_t* seq_slot;    // [n_seq] token slot of the sequence
    const int32_t* seq_byte;    // [n_seq] first byte taken in the token (2a for allele a with --splitPhased)
    const int32_t* seq_width;   // [n_seq] bytes per site (the token's width, or 1)
    const int64_t* lo;          // [n_win] first data line of the window
    const int64_t* hi;          // [n_win] one past its last
    int64_t R;
    int64_t* len;               // length pass: [R]
    // write pass
    const uint8_t* buf;
    const long long* starts;
    const uint32_t* tok;
    int n_slots;
    const int64_t* off;         // [R + 1]
    int64_t row0, x0, row1, x1; // the slab: cells [(row0, x0), (row1, x1))
    int64_t base;               // byte offset of cell (row0, x0)
    char* out;
};

__device__ __forceinline__ int ndigits(int64_t v) {
    int n = 1;
    while (v >= 10) {
        v /= 10;
        ++n;
    }
    return n;
}

__device__ __forceinline__ int prefix_len(const RowParams& rp, int k) {
    return (int)(rp.name_off[k + 1] - rp.name_off[k]) + (rp.fmt == 0 ? 2 : 3);
}

__global__ void k_seq_len(const __grid_constant__ RowParams rp) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < rp.R; r += (int64_t)gridDim.x * blockDim.x) {
        const int64_t w = r / rp.rpw;
        const int j = (int)(r - w * rp.rpw);
        const int64_t n = rp.hi[w] - rp.lo[w];
        if (rp.fmt == 1 && j == 0) rp.len[r] = 1 + ndigits(rp.n_seq) + 1 + ndigits(n * rp.maxw) + 1;     // " n L\n"
        else {
            const int k = j - rp.fmt;
            rp.len[r] = prefix_len(rp, k) + n * rp.seq_width[k] + 1;
        }
    }
}

__device__ __forceinline__ void put_int(char* o, int64_t v, int nd) {
    for (int i = nd - 1; i >= 0; --i) {
        o[i] = (char)('0' + v % 10);
        v /= 10;
    }
}

// the prefix and the final '\n' of rows row0 .. rlast
__global__ void k_seq_frame(const __grid_constant__ RowParams rp, int64_t rlast) {
    for (int64_t r = rp.row0 + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r <= rlast; r += (int64_t)gridDim.x * blockDim.x) {
        const int64_t w = r / rp.rpw;
        const int j = (int)(r - w * rp.rpw);
        const bool header = rp.fmt == 1 && j == 0;
        const int k = j - rp.fmt;
        const int64_t n = header ? 0 : rp.hi[w] - rp.lo[w];
        const int64_t P = header ? rp.off[r + 1] - rp.off[r] - 1 : prefix_len(rp, k);
        const int64_t wd = header ? 0 : rp.seq_width[k];
        char* o = rp.out + (rp.off[r] - rp.base);
        const bool pre = (r > rp.row0 || rp.x0 < 0) && (r < rp.row1 || rp.x1 >= 0);
        const bool suf = (r > rp.row0 || n >= rp.x0) && r < rp.row1;
        if (pre) {
            if (header) {                                        // " {n} {L}" (genomics.py:2243)
                const int a = ndigits(rp.n_seq), b = ndigits((rp.hi[w] - rp.lo[w]) * rp.maxw);
                o[0] = ' ';
                put_int(o + 1, rp.n_seq, a);
                o[1 + a] = ' ';
                put_int(o + 2 + a, (rp.hi[w] - rp.lo[w]) * rp.maxw, b);
            } else {
                const char* nm = rp.names + rp.name_off[k];
                const int nl = (int)(rp.name_off[k + 1] - rp.name_off[k]);
                int at = 0;
                if (rp.fmt == 0) o[at++] = '>';
                for (int i = 0; i < nl; ++i) o[at++] = nm[i];
                if (rp.fmt == 0) o[at++] = '\n';
                else o[at++] = ' ', o[at++] = ' ', o[at++] = ' ';
            }
        }
        if (suf) o[P + n * wd] = '\n';
    }
}

// the windows of a slab: sequences [k_lo, k_hi) and sites [s_lo, s_hi) of each, tiles tile0 .. tile0 + nq * ns
struct SeqTileWin {
    int64_t lo, row_base, s_lo, s_hi, tile0;
    int32_t k_lo, k_hi, nq, pad;
};

__global__ void __launch_bounds__(256) k_seq_tile(const __grid_constant__ RowParams rp, const SeqTileWin* __restrict__ ents,
                                                  int n_ent, int64_t n_tiles, int TS) {
    extern __shared__ uint8_t sm[];     // [TQ][TS * maxw]
    __shared__ int e_sh;
    const int pitch = TS * rp.maxw;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    for (int64_t t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        if (threadIdx.x == 0) {
            int a = 0, b = n_ent - 1;
            while (a < b) {
                const int mid = (a + b + 1) >> 1;
                if (ents[mid].tile0 <= t) a = mid;
                else b = mid - 1;
            }
            e_sh = a;
        }
        __syncthreads();
        const SeqTileWin E = ents[e_sh];
        const int64_t rel = t - E.tile0;
        const int tq = (int)(rel % E.nq);
        const int64_t i0 = E.s_lo + (rel / E.nq) * TS;
        const int k0 = E.k_lo + tq * TQ;
        const int nk = min(TQ, E.k_hi - k0);
        const int ni = (int)(E.s_hi - i0 < (int64_t)TS ? E.s_hi - i0 : (int64_t)TS);
        // stage: consecutive threads take consecutive sequences of one site, so a warp reads along one line of the text
        for (int idx = threadIdx.x; idx < TQ * ni; idx += blockDim.x) {
            const int q = idx % TQ, i = idx / TQ;
            if (q >= nk) continue;
            const int k = k0 + q;
            const int64_t r = E.row_base + rp.fmt + k, x = i0 + i;
            if (!((r > rp.row0 || x >= rp.x0) && (r < rp.row1 || x < rp.x1))) continue;
            const int64_t s = E.lo + x;
            const uint8_t* src = rp.buf + rp.starts[s] + rp.tok[(size_t)s * rp.n_slots + rp.seq_slot[k]] + rp.seq_byte[k];
            const int wd = rp.seq_width[k];
            uint8_t* dst = sm + q * pitch + i * wd;
            for (int b = 0; b < wd; ++b) {
                unsigned c = src[b];
                if (rp.nto_gap && (c == 'N' || c == 'n')) c = '-';      // missingtrans (genomics.py:42)
                dst[b] = (uint8_t)c;
            }
        }
        __syncthreads();
        // write: one warp per sequence, its sites as contiguous bytes
        for (int q = warp; q < nk; q += nwarps) {
            const int k = k0 + q;
            const int64_t r = E.row_base + rp.fmt + k;
            int64_t ia = 0, ib = ni;
            if (r == rp.row0) ia = max(ia, rp.x0 - i0);
            if (r == rp.row1) ib = min(ib, rp.x1 - i0);
            if (ib <= ia) continue;
            const int wd = rp.seq_width[k];
            char* dst = rp.out + (rp.off[r] - rp.base) + prefix_len(rp, k) + (i0 + ia) * wd;
            const uint8_t* src = sm + q * pitch + ia * wd;
            const int nb = (int)(ib - ia) * wd;
            for (int b = lane; b < nb; b += 32) dst[b] = (char)src[b];
        }
        __syncthreads();
    }
}

struct SeqState {
    uint64_t text_gen = 0;          // ctx->text_gen of the index
    int64_t S = -1;
    int n_slots = 0;
    PgBuf tok, meta, err, tab, win, off, cub, tiles, out;
    // the plan of pg_seq_plan
    bool planned = false;
    int fmt = 0, nto_gap = 0, n_seq = 0, rpw = 0, maxw = 0, TS = 1;
    int64_t n_win = 0, R = 0;
    size_t at_name_off = 0, at_names = 0, at_slot = 0, at_byte = 0, at_width = 0;
    std::vector<int64_t> h_off, n_sites, h_lo;   // host: row offsets [R + 1]; sites and first line of every window
    std::vector<int32_t> plen, width;    // host: prefix bytes and step of every sequence
};

SeqState* sstate(pg_ctx* ctx) {
    if (!ctx->seq_state) ctx->seq_state = new SeqState();
    return (SeqState*)ctx->seq_state;
}

RowParams row_params(pg_ctx* ctx, SeqState* ss) {
    RowParams rp;
    memset(&rp, 0, sizeof(rp));
    const char* t = (const char*)ss->tab.p;
    rp.fmt = ss->fmt;
    rp.nto_gap = ss->nto_gap;
    rp.n_seq = ss->n_seq;
    rp.rpw = ss->rpw;
    rp.maxw = ss->maxw;
    rp.name_off = (const int64_t*)(t + ss->at_name_off);
    rp.names = t + ss->at_names;
    rp.seq_slot = (const int32_t*)(t + ss->at_slot);
    rp.seq_byte = (const int32_t*)(t + ss->at_byte);
    rp.seq_width = (const int32_t*)(t + ss->at_width);
    rp.lo = (const int64_t*)ss->win.p;
    rp.hi = rp.lo + ss->n_win;
    rp.R = ss->R;
    rp.buf = (const uint8_t*)ctx->text.p;
    rp.starts = (const long long*)ctx->starts.p;
    rp.tok = (const uint32_t*)ss->tok.p;
    rp.n_slots = ss->n_slots;
    rp.off = (const int64_t*)ss->off.p;
    return rp;
}

}  // namespace

void pg_seq_free(pg_ctx* ctx) {
    SeqState* ss = (SeqState*)ctx->seq_state;
    if (!ss) return;
    PgBuf* bufs[] = {&ss->tok, &ss->meta, &ss->err, &ss->tab, &ss->win, &ss->off, &ss->cub, &ss->tiles, &ss->out};
    for (PgBuf* b : bufs) b->release();
    delete ss;
    ctx->seq_state = nullptr;
}

extern "C" int pg_seq_index(pg_ctx* ctx, const char* text, size_t len, const char* path, int64_t body_offset, int32_t n_cols,
                            const int32_t* col_slot, int32_t n_slots, const int32_t* slot_width, int32_t exact_cols,
                            int64_t* n_sites, int64_t* error) {
    PG_CHECK(ctx && (text || path || len == 0) && n_sites && error && (n_cols == 0 || col_slot) && (n_slots == 0 || slot_width),
             "pg_seq_index: null argument");
    PG_CHECK(n_cols >= 0 && n_slots >= 0 && n_slots <= n_cols, "pg_seq_index: %d slots for %d columns", n_slots, n_cols);
    {
        std::vector<char> seen((size_t)n_slots, 0);
        for (int c = 0; c < n_cols; ++c) {
            const int s = col_slot[c];
            if (s < 0) continue;
            PG_CHECK(s < n_slots && !seen[(size_t)s], "pg_seq_index: column %d has slot %d (slots must be distinct, below %d)", c,
                     s, n_slots);
            seen[(size_t)s] = 1;
        }
        for (int s = 0; s < n_slots; ++s) {
            PG_CHECK(seen[(size_t)s], "pg_seq_index: slot %d has no column", s);
            PG_CHECK(slot_width[s] >= 1 && slot_width[s] <= SEQ_MAX_WIDTH, "pg_seq_index: token width %d of slot %d (1 to %d)",
                     slot_width[s], s, SEQ_MAX_WIDTH);
        }
    }
    error[0] = error[1] = error[2] = 0;
    *n_sites = 0;
    PG_CUDA(cudaSetDevice(ctx->device));
    pg_timings_reset(ctx);
    SeqState* ss = sstate(ctx);
    ss->S = -1;
    ss->planned = false;
    int fd = -1;
    if (path) {
        fd = open(path, O_RDONLY);
        PG_CHECK(fd >= 0, "pg_seq_index: cannot open %s", path);
        struct stat st;
        if (fstat(fd, &st) != 0 || body_offset < 0 || (int64_t)st.st_size < body_offset) {
            close(fd);
            pg_set_error("pg_seq_index: cannot stat %s (or the body offset is past its end)", path);
            return PG_ERR;
        }
        len = (size_t)st.st_size - (size_t)body_offset;
    }
    int64_t S = 0;
    const int rc = pg_text_load(ctx, path ? nullptr : (text ? text : ""), fd, path ? (size_t)body_offset : 0, len, &S);
    if (fd >= 0) close(fd);
    PG_TRY(rc);
    ctx->ingest_sites = -1;             // the text no longer belongs to the resident matrix
    const size_t tok_bytes = (size_t)S * (size_t)n_slots * 4;
    {
        size_t free_b = 0, total_b = 0;
        PG_CUDA(cudaMemGetInfo(&free_b, &total_b));
        PG_CHECK(tok_bytes + (size_t)S * 13 < free_b + ss->tok.cap + ss->meta.cap,
                 "pg_seq_index: the token index of %lld lines x %d columns needs %zu bytes of device memory (%zu free)",
                 (long long)S, n_slots, tok_bytes, free_b);
    }
    PG_TRY(ss->tok.ensure(tok_bytes + 64));
    PG_TRY(ss->meta.ensure((size_t)std::max<int64_t>(S, 1) * 13 + 64));     // hash [S] int64, pos [S] int32, flags [S] int8
    PG_TRY(ss->err.ensure((size_t)std::max(n_cols, 1) * 8 + 64));
    unsigned long long* d_hash = (unsigned long long*)ss->meta.p;
    int32_t* d_pos = (int32_t*)(d_hash + S);
    int8_t* d_flags = (int8_t*)(d_pos + S);
    unsigned long long* d_err = (unsigned long long*)ss->err.p;
    int32_t* d_tab = (int32_t*)(d_err + 1);     // col_slot [n_cols], slot_width [n_slots]
    PG_CUDA(cudaMemsetAsync(d_err, 0xff, 8, ctx->stream));
    if (n_cols) PG_CUDA(cudaMemcpyAsync(d_tab, col_slot, (size_t)n_cols * 4, cudaMemcpyHostToDevice, ctx->stream));
    if (n_slots) PG_CUDA(cudaMemcpyAsync(d_tab + n_cols, slot_width, (size_t)n_slots * 4, cudaMemcpyHostToDevice, ctx->stream));
    if (S > 0) {
        TokParams tp;
        tp.buf = (const uint8_t*)ctx->text.p;
        tp.len = len;
        tp.starts = (const long long*)ctx->starts.p;
        tp.S = S;
        tp.n_cols = n_cols;
        tp.col_slot = d_tab;
        tp.n_slots = n_slots;
        tp.slot_width = d_tab + n_cols;
        tp.exact = exact_cols ? 1 : 0;
        tp.tok = (uint32_t*)ss->tok.p;
        tp.pos = d_pos;
        tp.hash = d_hash;
        tp.err = d_err;
        const unsigned grid = (unsigned)std::min<int64_t>((S + 7) / 8, (int64_t)ctx->sm_count * 64);
        PG_TRY(pg_timed(ctx, "seq_tokens", [&] { k_seq_tokens<<<grid, 256, 0, ctx->stream>>>(tp); }));
        PG_TRY(pg_scaffold_flags(ctx, d_hash, S, d_flags));
        ctx->launches += 2;
    }
    unsigned long long packed = ~0ull;
    PG_CUDA(cudaMemcpyAsync(&packed, d_err, 8, cudaMemcpyDeviceToHost, ctx->stream));
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    if (packed != ~0ull) {
        error[0] = (int64_t)(packed & 15ull);
        error[1] = (int64_t)(packed >> 28);
        error[2] = (int64_t)((packed >> 4) & 0xffffffull);
    }
    ss->S = S;
    ss->n_slots = n_slots;
    ss->text_gen = ctx->text_gen;
    *n_sites = S;
    return PG_OK;
}

extern "C" int pg_seq_meta(pg_ctx* ctx, int32_t* pos, int8_t* new_scaffold, int64_t* line_off) {
    PG_CHECK(ctx != nullptr, "pg_seq_meta: null ctx");
    SeqState* ss = sstate(ctx);
    PG_CHECK(ss->S >= 0 && ss->text_gen == ctx->text_gen, "pg_seq_meta: no pg_seq_index on the current text");
    const int64_t S = ss->S;
    if (S == 0) return PG_OK;
    PG_CUDA(cudaSetDevice(ctx->device));
    const unsigned long long* d_hash = (const unsigned long long*)ss->meta.p;
    const int32_t* d_pos = (const int32_t*)(d_hash + S);
    const int8_t* d_flags = (const int8_t*)(d_pos + S);
    if (pos) PG_CUDA(cudaMemcpyAsync(pos, d_pos, (size_t)S * 4, cudaMemcpyDeviceToHost, ctx->stream));
    if (new_scaffold) PG_CUDA(cudaMemcpyAsync(new_scaffold, d_flags, (size_t)S, cudaMemcpyDeviceToHost, ctx->stream));
    if (line_off) PG_CUDA(cudaMemcpyAsync(line_off, ctx->starts.p, (size_t)S * 8, cudaMemcpyDeviceToHost, ctx->stream));
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    return PG_OK;
}

extern "C" int pg_seq_plan(pg_ctx* ctx, int32_t fmt, int32_t nto_gap, int32_t n_seq, const char* names, const int64_t* name_off,
                           const int32_t* seq_slot, const int32_t* seq_byte, const int32_t* seq_width, int64_t n_win,
                           const int64_t* lo, const int64_t* hi, int64_t* n_rows, int64_t* win_bytes) {
    PG_CHECK(ctx && n_rows && (n_win == 0 || (lo && hi && win_bytes)), "pg_seq_plan: null argument");
    PG_CHECK(n_seq >= 1 && names && name_off && seq_slot && seq_byte && seq_width, "pg_seq_plan: no sequences");
    PG_CHECK(fmt == 0 || fmt == 1, "pg_seq_plan: format %d is not 0 (FASTA) or 1 (PHYLIP)", fmt);
    SeqState* ss = sstate(ctx);
    PG_CHECK(ss->S >= 0 && ss->text_gen == ctx->text_gen, "pg_seq_plan: no pg_seq_index on the current text");
    ss->planned = false;
    int maxw = 1;
    std::vector<int32_t> plen((size_t)n_seq), width(seq_width, seq_width + n_seq);
    PG_CHECK(name_off[0] == 0, "pg_seq_plan: name_off[0] must be 0");
    for (int k = 0; k < n_seq; ++k) {
        PG_CHECK(seq_slot[k] >= 0 && seq_slot[k] < ss->n_slots, "pg_seq_plan: sequence %d reads slot %d of %d", k, seq_slot[k],
                 ss->n_slots);
        PG_CHECK(seq_width[k] >= 1 && seq_width[k] <= SEQ_MAX_WIDTH && seq_byte[k] >= 0,
                 "pg_seq_plan: sequence %d takes %d bytes from byte %d", k, seq_width[k], seq_byte[k]);
        PG_CHECK(name_off[k + 1] >= name_off[k] && name_off[k + 1] - name_off[k] < (1 << 20), "pg_seq_plan: name %d", k);
        plen[(size_t)k] = (int32_t)(name_off[k + 1] - name_off[k]) + (fmt == 0 ? 2 : 3);
        maxw = std::max(maxw, (int)seq_width[k]);
    }
    std::vector<int64_t> n_sites((size_t)n_win);
    for (int64_t w = 0; w < n_win; ++w) {
        PG_CHECK(lo[w] >= 0 && lo[w] <= hi[w] && hi[w] <= ss->S, "pg_seq_plan: window %lld [%lld, %lld) outside the %lld lines",
                 (long long)w, (long long)lo[w], (long long)hi[w], (long long)ss->S);
        n_sites[(size_t)w] = hi[w] - lo[w];
    }
    const int rpw = n_seq + fmt;
    const int64_t R = n_win * rpw;
    PG_CHECK(R + 1 < (int64_t)INT32_MAX, "pg_seq_plan: %lld output rows in one plan (at most %d)", (long long)R, INT32_MAX - 2);
    PG_CUDA(cudaSetDevice(ctx->device));
    pg_timings_reset(ctx);
    // sequence tables: name offsets, slots, bytes, widths, then the names
    const size_t nb_names = (size_t)name_off[n_seq];
    size_t o = 0;
    auto take = [&](size_t bytes) {
        const size_t at = o;
        o += (bytes + 15) & ~(size_t)15;
        return at;
    };
    ss->at_name_off = take((size_t)(n_seq + 1) * 8);
    ss->at_slot = take((size_t)n_seq * 4);
    ss->at_byte = take((size_t)n_seq * 4);
    ss->at_width = take((size_t)n_seq * 4);
    ss->at_names = take(nb_names + 1);
    std::vector<char> h(o, 0);
    memcpy(h.data() + ss->at_name_off, name_off, (size_t)(n_seq + 1) * 8);
    memcpy(h.data() + ss->at_slot, seq_slot, (size_t)n_seq * 4);
    memcpy(h.data() + ss->at_byte, seq_byte, (size_t)n_seq * 4);
    memcpy(h.data() + ss->at_width, seq_width, (size_t)n_seq * 4);
    memcpy(h.data() + ss->at_names, names, nb_names);
    PG_TRY(ss->tab.ensure(o + 64));
    PG_CUDA(cudaMemcpyAsync(ss->tab.p, h.data(), o, cudaMemcpyHostToDevice, ctx->stream));
    PG_TRY(ss->win.ensure((size_t)std::max<int64_t>(n_win, 1) * 16 + 64));
    if (n_win) {
        PG_CUDA(cudaMemcpyAsync(ss->win.p, lo, (size_t)n_win * 8, cudaMemcpyHostToDevice, ctx->stream));
        PG_CUDA(cudaMemcpyAsync((int64_t*)ss->win.p + n_win, hi, (size_t)n_win * 8, cudaMemcpyHostToDevice, ctx->stream));
    }
    ss->fmt = fmt;
    ss->nto_gap = nto_gap ? 1 : 0;
    ss->n_seq = n_seq;
    ss->rpw = rpw;
    ss->maxw = maxw;
    ss->TS = std::max(1, std::min(TS_MAX, TILE_ROW / maxw));
    ss->n_win = n_win;
    ss->R = R;
    // row lengths -> exclusive scan -> offsets [R + 1]
    PG_TRY(ss->off.ensure((size_t)(R + 1) * 16 + 64));
    int64_t* d_off = (int64_t*)ss->off.p;
    int64_t* d_len = d_off + (R + 1);
    PG_CUDA(cudaMemsetAsync(d_len + R, 0, 8, ctx->stream));
    RowParams rp = row_params(ctx, ss);
    rp.len = d_len;
    if (R > 0) {
        const unsigned grid = (unsigned)std::min<int64_t>((R + 255) / 256, (int64_t)ctx->sm_count * 16);
        PG_TRY(pg_timed(ctx, "seq_len", [&] { k_seq_len<<<grid, 256, 0, ctx->stream>>>(rp); }));
    }
    size_t tmp = 0;
    PG_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tmp, d_len, d_off, (int)(R + 1), ctx->stream));
    PG_TRY(ss->cub.ensure(tmp + 64));
    PG_CUDA(cub::DeviceScan::ExclusiveSum(ss->cub.p, tmp, d_len, d_off, (int)(R + 1), ctx->stream));
    ctx->launches += 2;
    ss->h_off.resize((size_t)R + 1);
    PG_TRY(pg_d2h_staged(ctx, ss->h_off.data(), d_off, (size_t)(R + 1) * 8));
    ss->n_sites.swap(n_sites);
    ss->h_lo.assign(lo, lo + n_win);
    ss->plen.swap(plen);
    ss->width.swap(width);
    for (int64_t w = 0; w < n_win; ++w) win_bytes[w] = ss->h_off[(size_t)(w + 1) * rpw] - ss->h_off[(size_t)w * rpw];
    *n_rows = R;
    ss->planned = true;
    return PG_OK;
}

extern "C" int pg_seq_emit(pg_ctx* ctx, int64_t row0, int64_t part0, char* out, size_t cap, int64_t* row1, int64_t* part1,
                           size_t* bytes) {
    PG_CHECK(ctx && out && row1 && part1 && bytes, "pg_seq_emit: null argument");
    SeqState* ss = sstate(ctx);
    PG_CHECK(ss->planned && ss->text_gen == ctx->text_gen, "pg_seq_emit: no pg_seq_plan on the current text");
    const int64_t R = ss->R;
    PG_CHECK(row0 >= 0 && row0 <= R && part0 >= -1 && (row0 < R || part0 == -1), "pg_seq_emit: cell (%lld, %lld) out of range",
             (long long)row0, (long long)part0);
    *row1 = row0;
    *part1 = part0;
    *bytes = 0;
    if (row0 == R) return PG_OK;
    const std::vector<int64_t>& off = ss->h_off;
    const int fmt = ss->fmt, rpw = ss->rpw;
    auto header = [&](int64_t r) { return fmt == 1 && r % rpw == 0; };
    auto plen = [&](int64_t r) -> int64_t { return header(r) ? off[(size_t)r + 1] - off[(size_t)r] - 1 : ss->plen[(size_t)(r % rpw - fmt)]; };
    auto nsites = [&](int64_t r) -> int64_t { return header(r) ? 0 : ss->n_sites[(size_t)(r / rpw)]; };
    auto step = [&](int64_t r) -> int64_t { return header(r) ? 0 : ss->width[(size_t)(r % rpw - fmt)]; };
    auto byte_of = [&](int64_t r, int64_t x) { return r == R ? off[(size_t)R] : off[(size_t)r] + (x < 0 ? 0 : plen(r) + x * step(r)); };
    PG_CHECK(part0 <= nsites(row0), "pg_seq_emit: part %lld of row %lld (%lld sites)", (long long)part0, (long long)row0,
             (long long)nsites(row0));
    const int64_t base = byte_of(row0, part0), target = base + (int64_t)cap;
    // whole rows that fit; else cut row0 after as many sites as fit
    int64_t r1 = (int64_t)(std::upper_bound(off.begin() + row0 + 1, off.end(), target) - off.begin()) - 1;
    int64_t x1 = -1;
    if (r1 <= row0) {
        r1 = row0;
        const int64_t avail = target - off[(size_t)row0] - plen(row0);
        const int64_t st = step(row0);
        x1 = avail < 0 ? -2 : std::min(nsites(row0), st > 0 ? avail / st : nsites(row0));
        PG_CHECK(x1 > part0 && x1 >= 0, "pg_seq_emit: a buffer of %zu bytes cannot hold the name and one site of row %lld", cap,
                 (long long)row0);
    }
    const size_t nb = (size_t)(byte_of(r1, x1) - base);
    PG_CUDA(cudaSetDevice(ctx->device));
    pg_timings_reset(ctx);
    PG_TRY(ss->out.ensure(nb + 64));
    RowParams rp = row_params(ctx, ss);
    rp.row0 = row0;
    rp.x0 = part0;
    rp.row1 = r1;
    rp.x1 = x1;
    rp.base = base;
    rp.out = (char*)ss->out.p;
    const int64_t rlast = x1 >= 0 ? r1 : r1 - 1;
    // the slab's windows and their tiles
    std::vector<SeqTileWin> ents;
    int64_t n_tiles = 0;
    const int TS = ss->TS;
    for (int64_t w = row0 / rpw; w <= rlast / rpw; ++w) {
        const int64_t ra = std::max(w * rpw, row0), rb = std::min((w + 1) * rpw - 1, rlast);
        const int64_t k_lo = std::max<int64_t>(ra - w * rpw - fmt, 0), k_hi = rb - w * rpw - fmt + 1;
        const int64_t n = ss->n_sites[(size_t)w];
        int64_t s_lo = 0, s_hi = n;
        if (ra == rb && ra == row0 && part0 > 0) s_lo = part0;
        if (ra == rb && rb == r1 && x1 >= 0) s_hi = std::min(n, x1);
        if (k_hi <= k_lo || s_hi <= s_lo) continue;
        SeqTileWin e;
        e.lo = ss->h_lo[(size_t)w];
        e.row_base = w * rpw;
        e.s_lo = s_lo;
        e.s_hi = s_hi;
        e.tile0 = n_tiles;
        e.k_lo = (int32_t)k_lo;
        e.k_hi = (int32_t)k_hi;
        e.nq = (int32_t)((k_hi - k_lo + TQ - 1) / TQ);
        e.pad = 0;
        ents.push_back(e);
        n_tiles += (int64_t)e.nq * ((s_hi - s_lo + TS - 1) / TS);
    }
    PG_TRY(pg_timed(ctx, "seq_frame", [&] {
        const int64_t nr = rlast - row0 + 1;
        k_seq_frame<<<(unsigned)std::min<int64_t>((nr + 255) / 256, (int64_t)ctx->sm_count * 16), 256, 0, ctx->stream>>>(rp, rlast);
    }));
    ctx->launches += 1;
    if (n_tiles > 0) {
        PG_TRY(ss->tiles.ensure(ents.size() * sizeof(SeqTileWin) + 64));
        PG_CUDA(cudaMemcpyAsync(ss->tiles.p, ents.data(), ents.size() * sizeof(SeqTileWin), cudaMemcpyHostToDevice, ctx->stream));
        const int smem = TQ * TS * ss->maxw;
        const unsigned grid = (unsigned)std::min<int64_t>(n_tiles, (int64_t)ctx->sm_count * 8);
        PG_TRY(pg_timed(ctx, "seq_tile", [&] {
            k_seq_tile<<<grid, 256, smem, ctx->stream>>>(rp, (const SeqTileWin*)ss->tiles.p, (int)ents.size(), n_tiles, TS);
        }));
        ctx->launches += 1;
    }
    PG_CUDA(cudaMemcpyAsync(out, ss->out.p, nb, cudaMemcpyDeviceToHost, ctx->stream));
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    *row1 = r1;
    *part1 = x1;
    *bytes = nb;
    return PG_OK;
}
