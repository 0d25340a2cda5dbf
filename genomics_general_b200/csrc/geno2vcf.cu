// genoToVCF.py on the device: .geno genotypes -> VCF GT records, with REF from a reference FASTA (VCF_processing/genoToVCF.py
// makeVCFline, genomics.py GenomeSite / Genotype 317-378, 500-557, parseFasta 2256-2261).
//
// The reference FASTA is loaded once (pg_g2v_ref_load / pg_g2v_ref_index) by fasta.cu's shared loader: its text goes to
// HBM, k_fa_marks flags the '>' bytes and a CUB select gives the record starts; the host names the records from their header
// pieces; k_fa_keep flags the sequence bytes (after a record's first newline, not '\n', '\r' or ' ') and counts them per
// record, and a CUB select compacts them into one resident buffer.
// The body is streamed in chunks of complete lines.  Per chunk (pg_g2v_chunk, pg_g2v_sites, pg_g2v_emit):
//   ingest.cu's pg_text_load uploads the text and indexes its data lines;
//   k_g2v_tokens : ONE WARP PER DATA LINE (pg_warp_fields, which classifies a line as k_seq_tokens does): field 0 -> scaffold hash and span, field 1 -> POS as int64,
//                  field 2 + c -> the line-relative start of column c's token when a selected sample reads the column;
//   pg_scaffold_flags and a CUB select give the first line of every scaffold run, which the host maps to a FASTA record;
//   k_g2v_sites  : ONE WARP PER DATA LINE, lanes over the selected samples: each lane takes its samples' alleles and counts
//                  the A/C/G/T of the ones whose alleles all are A C G T N, a warp reduction sums them; lane 0 orders them
//                  (pg_freq_order), puts the reference base first and writes the row's byte length;
//   a CUB exclusive scan gives the row offsets, and k_g2v_emit writes the rows that meet a byte range into a slab (lane 0
//   the fixed columns, the sample fields placed by a warp prefix sum of their widths); a row may be cut between slabs.
// Errors go through one atomicMin word: (data line << 28) | (column << 4) | code, the column 0 for the line itself, k + 1 for
// selected sample k and n_sel + 1 for the reference lookup, so the first line, then the first column wins.
#include <algorithm>
#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>

#include "pgwin_internal.h"

namespace {

enum { GE_POS = 1, GE_NO_POS = 2, GE_POS_RANGE = 3, GE_TWO_FIELDS = 4, GE_BYTE = 5, GE_CR = 6, GE_MISSING = 7, GE_DIPLO = 8,
       GE_SCAFFOLD = 9, GE_OUTSIDE = 10 };

struct LineMeta {
    long long pos;
    uint32_t scaf_b, scaf_len;  // the scaffold token: first byte from the line start, length
    int32_t n_geno;             // genotype fields (fields - 2; 0 when fewer)
    int32_t bad;                // a line-level error was reported: the site pass skips the line
    unsigned long long L;       // the allele list: its length in bits 56..63, its bytes in bits 0..39
};

struct G2vParams {
    const uint8_t* buf;
    size_t len;
    const long long* starts;
    int64_t S;
    int fmt;                    // 0 phased, 1 diplo, 2 pairs
    int n_cols, n_slots, n_sel;
    const int32_t* col_slot;    // [n_cols] token slot of the column, or -1
    const int32_t* col_prev;    // [n_cols] the previous column of the same name, or -1
    const int32_t* sel_col;     // [n_sel] the last column of the selected sample's name
    uint32_t* tok;              // [S x n_slots]
    LineMeta* meta;             // [S]
    unsigned long long* hash;   // [S]
    unsigned long long* err;
    // the reference
    int use_ref;
    int64_t n_runs;
    const long long* run_line;  // [n_runs] first line of every scaffold run
    const int32_t* run_rec;     // [n_runs] its FASTA record, or -1
    const int64_t* rec_off;     // [n_rec] first byte of the record's sequence in seq
    const int64_t* rec_len;     // [n_rec]
    const uint8_t* seq;
    int64_t* len_out;           // [S + 1] row bytes
    // emit: rows [r0, r1) meet the bytes [b0, b1) of the output
    const int64_t* off;
    int64_t r0, r1, b0, b1;
    char* out;
};

__device__ __forceinline__ void report(const G2vParams& p, int code, int64_t line, int col) {
    atomicMin(p.err, ((unsigned long long)(line + 1) << 28) | ((unsigned long long)min(col, (1 << 24) - 1) << 4) |
                         (unsigned long long)code);
}

// diplo codes -> the two alleles (genomics.py:14-15 DIPLOTYPES / PAIRS), 0 for a byte that is not a code
__device__ __forceinline__ uint32_t diplo_pair(unsigned c) {
    switch (c) {
        case 'A': return 'A' | ('A' << 8);
        case 'C': return 'C' | ('C' << 8);
        case 'G': return 'G' | ('G' << 8);
        case 'K': return 'G' | ('T' << 8);
        case 'M': return 'A' | ('C' << 8);
        case 'N': return 'N' | ('N' << 8);
        case 'S': return 'C' | ('G' << 8);
        case 'R': return 'A' | ('G' << 8);
        case 'T': return 'T' | ('T' << 8);
        case 'W': return 'A' | ('T' << 8);
        case 'Y': return 'C' | ('T' << 8);
        default: return 0;
    }
}

__device__ __forceinline__ int base_code(unsigned c) {
    return c == 'A' ? 0 : c == 'C' ? 1 : c == 'G' ? 2 : c == 'T' ? 3 : c == 'N' ? 4 : -1;
}

// One sample's genotype on a line: its token (width w) in the text, its alleles and phase (genomics.py Genotype.__init__).
struct Geno {
    const uint8_t* t;
    int w, n;                   // token width, alleles
    unsigned phase;
    uint32_t pair;              // diplo: the two alleles
    __device__ __forceinline__ unsigned allele(int i) const {
        return pair ? (pair >> (8 * i)) & 0xffu : (unsigned)t[i * (n == w ? 1 : 2)];
    }
    __device__ __forceinline__ int field_width() const { return 2 * n - 1; }
};

// sample k of the line: -1 missing column, -2 bad diplo token, else 0 with g filled
__device__ __forceinline__ int sample_geno(const G2vParams& p, int64_t line, int n_geno, int k, Geno& g) {
    int c = p.sel_col[k];
    while (c >= 0 && c >= n_geno) c = p.col_prev[c];
    if (c < 0) return -1;
    g.t = p.buf + p.starts[line] + p.tok[(size_t)line * p.n_slots + p.col_slot[c]];
    int w = 0;
    while (true) {
        const unsigned b = g.t[w];
        if (b == '\n' || pg_sblank(b)) break;
        ++w;
    }
    g.w = w;
    g.pair = 0;
    g.phase = '/';
    if (p.fmt == 1) {                                   // diplo: haplo(token)
        g.pair = w == 1 ? diplo_pair(g.t[0]) : 0;
        if (!g.pair) return -2;
        g.n = 2;
    } else if (p.fmt == 0) {                            // phased: token[::2], phase token[1] for odd widths > 1
        g.n = (w + 1) / 2;
        if (w > 1 && (w & 1)) g.phase = g.t[1];
    } else {                                            // pairs: every byte an allele
        g.n = w;
    }
    return 0;
}

__device__ __forceinline__ int L_len(unsigned long long L) { return (int)(L >> 56); }
__device__ __forceinline__ unsigned L_at(unsigned long long L, int i) { return (unsigned)(L >> (8 * i)) & 0xffu; }
__device__ __forceinline__ int L_index(unsigned long long L, unsigned a) {
    const int n = L_len(L);
    for (int i = 0; i < n; ++i)
        if (L_at(L, i) == a) return i;
    return -1;
}

__device__ __forceinline__ int pos_digits(long long v) {
    unsigned long long u = v < 0 ? 0ull - (unsigned long long)v : (unsigned long long)v;
    int n = 1 + (v < 0);
    while (u >= 10) {
        u /= 10;
        ++n;
    }
    return n;
}

// fixed columns "scaffold\tPOS\t.\tREF\tALT\t.\t.\t.\tGT"
__device__ __forceinline__ int64_t fixed_len(const LineMeta& m) {
    const int nl = L_len(m.L);
    return (int64_t)m.scaf_len + pos_digits(m.pos) + (nl == 1 ? 1 : 2 * (nl - 1) - 1) + 15;
}

__global__ void __launch_bounds__(256) k_g2v_tokens(const __grid_constant__ G2vParams p) {
    const int lane = threadIdx.x & 31;
    const int64_t line = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (line >= p.S) return;
    {
        const size_t l0 = (size_t)p.starts[line];
        bool hi = false, lone_cr = false, pos_bad = false;
        const unsigned n_fields = pg_warp_fields(p.buf, p.len, l0, &hi, &lone_cr, [&](unsigned fidx, size_t q) {
            if (fidx == 0) {                                        // scaffold name -> hash and span
                unsigned long long h = 1469598103934665603ull;
                size_t j = q;
                for (;; ++j) {
                    const unsigned c = pg_byte_at(p.buf, p.len, j);
                    if (c == '\n' || pg_sblank(c)) break;
                    h = (h ^ c) * 1099511628211ull;
                }
                p.hash[line] = h;
                p.meta[line].scaf_b = (uint32_t)(q - l0);
                p.meta[line].scaf_len = (uint32_t)(j - q);
            } else if (fidx == 1) {                                 // POS: [+-]?[0-9]+ within int64
                size_t j = q;
                unsigned c = pg_byte_at(p.buf, p.len, j);
                bool neg = false;
                if (c == '-' || c == '+') {
                    neg = (c == '-');
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
                    report(p, GE_POS, line, 0);
                    pos_bad = true;
                } else if (over || v > (1ull << 63) - (neg ? 0 : 1)) {
                    report(p, GE_POS_RANGE, line, 0);
                    pos_bad = true;
                }
                p.meta[line].pos = neg ? (long long)(0ull - v) : (long long)v;
            } else {
                const int col = (int)fidx - 2;
                if (col >= p.n_cols) return;
                const int slot = p.col_slot[col];
                if (slot >= 0) p.tok[(size_t)line * p.n_slots + slot] = (uint32_t)(q - l0);
            }
        });
        pos_bad = __any_sync(0xffffffffu, pos_bad);
        if (lane == 0) {
            bool bad = pos_bad;
            if (hi) report(p, GE_BYTE, line, 0), bad = true;
            if (lone_cr) report(p, GE_CR, line, 0), bad = true;
            if (n_fields < 2) report(p, GE_NO_POS, line, 0), bad = true;
            else if (n_fields == 2) report(p, GE_TWO_FIELDS, line, 0), bad = true;
            if (n_fields == 0) p.hash[line] = 0;
            p.meta[line].n_geno = n_fields > 2 ? (int32_t)n_fields - 2 : 0;
            p.meta[line].bad = bad ? 1 : 0;
        }
    }
}

__global__ void __launch_bounds__(256) k_g2v_sites(const __grid_constant__ G2vParams p) {
    const int lane = threadIdx.x & 31;
    const int64_t line = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (line >= p.S) return;
    {
        if (p.meta[line].bad) {
            if (lane == 0) p.len_out[line] = 0;
            return;
        }
        int cnt[4] = {0, 0, 0, 0};
        int64_t fields = 0;
        for (int k = lane; k < p.n_sel; k += 32) {
            Geno g;
            const int r = sample_geno(p, line, p.meta[line].n_geno, k, g);
            if (r < 0) {
                report(p, r == -1 ? GE_MISSING : GE_DIPLO, line, k + 1);
                continue;
            }
            fields += 1 + g.field_width();
            int add[4] = {0, 0, 0, 0};                      // a genotype counts only when all its alleles are A C G T N
            bool all = true;
            for (int i = 0; i < g.n; ++i) {
                const int b = base_code(g.allele(i));
                if (b < 0) all = false;
                else if (b < 4) ++add[b];
            }
            if (all)
                for (int a = 0; a < 4; ++a) cnt[a] += add[a];
        }
#pragma unroll
        for (int d = 16; d >= 1; d >>= 1) {
            for (int a = 0; a < 4; ++a) cnt[a] += __shfl_xor_sync(0xffffffffu, cnt[a], d);
            fields += __shfl_xor_sync(0xffffffffu, fields, d);
        }
        if (lane != 0) return;
        LineMeta m = p.meta[line];
        int rank[4];
        const int nr = pg_freq_order(cnt, rank);
        unsigned long long L = 0;                           // the counted bases by frequency, else [N]
        int nl = 0;
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
            for (int a = 0; a < 4; ++a)
                if (r < nr && rank[a] == r) L |= (unsigned long long)((0x54474341u >> (8 * a)) & 0xffu) << (8 * nl++);
        if (nl == 0) L = 'N', nl = 1;
        if (p.use_ref) {                                    // L = [refBase] + (L without refBase)
            int64_t a = 0, b = p.n_runs - 1;
            while (a < b) {
                const int64_t mid = (a + b + 1) >> 1;
                if (p.run_line[mid] <= line) a = mid;
                else b = mid - 1;
            }
            const int rec = p.run_rec[a];
            if (rec < 0) {
                report(p, GE_SCAFFOLD, line, p.n_sel + 1);
                p.len_out[line] = 0;
                return;
            }
            const long long n = p.rec_len[rec];
            if (!(m.pos >= 1 - n && m.pos <= n)) {          // seq[pos - 1] with Python's indexing
                report(p, GE_OUTSIDE, line, p.n_sel + 1);
                p.len_out[line] = 0;
                return;
            }
            const unsigned rb = p.seq[p.rec_off[rec] + (m.pos - 1 < 0 ? m.pos - 1 + n : m.pos - 1)];
            unsigned long long t = rb;
            int n2 = 1;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const unsigned c = (unsigned)(L >> (8 * j)) & 0xffu;
                if (j < nl && c != rb) t |= (unsigned long long)c << (8 * n2++);
            }
            L = t;
            nl = n2;
        }
        L |= (unsigned long long)nl << 56;
        m.L = L;
        p.meta[line].L = L;
        p.len_out[line] = fixed_len(m) + fields + 1;
    }
}

__device__ __forceinline__ void put(const G2vParams& p, int64_t at, char c) {
    if (at >= 0 && at < p.b1 - p.b0) p.out[at] = c;
}

__global__ void __launch_bounds__(256) k_g2v_emit(const __grid_constant__ G2vParams p) {
    const int lane = threadIdx.x & 31;
    const int64_t line = p.r0 + (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (line >= p.r1) return;
    {
        const LineMeta m = p.meta[line];
        const int64_t o = p.off[line] - p.b0;
        const uint8_t* text = p.buf + p.starts[line];
        for (uint32_t i = lane; i < m.scaf_len; i += 32) put(p, o + i, (char)text[m.scaf_b + i]);
        int64_t at = fixed_len(m);
        if (lane == 0) {
            int64_t x = o + m.scaf_len;
            put(p, x++, '\t');
            const int nd = pos_digits(m.pos);
            unsigned long long u = m.pos < 0 ? 0ull - (unsigned long long)m.pos : (unsigned long long)m.pos;
            if (m.pos < 0) put(p, x, '-');
            for (int i = nd - 1; i >= (m.pos < 0); --i, u /= 10) put(p, x + i, (char)('0' + u % 10));
            x += nd;
            put(p, x++, '\t');
            put(p, x++, '.');
            put(p, x++, '\t');
            put(p, x++, (char)L_at(m.L, 0));
            put(p, x++, '\t');
            const int nl = L_len(m.L);
            if (nl == 1) put(p, x++, '.');
            for (int j = 1; j < nl; ++j) {
                if (j > 1) put(p, x++, ',');
                put(p, x++, (char)L_at(m.L, j));
            }
            const char tail[] = "\t.\t.\t.\tGT";
            for (int j = 0; j < 9; ++j) put(p, x++, tail[j]);
        }
        for (int k0 = 0; k0 < p.n_sel; k0 += 32) {
            const int k = k0 + lane;
            Geno g;
            int n = 0;
            if (k < p.n_sel) {
                sample_geno(p, line, m.n_geno, k, g);
                n = 1 + g.field_width();
            }
            int incl = n;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const int v = __shfl_up_sync(0xffffffffu, incl, d);
                if (lane >= d) incl += v;
            }
            if (k < p.n_sel) {                              // asCoded: the alleles' indices in L, all '.' when one is not in L
                int64_t x = o + at + (incl - n);
                put(p, x++, '\t');
                bool miss = false;
                for (int i = 0; i < g.n; ++i) miss |= L_index(m.L, g.allele(i)) < 0;
                for (int i = 0; i < g.n; ++i) {
                    if (i) put(p, x++, (char)g.phase);
                    put(p, x++, miss ? '.' : (char)('0' + L_index(m.L, g.allele(i))));
                }
            }
            at += __shfl_sync(0xffffffffu, incl, 31);
        }
        if (lane == 0) put(p, o + at, '\n');
    }
}


__global__ void k_g2v_run_off(const long long* __restrict__ starts, const long long* __restrict__ run_line, int64_t n_runs,
                              long long* __restrict__ run_off) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_runs; i += (int64_t)gridDim.x * blockDim.x)
        run_off[i] = starts[run_line[i]];
}

struct G2vState {
    // the reference: its text and flags until pg_g2v_ref_index, then the compacted sequences and {rec_off, rec_len}
    PgFasta ref;
    PgBuf cub;
    // the spec: col_slot [n_cols], col_prev [n_cols], sel_col [n_sel]
    PgBuf spec;
    int fmt = -1, n_cols = 0, n_slots = 0, n_sel = 0, use_ref = 0;
    // the current chunk: token starts, line records, row lengths and offsets (the scaffold hashes before them), scaffold
    // runs {line, offset, record}, the error word, the output slab
    PgBuf tok, meta, lens, runs, err, out;
    uint64_t text_gen = 0;
    size_t len = 0;
    int64_t S = -1, n_runs = 0, n_rows = 0;
    bool sited = false;
    std::vector<int64_t> h_off;
};

G2vState* gstate(pg_ctx* ctx) {
    if (!ctx->g2v_state) ctx->g2v_state = new G2vState();
    return (G2vState*)ctx->g2v_state;
}

G2vParams params(pg_ctx* ctx, G2vState* gs) {
    G2vParams p;
    memset(&p, 0, sizeof(p));
    p.buf = (const uint8_t*)ctx->text.p;
    p.len = gs->len;
    p.starts = (const long long*)ctx->starts.p;
    p.S = gs->S;
    p.fmt = gs->fmt;
    p.n_cols = gs->n_cols;
    p.n_slots = gs->n_slots;
    p.n_sel = gs->n_sel;
    p.col_slot = (const int32_t*)gs->spec.p;
    p.col_prev = p.col_slot + gs->n_cols;
    p.sel_col = p.col_prev + gs->n_cols;
    p.tok = (uint32_t*)gs->tok.p;
    p.meta = (LineMeta*)gs->meta.p;
    p.hash = (unsigned long long*)gs->lens.p;           // consumed by pg_scaffold_flags before the site pass writes lengths
    p.len_out = (int64_t*)gs->lens.p;
    p.off = p.len_out + (gs->S + 1);
    p.err = (unsigned long long*)gs->err.p;
    p.use_ref = gs->use_ref;
    p.n_runs = gs->n_runs;
    p.run_line = (const long long*)gs->runs.p;
    p.run_rec = (const int32_t*)(p.run_line + 2 * (gs->S + 1));
    p.rec_off = (const int64_t*)gs->ref.rec.p;
    p.rec_len = p.rec_off + gs->ref.n_rec;
    p.seq = (const uint8_t*)gs->ref.seq.p;
    return p;
}

}  // namespace

void pg_g2v_free(pg_ctx* ctx) {
    G2vState* gs = (G2vState*)ctx->g2v_state;
    if (!gs) return;
    gs->ref.release();
    PgBuf* bufs[] = {&gs->cub, &gs->spec, &gs->tok, &gs->meta, &gs->lens, &gs->runs, &gs->err, &gs->out};
    for (PgBuf* b : bufs) b->release();
    delete gs;
    ctx->g2v_state = nullptr;
}

extern "C" int pg_g2v_ref_load(pg_ctx* ctx, const char* text, size_t len, int64_t* n_rec) {
    PG_CHECK(ctx && (text || len == 0) && n_rec, "pg_g2v_ref_load: null argument");
    *n_rec = 0;
    PG_CUDA(cudaSetDevice(ctx->device));
    pg_timings_reset(ctx);
    G2vState* gs = gstate(ctx);
    return pg_fa_load(ctx, gs->ref, text, len, "g2v", n_rec);
}

extern "C" int pg_g2v_ref_starts(pg_ctx* ctx, int64_t* starts) {
    PG_CHECK(ctx && starts, "pg_g2v_ref_starts: null argument");
    G2vState* gs = gstate(ctx);
    PG_CHECK(!gs->ref.indexed, "pg_g2v_ref_starts: the record starts are gone after pg_g2v_ref_index");
    PG_CUDA(cudaSetDevice(ctx->device));
    return pg_fa_starts(ctx, gs->ref, starts);
}

extern "C" int pg_g2v_ref_index(pg_ctx* ctx, int64_t n_rec, const int64_t* lo, const int64_t* hi, int64_t* rec_len) {
    PG_CHECK(ctx && (n_rec == 0 || (lo && hi && rec_len)), "pg_g2v_ref_index: null argument");
    G2vState* gs = gstate(ctx);
    PG_CHECK(!gs->ref.indexed && n_rec == gs->ref.n_rec && n_rec > 0,
             "pg_g2v_ref_index: %lld records, the last pg_g2v_ref_load found %lld", (long long)n_rec, (long long)gs->ref.n_rec);
    for (int64_t k = 0; k < n_rec; ++k)
        PG_CHECK(lo[k] >= 0 && lo[k] <= hi[k] && hi[k] <= (int64_t)gs->ref.fa_len && (k == 0 || lo[k] >= hi[k - 1]),
                 "pg_g2v_ref_index: record %lld spans [%lld, %lld) (sorted, disjoint, inside the %zu bytes)", (long long)k,
                 (long long)lo[k], (long long)hi[k], gs->ref.fa_len);
    PG_CUDA(cudaSetDevice(ctx->device));
    pg_timings_reset(ctx);
    return pg_fa_index(ctx, gs->ref, n_rec, lo, hi, "g2v", rec_len);
}

extern "C" int pg_g2v_spec(pg_ctx* ctx, int32_t fmt, int32_t n_cols, const int32_t* col_slot, const int32_t* col_prev,
                           int32_t n_sel, const int32_t* sel_col, int32_t use_ref) {
    PG_CHECK(ctx && (n_cols == 0 || (col_slot && col_prev)) && sel_col, "pg_g2v_spec: null argument");
    PG_CHECK(fmt >= 0 && fmt <= 2, "pg_g2v_spec: format %d is not 0 (phased), 1 (diplo) or 2 (pairs)", fmt);
    PG_CHECK(n_sel >= 1 && n_cols >= 1, "pg_g2v_spec: %d selected samples of %d columns", n_sel, n_cols);
    G2vState* gs = gstate(ctx);
    PG_CHECK(!use_ref || gs->ref.indexed, "pg_g2v_spec: a reference lookup without pg_g2v_ref_index");
    int n_slots = 0;
    for (int c = 0; c < n_cols; ++c) {
        PG_CHECK(col_slot[c] == -1 || col_slot[c] == n_slots, "pg_g2v_spec: column %d has slot %d (slots number the slotted "
                 "columns in order)", c, col_slot[c]);
        n_slots += col_slot[c] >= 0;
        PG_CHECK(col_prev[c] >= -1 && col_prev[c] < c, "pg_g2v_spec: column %d follows column %d", c, col_prev[c]);
    }
    for (int k = 0; k < n_sel; ++k) {
        PG_CHECK(sel_col[k] >= 0 && sel_col[k] < n_cols, "pg_g2v_spec: sample %d reads column %d of %d", k, sel_col[k], n_cols);
        for (int c = sel_col[k]; c >= 0; c = col_prev[c])
            PG_CHECK(col_slot[c] >= 0, "pg_g2v_spec: column %d (read by sample %d) has no slot", c, k);
    }
    std::vector<int32_t> tab;
    tab.insert(tab.end(), col_slot, col_slot + n_cols);
    tab.insert(tab.end(), col_prev, col_prev + n_cols);
    tab.insert(tab.end(), sel_col, sel_col + n_sel);
    PG_CUDA(cudaSetDevice(ctx->device));
    PG_TRY(gs->spec.ensure(tab.size() * 4 + 64));
    PG_CUDA(cudaMemcpyAsync(gs->spec.p, tab.data(), tab.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    gs->fmt = fmt;
    gs->n_cols = n_cols;
    gs->n_slots = n_slots;
    gs->n_sel = n_sel;
    gs->use_ref = use_ref ? 1 : 0;
    gs->S = -1;
    return PG_OK;
}

extern "C" int pg_g2v_chunk(pg_ctx* ctx, const char* text, size_t len, int64_t* n_lines, int64_t* n_runs) {
    PG_CHECK(ctx && (text || len == 0) && n_lines && n_runs, "pg_g2v_chunk: null argument");
    G2vState* gs = gstate(ctx);
    PG_CHECK(gs->fmt >= 0, "pg_g2v_chunk: no pg_g2v_spec");
    PG_CHECK(len < ((size_t)1 << 32), "pg_g2v_chunk: a chunk of %zu bytes (a line of 4 GiB or more; token offsets are 32-bit)",
             len);
    *n_lines = *n_runs = 0;
    PG_CUDA(cudaSetDevice(ctx->device));
    pg_timings_reset(ctx);
    gs->S = -1;
    gs->sited = false;
    int64_t S = 0;
    PG_TRY(pg_text_load(ctx, text ? text : "", -1, 0, len, &S));
    ctx->ingest_sites = -1;                             // the text no longer belongs to the resident matrix
    PG_TRY(gs->tok.ensure((size_t)S * gs->n_slots * 4 + 64));
    PG_TRY(gs->meta.ensure((size_t)S * sizeof(LineMeta) + 64));
    PG_TRY(gs->lens.ensure((size_t)(S + 1) * 16 + 64));
    PG_TRY(gs->runs.ensure((size_t)(S + 1) * 20 + 64));
    PG_TRY(gs->err.ensure((size_t)S + 128));            // the error word, the selected count, the scaffold flags
    unsigned long long* d_err = (unsigned long long*)gs->err.p;
    int64_t* d_n = (int64_t*)(d_err + 1);
    int8_t* d_flags = (int8_t*)(d_n + 1);
    PG_CUDA(cudaMemsetAsync(d_err, 0xff, 8, ctx->stream));
    gs->len = len;
    gs->S = S;
    gs->n_runs = 0;
    gs->text_gen = ctx->text_gen;
    if (S > 0) {
        G2vParams p = params(ctx, gs);
        const unsigned grid = (unsigned)((S + 7) / 8);                 // one warp per line
        PG_TRY(pg_timed(ctx, "g2v_tokens", [&] { k_g2v_tokens<<<grid, 256, 0, ctx->stream>>>(p); }));
        PG_TRY(pg_scaffold_flags(ctx, p.hash, S, d_flags));
        long long* d_run_line = (long long*)gs->runs.p;
        thrust::counting_iterator<long long> idx(0);
        size_t tmp = 0;
        PG_CUDA(cub::DeviceSelect::Flagged(nullptr, tmp, idx, d_flags, d_run_line, d_n, S, ctx->stream));
        PG_TRY(gs->cub.ensure(tmp + 64));
        PG_TRY(pg_timed(ctx, "g2v_runs", [&] {
            cub::DeviceSelect::Flagged(gs->cub.p, tmp, idx, d_flags, d_run_line, d_n, S, ctx->stream);
        }));
        int64_t nr = 0;
        PG_CUDA(cudaMemcpyAsync(&nr, d_n, 8, cudaMemcpyDeviceToHost, ctx->stream));
        PG_CUDA(cudaStreamSynchronize(ctx->stream));
        gs->n_runs = nr;
        PG_TRY(pg_timed(ctx, "g2v_runs", [&] {
            k_g2v_run_off<<<(unsigned)std::min<int64_t>((nr + 255) / 256, 1024), 256, 0, ctx->stream>>>(
                (const long long*)ctx->starts.p, d_run_line, nr, d_run_line + (S + 1));
        }));
        ctx->launches += 4;
    }
    *n_lines = S;
    *n_runs = gs->n_runs;
    return PG_OK;
}

extern "C" int pg_g2v_runs(pg_ctx* ctx, int64_t* run_line, int64_t* run_off) {
    PG_CHECK(ctx && run_line && run_off, "pg_g2v_runs: null argument");
    G2vState* gs = gstate(ctx);
    PG_CHECK(gs->S >= 0 && gs->text_gen == ctx->text_gen, "pg_g2v_runs: no pg_g2v_chunk on the current text");
    if (gs->n_runs == 0) return PG_OK;
    PG_CUDA(cudaSetDevice(ctx->device));
    const long long* d = (const long long*)gs->runs.p;
    PG_CUDA(cudaMemcpyAsync(run_line, d, (size_t)gs->n_runs * 8, cudaMemcpyDeviceToHost, ctx->stream));
    PG_CUDA(cudaMemcpyAsync(run_off, d + (gs->S + 1), (size_t)gs->n_runs * 8, cudaMemcpyDeviceToHost, ctx->stream));
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    return PG_OK;
}

extern "C" int pg_g2v_sites(pg_ctx* ctx, const int32_t* run_rec, int64_t* n_rows, int64_t* n_bytes, int64_t* error) {
    PG_CHECK(ctx && n_rows && n_bytes && error, "pg_g2v_sites: null argument");
    G2vState* gs = gstate(ctx);
    PG_CHECK(gs->S >= 0 && gs->text_gen == ctx->text_gen, "pg_g2v_sites: no pg_g2v_chunk on the current text");
    PG_CHECK(!gs->use_ref || gs->n_runs == 0 || run_rec, "pg_g2v_sites: no record for the scaffold runs");
    const int64_t S = gs->S;
    for (int k = 0; k < 4; ++k) error[k] = 0;
    *n_rows = *n_bytes = 0;
    PG_CUDA(cudaSetDevice(ctx->device));
    pg_timings_reset(ctx);
    if (gs->use_ref)
        for (int64_t i = 0; i < gs->n_runs; ++i)
            PG_CHECK(run_rec[i] >= -1 && run_rec[i] < gs->ref.n_rec, "pg_g2v_sites: run %lld maps to record %d of %lld",
                     (long long)i, run_rec[i], (long long)gs->ref.n_rec);
    G2vParams p = params(ctx, gs);
    if (gs->use_ref && gs->n_runs)
        PG_CUDA(cudaMemcpyAsync((void*)p.run_rec, run_rec, (size_t)gs->n_runs * 4, cudaMemcpyHostToDevice, ctx->stream));
    PG_CUDA(cudaMemsetAsync(p.len_out + S, 0, 8, ctx->stream));
    if (S > 0) {
        const unsigned grid = (unsigned)((S + 7) / 8);                 // one warp per line
        PG_TRY(pg_timed(ctx, "g2v_sites", [&] { k_g2v_sites<<<grid, 256, 0, ctx->stream>>>(p); }));
    }
    size_t tmp = 0;
    int64_t* d_off = (int64_t*)p.off;
    PG_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tmp, p.len_out, d_off, S + 1, ctx->stream));
    PG_TRY(gs->cub.ensure(tmp + 64));
    PG_TRY(pg_timed(ctx, "g2v_scan", [&] {
        cub::DeviceScan::ExclusiveSum(gs->cub.p, tmp, p.len_out, d_off, S + 1, ctx->stream);
    }));
    ctx->launches += 2;
    unsigned long long w = ~0ull;
    PG_CUDA(cudaMemcpyAsync(&w, p.err, 8, cudaMemcpyDeviceToHost, ctx->stream));
    gs->h_off.resize((size_t)S + 1);
    PG_TRY(pg_d2h_staged(ctx, gs->h_off.data(), d_off, (size_t)(S + 1) * 8));
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    int64_t rows = S;
    if (w != ~0ull) {
        rows = (int64_t)(w >> 28) - 1;
        error[0] = (int64_t)(w & 15ull);
        error[1] = rows;
        error[2] = (int64_t)((w >> 4) & 0xffffffull);
        long long off = 0;
        PG_CUDA(cudaMemcpy(&off, (const long long*)ctx->starts.p + rows, 8, cudaMemcpyDeviceToHost));
        error[3] = off;
    }
    gs->n_rows = rows;
    gs->sited = true;
    *n_rows = rows;
    *n_bytes = gs->h_off[(size_t)rows];
    return PG_OK;
}

extern "C" int pg_g2v_emit(pg_ctx* ctx, int64_t byte0, char* out, size_t cap, size_t* bytes) {
    PG_CHECK(ctx && out && bytes, "pg_g2v_emit: null argument");
    G2vState* gs = gstate(ctx);
    PG_CHECK(gs->sited && gs->text_gen == ctx->text_gen, "pg_g2v_emit: no pg_g2v_sites on the current text");
    const std::vector<int64_t>& off = gs->h_off;
    const int64_t end = off[(size_t)gs->n_rows];
    PG_CHECK(byte0 >= 0 && byte0 <= end && cap > 0, "pg_g2v_emit: byte %lld of %lld", (long long)byte0, (long long)end);
    *bytes = 0;
    if (byte0 == end) return PG_OK;
    const int64_t b1 = std::min<int64_t>(end, byte0 + (int64_t)cap);
    const auto first = off.begin(), last = off.begin() + gs->n_rows + 1;
    const int64_t r0 = (int64_t)(std::upper_bound(first, last, byte0) - first) - 1;     // the row that holds byte0
    const int64_t r1 = (int64_t)(std::lower_bound(first, last, b1) - first);            // the first row at or after b1
    PG_CUDA(cudaSetDevice(ctx->device));
    pg_timings_reset(ctx);
    PG_TRY(gs->out.ensure((size_t)(b1 - byte0) + 64));
    G2vParams p = params(ctx, gs);
    p.r0 = r0;
    p.r1 = r1;
    p.b0 = byte0;
    p.b1 = b1;
    p.out = (char*)gs->out.p;
    const unsigned grid = (unsigned)((r1 - r0 + 7) / 8);               // one warp per row
    PG_TRY(pg_timed(ctx, "g2v_emit", [&] { k_g2v_emit<<<grid, 256, 0, ctx->stream>>>(p); }));
    ctx->launches += 1;
    PG_CUDA(cudaMemcpyAsync(out, gs->out.p, (size_t)(b1 - byte0), cudaMemcpyDeviceToHost, ctx->stream));
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    *bytes = (size_t)(b1 - byte0);
    return PG_OK;
}
