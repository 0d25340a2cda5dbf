// parseVCF.py on the device: VCF text -> .geno rows (VCF_processing/parseVCF.py:13-237, 350-391).
//
//   k_vcf_count_starts / k_vcf_write_starts : data-line start offsets, as ingest.cu's two passes around an exclusive scan,
//                    with the VCF line rule (universal newlines: '\n', '\r\n' and a lone '\r' end a line; blank lines and
//                    lines whose first field starts with '#' are skipped; str.split() blanks include \x1c-\x1f)
//   k_vcf_records  : ONE WARP PER LINE, as k_parse_lines: lanes classify 4 bytes per step, a warp prefix sum numbers the
//                    fields.  Fields 0-8 give the CHROM / POS / REF / ALT / QUAL / FORMAT spans; the start of every
//                    sample column a selected sample may read goes to a per-line slot table.  Lane 0 then parses POS
//                    (int64, fast path), the ALTs (count, every allele as long as REF), QUAL against --minQual and the
//                    FORMAT keys (one bit mask of positions per looked-up key).  Lines with a byte >= 0x80 are flagged.
//   k_vcf_links    : one thread per line: --excludeDuplicates compares CHROM and POS text with the data line before.
//   k_vcf_genotypes: ONE THREAD PER (kept row, selected sample): GT, the genotype filters, the ploidy; writes a verdict
//                    byte and the GT (or --field) span, no text.  Tokens off the fast number path are left to the host.
//   k_vcf_emit     : ONE WARP PER KEPT ROW, as k_filter_emit: lengths, a CUB exclusive scan, then the bytes of a slab.
#include <algorithm>
#include <cub/cub.cuh>

#include "pgwin_internal.h"

namespace {

constexpr int CS_THREADS = 256;
constexpr int CS_BYTES_PER_THREAD = 16;
constexpr int CS_BLOCK_BYTES = CS_THREADS * CS_BYTES_PER_THREAD;
constexpr int VCF_MAX_KEYS = 40;

__device__ __forceinline__ bool vws(unsigned c) { return c == ' ' || c == '\t' || c == '\v' || c == '\f' || (c >= 0x1c && c <= 0x1f); }
__device__ __forceinline__ bool vterm(unsigned c) { return c == '\n' || c == '\r'; }
__device__ __forceinline__ bool vblank(unsigned c) { return vws(c) || vterm(c); }

// i is the first byte of a line ('\n' right after '\r' belongs to the '\r\n' before it)
__device__ __forceinline__ bool vcf_line_begins(const uint8_t* __restrict__ b, size_t i) {
    if (i == 0) return true;
    const unsigned p = b[i - 1];
    return p == '\n' || (p == '\r' && b[i] != '\n');
}

// a data line starts at i: a line begins there, holds a non-blank byte, and its first field does not start with '#'
__device__ __forceinline__ bool vcf_line_start_at(const uint8_t* __restrict__ b, size_t len, size_t i) {
    if (i >= len || !vcf_line_begins(b, i)) return false;
    for (size_t j = i; j < len; ++j) {
        const unsigned c = b[j];
        if (vterm(c)) return false;
        if (!vws(c)) return c != '#';
    }
    return false;
}

__global__ void __launch_bounds__(CS_THREADS) k_vcf_count_starts(const uint8_t* __restrict__ buf, size_t len,
                                                                 unsigned* __restrict__ block_counts) {
    typedef cub::BlockReduce<unsigned, CS_THREADS> BR;
    __shared__ typename BR::TempStorage tmp;
    const size_t base = (size_t)blockIdx.x * CS_BLOCK_BYTES + (size_t)threadIdx.x * CS_BYTES_PER_THREAD;
    unsigned n = 0;
    for (int k = 0; k < CS_BYTES_PER_THREAD; ++k) n += vcf_line_start_at(buf, len, base + k) ? 1u : 0u;
    const unsigned tot = BR(tmp).Sum(n);
    if (threadIdx.x == 0) block_counts[blockIdx.x] = tot;
}

__global__ void __launch_bounds__(CS_THREADS) k_vcf_write_starts(const uint8_t* __restrict__ buf, size_t len,
                                                                 const unsigned long long* __restrict__ block_base,
                                                                 long long* __restrict__ starts) {
    typedef cub::BlockScan<unsigned, CS_THREADS> BS;
    __shared__ typename BS::TempStorage tmp;
    const size_t base = (size_t)blockIdx.x * CS_BLOCK_BYTES + (size_t)threadIdx.x * CS_BYTES_PER_THREAD;
    unsigned flags = 0, n = 0;
    for (int k = 0; k < CS_BYTES_PER_THREAD; ++k)
        if (vcf_line_start_at(buf, len, base + k)) {
            flags |= 1u << k;
            ++n;
        }
    unsigned off;
    BS(tmp).ExclusiveSum(n, off);
    unsigned long long o = block_base[blockIdx.x] + off;
    for (int k = 0; k < CS_BYTES_PER_THREAD; ++k)
        if (flags & (1u << k)) starts[o++] = (long long)(base + k);
}

// ---- numbers -------------------------------------------------------------------------------------------------------

enum { NUM_OK = 0, NUM_INVALID = 1, NUM_UNRESOLVED = 2 };

__device__ __forceinline__ bool lower_eq(const uint8_t* t, int n, const char* w) {
    for (int i = 0; i < n; ++i) {
        unsigned c = t[i];
        if (c >= 'A' && c <= 'Z') c += 32;
        if (c != (unsigned)w[i]) return false;
    }
    return w[n] == 0;
}

// Python float() of the token t[0, n): NUM_OK with the exact double on the fast path (ASCII decimal with a significand below
// 2^53 and a power of ten of at most 22 either way: one correctly rounded multiply or divide, Clinger's exact case; inf,
// infinity and nan in any case, signed); NUM_INVALID for tokens float() certainly rejects; NUM_UNRESOLVED otherwise
// ('_', more digits, larger exponents, non-ASCII digits), which the host settles with float().
__device__ int parse_double(const uint8_t* t, int n, double& v) {
    if (n == 0) return NUM_INVALID;
    for (int i = 0; i < n; ++i) {
        const unsigned c = t[i];
        if (c >= 0x80) return NUM_UNRESOLVED;
        const bool can = (c >= '0' && c <= '9') || c == '+' || c == '-' || c == '.' || c == '_' || c == 'e' || c == 'E' ||
                         c == 'i' || c == 'I' || c == 'n' || c == 'N' || c == 'f' || c == 'F' || c == 't' || c == 'T' ||
                         c == 'y' || c == 'Y' || c == 'a' || c == 'A';
        if (!can) return NUM_INVALID;
    }
    int i = 0;
    bool neg = false;
    if (t[0] == '+' || t[0] == '-') {
        neg = t[0] == '-';
        i = 1;
    }
    const uint8_t* r = t + i;
    const int rn = n - i;
    if (lower_eq(r, rn, "inf") || lower_eq(r, rn, "infinity")) {
        v = neg ? -INFINITY : INFINITY;
        return NUM_OK;
    }
    if (lower_eq(r, rn, "nan")) {
        v = NAN;
        return NUM_OK;
    }
    unsigned long long m = 0;
    int sig = 0, frac = 0, digits = 0;
    bool dot = false;
    for (; i < n; ++i) {
        const unsigned c = t[i];
        if (c >= '0' && c <= '9') {
            ++digits;
            if (m == 0 && c == '0') {
                if (dot) ++frac;
                continue;
            }
            if (++sig > 19) return NUM_UNRESOLVED;
            m = m * 10 + (c - '0');
            if (dot) ++frac;
        } else if (c == '.' && !dot) {
            dot = true;
        } else {
            break;
        }
    }
    if (digits == 0) return NUM_INVALID;            // float() needs a digit before the exponent
    int e = 0;
    if (i < n) {
        if (t[i] != 'e' && t[i] != 'E') return NUM_UNRESOLVED;
        ++i;
        bool eneg = false;
        if (i < n && (t[i] == '+' || t[i] == '-')) {
            eneg = t[i] == '-';
            ++i;
        }
        if (i == n) return NUM_UNRESOLVED;
        for (; i < n; ++i) {
            const unsigned c = t[i];
            if (c < '0' || c > '9') return NUM_UNRESOLVED;
            if (e < 100000) e = e * 10 + (int)(c - '0');
        }
        if (eneg) e = -e;
    }
    if (m == 0) {
        v = neg ? -0.0 : 0.0;
        return NUM_OK;
    }
    if (m > (1ull << 53)) return NUM_UNRESOLVED;
    const int p = e - frac;
    if (p > 22 || p < -22) return NUM_UNRESOLVED;
    const double p10[23] = {1e0,  1e1,  1e2,  1e3,  1e4,  1e5,  1e6,  1e7,  1e8,  1e9,  1e10, 1e11,
                            1e12, 1e13, 1e14, 1e15, 1e16, 1e17, 1e18, 1e19, 1e20, 1e21, 1e22};
    double x = (double)m;
    x = p >= 0 ? x * p10[p] : x / p10[-p];
    v = neg ? -x : x;
    return NUM_OK;
}

// Python int() of POS on the fast path: sign, ASCII digits with single '_' between digits, at most 18 digits
__device__ bool parse_pos(const uint8_t* t, int n, long long& v) {
    int i = 0;
    bool neg = false;
    if (n > 0 && (t[0] == '+' || t[0] == '-')) {
        neg = t[0] == '-';
        i = 1;
    }
    if (i >= n) return false;
    long long x = 0;
    int nd = 0;
    bool prev_digit = false;
    for (; i < n; ++i) {
        const unsigned c = t[i];
        if (c >= '0' && c <= '9') {
            x = x * 10 + (c - '0');
            if (x != 0 && ++nd > 18) return false;
            prev_digit = true;
        } else if (c == '_' && prev_digit && i + 1 < n && t[i + 1] >= '0' && t[i + 1] <= '9') {
            prev_digit = false;
        } else {
            return false;
        }
    }
    v = neg ? -x : x;
    return true;
}

// ---- per-line records ----------------------------------------------------------------------------------------------

struct RecParams {
    const uint8_t* buf;
    size_t len;
    const long long* starts;
    int64_t S;
    int n_cols;
    const int32_t* col_slot;
    int n_slots;
    uint32_t* slots;                // [S x n_slots] offset of the column's first byte from the line start
    int n_keys;
    const int32_t* key_off;         // [n_keys + 1] into key_chars
    const uint8_t* key_chars;
    unsigned long long* key_mask;   // [S x n_keys] bit j: FORMAT key j is this key
    int has_min_qual;
    double min_qual;
    pg_vcf_line* lines;
};

__device__ __forceinline__ unsigned vbyte(const RecParams& rp, size_t i) { return i < rp.len ? rp.buf[i] : (unsigned)'\n'; }

__global__ void __launch_bounds__(256) k_vcf_records(const __grid_constant__ RecParams rp) {
    __shared__ uint32_t span[8][9][2];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int64_t warps = (int64_t)gridDim.x * 8;
    for (int64_t line = (int64_t)blockIdx.x * 8 + wid; line < rp.S; line += warps) {
        const size_t l0 = (size_t)rp.starts[line];
        if (lane < 18) span[wid][lane / 2][lane & 1] = 0;
        __syncwarp();
        unsigned fields_before = 0;
        bool prev_ws = true, high = false, done = false;
        size_t line_end = rp.len;
        for (size_t step = 0; !done; ++step) {
            const size_t wbase = l0 + step * 128 + (size_t)lane * 4;
            unsigned ws = 0, nl = 0, hi = 0;
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const unsigned c = vbyte(rp, wbase + k);
                if (vws(c)) ws |= 1u << k;
                else if (vterm(c)) nl |= 1u << k;
                if (c >= 0x80) hi |= 1u << k;
            }
            // everything from the first terminator of the line on is outside the line
            const unsigned nl_lanes = __ballot_sync(0xffffffffu, nl != 0);
            if (nl_lanes) {
                const int first = __ffs(nl_lanes) - 1;
                if (lane > first) ws = 0xfu, nl = 0, hi = 0;
                else if (lane == first) {
                    const unsigned from = nl & (0u - nl);
                    ws |= ~(from - 1u) & 0xfu;
                    hi &= from - 1u;
                }
                line_end = __shfl_sync(0xffffffffu, (unsigned long long)(wbase + (__ffs(nl | 16u) - 1)), first);
                done = true;
            }
            high |= hi != 0;
            const unsigned last_ws = (ws >> 3) & 1u;
            unsigned pw = __shfl_up_sync(0xffffffffu, last_ws, 1);
            if (lane == 0) pw = prev_ws ? 1u : 0u;
            const unsigned st = ~ws & (((ws << 1) | pw) & 0xfu) & 0xfu;
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
                if (fidx < 9) {
                    size_t e = q;
                    if (fidx != 7)
                        while (!vblank(vbyte(rp, e))) ++e;
                    span[wid][fidx][0] = (uint32_t)(q - l0);
                    span[wid][fidx][1] = (uint32_t)(e - q);
                } else if ((int)fidx < rp.n_cols) {
                    const int s = rp.col_slot[fidx];
                    if (s >= 0) rp.slots[line * rp.n_slots + s] = (uint32_t)(q - l0);
                }
            }
        }
        // a byte >= 0x80 before the line's end (the lanes past the terminator dropped theirs above)
        const bool any_high = __any_sync(0xffffffffu, high);
        __syncwarp();
        if (lane == 0) {
            pg_vcf_line L;
            L.start = (int64_t)l0;
            L.end = (int64_t)line_end;
            L.n_fields = (int32_t)fields_before;
            uint32_t fl = any_high ? PG_VCF_NONASCII : 0u;
            const uint32_t(*sp)[2] = span[wid];
            L.chrom_off = sp[0][0]; L.chrom_len = sp[0][1];
            L.pos_off = sp[1][0];   L.pos_len = sp[1][1];
            L.ref_off = sp[3][0];   L.ref_len = sp[3][1];
            L.alt_off = sp[4][0];   L.alt_len = sp[4][1];
            L.qual_off = sp[5][0];  L.qual_len = sp[5][1];
            L.fmt_off = sp[8][0];   L.fmt_len = sp[8][1];
            const uint8_t* t = rp.buf + l0;
            long long pos = 0;
            if (L.n_fields < 2 || !parse_pos(t + L.pos_off, (int)L.pos_len, pos)) fl |= PG_VCF_POS_UNRESOLVED;
            L.pos = pos;
            // ALT: "." is no ALT; otherwise comma-separated alleles, each compared in length with REF
            int nalt = 0;
            bool same_len = true;
            if (L.n_fields >= 5 && !(L.alt_len == 1 && t[L.alt_off] == '.')) {
                uint32_t a = 0;
                nalt = 1;
                for (uint32_t i = 0; i < L.alt_len; ++i)
                    if (t[L.alt_off + i] == ',') {
                        same_len &= (a == L.ref_len);
                        a = 0;
                        ++nalt;
                    } else {
                        ++a;
                    }
                same_len &= (a == L.ref_len);
            }
            L.n_alt = nalt;
            if (same_len) fl |= PG_VCF_SAME_LEN;
            if (rp.has_min_qual && L.n_fields >= 6) {
                double q = 0;
                const int r = parse_double(t + L.qual_off, (int)L.qual_len, q);
                if (r == NUM_UNRESOLVED) fl |= PG_VCF_QUAL_UNRESOLVED;
                else if (r == NUM_OK && q < rp.min_qual) fl |= PG_VCF_QUAL_DROP;
            }
            // FORMAT keys: bit j of key k's mask = the j-th key is k
            unsigned long long* km = rp.key_mask + line * rp.n_keys;
            for (int k = 0; k < rp.n_keys; ++k) km[k] = 0;
            if (L.n_fields >= 9) {
                uint32_t a = 0;
                int j = 0;
                for (uint32_t i = 0; i <= L.fmt_len; ++i) {
                    if (i < L.fmt_len && t[L.fmt_off + i] != ':') continue;
                    const int kl = (int)(i - a);
                    for (int k = 0; k < rp.n_keys; ++k) {
                        const int o = rp.key_off[k];
                        if (rp.key_off[k + 1] - o != kl) continue;
                        bool eq = true;
                        for (int c = 0; c < kl && eq; ++c) eq = rp.key_chars[o + c] == t[L.fmt_off + a + c];
                        if (eq) {
                            if (j >= 64) fl |= PG_VCF_FORMAT_WIDE;
                            else km[k] |= 1ull << j;
                        }
                    }
                    ++j;
                    a = i + 1;
                }
            }
            L.flags = fl;
            rp.lines[line] = L;
        }
        __syncwarp();
    }
}

__device__ __forceinline__ bool same_text(const uint8_t* a, uint32_t an, const uint8_t* b, uint32_t bn) {
    if (an != bn) return false;
    for (uint32_t i = 0; i < an; ++i)
        if (a[i] != b[i]) return false;
    return true;
}

// --excludeDuplicates: CHROM and POS text equal to those of the data line before (line 0: the previous chunk's last one)
__global__ void k_vcf_links(const uint8_t* __restrict__ buf, pg_vcf_line* __restrict__ lines, int64_t S,
                            const uint8_t* __restrict__ prev, uint32_t prev_chrom, uint32_t prev_pos) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < S; i += (int64_t)gridDim.x * blockDim.x) {
        pg_vcf_line& L = lines[i];
        if (L.n_fields < 2) continue;
        const uint8_t* t = buf + L.start;
        bool dup;
        if (i == 0) {
            dup = prev != nullptr && same_text(t + L.chrom_off, L.chrom_len, prev, prev_chrom) &&
                  same_text(t + L.pos_off, L.pos_len, prev + prev_chrom, prev_pos);
        } else {
            const pg_vcf_line& P = lines[i - 1];
            const uint8_t* u = buf + P.start;
            dup = P.n_fields >= 2 && same_text(t + L.chrom_off, L.chrom_len, u + P.chrom_off, P.chrom_len) &&
                  same_text(t + L.pos_off, L.pos_len, u + P.pos_off, P.pos_len);
        }
        if (dup) L.flags |= PG_VCF_DUPLICATE;
    }
}

// ---- genotypes -----------------------------------------------------------------------------------------------------

enum { V_FAIL = 1, V_UNRESOLVED = 2, V_PLOIDY = 4, V_PHASED = 8, V_ABSENT = 16, V_PHASE_FIELD = 32 };

struct IsUnresolved {
    __device__ int64_t operator()(uint8_t v) const { return (v & V_UNRESOLVED) ? 1 : 0; }
};
enum { GERR_NO_GT = 1, GERR_PLOIDY = 2 };

struct GenoParams {
    const uint8_t* buf;
    const pg_vcf_line* lines;
    const uint32_t* slots;
    int n_slots;
    const unsigned long long* key_mask;
    int n_keys;
    const int64_t* rows;            // [R] line of every kept row
    const int64_t* pos;             // [R] its POS
    int64_t R;
    int n_samp;
    const int32_t* samp_col;
    const int32_t* col_prev;
    const int32_t* col_slot;
    const int32_t* samp_ploidy;
    int field_key, field_phase;     // --field: key index (-1: genotypes); field_phase: --field phase
    int n_filt;
    const int32_t* filt_key;
    const double* filt_min;
    const double* filt_max;
    const uint8_t* filt_site;
    const uint8_t* filt_gt;
    const uint8_t* filt_samp;       // [n_filt x n_samp]
    const uint8_t* missing;
    int missing_len;
    const uint8_t* sep;
    int sep_len;
    int skip_indels, keep_partial, p2m, add_ref;
    uint8_t* verdict;               // [R x n_samp]
    uint2* span;                    // [R x n_samp] GT (or --field) value: offset from the line start, length
    unsigned long long* err;
    unsigned long long* n_unres;
    // emission
    const int64_t* off;
    char* out;
    int64_t row0, nrows;
    int64_t* len;
};

// j-th ':' subfield of the sample text [a, e): its offset and length
__device__ __forceinline__ bool subfield(const uint8_t* t, uint32_t a, uint32_t e, int j, uint32_t& o, uint32_t& n) {
    uint32_t i = a;
    for (int k = 0; k < j; ++k) {
        while (i < e && t[i] != ':') ++i;
        if (i >= e) return false;
        ++i;
    }
    uint32_t b = i;
    while (b < e && t[b] != ':') ++b;
    o = i;
    n = b - i;
    return true;
}

// the value of key k for a sample with nv subfields: dict(zip(keys, values)) keeps the last key within the values
__device__ __forceinline__ int key_index(unsigned long long mask, int nv) {
    if (nv < 64) mask &= (1ull << nv) - 1ull;
    return mask ? 63 - __clzll(mask) : -1;
}

__device__ __forceinline__ void report(const GenoParams& gp, int64_t line, int s, int code) {
    const unsigned long long s1 = (unsigned long long)min(s, (1 << 21) - 1);
    atomicMin(gp.err, ((unsigned long long)(line + 1) << 24) | (s1 << 3) | (unsigned long long)code);
}

__global__ void __launch_bounds__(256) k_vcf_genotypes(const __grid_constant__ GenoParams gp) {
    const int64_t total = gp.R * gp.n_samp;
    for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < total; g += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = g / gp.n_samp;
        const int s = (int)(g - r * gp.n_samp);
        const int64_t line = gp.rows[r];
        const pg_vcf_line L = gp.lines[line];
        const uint8_t* t = gp.buf + L.start;
        int c = gp.samp_col[s];
        while (c >= L.n_fields) c = gp.col_prev[c];
        const uint32_t a = gp.slots[line * gp.n_slots + gp.col_slot[c]];
        uint32_t e = a;
        int nv = 1;
        while (!vblank(t[e])) nv += t[e++] == ':';
        const unsigned long long* km = gp.key_mask + line * gp.n_keys;
        uint8_t v = 0;
        uint32_t go = 0, gn = 0;
        const int jg = key_index(km[0], nv);
        const bool has_gt = jg >= 0 && subfield(t, a, e, jg, go, gn);
        bool phased = false;
        int n_al = 1;
        for (uint32_t i = 0; has_gt && i < gn; ++i) {
            const unsigned ch = t[go + i];
            phased |= ch == '|';
            n_al += ch == '|' || ch == '/';
        }
        if (phased) v |= V_PHASED;
        if (gp.field_key >= 0) {                             // getGenoField (parseVCF.py:183-190)
            uint32_t fo = 0, fn = 0;
            const int jf = key_index(km[gp.field_key], nv);
            if (gp.field_phase && has_gt) {
                v |= V_PHASE_FIELD;                         // genoData["phase"], set with the GT (97)
            } else if (!(jf >= 0 && subfield(t, a, e, jf, fo, fn))) {
                v |= V_ABSENT;
            }
            gp.verdict[g] = v;
            gp.span[g] = make_uint2(fo, fn);
            continue;
        }
        if (!has_gt) {
            report(gp, line, s, GERR_NO_GT);
            gp.verdict[g] = V_FAIL;
            continue;
        }
        // GTtype (parseVCF.py:13-18): all alleles the same text?  then "0" / "." / other
        uint32_t l0 = 0;
        while (l0 < gn && t[go + l0] != '/' && t[go + l0] != '|') ++l0;
        bool het = false;
        {
            uint32_t i = l0;
            while (i < gn && !het) {
                const uint32_t b = ++i;
                while (i < gn && t[go + i] != '/' && t[go + i] != '|') ++i;
                het = !same_text(t + go, l0, t + go + b, i - b);
            }
        }
        const unsigned gtbit = het ? 1u : (l0 == 1 && t[go] == '0' ? 2u : (l0 == 1 && t[go] == '.' ? 4u : 8u));
        const unsigned sitebit = L.n_alt == 0 ? 1u : ((L.flags & PG_VCF_SAME_LEN) ? 2u : 4u);
        for (int f = 0; f < gp.n_filt; ++f) {                 // parseVCF.py:118-131
            if (!(gp.filt_site[f] & sitebit) || !(gp.filt_gt[f] & gtbit) || !gp.filt_samp[(size_t)f * gp.n_samp + s]) continue;
            bool pass = false;
            uint32_t vo, vn;
            const int k = gp.filt_key[f];
            const int j = k >= 0 ? key_index(km[k], nv) : -1;
            if (j >= 0 && subfield(t, a, e, j, vo, vn)) {
                pass = true;
                uint32_t i = vo;
                for (;;) {
                    uint32_t b = i;
                    while (b < vo + vn && t[b] != ',') ++b;
                    double x = 0;
                    const int rc = parse_double(t + i, (int)(b - i), x);
                    if (rc == NUM_UNRESOLVED) {
                        v |= V_UNRESOLVED;
                        break;
                    }
                    if (rc == NUM_INVALID || !(gp.filt_min[f] <= x && x <= gp.filt_max[f])) {
                        pass = false;
                        break;
                    }
                    if (b >= vo + vn) break;
                    i = b + 1;
                }
            }
            if (v & V_UNRESOLVED) break;
            if (!pass) {
                v |= V_FAIL;
                break;
            }
        }
        if (n_al != gp.samp_ploidy[s]) {                      // 133-139
            if (gp.p2m) v |= V_PLOIDY;
            else report(gp, line, s, GERR_PLOIDY);
        }
        gp.verdict[g] = v;
        gp.span[g] = make_uint2(go, gn);
    }
}

// ---- emission ------------------------------------------------------------------------------------------------------

// allele a of the line: REF (a = 0) or the a-th ALT
__device__ __forceinline__ void allele_text(const uint8_t* t, const pg_vcf_line& L, int a, uint32_t& o, uint32_t& n) {
    if (a == 0) {
        o = L.ref_off;
        n = L.ref_len;
        return;
    }
    uint32_t i = L.alt_off;
    for (int k = 1; k < a; ++k) {
        while (t[i] != ',') ++i;
        ++i;
    }
    uint32_t b = i;
    while (b < L.alt_off + L.alt_len && t[b] != ',') ++b;
    o = i;
    n = b - i;
}

// the allele key "0".."nALT" of the text, or -1 (the lookup in alleleDict raises, parseVCF.py:145)
__device__ __forceinline__ int allele_key(const uint8_t* k, uint32_t n, int nalt) {
    if (n == 0 || n > 9 || (n > 1 && k[0] == '0')) return -1;
    int x = 0;
    for (uint32_t i = 0; i < n; ++i) {
        if (k[i] < '0' || k[i] > '9') return -1;
        x = x * 10 + (k[i] - '0');
    }
    return x <= nalt ? x : -1;
}

__device__ __forceinline__ void put(char* o, int& n, const uint8_t* src, uint32_t len) {
    if (o)
        for (uint32_t i = 0; i < len; ++i) o[n + i] = (char)src[i];
    n += (int)len;
}

// text of genotype (row, sample): getGenotype (parseVCF.py:141-163) or getGenoField; writes it at o when o != nullptr
__device__ int geno_text(const GenoParams& gp, const uint8_t* t, const pg_vcf_line& L, int64_t g, int s, char* o) {
    const uint8_t v = gp.verdict[g];
    const uint2 sp = gp.span[g];
    int n = 0;
    const uint8_t ph = (v & V_PHASED) ? '|' : '/';
    if (gp.field_key >= 0) {
        if (v & V_ABSENT) put(o, n, gp.missing, gp.missing_len);
        else if (v & V_PHASE_FIELD) put(o, n, &ph, 1);
        else put(o, n, t + sp.x, sp.y);
        return n;
    }
    bool all_missing = (v & (V_FAIL | V_PLOIDY)) != 0;
    const int pl = gp.samp_ploidy[s];
    if (!all_missing) {
        // first walk: every key must look up, and (without --keepPartial) no allele may read as the missing string
        bool any_missing = false;
        for (uint32_t i = 0; i <= sp.y && !all_missing;) {
            uint32_t b = i;
            while (b < sp.y && t[sp.x + b] != '/' && t[sp.x + b] != '|') ++b;
            const int k = allele_key(t + sp.x + i, b - i, L.n_alt);
            if (k < 0) {
                all_missing = true;
                break;
            }
            uint32_t ao, an;
            allele_text(t, L, k, ao, an);
            if (gp.skip_indels && an != L.ref_len) any_missing = true;
            else any_missing |= same_text(t + ao, an, gp.missing, (uint32_t)gp.missing_len);
            i = b + 1;
        }
        if (any_missing && !gp.keep_partial) all_missing = true;
        if (!all_missing) {
            bool first = true;
            for (uint32_t i = 0; i <= sp.y;) {
                uint32_t b = i;
                while (b < sp.y && t[sp.x + b] != '/' && t[sp.x + b] != '|') ++b;
                const int k = allele_key(t + sp.x + i, b - i, L.n_alt);
                uint32_t ao, an;
                allele_text(t, L, k, ao, an);
                if (!first) put(o, n, &ph, 1);
                first = false;
                if (gp.skip_indels && an != L.ref_len) put(o, n, gp.missing, gp.missing_len);
                else put(o, n, t + ao, an);
                i = b + 1;
            }
            return n;
        }
    }
    for (int k = 0; k < pl; ++k) {                            // [missing] * ploidy
        if (k) put(o, n, &ph, 1);
        put(o, n, gp.missing, gp.missing_len);
    }
    return n;
}

__device__ __forceinline__ int dec_len(long long x, char* o) {
    char d[24];
    int n = 0;
    unsigned long long u = x < 0 ? 0ull - (unsigned long long)x : (unsigned long long)x;
    do {
        d[n++] = (char)('0' + u % 10);
        u /= 10;
    } while (u);
    int w = 0;
    if (x < 0) {
        if (o) o[w] = '-';
        ++w;
    }
    for (int i = n - 1; i >= 0; --i, ++w)
        if (o) o[w] = d[i];
    return w;
}

template <bool WRITE>
__global__ void __launch_bounds__(256) k_vcf_emit(const __grid_constant__ GenoParams gp) {
    const int lane = threadIdx.x & 31;
    for (int64_t r = gp.row0 + (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5); r < gp.row0 + gp.nrows; r += (int64_t)gridDim.x * 8) {
        const int64_t line = gp.rows[r];
        const pg_vcf_line L = gp.lines[line];
        const uint8_t* t = gp.buf + L.start;
        char* o = WRITE ? gp.out + (gp.off[r] - gp.off[gp.row0]) : nullptr;
        // CHROM sep str(POS) [sep REF]
        int at = 0;
        if (lane == 0) {
            put(o, at, t + L.chrom_off, L.chrom_len);
            put(o, at, gp.sep, gp.sep_len);
            at += dec_len(gp.pos[r], o ? o + at : nullptr);
            if (gp.add_ref) {
                put(o, at, gp.sep, gp.sep_len);
                put(o, at, t + L.ref_off, L.ref_len);
            }
        }
        int64_t base = __shfl_sync(0xffffffffu, at, 0);
        for (int s0 = 0; s0 < gp.n_samp; s0 += 32) {
            const int s = s0 + lane;
            const int64_t g = r * gp.n_samp + s;
            const int n = s < gp.n_samp ? gp.sep_len + geno_text(gp, t, L, g, s, nullptr) : 0;
            int incl = n;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const int x = __shfl_up_sync(0xffffffffu, incl, d);
                if (lane >= d) incl += x;
            }
            if (WRITE && s < gp.n_samp) {
                char* q = o + base + (incl - n);
                int w = 0;
                put(q, w, gp.sep, gp.sep_len);
                geno_text(gp, t, L, g, s, q + w);
            }
            base += __shfl_sync(0xffffffffu, incl, 31);
        }
        if (lane == 0) {
            if (WRITE) o[base] = '\n';
            else gp.len[r] = base + 1;
        }
    }
}

// ---- host side -----------------------------------------------------------------------------------------------------

// blocks of the spec table on the device (pg_vcf_set_spec), in this order
enum { B_COL_SLOT, B_KEY_OFF, B_KEY_CHARS, B_SAMP_COL, B_COL_PREV, B_PLOIDY, B_FKEY, B_FMIN, B_FMAX, B_FSITE, B_FGT, B_FSAMP,
       B_MISSING, B_SEP, B_PREV, N_BLOCKS };

struct VcfState {
    bool have_spec = false;
    int n_cols = 0, n_slots = 0, n_keys = 0, n_samp = 0, n_filt = 0, field_key = -1, field_phase = 0;
    int has_min_qual = 0;
    double min_qual = 0;
    int skip_indels = 0, keep_partial = 0, p2m = 0, add_ref = 0, missing_len = 0, sep_len = 0;
    size_t at[N_BLOCKS] = {};       // byte offset of every block in `tab`
    PgBuf tab, text, starts, lines, slots, masks, rows, verdict, span, off, out, cub, scratch;
    size_t len = 0;
    int64_t S = -1, R = -1;
    bool offsets_ready = false;
    std::vector<int64_t> h_off;
    const char* block(int b) const { return (const char*)tab.p + at[b]; }
};

VcfState* vstate(pg_ctx* ctx) {
    if (!ctx->vcf_state) ctx->vcf_state = new VcfState();
    return (VcfState*)ctx->vcf_state;
}

GenoParams geno_params(VcfState* vs) {
    GenoParams gp;
    memset(&gp, 0, sizeof(gp));
    gp.buf = (const uint8_t*)vs->text.p;
    gp.lines = (const pg_vcf_line*)vs->lines.p;
    gp.slots = (const uint32_t*)vs->slots.p;
    gp.n_slots = vs->n_slots;
    gp.key_mask = (const unsigned long long*)vs->masks.p;
    gp.n_keys = vs->n_keys;
    gp.rows = (const int64_t*)vs->rows.p;
    gp.pos = (const int64_t*)vs->rows.p + std::max<int64_t>(vs->R, 1);
    gp.R = vs->R;
    gp.n_samp = vs->n_samp;
    gp.samp_col = (const int32_t*)vs->block(B_SAMP_COL);
    gp.col_prev = (const int32_t*)vs->block(B_COL_PREV);
    gp.col_slot = (const int32_t*)vs->block(B_COL_SLOT);
    gp.samp_ploidy = (const int32_t*)vs->block(B_PLOIDY);
    gp.field_key = vs->field_key;
    gp.field_phase = vs->field_phase;
    gp.n_filt = vs->n_filt;
    gp.filt_key = (const int32_t*)vs->block(B_FKEY);
    gp.filt_min = (const double*)vs->block(B_FMIN);
    gp.filt_max = (const double*)vs->block(B_FMAX);
    gp.filt_site = (const uint8_t*)vs->block(B_FSITE);
    gp.filt_gt = (const uint8_t*)vs->block(B_FGT);
    gp.filt_samp = (const uint8_t*)vs->block(B_FSAMP);
    gp.missing = (const uint8_t*)vs->block(B_MISSING);
    gp.missing_len = vs->missing_len;
    gp.sep = (const uint8_t*)vs->block(B_SEP);
    gp.sep_len = vs->sep_len;
    gp.skip_indels = vs->skip_indels;
    gp.keep_partial = vs->keep_partial;
    gp.p2m = vs->p2m;
    gp.add_ref = vs->add_ref;
    gp.verdict = (uint8_t*)vs->verdict.p;
    gp.span = (uint2*)vs->span.p;
    return gp;
}

}  // namespace

void pg_vcf_free(pg_ctx* ctx) {
    VcfState* vs = (VcfState*)ctx->vcf_state;
    if (!vs) return;
    PgBuf* bufs[] = {&vs->tab, &vs->text, &vs->starts, &vs->lines, &vs->slots, &vs->masks, &vs->rows, &vs->verdict,
                     &vs->span, &vs->off, &vs->out, &vs->cub, &vs->scratch};
    for (PgBuf* b : bufs) b->release();
    delete vs;
    ctx->vcf_state = nullptr;
}

extern "C" int pg_vcf_set_spec(pg_ctx* ctx, const pg_vcf_spec* sp) {
    PG_CHECK(ctx && sp, "pg_vcf_set_spec: null argument");
    PG_CHECK(sp->n_cols >= 9 && sp->col_slot && sp->col_prev, "pg_vcf_set_spec: the header must hold the nine fixed columns");
    PG_CHECK(sp->n_keys >= 1 && sp->n_keys <= VCF_MAX_KEYS && sp->key_off && sp->key_chars,
             "pg_vcf_set_spec: %d FORMAT keys (1 to %d)", sp->n_keys, VCF_MAX_KEYS);
    PG_CHECK(sp->n_samp >= 0 && (sp->n_samp == 0 || (sp->samp_col && sp->samp_ploidy)), "pg_vcf_set_spec: no sample table");
    PG_CHECK(sp->n_filt >= 0 && sp->field_key >= -1 && sp->field_key < sp->n_keys, "pg_vcf_set_spec: bad filter or field key");
    PG_CHECK(sp->missing_len >= 0 && sp->sep_len >= 0, "pg_vcf_set_spec: bad missing or separator string");
    int n_slots = 0;
    for (int c = 0; c < sp->n_cols; ++c) {
        PG_CHECK(sp->col_prev[c] < c && (sp->col_prev[c] >= 9 || sp->col_prev[c] == -1), "pg_vcf_set_spec: column %d", c);
        if (sp->col_slot[c] >= 0) {
            PG_CHECK(c >= 9 && sp->col_slot[c] == n_slots, "pg_vcf_set_spec: slots must number the wanted columns in order");
            ++n_slots;
        }
    }
    for (int s = 0; s < sp->n_samp; ++s) {
        PG_CHECK(sp->samp_col[s] >= 9 && sp->samp_col[s] < sp->n_cols, "pg_vcf_set_spec: sample %d column", s);
        for (int c = sp->samp_col[s]; c >= 0; c = sp->col_prev[c])
            PG_CHECK(sp->col_slot[c] >= 0, "pg_vcf_set_spec: column %d of sample %d has no slot", c, s);
    }
    for (int f = 0; f < sp->n_filt; ++f)
        PG_CHECK(sp->filt_key[f] >= -1 && sp->filt_key[f] < sp->n_keys, "pg_vcf_set_spec: filter %d key", f);
    VcfState* vs = vstate(ctx);
    const int nk = sp->n_keys, ns = sp->n_samp, nf = sp->n_filt, nc = sp->n_cols;
    struct Block {
        const void* src;
        size_t bytes;
    };
    const Block blocks[] = {{sp->col_slot, (size_t)nc * 4},           {sp->key_off, (size_t)(nk + 1) * 4},
                            {sp->key_chars, (size_t)sp->key_off[nk]}, {sp->samp_col, (size_t)ns * 4},
                            {sp->col_prev, (size_t)nc * 4},           {sp->samp_ploidy, (size_t)ns * 4},
                            {sp->filt_key, (size_t)nf * 4},           {sp->filt_min, (size_t)nf * 8},
                            {sp->filt_max, (size_t)nf * 8},           {sp->filt_site, (size_t)nf},
                            {sp->filt_gt, (size_t)nf},                {sp->filt_samp, (size_t)nf * ns},
                            {sp->missing, (size_t)sp->missing_len},   {sp->sep, (size_t)sp->sep_len},
                            {nullptr, 4096}};
    constexpr int NB = (int)(sizeof(blocks) / sizeof(blocks[0]));
    static_assert(NB == N_BLOCKS, "one block per B_* index");
    size_t at[NB], o = 0;
    for (int i = 0; i < NB; ++i) {
        at[i] = o;
        o += (blocks[i].bytes + 16 + 15) & ~(size_t)15;
    }
    PG_CUDA(cudaSetDevice(ctx->device));
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    PG_TRY(vs->tab.ensure(o));
    std::vector<char> h(o, 0);
    for (int i = 0; i < NB; ++i)
        if (blocks[i].src && blocks[i].bytes) memcpy(h.data() + at[i], blocks[i].src, blocks[i].bytes);
    PG_CUDA(cudaMemcpy(vs->tab.p, h.data(), o, cudaMemcpyHostToDevice));
    std::copy(at, at + NB, vs->at);
    vs->n_cols = nc;
    vs->n_slots = n_slots;
    vs->n_keys = nk;
    vs->n_samp = ns;
    vs->n_filt = nf;
    vs->field_key = sp->field_key;
    vs->field_phase = sp->field_phase;
    vs->has_min_qual = sp->has_min_qual;
    vs->min_qual = sp->min_qual;
    vs->skip_indels = sp->skip_indels;
    vs->keep_partial = sp->keep_partial;
    vs->p2m = sp->ploidy_mismatch_to_missing;
    vs->add_ref = sp->add_ref_track;
    vs->missing_len = sp->missing_len;
    vs->sep_len = sp->sep_len;
    vs->have_spec = true;
    vs->S = vs->R = -1;
    return PG_OK;
}

extern "C" int pg_vcf_load(pg_ctx* ctx, const char* text, size_t len, const char* prev, int32_t prev_chrom, int32_t prev_pos,
                           int64_t* n_lines) {
    PG_CHECK(ctx && (text || len == 0) && n_lines, "pg_vcf_load: null argument");
    VcfState* vs = vstate(ctx);
    PG_CHECK(vs->have_spec, "pg_vcf_load: no pg_vcf_set_spec");
    PG_CHECK(!prev || (prev_chrom >= 0 && prev_pos >= 0 && prev_chrom + prev_pos <= 4000), "pg_vcf_load: previous line too long");
    PG_CHECK(len < ((size_t)1 << 32), "pg_vcf_load: %zu bytes in one chunk (at most 4 GiB)", len);
    PG_CUDA(cudaSetDevice(ctx->device));
    pg_timings_reset(ctx);
    *n_lines = 0;
    vs->S = vs->R = -1;
    vs->len = len;
    PG_TRY(vs->text.ensure(len + 256));
    uint8_t* d_text = (uint8_t*)vs->text.p;
    {
        const int ti = pg_time_begin(ctx, "vcf_text_h2d");
        if (len) PG_CUDA(cudaMemcpyAsync(d_text, text, len, cudaMemcpyHostToDevice, ctx->stream));
        PG_CUDA(cudaMemsetAsync(d_text + len, '\n', 256, ctx->stream));
        pg_time_end(ctx, ti);
    }
    if (prev) PG_CUDA(cudaMemcpyAsync((char*)vs->block(B_PREV), prev, (size_t)(prev_chrom + prev_pos),
                                      cudaMemcpyHostToDevice, ctx->stream));
    const size_t nblk = (len + CS_BLOCK_BYTES - 1) / CS_BLOCK_BYTES;
    int64_t S = 0;
    if (nblk > 0) {
        size_t scan_tmp = 0;
        cub::DeviceScan::ExclusiveSum(nullptr, scan_tmp, (unsigned*)nullptr, (unsigned long long*)nullptr, (int)nblk + 1,
                                      ctx->stream);
        const size_t o_base = ((nblk + 1) * 4 + 255) & ~(size_t)255;
        const size_t o_tmp = o_base + (((nblk + 1) * 8 + 255) & ~(size_t)255);
        PG_TRY(vs->scratch.ensure(o_tmp + scan_tmp + 64));
        unsigned* d_cnt = (unsigned*)vs->scratch.p;
        unsigned long long* d_base = (unsigned long long*)((char*)vs->scratch.p + o_base);
        PG_CUDA(cudaMemsetAsync(d_cnt + nblk, 0, 4, ctx->stream));
        PG_TRY(pg_timed(ctx, "vcf_index", [&] { k_vcf_count_starts<<<(unsigned)nblk, CS_THREADS, 0, ctx->stream>>>(d_text, len, d_cnt); }));
        PG_CUDA(cub::DeviceScan::ExclusiveSum((char*)vs->scratch.p + o_tmp, scan_tmp, d_cnt, d_base, (int)nblk + 1, ctx->stream));
        unsigned long long total = 0;
        PG_CUDA(cudaMemcpyAsync(&total, d_base + nblk, 8, cudaMemcpyDeviceToHost, ctx->stream));
        PG_CUDA(cudaStreamSynchronize(ctx->stream));
        S = (int64_t)total;
        PG_TRY(vs->starts.ensure((size_t)std::max<int64_t>(S, 1) * 8 + 64));
        if (S > 0)
            PG_TRY(pg_timed(ctx, "vcf_index", [&] {
                k_vcf_write_starts<<<(unsigned)nblk, CS_THREADS, 0, ctx->stream>>>(d_text, len, d_base, (long long*)vs->starts.p);
            }));
        ctx->launches += 3;
    }
    vs->S = S;
    *n_lines = S;
    if (S == 0) return PG_OK;
    PG_TRY(vs->lines.ensure((size_t)S * sizeof(pg_vcf_line) + 64));
    PG_TRY(vs->slots.ensure((size_t)S * std::max(vs->n_slots, 1) * 4 + 64));
    PG_TRY(vs->masks.ensure((size_t)S * vs->n_keys * 8 + 64));
    RecParams rp;
    rp.buf = d_text;
    rp.len = len;
    rp.starts = (const long long*)vs->starts.p;
    rp.S = S;
    rp.n_cols = vs->n_cols;
    rp.col_slot = (const int32_t*)vs->block(B_COL_SLOT);
    rp.n_slots = vs->n_slots;
    rp.slots = (uint32_t*)vs->slots.p;
    rp.n_keys = vs->n_keys;
    rp.key_off = (const int32_t*)vs->block(B_KEY_OFF);
    rp.key_chars = (const uint8_t*)vs->block(B_KEY_CHARS);
    rp.key_mask = (unsigned long long*)vs->masks.p;
    rp.has_min_qual = vs->has_min_qual;
    rp.min_qual = vs->min_qual;
    rp.lines = (pg_vcf_line*)vs->lines.p;
    const unsigned grid = (unsigned)std::min<int64_t>((S + 7) / 8, (int64_t)ctx->sm_count * 64);
    PG_TRY(pg_timed(ctx, "vcf_records", [&] { k_vcf_records<<<grid, 256, 0, ctx->stream>>>(rp); }));
    PG_TRY(pg_timed(ctx, "vcf_links", [&] {
        k_vcf_links<<<(unsigned)std::min<int64_t>((S + 255) / 256, 4096), 256, 0, ctx->stream>>>(
            d_text, (pg_vcf_line*)vs->lines.p, S, prev ? (const uint8_t*)vs->block(B_PREV) : nullptr, (uint32_t)prev_chrom,
            (uint32_t)prev_pos);
    }));
    ctx->launches += 2;
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    return PG_OK;
}

extern "C" int pg_vcf_lines(pg_ctx* ctx, int64_t line0, int64_t n, pg_vcf_line* out) {
    PG_CHECK(ctx && (out || n == 0), "pg_vcf_lines: null argument");
    VcfState* vs = vstate(ctx);
    PG_CHECK(vs->S >= 0 && line0 >= 0 && n >= 0 && line0 + n <= vs->S, "pg_vcf_lines: lines out of range (or no pg_vcf_load)");
    if (n == 0) return PG_OK;
    PG_CUDA(cudaSetDevice(ctx->device));
    PG_CUDA(cudaMemcpyAsync(out, (const pg_vcf_line*)vs->lines.p + line0, (size_t)n * sizeof(pg_vcf_line), cudaMemcpyDeviceToHost,
                            ctx->stream));
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    return PG_OK;
}

extern "C" int pg_vcf_genotypes(pg_ctx* ctx, int64_t n_rows, const int64_t* rows, const int64_t* pos, int64_t* n_unresolved,
                                uint64_t* error) {
    PG_CHECK(ctx && (n_rows == 0 || (rows && pos)) && n_unresolved && error, "pg_vcf_genotypes: null argument");
    VcfState* vs = vstate(ctx);
    PG_CHECK(vs->S >= 0, "pg_vcf_genotypes: no pg_vcf_load");
    PG_CHECK(n_rows >= 0 && n_rows < (int64_t)INT32_MAX, "pg_vcf_genotypes: %lld rows in one chunk", (long long)n_rows);
    for (int64_t r = 0; r < n_rows; ++r) PG_CHECK(rows[r] >= 0 && rows[r] < vs->S, "pg_vcf_genotypes: row %lld line", (long long)r);
    PG_CUDA(cudaSetDevice(ctx->device));
    pg_timings_reset(ctx);
    *n_unresolved = 0;
    *error = 0;
    vs->R = n_rows;
    vs->offsets_ready = false;
    const int64_t G = n_rows * vs->n_samp;
    PG_TRY(vs->rows.ensure((size_t)std::max<int64_t>(n_rows, 1) * 16 + 64));
    PG_TRY(vs->verdict.ensure((size_t)G + 64));
    PG_TRY(vs->span.ensure((size_t)G * 8 + 64));
    PG_TRY(vs->off.ensure(64));
    if (n_rows) {
        PG_CUDA(cudaMemcpyAsync(vs->rows.p, rows, (size_t)n_rows * 8, cudaMemcpyHostToDevice, ctx->stream));
        PG_CUDA(cudaMemcpyAsync((int64_t*)vs->rows.p + n_rows, pos, (size_t)n_rows * 8, cudaMemcpyHostToDevice, ctx->stream));
    }
    unsigned long long* d_w = (unsigned long long*)vs->off.p;
    PG_CUDA(cudaMemsetAsync(d_w, 0xff, 8, ctx->stream));
    PG_CUDA(cudaMemsetAsync(d_w + 1, 0, 8, ctx->stream));
    GenoParams gp = geno_params(vs);
    gp.err = d_w;
    if (G > 0) {
        const unsigned grid = (unsigned)std::min<int64_t>((G + 255) / 256, (int64_t)ctx->sm_count * 16);
        PG_TRY(pg_timed(ctx, "vcf_genotypes", [&] { k_vcf_genotypes<<<grid, 256, 0, ctx->stream>>>(gp); }));
        ctx->launches += 1;
    }
    unsigned long long w = ~0ull;
    PG_CUDA(cudaMemcpyAsync(&w, d_w, 8, cudaMemcpyDeviceToHost, ctx->stream));
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    *error = w == ~0ull ? 0 : (uint64_t)w;
    if (G > 0 && vs->field_key < 0 && vs->n_filt > 0) {
        // genotypes whose filter values left the fast number path: the host settles them (pg_vcf_verdicts)
        size_t tmp = 0;
        int64_t* d_cnt = (int64_t*)(d_w + 2);
        cub::TransformInputIterator<int64_t, IsUnresolved, const uint8_t*> it((const uint8_t*)vs->verdict.p, IsUnresolved());
        PG_CUDA(cub::DeviceReduce::Sum(nullptr, tmp, it, d_cnt, (int)G, ctx->stream));
        PG_TRY(vs->cub.ensure(tmp + 64));
        PG_CUDA(cub::DeviceReduce::Sum(vs->cub.p, tmp, it, d_cnt, (int)G, ctx->stream));
        int64_t nu = 0;
        PG_CUDA(cudaMemcpyAsync(&nu, d_cnt, 8, cudaMemcpyDeviceToHost, ctx->stream));
        PG_CUDA(cudaStreamSynchronize(ctx->stream));
        *n_unresolved = nu;
    }
    return PG_OK;
}

extern "C" int pg_vcf_verdicts(pg_ctx* ctx, uint8_t* get, const uint8_t* put) {
    PG_CHECK(ctx != nullptr, "pg_vcf_verdicts: null ctx");
    VcfState* vs = vstate(ctx);
    PG_CHECK(vs->R >= 0, "pg_vcf_verdicts: no pg_vcf_genotypes");
    const size_t G = (size_t)vs->R * vs->n_samp;
    if (G == 0) return PG_OK;
    PG_CUDA(cudaSetDevice(ctx->device));
    if (get) PG_CUDA(cudaMemcpyAsync(get, vs->verdict.p, G, cudaMemcpyDeviceToHost, ctx->stream));
    if (put) {
        PG_CUDA(cudaMemcpyAsync(vs->verdict.p, put, G, cudaMemcpyHostToDevice, ctx->stream));
        vs->offsets_ready = false;
    }
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    return PG_OK;
}

extern "C" int pg_vcf_emit(pg_ctx* ctx, int64_t row0, char* out, size_t cap, int64_t* rows, size_t* bytes) {
    PG_CHECK(ctx && out && rows && bytes, "pg_vcf_emit: null argument");
    VcfState* vs = vstate(ctx);
    PG_CHECK(vs->R >= 0, "pg_vcf_emit: no pg_vcf_genotypes");
    PG_CHECK(row0 >= 0 && row0 <= vs->R, "pg_vcf_emit: row %lld out of range", (long long)row0);
    *rows = 0;
    *bytes = 0;
    if (row0 == vs->R) return PG_OK;
    PG_CUDA(cudaSetDevice(ctx->device));
    pg_timings_reset(ctx);
    const int64_t R = vs->R;
    GenoParams gp = geno_params(vs);
    if (!vs->offsets_ready) {
        PG_TRY(vs->off.ensure((size_t)(R + 1) * 16 + 64));
        int64_t* d_off = (int64_t*)vs->off.p;
        int64_t* d_len = d_off + (R + 1);
        PG_CUDA(cudaMemsetAsync(d_len + R, 0, 8, ctx->stream));
        gp.row0 = 0;
        gp.nrows = R;
        gp.len = d_len;
        PG_TRY(pg_timed(ctx, "vcf_emit_len", [&] {
            k_vcf_emit<false><<<(unsigned)std::min<int64_t>((R + 7) / 8, (int64_t)ctx->sm_count * 32), 256, 0, ctx->stream>>>(gp);
        }));
        size_t tmp = 0;
        PG_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tmp, d_len, d_off, (int)(R + 1), ctx->stream));
        PG_TRY(vs->cub.ensure(tmp + 64));
        PG_CUDA(cub::DeviceScan::ExclusiveSum(vs->cub.p, tmp, d_len, d_off, (int)(R + 1), ctx->stream));
        vs->h_off.resize((size_t)R + 1);
        PG_CUDA(cudaMemcpyAsync(vs->h_off.data(), d_off, (size_t)(R + 1) * 8, cudaMemcpyDeviceToHost, ctx->stream));
        PG_CUDA(cudaStreamSynchronize(ctx->stream));
        vs->offsets_ready = true;
        ctx->launches += 2;
    }
    const int64_t base = vs->h_off[(size_t)row0];
    const int64_t row1 =
        (int64_t)(std::upper_bound(vs->h_off.begin() + row0, vs->h_off.end(), base + (int64_t)cap) - vs->h_off.begin()) - 1;
    PG_CHECK(row1 > row0, "pg_vcf_emit: row %lld needs %lld bytes, more than the %zu of the buffer", (long long)row0,
             (long long)(vs->h_off[(size_t)row0 + 1] - base), cap);
    const size_t nb = (size_t)(vs->h_off[(size_t)row1] - base);
    PG_TRY(vs->out.ensure(nb + 64));
    gp.row0 = row0;
    gp.nrows = row1 - row0;
    gp.off = (const int64_t*)vs->off.p;
    gp.out = (char*)vs->out.p;
    PG_TRY(pg_timed(ctx, "vcf_emit", [&] {
        k_vcf_emit<true><<<(unsigned)std::min<int64_t>((gp.nrows + 7) / 8, (int64_t)ctx->sm_count * 32), 256, 0, ctx->stream>>>(gp);
    }));
    ctx->launches += 1;
    PG_CUDA(cudaMemcpyAsync(out, vs->out.p, nb, cudaMemcpyDeviceToHost, ctx->stream));
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    *rows = row1 - row0;
    *bytes = nb;
    return PG_OK;
}
