// Device-side .geno TEXT ingest: the text goes to HBM as it is (one H2D stream of the file's bytes) and is tokenised
// there, straight into the resident pitched one-hot genotype matrix.
//
// Replaces parseGenoLine / GenoFileReader.nextSite (genomics.py:1884-1945) + splitSeq / haplo / forceHomo
// (genomics.py:390-396, 27, 407) + seqArrayToNumArray (74-77) for a whole file.  Same grammar as the host tokenizer
// (geno_parse.cpp), which stays as the path for files larger than device memory and for the generator API:
//   line   := scaffold WS position WS token (WS token)*        ('#' lines and blank lines are skipped)
//   phased : alleles are the characters 0,2,4.. of the token   ("A|T", "A/N", "G")
//   pairs  : two letters, no separator;  diplo : one IUPAC letter -> two alleles (genomics.py:14-15);  haplo : one letter
//
//   k_count_starts / k_write_starts : data-line start offsets (two passes around an exclusive scan of block counts)
//   k_parse_lines                   : ONE WARP PER LINE; each lane classifies 4 bytes per step, a warp prefix sum of the
//                                     token-start flags numbers the fields, the lane that owns a field start decodes it:
//                                     field 0 -> 64-bit hash of the scaffold name, field 1 -> int32 position,
//                                     field 2+c -> alleles of genotype column c, stored as one-hot bytes at
//                                     geno[site * pitch + first_hap(c) + a]
//   k_scaffold_flags                : new_scaffold[i] = hash[i] != hash[i-1]
// Bound: the H2D copy of the text (PCIe); the kernels read the text once and write the matrix once.
#include <fcntl.h>
#include <stdlib.h>
#include <sys/stat.h>
#include <unistd.h>

#include <algorithm>
#include <cub/cub.cuh>
#include <thread>

#include "pgwin_internal.h"

namespace {

constexpr int CS_THREADS = 256;
constexpr int CS_BYTES_PER_THREAD = 16;
constexpr int CS_BLOCK_BYTES = CS_THREADS * CS_BYTES_PER_THREAD;

__device__ __forceinline__ bool is_ws_dev(unsigned c) { return c == ' ' || c == '\t' || c == '\r' || c == '\v' || c == '\f'; }

// A data line starts at i iff i is the first byte of a line, the line is not a '#' comment and holds a non-blank byte.
__device__ __forceinline__ bool line_start_at(const uint8_t* __restrict__ buf, size_t len, size_t i) {
    if (i >= len) return false;
    if (i > 0 && buf[i - 1] != '\n') return false;
    unsigned c = buf[i];
    if (c == '#' || c == '\n') return false;
    if (!is_ws_dev(c)) return true;
    for (size_t j = i + 1; j < len; ++j) {      // leading blanks (rare): look for a non-blank byte before the line ends
        c = buf[j];
        if (c == '\n') return false;
        if (!is_ws_dev(c)) return true;
    }
    return false;
}

__global__ void __launch_bounds__(CS_THREADS) k_count_starts(const uint8_t* __restrict__ buf, size_t len,
                                                             unsigned* __restrict__ block_counts) {
    typedef cub::BlockReduce<unsigned, CS_THREADS> BR;
    __shared__ typename BR::TempStorage tmp;
    const size_t base = (size_t)blockIdx.x * CS_BLOCK_BYTES + (size_t)threadIdx.x * CS_BYTES_PER_THREAD;
    unsigned n = 0;
    if (base < len) {
        // a line start needs '\n' right before it: test the cheap condition first
#pragma unroll 4
        for (int k = 0; k < CS_BYTES_PER_THREAD; ++k) {
            const size_t i = base + k;
            if (i < len && (i == 0 || buf[i - 1] == '\n')) n += line_start_at(buf, len, i) ? 1u : 0u;
        }
    }
    const unsigned tot = BR(tmp).Sum(n);
    if (threadIdx.x == 0) block_counts[blockIdx.x] = tot;
}

__global__ void __launch_bounds__(CS_THREADS) k_write_starts(const uint8_t* __restrict__ buf, size_t len,
                                                             const unsigned long long* __restrict__ block_base,
                                                             long long* __restrict__ starts) {
    typedef cub::BlockScan<unsigned, CS_THREADS> BS;
    __shared__ typename BS::TempStorage tmp;
    const size_t base = (size_t)blockIdx.x * CS_BLOCK_BYTES + (size_t)threadIdx.x * CS_BYTES_PER_THREAD;
    unsigned flags = 0, n = 0;
    if (base < len) {
#pragma unroll 4
        for (int k = 0; k < CS_BYTES_PER_THREAD; ++k) {
            const size_t i = base + k;
            if (i < len && (i == 0 || buf[i - 1] == '\n') && line_start_at(buf, len, i)) {
                flags |= 1u << k;
                ++n;
            }
        }
    }
    unsigned off;
    BS(tmp).ExclusiveSum(n, off);
    unsigned long long o = block_base[blockIdx.x] + off;
    for (int k = 0; k < CS_BYTES_PER_THREAD; ++k)
        if (flags & (1u << k)) starts[o++] = (long long)(base + k);
}

struct ParseParams {
    const uint8_t* buf;
    size_t len;
    const long long* starts;    // [S]
    int64_t S;
    int fmt;                    // 0 phased, 1 diplo, 2 pairs, 3 haplo
    int n_cols;                 // genotype columns the caller described
    const int32_t* col_hap;     // [n_cols] first output haplotype of the column, or -1 (column not wanted)
    const int8_t* col_ploidy;   // [n_cols]
    int n_wanted;               // columns with col_hap >= 0: every line must hold all of them
    uint8_t* geno;              // resident one-hot matrix
    int pitch;
    int32_t* pos;
    unsigned long long* scaf_hash;
    unsigned long long* err;    // all ones = ok, else (data line << 28) | (genotype column << 4) | code, 1-based
    // strict tokens (pg_ingest_set_strict): 1 = a token must be exactly as wide as the sample's ploidy and hold only A C G T N
    // (phased / pairs) or a letter of genomics.py:14 DIPLOTYPES (diplo, diploid samples only); the phase character of each
    // sample (token[1] of a phased token of ploidy >= 2, else '/', genomics.py:335) goes to aux[line * H + first_hap].
    // 2 = the width test only: other characters are read as without it (missing unless A C G T)
    int strict;
    uint8_t* aux;
    int aux_stride;
};

enum { ERR_NONE = 0, ERR_POS = 1, ERR_PLOIDY = 2, ERR_MISSING_COLS = 3, ERR_NO_POS = 4, ERR_CHAR = 5, ERR_POS_RANGE = 6 };

__device__ __forceinline__ bool acgtn(unsigned c) { return c == 'A' || c == 'C' || c == 'G' || c == 'T' || c == 'N'; }
__device__ __forceinline__ bool diplotype(unsigned c) {
    return acgtn(c) || c == 'K' || c == 'M' || c == 'S' || c == 'R' || c == 'W' || c == 'Y';
}

__device__ __forceinline__ unsigned onehot(unsigned c) {
    return c == 'A' ? 0x01u : (c == 'C' ? 0x04u : (c == 'G' ? 0x10u : (c == 'T' ? 0x40u : 0u)));
}
// IUPAC diplotype -> the two alleles (genomics.py:14-15 DIPLOTYPES/PAIRS); anything else: missing, missing
__device__ __forceinline__ void diplo_alleles(unsigned c, unsigned& a0, unsigned& a1) {
    a0 = a1 = 'N';
    switch (c) {
        case 'A': a0 = 'A'; a1 = 'A'; break;
        case 'C': a0 = 'C'; a1 = 'C'; break;
        case 'G': a0 = 'G'; a1 = 'G'; break;
        case 'T': a0 = 'T'; a1 = 'T'; break;
        case 'K': a0 = 'G'; a1 = 'T'; break;
        case 'M': a0 = 'A'; a1 = 'C'; break;
        case 'S': a0 = 'C'; a1 = 'G'; break;
        case 'R': a0 = 'A'; a1 = 'G'; break;
        case 'W': a0 = 'A'; a1 = 'T'; break;
        case 'Y': a0 = 'C'; a1 = 'T'; break;
        default: break;
    }
}

__device__ __forceinline__ void report(const ParseParams& pp, int code, int64_t line, int col) {
    // the first offending line wins (then the lowest column): line, column and code packed into one word for atomicMin
    const unsigned long long c1 = (unsigned long long)min(max(col + 1, 0), (1 << 24) - 1);
    atomicMin(pp.err, ((unsigned long long)(line + 1) << 28) | (c1 << 4) | (unsigned long long)code);
}

// byte at absolute offset i of the text ('\n' past the end, so that every field terminates)
__device__ __forceinline__ unsigned byte_at(const ParseParams& pp, size_t i) { return i < pp.len ? pp.buf[i] : (unsigned)'\n'; }

__global__ void __launch_bounds__(256) k_parse_lines(const __grid_constant__ ParseParams pp) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
    for (int64_t line = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); line < pp.S; line += warps) {
        const size_t l0 = (size_t)pp.starts[line];
        const size_t a0 = l0 & ~(size_t)3;                  // aligned base of the 128-byte steps
        unsigned fields_before = 0;                         // fields that started in earlier steps
        bool prev_ws = true;                                // class of the byte before this step's first byte
        unsigned found = 0;                                 // wanted genotype columns decoded by this lane
        bool have_pos = false;
        bool done = false;
        for (size_t step = 0; !done; ++step) {
            const size_t wbase = a0 + step * 128 + (size_t)lane * 4;
            uint32_t w = 0x0a0a0a0au;                       // bytes outside the buffer read as '\n'
            if (wbase + 4 <= pp.len) w = *reinterpret_cast<const uint32_t*>(pp.buf + wbase);
            else if (wbase < pp.len) {
                for (int k = 0; k < 4; ++k)
                    if (wbase + k < pp.len) w = (w & ~(0xffu << (8 * k))) | ((uint32_t)pp.buf[wbase + k] << (8 * k));
            }
            // classify the 4 bytes: bit k of ws / nl
            unsigned ws = 0, nl = 0;
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const unsigned c = (w >> (8 * k)) & 0xffu;
                const bool before = (wbase + k) < l0;       // bytes of the previous line inside the first aligned word
                if (before || is_ws_dev(c)) ws |= 1u << k;
                else if (c == '\n') nl |= 1u << k;
            }
            // everything from the first '\n' of the line on is outside the line
            const unsigned nl_lanes = __ballot_sync(0xffffffffu, nl != 0);
            if (nl_lanes) {
                const int first = __ffs(nl_lanes) - 1;
                if (lane > first) ws = 0xfu, nl = 0;
                else if (lane == first) {
                    const unsigned from = nl & (0u - nl);               // lowest set bit
                    ws |= ~(from - 1u) & 0xfu;                          // that byte and the ones after it: blank
                }
                done = true;
            }
            // field starts: non-blank byte whose predecessor is blank
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
            unsigned fidx = fields_before + incl - cnt;                 // index of this lane's first field start
            fields_before += __shfl_sync(0xffffffffu, incl, 31);
            prev_ws = (__shfl_sync(0xffffffffu, last_ws, 31) != 0);
            // decode the fields that start in this lane's bytes
            for (unsigned m = st; m; m &= m - 1, ++fidx) {
                const int k = __ffs(m) - 1;
                const size_t q = wbase + k;
                if (fidx == 0) {                                        // scaffold name -> hash
                    unsigned long long h = 1469598103934665603ull;
                    for (size_t j = q;; ++j) {
                        const unsigned c = byte_at(pp, j);
                        if (c == '\n' || is_ws_dev(c)) break;
                        h = (h ^ c) * 1099511628211ull;
                    }
                    pp.scaf_hash[line] = h;
                } else if (fidx == 1) {                                 // position
                    size_t j = q;
                    unsigned c = byte_at(pp, j);
                    bool neg = false;
                    if (c == '-' || c == '+') {
                        neg = (c == '-');
                        c = byte_at(pp, ++j);
                    }
                    // position errors take column -1, so that they precede any genotype column's error of the line
                    if (c < '0' || c > '9') report(pp, ERR_POS, line, -1);
                    long long v = 0;
                    while (c >= '0' && c <= '9') {
                        if (v <= (1ll << 31)) v = v * 10 + (long long)(c - '0');    // past the limit it stays out of range
                        c = byte_at(pp, ++j);
                    }
                    if (v > (1ll << 31) - (neg ? 0 : 1)) report(pp, ERR_POS_RANGE, line, -1);
                    pp.pos[line] = (int32_t)(neg ? -v : v);
                    have_pos = true;
                } else {
                    const int col = (int)fidx - 2;
                    if (col >= pp.n_cols) continue;
                    const int hap0 = pp.col_hap[col];
                    if (hap0 < 0) continue;
                    const int pl = pp.col_ploidy[col];
                    uint8_t* o = pp.geno + (size_t)line * pp.pitch + hap0;
                    // token length, up to what the format can use
                    int tl = 0;
                    const int tmax = 2 * pl + 1;
                    while (tl < tmax) {
                        const unsigned c = byte_at(pp, q + tl);
                        if (c == '\n' || is_ws_dev(c)) break;
                        ++tl;
                    }
                    if (pp.strict) {
                        const int want = pp.fmt == 0 ? 2 * pl - 1 : (pp.fmt == 1 ? 1 : pl);
                        if (tl != want || (pp.fmt == 1 && pl != 2)) {
                            report(pp, ERR_PLOIDY, line, col);
                            continue;
                        }
                    }
                    if (pp.strict == 1) {
                        bool ok = true;
                        if (pp.fmt == 1) ok = diplotype(byte_at(pp, q));
                        else
                            for (int a = 0; a < pl; ++a) ok = ok && acgtn(byte_at(pp, q + (pp.fmt == 0 ? 2 * a : a)));
                        if (!ok) {
                            report(pp, ERR_CHAR, line, col);
                            continue;
                        }
                        pp.aux[(size_t)line * pp.aux_stride + hap0] =
                            (uint8_t)(pp.fmt == 0 && pl >= 2 ? byte_at(pp, q + 1) : (unsigned)'/');
                    }
                    if (pp.fmt == 0) {                                  // phased: characters 0,2,4,...
                        if ((tl + 1) / 2 != pl) {
                            report(pp, ERR_PLOIDY, line, col);
                            continue;
                        }
                        for (int a = 0; a < pl; ++a) o[a] = (uint8_t)onehot(byte_at(pp, q + 2 * a));
                    } else if (pp.fmt == 2) {                           // pairs
                        if (tl != pl) {
                            report(pp, ERR_PLOIDY, line, col);
                            continue;
                        }
                        for (int a = 0; a < pl; ++a) o[a] = (uint8_t)onehot(byte_at(pp, q + a));
                    } else if (pp.fmt == 1) {                           // diplo
                        unsigned x0, x1;
                        diplo_alleles(byte_at(pp, q), x0, x1);
                        if (pl == 1) o[0] = (uint8_t)(x0 == x1 ? onehot(x0) : 0u);   // forceHomo (genomics.py:407)
                        else if (pl == 2) {
                            o[0] = (uint8_t)onehot(x0);
                            o[1] = (uint8_t)onehot(x1);
                        } else {
                            report(pp, ERR_PLOIDY, line, col);
                            continue;
                        }
                    } else {                                            // haplo
                        if (pl != 1) {
                            report(pp, ERR_PLOIDY, line, col);
                            continue;
                        }
                        o[0] = (uint8_t)onehot(byte_at(pp, q));
                    }
                    ++found;
                }
            }
        }
        // every wanted column must have been present; the line must have a position
#pragma unroll
        for (int d = 16; d >= 1; d >>= 1) found += __shfl_xor_sync(0xffffffffu, found, d);
        const bool any_pos = __any_sync(0xffffffffu, have_pos);
        if (lane == 0) {
            if (!any_pos) report(pp, ERR_NO_POS, line, 0);
            // one past the last genotype column: an error of any column of the line comes first
            else if ((int)found != pp.n_wanted) report(pp, ERR_MISSING_COLS, line, (int)fields_before - 2);
        }
    }
}

__global__ void k_scaffold_flags(const unsigned long long* __restrict__ h, int64_t S, int8_t* __restrict__ flags) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < S; i += (int64_t)gridDim.x * blockDim.x)
        flags[i] = (i == 0 || h[i] != h[i - 1]) ? 1 : 0;
}

}  // namespace

namespace {

// bytes [off, off + n) of the source (memory or file) -> dst (pinned), split over a few host threads: a single thread
// copies ~5-10 GB/s out of pageable memory or the page cache, the H2D engine moves ~55 GB/s
int fill_slab(const char* mem, int fd, size_t file_off, size_t off, size_t n, char* dst, int n_threads) {
    if (n_threads < 1) n_threads = 1;
    std::vector<std::thread> th;
    std::vector<int> rc((size_t)n_threads, 0);
    auto work = [&](int t) {
        const size_t a = n * (size_t)t / (size_t)n_threads, b = n * (size_t)(t + 1) / (size_t)n_threads;
        if (mem) {
            memcpy(dst + a, mem + off + a, b - a);
            return;
        }
        size_t done = a;
        while (done < b) {
            const ssize_t r = pread(fd, dst + done, b - done, (off_t)(file_off + off + done));
            if (r <= 0) {
                rc[(size_t)t] = 1;
                return;
            }
            done += (size_t)r;
        }
    };
    for (int t = 1; t < n_threads; ++t) th.emplace_back(work, t);
    work(0);
    for (auto& x : th) x.join();
    for (int v : rc)
        if (v) return 1;
    return 0;
}

int ingest_core(pg_ctx* ctx, const char* mem, int fd, size_t file_off, size_t len, int32_t fmt, int32_t n_cols,
                const int32_t* col_hap, const int8_t* col_ploidy, int32_t H_out, int64_t* n_sites);

}  // namespace

// Text (complete lines, no header line) -> resident matrix of this ctx.  Afterwards the ctx holds *n_sites sites of
// H_out haplotypes; positions, new-scaffold flags and line offsets are read back with pg_ingest_meta.
extern "C" int pg_ingest_text(pg_ctx* ctx, const char* buf, size_t len, int32_t fmt, int32_t n_cols, const int32_t* col_hap,
                              const int8_t* col_ploidy, int32_t H_out, int64_t* n_sites) {
    PG_CHECK(ctx && (buf || len == 0) && col_hap && col_ploidy && n_sites, "pg_ingest_text: null argument");
    return ingest_core(ctx, buf ? buf : "", -1, 0, len, fmt, n_cols, col_hap, col_ploidy, H_out, n_sites);
}

// The same for a file on disk: bytes [body_offset, EOF) of `path` (body_offset = length of the header line, or 0) are read
// straight into the pinned staging buffers by a few host threads — no intermediate copy of the file in host memory.
extern "C" int pg_ingest_file(pg_ctx* ctx, const char* path, int64_t body_offset, int32_t fmt, int32_t n_cols,
                              const int32_t* col_hap, const int8_t* col_ploidy, int32_t H_out, int64_t* n_sites) {
    PG_CHECK(ctx && path && col_hap && col_ploidy && n_sites, "pg_ingest_file: null argument");
    const int fd = open(path, O_RDONLY);
    PG_CHECK(fd >= 0, "pg_ingest_file: cannot open %s", path);
    struct stat st;
    if (fstat(fd, &st) != 0 || body_offset < 0 || (int64_t)st.st_size < body_offset) {
        close(fd);
        pg_set_error("pg_ingest_file: cannot stat %s (or the body offset is past its end)", path);
        return PG_ERR;
    }
    const int rc = ingest_core(ctx, nullptr, fd, (size_t)body_offset, (size_t)st.st_size - (size_t)body_offset, fmt, n_cols,
                               col_hap, col_ploidy, H_out, n_sites);
    close(fd);
    return rc;
}

// Bytes [byte_lo, byte_hi) of the file (both at line starts; byte_hi < 0: end of file): one rank's share of the data lines in
// the multi-GPU command lines.  line_off values of pg_ingest_meta are relative to byte_lo.
extern "C" int pg_ingest_file_range(pg_ctx* ctx, const char* path, int64_t byte_lo, int64_t byte_hi, int32_t fmt, int32_t n_cols,
                                    const int32_t* col_hap, const int8_t* col_ploidy, int32_t H_out, int64_t* n_sites) {
    PG_CHECK(ctx && path && col_hap && col_ploidy && n_sites, "pg_ingest_file_range: null argument");
    const int fd = open(path, O_RDONLY);
    PG_CHECK(fd >= 0, "pg_ingest_file_range: cannot open %s", path);
    struct stat st;
    if (fstat(fd, &st) != 0) {
        close(fd);
        pg_set_error("pg_ingest_file_range: cannot stat %s", path);
        return PG_ERR;
    }
    if (byte_hi < 0 || byte_hi > (int64_t)st.st_size) byte_hi = (int64_t)st.st_size;
    if (byte_lo < 0 || byte_lo > byte_hi) {
        close(fd);
        pg_set_error("pg_ingest_file_range: bad byte range [%lld, %lld)", (long long)byte_lo, (long long)byte_hi);
        return PG_ERR;
    }
    const int rc = ingest_core(ctx, nullptr, fd, (size_t)byte_lo, (size_t)(byte_hi - byte_lo), fmt, n_cols, col_hap, col_ploidy,
                               H_out, n_sites);
    close(fd);
    return rc;
}

// The text -> ctx->text (then 256 bytes of '\n'), the start of every data line -> ctx->starts, *n_lines = data lines.  The
// source is memory (mem) or bytes [file_off, file_off + len) of the open file fd.  Shared by the .geno ingest and genoToSeq
// (seq.cu); bumps ctx->text_gen.
int pg_text_load(pg_ctx* ctx, const char* mem, int fd, size_t file_off, size_t len, int64_t* n_lines) {
    *n_lines = 0;
    ctx->text_gen += 1;
    size_t free_b = 0, total_b = 0;
    PG_CUDA(cudaMemGetInfo(&free_b, &total_b));
    PG_CHECK(len + ((size_t)1 << 30) < free_b + ctx->text.cap, "pg_ingest_text: %zu bytes of text do not fit in device memory "
             "(%zu free) — use the host tokenizer (pg_geno_parse) and pg_upload", len, free_b);
    PG_TRY(ctx->text.ensure(len + 256));
    uint8_t* d_text = (uint8_t*)ctx->text.p;
    // H2D of the text: host threads fill two pinned staging buffers in turn, the copy engine drains them
    {
        const size_t slab = (size_t)64 << 20;
        // a few threads saturate the copy into pinned memory, more only contend (PG_INGEST_THREADS overrides; tools/ingest_threads.py
        // sweeps it)
        int n_threads = std::max(1, std::min(4, (int)std::thread::hardware_concurrency() / 2));
        if (const char* e = getenv("PG_INGEST_THREADS")) n_threads = std::max(1, std::min(128, atoi(e)));
        if (!ctx->h_text[0]) {
            for (int k = 0; k < 2; ++k) {
                PG_CUDA(cudaHostAlloc(&ctx->h_text[k], slab, cudaHostAllocDefault));
                PG_CUDA(cudaEventCreateWithFlags(&ctx->h_text_free[k], cudaEventDisableTiming));
            }
        }
        const int ti = pg_time_begin(ctx, "text_h2d");
        ctx->ingest_geom[0] = (int64_t)((len + slab - 1) / slab);
        ctx->ingest_geom[1] = (int64_t)slab;
        ctx->ingest_geom[2] = CS_BLOCK_BYTES;
        ctx->ingest_geom[3] = ctx->ingest_geom[4] = 0;
        int k = 0;
        for (size_t o = 0; o < len; o += slab, ++k) {
            const size_t n = std::min(slab, len - o);
            const int b = k & 1;
            if (k >= 2) PG_CUDA(cudaEventSynchronize(ctx->h_text_free[b]));
            PG_CHECK(fill_slab(mem, fd, file_off, o, n, (char*)ctx->h_text[b], n_threads) == 0,
                     "pg_ingest: reading the text failed at byte %zu", o);
            PG_CUDA(cudaMemcpyAsync(d_text + o, ctx->h_text[b], n, cudaMemcpyHostToDevice, ctx->stream));
            PG_CUDA(cudaEventRecord(ctx->h_text_free[b], ctx->stream));
        }
        PG_CUDA(cudaMemsetAsync(d_text + len, '\n', 256, ctx->stream));
        pg_time_end(ctx, ti);
    }
    const size_t nblk = (len + CS_BLOCK_BYTES - 1) / CS_BLOCK_BYTES;
    int64_t S = 0;
    if (nblk > 0) {
        PG_CHECK(nblk < ((size_t)1 << 31), "pg_ingest_text: text too large for one call");
        // block counts -> exclusive scan (64-bit) -> starts
        size_t scan_tmp = 0;
        cub::DeviceScan::ExclusiveSum(nullptr, scan_tmp, (unsigned*)nullptr, (unsigned long long*)nullptr, (int)nblk + 1,
                                      ctx->stream);
        PG_TRY(ctx->misc.ensure((nblk + 1) * 4 + 64));
        PG_TRY(ctx->misc2.ensure((nblk + 1) * 8 + 64));
        PG_TRY(ctx->misc3.ensure(scan_tmp + 64));
        unsigned* d_cnt = (unsigned*)ctx->misc.p;
        unsigned long long* d_base = (unsigned long long*)ctx->misc2.p;
        PG_CUDA(cudaMemsetAsync(d_cnt + nblk, 0, 4, ctx->stream));
        {
            const int ti = pg_time_begin(ctx, "ingest_index");
            k_count_starts<<<(unsigned)nblk, CS_THREADS, 0, ctx->stream>>>(d_text, len, d_cnt);
            pg_time_end(ctx, ti);
            PG_CUDA(cudaGetLastError());
        }
        PG_CUDA(cub::DeviceScan::ExclusiveSum(ctx->misc3.p, scan_tmp, d_cnt, d_base, (int)nblk + 1, ctx->stream));
        ctx->launches += 1;
        unsigned long long total = 0;
        PG_CUDA(cudaMemcpyAsync(&total, d_base + nblk, 8, cudaMemcpyDeviceToHost, ctx->stream));
        PG_CUDA(cudaStreamSynchronize(ctx->stream));
        S = (int64_t)total;
        PG_TRY(ctx->starts.ensure((size_t)std::max<int64_t>(S, 1) * 8 + 64));
        long long* d_starts = (long long*)ctx->starts.p;
        if (S > 0) {
            const int ti = pg_time_begin(ctx, "ingest_index");
            k_write_starts<<<(unsigned)nblk, CS_THREADS, 0, ctx->stream>>>(d_text, len, d_base, d_starts);
            pg_time_end(ctx, ti);
            PG_CUDA(cudaGetLastError());
        }
    }
    PG_TRY(ctx->starts.ensure((size_t)std::max<int64_t>(S, 1) * 8 + 64));
    *n_lines = S;
    return PG_OK;
}

// new_scaffold[i] = hash[i] != hash[i - 1] for S lines (ctx stream)
int pg_scaffold_flags(pg_ctx* ctx, const unsigned long long* d_hash, int64_t S, int8_t* d_flags) {
    const unsigned fgrid = (unsigned)std::min<int64_t>((S + 255) / 256, 4096);
    k_scaffold_flags<<<fgrid, 256, 0, ctx->stream>>>(d_hash, S, d_flags);
    PG_CUDA(cudaGetLastError());
    return PG_OK;
}

namespace {
int ingest_core(pg_ctx* ctx, const char* mem, int fd, size_t file_off, size_t len, int32_t fmt, int32_t n_cols,
                const int32_t* col_hap, const int8_t* col_ploidy, int32_t H_out, int64_t* n_sites) {
    PG_CHECK(fmt >= 0 && fmt <= 3, "pg_ingest: unknown format %d", fmt);
    PG_CHECK(n_cols >= 1 && H_out >= 1, "pg_ingest: no genotype columns requested");
    int n_wanted = 0;
    {
        std::vector<char> used((size_t)H_out, 0);
        for (int c = 0; c < n_cols; ++c) {
            if (col_hap[c] < 0) continue;
            PG_CHECK(col_ploidy[c] >= 1 && col_ploidy[c] <= 8, "pg_ingest: ploidy %d of column %d unsupported",
                     (int)col_ploidy[c], c);
            PG_CHECK(col_hap[c] + col_ploidy[c] <= H_out, "pg_ingest: column %d maps outside the %d output haplotypes", c, H_out);
            for (int a = 0; a < col_ploidy[c]; ++a) {
                PG_CHECK(!used[col_hap[c] + a], "pg_ingest: output haplotype %d is written by two columns", col_hap[c] + a);
                used[col_hap[c] + a] = 1;
            }
            ++n_wanted;
        }
        for (int h = 0; h < H_out; ++h) PG_CHECK(used[h], "pg_ingest: output haplotype %d has no source column", h);
    }
    PG_CUDA(cudaSetDevice(ctx->device));
    pg_timings_reset(ctx);
    *n_sites = 0;
    int64_t S = 0;
    PG_TRY(pg_text_load(ctx, mem, fd, file_off, len, &S));
    const uint8_t* d_text = (const uint8_t*)ctx->text.p;
    const long long* d_starts = (const long long*)ctx->starts.p;
    PG_TRY(pg_alloc_sites(ctx, S, H_out));
    ctx->epoch += 1;
    *n_sites = S;
    ctx->ingest_sites = S;
    if (S == 0) return PG_OK;
    // column tables + per-line scratch
    PG_TRY(ctx->misc4.ensure((size_t)n_cols * 5 + 64 + 32));
    int32_t* d_col_hap = (int32_t*)ctx->misc4.p;
    int8_t* d_col_pl = (int8_t*)(d_col_hap + n_cols);
    PG_CUDA(cudaMemcpyAsync(d_col_hap, col_hap, (size_t)n_cols * 4, cudaMemcpyHostToDevice, ctx->stream));
    PG_CUDA(cudaMemcpyAsync(d_col_pl, col_ploidy, (size_t)n_cols, cudaMemcpyHostToDevice, ctx->stream));
    PG_TRY(ctx->meta.ensure((size_t)S * 9 + 64));
    unsigned long long* d_hash = (unsigned long long*)ctx->meta.p;
    int8_t* d_flags = (int8_t*)(d_hash + S);
    PG_TRY(ctx->out_i.ensure(64));
    unsigned long long* d_err = (unsigned long long*)ctx->out_i.p;
    PG_CUDA(cudaMemsetAsync(d_err, 0xff, 8, ctx->stream));       // no error: all ones
    ParseParams pp;
    pp.buf = d_text;
    pp.len = len;
    pp.starts = d_starts;
    pp.S = S;
    pp.fmt = fmt;
    pp.n_cols = n_cols;
    pp.col_hap = d_col_hap;
    pp.col_ploidy = d_col_pl;
    pp.n_wanted = n_wanted;
    pp.geno = (uint8_t*)ctx->d_geno;
    pp.pitch = ctx->pitch;
    pp.pos = ctx->d_pos;
    pp.scaf_hash = d_hash;
    pp.err = d_err;
    pp.strict = ctx->ingest_strict;
    pp.aux = nullptr;
    pp.aux_stride = H_out;
    if (pp.strict == 1) {
        PG_TRY(ctx->flt_aux.ensure((size_t)S * H_out + 64));
        pp.aux = (uint8_t*)ctx->flt_aux.p;
    }
    ctx->ingest_fmt = fmt;
    {
        const int ti = pg_time_begin(ctx, "ingest_parse");
        const unsigned grid = (unsigned)std::min<int64_t>((S + 7) / 8, (int64_t)ctx->sm_count * 64);
        k_parse_lines<<<grid, 256, 0, ctx->stream>>>(pp);
        pg_time_end(ctx, ti);
        PG_CUDA(cudaGetLastError());
        const unsigned fgrid = (unsigned)std::min<int64_t>((S + 255) / 256, 4096);
        PG_TRY(pg_scaffold_flags(ctx, d_hash, S, d_flags));
        ctx->ingest_geom[3] = (int64_t)grid * 8;
        ctx->ingest_geom[4] = (int64_t)fgrid * 256;
        ctx->launches += 1;
    }
    PG_TRY(pg_pack_rows(ctx, 0, S));
    unsigned long long packed = ~0ull;
    PG_CUDA(cudaMemcpyAsync(&packed, d_err, 8, cudaMemcpyDeviceToHost, ctx->stream));
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    ctx->ingest_sites = S;
    // [0] = code, [1] = data line (1-based), [2] = genotype column (1-based)
    const unsigned long long h_err[3] = {packed == ~0ull ? 0ull : (packed & 15ull), packed >> 28, (packed >> 4) & 0xffffffull};
    switch ((int)h_err[0]) {
        case ERR_NONE: break;
        case ERR_POS:
            pg_set_error("pg_ingest_text: data line %llu: position is not an integer", h_err[1]);
            return PG_ERR;
        case ERR_NO_POS:
            pg_set_error("pg_ingest_text: data line %llu: no position field", h_err[1]);
            return PG_ERR;
        case ERR_POS_RANGE:
            pg_set_error("pg_ingest_text: data line %llu: position outside the int32 range", h_err[1]);
            return PG_ERR;
        case ERR_PLOIDY:
            pg_set_error("pg_ingest_text: data line %llu, genotype column %llu: the token's allele count does not match the "
                         "sample's ploidy (genomics.py:1111 asserts the same)", h_err[1], h_err[2]);
            return PG_ERR;
        case ERR_CHAR:
            pg_set_error("pg_ingest_text: data line %llu, genotype column %llu: a character other than A, C, G, T or N (the "
                         "reference makes such a genotype missing but writes it out unchanged)", h_err[1], h_err[2]);
            return PG_ERR;
        default:
            pg_set_error("pg_ingest_text: data line %llu: %llu genotype columns, not every requested sample found", h_err[1],
                         h_err[2] - 1);
            return PG_ERR;
    }
    return PG_OK;
}

}  // namespace

// positions int32 [S], new_scaffold int8 [S] (1 where the scaffold field differs from the previous data line),
// line_off int64 [S] (byte offset of each data line in the text) of the last pg_ingest_text; any may be NULL.
extern "C" int pg_ingest_meta(pg_ctx* ctx, int32_t* pos, int8_t* new_scaffold, int64_t* line_off) {
    PG_CHECK(ctx != nullptr, "pg_ingest_meta: null ctx");
    const int64_t S = ctx->ingest_sites;
    PG_CHECK(S == ctx->S, "pg_ingest_meta: no text ingest on this ctx (or the matrix was replaced since)");
    PG_CUDA(cudaSetDevice(ctx->device));
    if (S == 0) return PG_OK;
    if (pos) PG_CUDA(cudaMemcpyAsync(pos, ctx->d_pos, (size_t)S * 4, cudaMemcpyDeviceToHost, ctx->stream));
    if (new_scaffold)
        PG_CUDA(cudaMemcpyAsync(new_scaffold, (const int8_t*)((const unsigned long long*)ctx->meta.p + S), (size_t)S,
                                cudaMemcpyDeviceToHost, ctx->stream));
    if (line_off) PG_CUDA(cudaMemcpyAsync(line_off, ctx->starts.p, (size_t)S * 8, cudaMemcpyDeviceToHost, ctx->stream));
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    return PG_OK;
}

// Strict tokens for the next ingests of this ctx (off by default): see ParseParams::strict.
extern "C" int pg_ingest_set_strict(pg_ctx* ctx, int32_t on) {
    PG_CHECK(ctx != nullptr, "pg_ingest_set_strict: null ctx");
    PG_CHECK(on >= 0 && on <= 2, "pg_ingest_set_strict: level %d is not 0, 1 or 2", on);
    ctx->ingest_strict = on;
    return PG_OK;
}

extern "C" int pg_debug_ingest(pg_ctx* ctx, int64_t* out) {
    PG_CHECK(ctx && out, "pg_debug_ingest: null argument");
    for (int k = 0; k < 5; ++k) out[k] = ctx->ingest_geom[k];
    return PG_OK;
}

// Frees the device copy of the text (it is kept after pg_ingest_text so that repeated ingests reuse the allocation).
extern "C" int pg_ingest_release(pg_ctx* ctx) {
    PG_CHECK(ctx != nullptr, "pg_ingest_release: null ctx");
    PG_CUDA(cudaSetDevice(ctx->device));
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    ctx->text.release();
    ctx->starts.release();
    ctx->meta.release();
    ctx->ingest_sites = -1;
    ctx->text_gen += 1;
    return PG_OK;
}
