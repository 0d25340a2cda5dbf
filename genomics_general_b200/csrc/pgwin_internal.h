// Internal declarations shared by the translation units of libpgwin.so (not part of the C-ABI).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <string>
#include <vector>

#include "../../include/pgwin.h"

#define PG_OK 0
#define PG_ERR 1

void pg_set_error(const char* fmt, ...);

#define PG_CUDA(call)                                                                                  \
    do {                                                                                               \
        cudaError_t _e = (call);                                                                       \
        if (_e != cudaSuccess) {                                                                       \
            pg_set_error("%s:%d: %s failed: %s", __FILE__, __LINE__, #call, cudaGetErrorString(_e));  \
            return PG_ERR;                                                                             \
        }                                                                                              \
    } while (0)

#define PG_CHECK(cond, ...)                 \
    do {                                    \
        if (!(cond)) {                      \
            pg_set_error(__VA_ARGS__);      \
            return PG_ERR;                  \
        }                                   \
    } while (0)

#define PG_TRY(expr)                 \
    do {                             \
        int _r = (expr);             \
        if (_r != PG_OK) return _r;  \
    } while (0)

struct PgTiming {
    char name[32];
    cudaEvent_t start, stop;
    int launches;
};

// grow-only device scratch buffer
struct PgBuf {
    void* p = nullptr;
    size_t cap = 0;
    int ensure(size_t bytes);
    void release();
};

static constexpr int PG_MAX_K1_POPS = 8;     // K1 keeps per-pop counts in registers: P <= 8
static constexpr int PG_MAX_POPS = 64;       // K2 block epilogue

// K1 launch geometry for one (S, H): see DESIGN.md "K1 tiling".
struct K1Plan {
    int pitch;        // bytes per site row on the device = 16 * chunks, chunks odd (bank-conflict-free LDS.128)
    int chunks;       // 16-byte chunks per row
    int G;            // lanes cooperating on one site (power of two, <= 32)
    int I;            // sites per lane per tile
    int wpt;          // consumer warps per tile (a "team"); nw / wpt teams work on different tiles
    int nw;           // consumer warps per CTA (8 or 12)
    int T;            // sites per tile = (32 * wpt / G) * I
    int stages;       // TMA ring depth
    int tile_bytes;   // T * pitch
    int smem_bytes;   // dynamic shared memory of the kernel
    int64_t num_tiles;
    int ctas;         // persistent CTAs, each owning a contiguous tile range
};
K1Plan pg_make_k1_plan(int64_t S, int H, int sm_count, int table_bytes, int nw = 8, int force_G = 0);
// rows of `pitch` bytes
K1Plan pg_make_k1_plan_rows(int64_t S, int pitch, int sm_count, int table_bytes, int nw, int force_G);
int pg_k1_ring_stages(int tile_bytes, int table_bytes);   // ring depth for stages of tile_bytes (< 2: does not fit)
int pg_k1_plan_ok(const K1Plan& p);   // 1 if the site-pass kernels can run this plan
int pg_pitch_for(int H);
int pg_packed_pitch_for(int H);       // bytes per row of the packed companion

// Site class of a packed row over its H haplotypes: every haplotype carries allele A / C / G / T, every haplotype is missing,
// every haplotype is called and exactly two alleles are present ("complete biallelic": VARIED2 when the two codes differ in
// their low bit only, so that plane B0 tells them apart; VARIED2_B1 when they differ in the high bit, so that plane B1 does,
// the higher code carrying the set bit either way), or anything else.  Zeroed memory reads as "varied", which is always safe
// to walk.
enum { PG_CLS_VARIED = 0, PG_CLS_A = 1, PG_CLS_C = 2, PG_CLS_G = 3, PG_CLS_T = 4, PG_CLS_MISSING = 5, PG_CLS_VARIED2 = 6,
       PG_CLS_VARIED2_B1 = 7 };
__host__ __device__ inline bool pg_cls_varied(unsigned c) { return c == PG_CLS_VARIED || c >= PG_CLS_VARIED2; }
__host__ __device__ inline bool pg_cls_biallelic(unsigned c) { return c >= PG_CLS_VARIED2; }

struct pg_ctx {
    int device = 0;
    int sm_count = 132;
    cudaStream_t stream = nullptr;
    // genotype matrix
    int8_t* d_geno = nullptr;
    int32_t* d_pos = nullptr;
    int64_t S = 0;
    int32_t H = 0;
    int32_t pitch = 0;
    size_t geno_cap = 0, pos_cap = 0;
    // packed companion of the resident matrix (DESIGN.md "Packed companion"): per site three planes of ceil(H / 32) words
    // (valid bits, low and high bit of the allele code), rows of packed_pitch bytes.  Every writer of d_geno rebuilds the
    // rows it wrote (pg_pack_rows); nullptr when it could not be allocated, and the popgen site pass then reads the bytes.
    uint32_t* d_packed = nullptr;
    int32_t packed_pitch = 0;
    size_t packed_cap = 0;
    // one class byte per packed row (PG_CLS_*), written by pg_pack_rows with the row; allocated, grown and dropped with
    // d_packed (nullptr: no classes, and the popgen pass streams every row)
    uint8_t* d_site_cls = nullptr;
    size_t cls_cap = 0;
    // populations
    int32_t P = 0;
    std::vector<int32_t> hap_pop;
    // windows (host copies) + segments
    int64_t W = 0;
    std::vector<int64_t> win_lo, win_hi;
    std::vector<int64_t> brk;                 // segment breakpoints, brk[0]=0 .. brk[nseg]=S
    std::vector<int32_t> win_seg_lo, win_seg_hi;
    // timings of the last statistics call
    std::vector<PgTiming> timings;
    std::vector<cudaEvent_t> event_pool;
    size_t events_used = 0;
    int64_t launches = 0;
    // scratch
    PgBuf tables, part, segmeta, winmeta, out_d, out_i, planes, planes2, pairs, misc, misc2, misc3, misc4, misc5;
    PgBuf text, starts, meta;                 // device-side text ingest (ingest.cu)
    int64_t ingest_sites = -1;
    int32_t ingest_fmt = 0;                   // format of the last text ingest
    int32_t ingest_strict = 0;                // pg_ingest_set_strict
    int64_t ingest_geom[5] = {0, 0, 0, 0, 0}; // geometry of the last text ingest (pg_debug_ingest)
    uint64_t text_gen = 0;                    // bumped by every load or release of ctx->text (pg_text_load)
    // filterGenotypes (filter.cu): phase character per sample of the strict ingest, sample tables, per-site statistics,
    // kept rows, their byte offsets and the output slab
    PgBuf flt_aux, flt_tab, flt_stats, flt_rows, flt_off, flt_out, flt_cub;
    void* flt_state = nullptr;                // host-side state of the last pg_filter (owned by filter.cu)
    void* vcf_state = nullptr;                // parseVCF buffers and spec (owned by vcf.cu)
    void* seq_state = nullptr;                // genoToSeq token index and row plan (owned by seq.cu)
    void* g2v_state = nullptr;                // genoToVCF reference sequences, spec and chunk state (owned by geno2vcf.cu)
    void* s2g_state = nullptr;                // seqToGeno sequences, line table and row plan (owned by seq2geno.cu)
    void* ws_state = nullptr;                 // windowStats values, positions and chunk state (owned by wstats.cu)
    void* merge_state = nullptr;              // mergeGeno scaffold table, per-file chunks and the rows (owned by merge.cu)
    void* h_text[2] = {nullptr, nullptr};     // pinned staging of the text
    cudaEvent_t h_text_free[2] = {nullptr, nullptr};
    // upload pipeline: copy stream + two staging buffers
    cudaStream_t copy_stream = nullptr;
    PgBuf stage[2];
    cudaEvent_t stage_full[2] = {nullptr, nullptr}, stage_free[2] = {nullptr, nullptr};
    bool want_freq = false;                   // carry the popFreq counters in the popgen site pass
    uint64_t epoch = 1;                       // bumped by every change of data shape / populations / windows
    uint64_t data_gen = 1;                    // bumped by every write of the resident matrix or the population map (also
                                              // an upload of the same shape, which keeps `epoch`)
    void* k1_cache[3] = {nullptr, nullptr, nullptr};   // cached launch state (popgen, abba, fourpop) — owned by k1.cu
    std::vector<unsigned long long> h_rec;    // host copy of the per-window records
    // native NCCL gather (nccl_gather.cu)
    void* nccl_comm = nullptr;
    int nccl_ranks = 1, nccl_rank = 0;
    PgBuf gather;
    PgBuf gather_flag;                        // one int64 all-reduced by the pipelined gather's collective refusal
    // pipelined gather (pg_popgen_gather_begin / _end): two record tables, exchange + read-back on a side stream
    cudaStream_t gather_stream = nullptr;
    cudaEvent_t g_rec[2] = {nullptr, nullptr}, g_done[2] = {nullptr, nullptr};
    PgBuf gslot[2];
    void* gslot_host[2] = {nullptr, nullptr};
    size_t gslot_host_cap[2] = {0, 0}, gslot_words[2] = {0, 0};
    int64_t gslot_wmax[2] = {0, 0};
    int32_t gslot_min_sites[2] = {0, 0};
    double gslot_min_data[2] = {0, 0};
    // what `end` needs of the batch as it was at `begin`: window count, record width (from P), bounds, data generation
    int64_t gslot_W[2] = {0, 0};
    int32_t gslot_RC[2] = {0, 0};
    std::vector<int64_t> gslot_lo[2], gslot_hi[2];
    uint64_t gslot_gen[2] = {0, 0};
    void* h_pinned = nullptr;                 // small pinned staging for result read-back
    size_t h_pinned_cap = 0;
    // sparse spectra (pg_sfs_sparse / pg_sfs_tables_sparse, k1.cu): the runs accumulated so far (keys + {count, first})
    // and the next merge's output, the slab's entries, the merge and CUB scratch.  The result waits in
    // sfs_acc_*[sfs_cur] until pg_sfs_sparse_fetch; sfs_total = its entries, -1 = none pending.
    PgBuf sfs_acc_k[2], sfs_acc_r[2], sfs_slab, sfs_merge, sfs_cub;
    int sfs_cur = 0;
    int64_t sfs_total = -1;
};

// timing helpers: every kernel launch is bracketed by events on ctx->stream
void pg_timings_reset(pg_ctx* ctx);
int pg_time_begin(pg_ctx* ctx, const char* name);   // returns timing index
void pg_time_end(pg_ctx* ctx, int idx);
int pg_pinned(pg_ctx* ctx, size_t bytes, void** out);
int pg_d2h_staged(pg_ctx* ctx, void* dst, const void* src, size_t bytes);   // large device -> pageable host copy
int pg_build_segments(pg_ctx* ctx);
int pg_pack_rows(pg_ctx* ctx, int64_t s0, int64_t n);   // rows [s0, s0 + n) of the packed companion from d_geno (ctx stream)

// launch() (one launch, or a few that share the label) bracketed by the timing label `name`, then the launch error check
template <class Launch>
int pg_timed(pg_ctx* ctx, const char* name, Launch&& launch) {
    const int ti = pg_time_begin(ctx, name);
    launch();
    pg_time_end(ctx, ti);
    PG_CUDA(cudaGetLastError());
    return PG_OK;
}

// Kernels that take more dynamic shared memory than the default limit need an attribute, which is per device: set it once per
// kernel and per device.  Only for a fixed `bytes` per kernel.
template <auto Kern>
int pg_smem_limit(const pg_ctx* ctx, int bytes) {
    static bool set[64] = {};
    if (!set[ctx->device & 63]) {
        PG_CUDA(cudaFuncSetAttribute(Kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
        set[ctx->device & 63] = true;
    }
    return PG_OK;
}

// tensor-core pairwise path (k2t.cu): bit-packed operand planes of one site span
struct K2TPlanes {
    int Hk = 0, R = 0;                 // plane rows (haplotypes in `order`), rows allocated (multiple of 16, pad rows zero)
    int64_t site_base = 0;             // first site of valid-plane chunk 0 (multiple of 64)
    int64_t nchunk_v = 0;
    const uint64_t* vplane = nullptr;  // [nchunk_v][R]: bit b of word (c, r) = haplotype r non-missing at site site_base + 64 c + b
    const int32_t* cps = nullptr;      // [64 nchunk_v + 1]: pseudo-sites before each site of the span
    int64_t npseudo = 0;
    const uint64_t* pq = nullptr;      // [ceil(npseudo / 64)][2][R]: P and Q planes of the pseudo-sites
    // n_ij is computed over "mask rows": one per plane row, or — when rows 2k and 2k+1 have identical valid planes (the two
    // haplotypes of a sample with per-genotype missingness) — one per pair of rows
    int Hm = 0, R2 = 0;
    const uint64_t* vpair = nullptr;   // [nchunk_v][R2] valid words of the even rows (nullptr: every row is its own mask row)
    const int32_t* d_mid = nullptr;    // [Hk] mask row of each plane row
};
bool pg_k2_use_tensor();               // false when PG_K2_POPC is set (the bit-plane POPC kernels, kept as a checker)
// can the tensor path's plane builders take Hk plane rows of `pitch`-byte site rows?  They stage 16 bytes per column and 8 per
// plane row in 96 KiB of shared memory: beyond about 4000 haplotype columns only the POPC kernels (any width) build planes
inline bool pg_k2t_fits(int pitch, int Hk) { return (size_t)16 * pitch + (size_t)((Hk + 15) / 16 * 16) * 8 <= 96 * 1024; }
int pg_k2t_build(pg_ctx* ctx, const std::vector<int32_t>& order, int64_t lo, int64_t hi, K2TPlanes& ps);
int pg_k2t_pairs(pg_ctx* ctx, const K2TPlanes& ps, const int64_t* d_lo, const int64_t* d_hi, int nb, int32_t* d_diff,
                 int32_t* d_n);
int pg_k2t_seq_nonnan(pg_ctx* ctx, const K2TPlanes& ps, const int64_t* d_lo, const int64_t* d_hi, int nb, long long* d_out);
int pg_k2t_het(pg_ctx* ctx, const K2TPlanes& ps, const int64_t* d_lo, const int64_t* d_hi, int nb, const int32_t* d_ind_start,
               int n_ind, int min_sites, double* d_out);

// Frequency order of a site's alleles A, C, G, T from their counts c: np.argsort(counts)[::-1] over the counted alleles
// (genomics.py:556) as a stable sort gives it — descending count, ties to the later allele.  rank[a] = place of allele a in
// the order (4 when its count is 0); returns the number of counted alleles.  Shared by filterGenotypes' row emission
// (filter.cu) and genoToVCF's allele lists (geno2vcf.cu).
__device__ __forceinline__ int pg_freq_order(const int c[4], int rank[4]) {
    int nr = 0;
    for (int a = 0; a < 4; ++a) {
        rank[a] = 4;
        if (c[a] <= 0) continue;
        int before = 0;
        for (int b = 0; b < 4; ++b)
            if (c[b] > 0 && (c[b] > c[a] || (c[b] == c[a] && b > a))) ++before;
        rank[a] = before;
        ++nr;
    }
    return nr;
}

// str.split() blanks of ASCII text ('\n' ends the line)
__device__ __forceinline__ bool pg_sblank(unsigned c) {
    return c == ' ' || c == '\t' || c == '\r' || c == '\v' || c == '\f' || (c >= 0x1c && c <= 0x1f);
}

// byte i of a text of len bytes, '\n' past its end
__device__ __forceinline__ unsigned pg_byte_at(const uint8_t* buf, size_t len, size_t i) { return i < len ? buf[i] : (unsigned)'\n'; }

// ONE WARP walks the line that starts at byte l0 of buf (len bytes) as str.split() reads it: each lane classifies 4 bytes per
// step and a warp prefix sum of the token-start flags numbers the fields.  The lane that owns the start q of field f calls
// on_field(f, q) (in field order within a lane).  Returns the line's field count to every lane; *hi = the line holds a byte
// >= 0x80, *lone_cr = a '\r' in it is not followed by '\n' (a line end of its own under universal newlines).  The
// classification is seq.cu's k_seq_tokens'; the caller gives every line its own warp.  Shared by genoToVCF's token pass
// (geno2vcf.cu) and seqToGeno's PHYLIP line pass (seq2geno.cu).
template <class OnField>
__device__ __forceinline__ unsigned pg_warp_fields(const uint8_t* buf, size_t len, size_t l0, bool* hi, bool* lone_cr,
                                                   OnField&& on_field) {
    const int lane = threadIdx.x & 31;
    const size_t a0 = l0 & ~(size_t)3;
    unsigned fields_before = 0;
    bool prev_ws = true, any_hi = false, any_cr = false, done = false;
    for (size_t step = 0; !done; ++step) {
        const size_t wbase = a0 + step * 128 + (size_t)lane * 4;
        uint32_t w = 0x0a0a0a0au;
        if (wbase + 4 <= len) w = *reinterpret_cast<const uint32_t*>(buf + wbase);
        else if (wbase < len) {
            for (int k = 0; k < 4; ++k)
                if (wbase + k < len) w = (w & ~(0xffu << (8 * k))) | ((uint32_t)buf[wbase + k] << (8 * k));
        }
        unsigned ws = 0, nl = 0, hb = 0, cr = 0;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const unsigned c = (w >> (8 * k)) & 0xffu;
            const bool before = (wbase + k) < l0;
            if (before || pg_sblank(c)) ws |= 1u << k;
            else if (c == '\n') nl |= 1u << k;
            if (!before && c >= 0x80u) hb |= 1u << k;
            if (!before && c == '\r') cr |= 1u << k;
        }
        const unsigned nl_lanes = __ballot_sync(0xffffffffu, nl != 0);
        if (nl_lanes) {
            const int first = __ffs(nl_lanes) - 1;
            if (lane > first) ws = 0xfu, nl = 0, hb = 0, cr = 0;
            else if (lane == first) {
                const unsigned from = nl & (0u - nl);
                ws |= ~(from - 1u) & 0xfu;
                hb &= from - 1u;
                cr &= from - 1u;
            }
            done = true;
        }
        any_hi |= hb != 0;
        for (unsigned m = cr; m; m &= m - 1)
            if (pg_byte_at(buf, len, wbase + __ffs(m)) != '\n') any_cr = true;
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
        for (unsigned m = st; m; m &= m - 1, ++fidx) on_field(fidx, wbase + (__ffs(m) - 1));
    }
    *hi = __any_sync(0xffffffffu, any_hi);
    *lone_cr = __any_sync(0xffffffffu, any_cr);
    return fields_before;
}

// implemented in k1.cu / k2.cu
// pairwise statistics for the listed windows, written into the DEVICE record table (stride RC words); window w spans sites
// [win_lo[w], win_hi[w]) of the resident matrix
int pg_k2_popgen_windows(pg_ctx* ctx, const std::vector<int64_t>& wins, const int64_t* win_lo, const int64_t* win_hi,
                         int32_t min_sites, double min_data, void* d_rec, int RC);
void pg_k1_cache_free(pg_ctx* ctx);
void pg_filter_free(pg_ctx* ctx);        // filter.cu
void pg_vcf_free(pg_ctx* ctx);           // vcf.cu
void pg_seq_free(pg_ctx* ctx);           // seq.cu
void pg_g2v_free(pg_ctx* ctx);           // geno2vcf.cu
void pg_s2g_free(pg_ctx* ctx);           // seq2geno.cu
void pg_ws_free(pg_ctx* ctx);            // wstats.cu
void pg_merge_free(pg_ctx* ctx);         // merge.cu
// fasta.cu: the FASTA loader of genoToVCF's reference and seqToGeno's input (genomics.parseFasta after universal newlines).
// pg_fa_load: the text -> fa, the byte offsets of its '>' bytes -> rec, *n_rec = their count; pg_fa_starts reads them back.
// pg_fa_index: record k's sequence is bytes [lo[k], hi[k]) of the text without '\n', '\r' and ' ', compacted into seq with
// {rec_off [n_rec], rec_len [n_rec]} in rec (int64); the text is released.  `tag` prefixes the timing labels (tag_fa_h2d,
// tag_fa_marks, tag_fa_keep, tag_fa_select); the caller resets the timings.
struct PgFasta {
    PgBuf fa, flags, seq, rec, scratch, cub;
    size_t fa_len = 0;
    int64_t n_rec = 0;
    bool indexed = false;
    void release();
};
int pg_fa_load(pg_ctx* ctx, PgFasta& fs, const char* text, size_t len, const char* tag, int64_t* n_rec);
int pg_fa_starts(pg_ctx* ctx, PgFasta& fs, int64_t* starts);
int pg_fa_index(pg_ctx* ctx, PgFasta& fs, int64_t n_rec, const int64_t* lo, const int64_t* hi, const char* tag,
                int64_t* rec_len);
// ingest.cu: the text (memory, or bytes [file_off, file_off + len) of the open file fd) -> ctx->text, the start of every data
// line -> ctx->starts, *n_lines = data lines; and the new-scaffold flags of S per-line scaffold hashes (both on ctx->stream)
int pg_text_load(pg_ctx* ctx, const char* mem, int fd, size_t file_off, size_t len, int64_t* n_lines);
int pg_scaffold_flags(pg_ctx* ctx, const unsigned long long* d_hash, int64_t S, int8_t* d_flags);
int pg_nccl_allreduce_i64(pg_ctx* ctx, void* d_buf, size_t count);   // nccl_gather.cu
int pg_popgen_enqueue(pg_ctx* ctx, int32_t min_sites, double min_data, int32_t force_path, void* d_rec, int** h_count);
int pg_popgen_resolve(pg_ctx* ctx, int32_t min_sites, double min_data, void* d_rec, int nk2);
int pg_abba_enqueue(pg_ctx* ctx, const int* sel, double min_data, void* d_rec);                 // records [W x 8]
int pg_fourpop_enqueue(pg_ctx* ctx, const int* sel, double min_data, int mode, void* d_rec);    // records [W x 17]
