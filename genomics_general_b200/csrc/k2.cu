// K2 — the pairwise path: per-window haplotype-pair matrices diff_ij / n_ij (integers), then the reference's
// mean-of-ratios epilogues.  The matrices come from one of two sets of operand planes:
//   - the tensor-core path (k2t.cu), the default: bit-packed planes and wgmma Gram kernels;
//   - the POPC path (this file), where the tensor path's plane builders cannot take the width (pg_k2t_fits, about 4000
//     haplotype columns) or PG_K2_POPC is set; the tests also compare the tensor path against it:
//       k2_build_planes : int8 [S x pitch] -> 3 bit-planes per haplotype (allele bit0, allele bit1, valid),
//                         haplotype-major, 32 sites per word           -- replaces Alignment.nanMask/numArray rows
//       k2_hash_rows / k2_verify_rows : plane rows with identical valid planes share one mask row of n_ij
//       k2_pair         : diff_ij = popc(((b0_i^b0_j)|(b1_i^b1_j)) & m_i & m_j), n_ij = popc(m_i & m_j) summed over
//                         the window's words; 64x64 haplotype tiles, 4x4 pairs per thread, cp.async ring
//                         -- replaces distMatrix + pairNonNan (genomics.py:907-916, 1042-1047)
//       k2_het, k2_seq_nonnan : sampleHet / seqNonNan from the bit-planes
//     These kernels are integer-issue bound (LOP3/POPC), not HBM bound (DESIGN.md §K2).
// The epilogues here read the matrices of either path:
//   k2_popgen_epi_* : d_ij = diff/n, minSites mask, nanmean_min block means -> pi / dxy / Fst (genomics.py:956-995)
//   k2_ind_epi      : individual x individual nanmean of ploidy blocks (genomics.py:934-954)
//   k2_hap_epi      : H12 / H2 clustering (genomics.py:1079-1098)
//   k2_reduce_pairs, k2_ind_epi64 : --windType cat, chunk matrices summed as int64
// The host half at the end of this file serves both paths: the entry points, their window batches and their scratch.
#include <stdlib.h>

#include <algorithm>
#include <cmath>

#include "pgwin_internal.h"

namespace {

constexpr int TS = 64;          // haplotypes per tile side
constexpr int TSP = TS + 1;     // padded (16-byte units) -> conflict-free STS/LDS
constexpr int KW = 16;          // words (32 sites each) per pipeline stage
constexpr int K4 = KW / 4;
constexpr int NST = 3;          // cp.async ring depth
enum { PAIR_DIFF = 0, PAIR_N = 1 };
template <int WHAT>
struct PairGeom {
    static constexpr int NP = (WHAT == PAIR_DIFF) ? 3 : 1;      // planes staged per operand
    static constexpr int OPND_BYTES = NP * K4 * TSP * 16;
    static constexpr int STAGE_BYTES = 2 * OPND_BYTES;
    static constexpr int SMEM = NST * STAGE_BYTES;
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void cp_async16(void* dst, const void* src, bool valid) {
    const int sz = valid ? 16 : 0;
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(dst)), "l"(src), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
    asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

// ------------------------------------------------------------------------------------------------
// bit-plane build
// ------------------------------------------------------------------------------------------------
constexpr int BP_SITES = 256, BP_COLS = 128, BP_ROWW = BP_COLS / 4 + 1;   // 33 words per site row (odd: no conflicts)
constexpr int BP_OUTW = 3 * BP_COLS + 4;                                     // words per warp in the ballot staging (+pad)
constexpr int BP_SMEM = BP_SITES * BP_ROWW * 4 + 8 * BP_OUTW * 4 + BP_COLS * 4 + 64;

// Resident code: A 0x01, C 0x04, G 0x10, T 0x40, missing 0x00  ->  bit0 = C|T (0x44), bit1 = G|T (0x50), valid = !=0
// Each warp transposes 32 sites (lane = site): one LDS.32 brings 4 columns, a predicate LOP3 + VOTE per byte and plane
// yields the 32-site word of that (plane, column); the 4 ballots of a plane leave as one STS.128.
__global__ void __launch_bounds__(256) k2_build_planes(const uint8_t* __restrict__ geno, int pitch, int64_t S,
                                                       int64_t site_base, const int32_t* __restrict__ col_to_row,
                                                       uint32_t* __restrict__ planes, int Hk, int64_t NWp) {
    extern __shared__ __align__(16) uint8_t bsm[];
    uint32_t* tile = reinterpret_cast<uint32_t*>(bsm);                          // [256][33]
    uint32_t* outp = tile + BP_SITES * BP_ROWW;                                  // [8 warps][3 planes][128 cols] (+pad)
    int32_t* s_c2r = reinterpret_cast<int32_t*>(outp + 8 * BP_OUTW);            // [128] plane row of a local column
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int col0 = blockIdx.x * BP_COLS;
    const int64_t sblk = blockIdx.y;
    const int64_t site0 = site_base + sblk * BP_SITES;

    if (tid < BP_COLS) {
        const int col = col0 + tid;
        s_c2r[tid] = (col < pitch) ? col_to_row[col] : -1;
    }
    // 256 sites x 128 columns: 8 lanes cover one row segment; all 8 passes are in flight together
    {
        uint4 v[8];
#pragma unroll
        for (int pass = 0; pass < 8; ++pass) {
            const int r = pass * 32 + warp * 4 + (lane >> 3);
            const int64_t site = site0 + r;
            const int col = col0 + (lane & 7) * 16;
            v[pass] = make_uint4(0u, 0u, 0u, 0u);
            if (site < S && col < pitch) v[pass] = *reinterpret_cast<const uint4*>(geno + site * pitch + col);
        }
#pragma unroll
        for (int pass = 0; pass < 8; ++pass) {
            const int r = pass * 32 + warp * 4 + (lane >> 3);
            uint32_t* d = tile + r * BP_ROWW + (lane & 7) * 4;
            d[0] = v[pass].x;
            d[1] = v[pass].y;
            d[2] = v[pass].z;
            d[3] = v[pass].w;
        }
    }
    __syncthreads();
    const uint32_t* myrow = tile + (warp * 32 + lane) * BP_ROWW;
    uint32_t* myout = outp + warp * BP_OUTW;
#pragma unroll 2
    for (int cw = 0; cw < BP_COLS / 4; ++cw) {
        // skip words whose 4 columns are all unused (warp-uniform)
        const int4 rr = *reinterpret_cast<const int4*>(s_c2r + cw * 4);
        if ((rr.x & rr.y & rr.z & rr.w) < 0) continue;
        const uint32_t w = myrow[cw];
        uint4 m, b0, b1;
        m.x = __ballot_sync(0xffffffffu, (w & 0x000000ffu) != 0u);
        m.y = __ballot_sync(0xffffffffu, (w & 0x0000ff00u) != 0u);
        m.z = __ballot_sync(0xffffffffu, (w & 0x00ff0000u) != 0u);
        m.w = __ballot_sync(0xffffffffu, (w & 0xff000000u) != 0u);
        b0.x = __ballot_sync(0xffffffffu, (w & 0x00000044u) != 0u);
        b0.y = __ballot_sync(0xffffffffu, (w & 0x00004400u) != 0u);
        b0.z = __ballot_sync(0xffffffffu, (w & 0x00440000u) != 0u);
        b0.w = __ballot_sync(0xffffffffu, (w & 0x44000000u) != 0u);
        b1.x = __ballot_sync(0xffffffffu, (w & 0x00000050u) != 0u);
        b1.y = __ballot_sync(0xffffffffu, (w & 0x00005000u) != 0u);
        b1.z = __ballot_sync(0xffffffffu, (w & 0x00500000u) != 0u);
        b1.w = __ballot_sync(0xffffffffu, (w & 0x50000000u) != 0u);
        if (lane == 0) {
            *reinterpret_cast<uint4*>(myout + 0 * BP_COLS + cw * 4) = b0;
            *reinterpret_cast<uint4*>(myout + 1 * BP_COLS + cw * 4) = b1;
            *reinterpret_cast<uint4*>(myout + 2 * BP_COLS + cw * 4) = m;
        }
    }
    __syncthreads();
    // (plane, column) -> 8 consecutive words (one per warp) = 32 bytes of the plane row
    for (int idx = tid; idx < 3 * BP_COLS; idx += 256) {
        const int p = idx / BP_COLS, cl = idx % BP_COLS;
        const int r = s_c2r[cl];
        if (r < 0) continue;
        uint32_t v[8];
#pragma unroll
        for (int wv = 0; wv < 8; ++wv) v[wv] = outp[wv * BP_OUTW + p * BP_COLS + cl];
        uint4* dst = reinterpret_cast<uint4*>(planes + ((size_t)p * Hk + r) * NWp + sblk * 8);
        dst[0] = make_uint4(v[0], v[1], v[2], v[3]);
        dst[1] = make_uint4(v[4], v[5], v[6], v[7]);
    }
}

// ------------------------------------------------------------------------------------------------
// pair kernel
// ------------------------------------------------------------------------------------------------
struct PairParams {
    const uint32_t* planes;   // [3][Hk][NWp]
    int Hk;                   // rows per plane in storage
    int64_t NWp;
    int64_t site_base;
    const int64_t* win_lo;    // [nb] absolute site indices (non-empty windows only)
    const int64_t* win_hi;
    int ntile;
    int n_rows;               // logical rows of this pass (haplotypes for DIFF, unique valid-masks for N)
    const int32_t* row_map;   // logical row -> plane row (nullptr = identity)
    int32_t* out;             // [nb][n_rows][n_rows]
};

// One pass over a window for one 64x64 tile pair.
//   PAIR_DIFF: diff_ij = sum popc(((b0_i^b0_j)|(b1_i^b1_j)) & m_i & m_j)      (3 planes)
//   PAIR_N   : n_ij    = sum popc(m_i & m_j)                                   (valid plane only, unique masks)
// DIAG: the tile pair is on the diagonal -> pairs with a > b are mirror images, skip them.
template <int WHAT, bool DIAG>
__device__ __forceinline__ void pair_accumulate(const uint8_t* sb, int ty, int tx, int (&acc)[4][4]) {
    using G = PairGeom<WHAT>;
    const uint4* I4 = reinterpret_cast<const uint4*>(sb);
    const uint4* J4 = reinterpret_cast<const uint4*>(sb + G::OPND_BYTES);
#pragma unroll
    for (int k4 = 0; k4 < K4; ++k4) {
        if (WHAT == PAIR_DIFF) {
            uint4 B0[4], B1[4], BM[4];
#pragma unroll
            for (int b = 0; b < 4; ++b) {
                B0[b] = J4[(0 * K4 + k4) * TSP + tx + 16 * b];
                B1[b] = J4[(1 * K4 + k4) * TSP + tx + 16 * b];
                BM[b] = J4[(2 * K4 + k4) * TSP + tx + 16 * b];
            }
#pragma unroll
            for (int a = 0; a < 4; ++a) {
                const uint4 A0 = I4[(0 * K4 + k4) * TSP + ty + 16 * a];
                const uint4 A1 = I4[(1 * K4 + k4) * TSP + ty + 16 * a];
                const uint4 AM = I4[(2 * K4 + k4) * TSP + ty + 16 * a];
#pragma unroll
                for (int b = 0; b < 4; ++b) {
                    if (DIAG && a > b) continue;
#define K2_DIFF_WORD(C) acc[a][b] += __popc(((A0.C ^ B0[b].C) | (A1.C ^ B1[b].C)) & AM.C & BM[b].C);
                    K2_DIFF_WORD(x)
                    K2_DIFF_WORD(y)
                    K2_DIFF_WORD(z)
                    K2_DIFF_WORD(w)
#undef K2_DIFF_WORD
                }
            }
        } else {
            uint4 BM[4];
#pragma unroll
            for (int b = 0; b < 4; ++b) BM[b] = J4[k4 * TSP + tx + 16 * b];
#pragma unroll
            for (int a = 0; a < 4; ++a) {
                const uint4 AM = I4[k4 * TSP + ty + 16 * a];
#pragma unroll
                for (int b = 0; b < 4; ++b) {
                    if (DIAG && a > b) continue;
                    acc[a][b] += __popc(AM.x & BM[b].x) + __popc(AM.y & BM[b].y) + __popc(AM.z & BM[b].z) +
                                 __popc(AM.w & BM[b].w);
                }
            }
        }
    }
}

template <int WHAT>
__global__ void __launch_bounds__(256, 2) k2_pair(const __grid_constant__ PairParams pp) {
    using G = PairGeom<WHAT>;
    extern __shared__ __align__(16) uint8_t psm[];
    const int tid = threadIdx.x;
    const int ty = tid >> 4, tx = tid & 15;
    // decode the upper-triangular tile pair
    int tp = blockIdx.x, ti = 0;
    while (tp >= pp.ntile - ti) {
        tp -= pp.ntile - ti;
        ++ti;
    }
    const int tj = ti + tp;
    const int wb = blockIdx.y;
    const int64_t rel_lo = pp.win_lo[wb] - pp.site_base, rel_hi = pp.win_hi[wb] - pp.site_base;
    const int64_t w_first = rel_lo >> 5, w_last = (rel_hi - 1) >> 5;
    const uint32_t mask_first = 0xffffffffu << (rel_lo & 31);
    const uint32_t mask_last = 0xffffffffu >> (31 - (int)((rel_hi - 1) & 31));
    const int64_t k_begin = w_first & ~(int64_t)3;
    const int nchunk = (int)((w_last - k_begin) / KW) + 1;
    constexpr int VALID_PLANE = (WHAT == PAIR_DIFF) ? 2 : 0;    // index of the valid plane inside a staged operand

    auto fill = [&](int chunk, int stage) {
        const int64_t k0 = k_begin + (int64_t)chunk * KW;
        uint8_t* sb = psm + stage * G::STAGE_BYTES;
#pragma unroll
        for (int it = 0; it < (2 * G::NP * TS * K4 + 255) / 256; ++it) {
            const int item = tid + it * 256;
            if (item >= 2 * G::NP * TS * K4) break;
            const int k4 = item & (K4 - 1);
            const int hap = (item / K4) & (TS - 1);
            const int p = (item / (K4 * TS)) % G::NP;
            const int opnd = item / (K4 * TS * G::NP);
            const int gh = (opnd == 0 ? ti : tj) * TS + hap;
            const bool valid = gh < pp.n_rows;
            int prow = valid ? gh : 0;
            if (pp.row_map) prow = pp.row_map[prow];
            const int plane = (WHAT == PAIR_DIFF) ? p : 2;
            const uint32_t* src = pp.planes + ((size_t)plane * pp.Hk + prow) * pp.NWp + k0 + 4 * k4;
            cp_async16(sb + opnd * G::OPND_BYTES + ((p * K4 + k4) * TSP + hap) * 16, src, valid);
        }
    };

    int acc[4][4];
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) acc[a][b] = 0;

    for (int s = 0; s < NST - 1; ++s) {
        if (s < nchunk) fill(s, s);
        cp_async_commit();
    }
    for (int ch = 0; ch < nchunk; ++ch) {
        cp_async_wait<NST - 2>();
        __syncthreads();
        {   // prefetch chunk ch+NST-1 into the stage consumed at iteration ch-1 (all threads are past it)
            const int nxt = ch + NST - 1;
            if (nxt < nchunk) fill(nxt, nxt % NST);
            cp_async_commit();
        }
        uint8_t* sb = psm + (ch % NST) * G::STAGE_BYTES;
        const int64_t k0 = k_begin + (int64_t)ch * KW;
        const bool need_fix = (k0 <= w_first) || (k0 + KW - 1 >= w_last);
        if (need_fix) {   // block-uniform: clip the J operand's valid plane to the window
            if (tid < TS) {
                for (int kk = 0; kk < KW; ++kk) {
                    const int64_t word = k0 + kk;
                    uint32_t mk = 0xffffffffu;
                    if (word < w_first || word > w_last) mk = 0;
                    else {
                        if (word == w_first) mk &= mask_first;
                        if (word == w_last) mk &= mask_last;
                    }
                    if (mk != 0xffffffffu) {
                        uint32_t* wp = reinterpret_cast<uint32_t*>(sb + G::OPND_BYTES +
                                                                   ((VALID_PLANE * K4 + (kk >> 2)) * TSP + tid) * 16) + (kk & 3);
                        *wp &= mk;
                    }
                }
            }
            __syncthreads();
        }
        if (ti == tj) pair_accumulate<WHAT, true>(sb, ty, tx, acc);
        else pair_accumulate<WHAT, false>(sb, ty, tx, acc);
    }
    cp_async_wait<0>();
    const size_t RR = (size_t)pp.n_rows * pp.n_rows;
    int32_t* o = pp.out + (size_t)wb * RR;
#pragma unroll
    for (int a = 0; a < 4; ++a) {
        const int i = ti * TS + ty + 16 * a;
#pragma unroll
        for (int b = 0; b < 4; ++b) {
            if (ti == tj && a > b) continue;             // written as the mirror of the (b, a) pair of thread (tx, ty)
            const int j = tj * TS + tx + 16 * b;
            if (i < pp.n_rows && j < pp.n_rows) {
                o[(size_t)i * pp.n_rows + j] = acc[a][b];
                o[(size_t)j * pp.n_rows + i] = acc[a][b];
            }
        }
    }
}

// ---- haplotypes with identical valid planes share their n_ij -------------------------------------------
__device__ __forceinline__ unsigned long long mixu64(unsigned long long x) {
    x ^= x >> 30;
    x *= 0xBF58476D1CE4E5B9ull;
    x ^= x >> 27;
    x *= 0x94D049BB133111EBull;
    x ^= x >> 31;
    return x;
}
__global__ void __launch_bounds__(256) k2_hash_rows(const uint32_t* __restrict__ mplane, int64_t NWp,
                                                    unsigned long long* __restrict__ hash) {
    __shared__ unsigned long long sh[8];
    const uint32_t* row = mplane + (size_t)blockIdx.x * NWp;
    unsigned long long h = 0;
    for (int64_t j = threadIdx.x; j < NWp; j += 256) h += mixu64(((unsigned long long)row[j] << 32) ^ (unsigned long long)j);
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) h += __shfl_xor_sync(0xffffffffu, h, d);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = h;
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned long long t = 0;
        for (int w = 0; w < 8; ++w) t += sh[w];
        hash[blockIdx.x] = t;
    }
}
__global__ void __launch_bounds__(256) k2_verify_rows(const uint32_t* __restrict__ mplane, int64_t NWp,
                                                      const int32_t* __restrict__ rep, int* __restrict__ mismatch) {
    const int r = blockIdx.x, q = rep[r];
    if (q == r) return;
    const uint32_t* a = mplane + (size_t)r * NWp;
    const uint32_t* b = mplane + (size_t)q * NWp;
    bool bad = false;
    for (int64_t j = threadIdx.x; j < NWp; j += 256) bad |= (a[j] != b[j]);
    if (bad) atomicOr(mismatch, 1);
}

// ------------------------------------------------------------------------------------------------
// epilogues
// ------------------------------------------------------------------------------------------------
// The pair matrices are symmetric; the tensor-core kernel writes the upper triangle only (i <= j), so every read goes
// through (min, max).
__device__ __forceinline__ size_t upper_idx(int i, int j, int ld) {
    return (i <= j) ? (size_t)i * ld + j : (size_t)j * ld + i;
}
__device__ __forceinline__ double nan_d() { return __longlong_as_double(0x7ff8000000000000ll); }

// deterministic block-wide sum: butterfly inside warps, then warp 0 adds the 8 partials in order
__device__ __forceinline__ void block_sum(double& s, long long& c, double* sh_s, long long* sh_c) {
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) {
        s += __shfl_xor_sync(0xffffffffu, s, d);
        c += __shfl_xor_sync(0xffffffffu, c, d);
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    __syncthreads();
    if (lane == 0) {
        sh_s[warp] = s;
        sh_c[warp] = c;
    }
    __syncthreads();
    double ts = 0.0;
    long long tc = 0;
    for (int w = 0; w < 8; ++w) {
        ts += sh_s[w];
        tc += sh_c[w];
    }
    s = ts;
    c = tc;
}

struct PopEpiParams {
    const int32_t* diff;       // [nb][Hk][Hk]
    const int32_t* n;          // [nb][Hm][Hm] over unique valid-masks
    const int32_t* mid;        // [Hk] mask id of each plane row
    int Hm;
    int Hk, P;
    const int32_t* pop_start;   // [P+1] plane-row offsets (rows sorted by population)
    int min_sites;
    double min_data;
    unsigned long long* rec;    // device record table [W x RC]: pi at word 3, then dxy, then fst
    int RC;
    const int64_t* win_idx;     // [nb] global window index of each batch entry
    double* blk_s;              // [nb][P(P+1)/2] block sums (stage 1 -> stage 2)
    long long* blk_c;           // [nb][P(P+1)/2] block counts
};

__device__ __forceinline__ double nanmean_min_dev(double sum, double nonnan, double size, double min_data) {
    // genomics.py:88-90 on a block with `nonnan` finite entries out of `size`
    if (size <= 0) return nan_d();
    const double nan_cnt = size - nonnan;
    if (1.0 - (1.0 * nan_cnt / size) < min_data) return nan_d();
    if (nonnan <= 0) return nan_d();
    return sum / nonnan;
}

// Stage 1: one CTA per (population block X <= Y, window) sums d_ij = diff/n over the block's valid pairs in a fixed order.
__global__ void __launch_bounds__(256) k2_popgen_epi_blocks(const __grid_constant__ PopEpiParams ep) {
    __shared__ double sh_s[8];
    __shared__ long long sh_c[8];
    const int P = ep.P;
    const int wb = blockIdx.y;
    int bi = blockIdx.x, X = 0;
    while (bi >= P - X) {           // decode the upper-triangular block index
        bi -= P - X;
        ++X;
    }
    const int Y = X + bi;
    const size_t HH = (size_t)ep.Hk * ep.Hk;
    const int32_t* D = ep.diff + (size_t)wb * HH;
    const int32_t* N = ep.n + (size_t)wb * ep.Hm * ep.Hm;
    const int r0 = ep.pop_start[X], r1 = ep.pop_start[X + 1];
    const int c0 = ep.pop_start[Y], c1 = ep.pop_start[Y + 1];
    const int nr = r1 - r0, nc = c1 - c0;
    double s = 0.0;
    long long c = 0;
    // a warp walks one matrix row at a time, lanes along the columns (coalesced, no integer division per element); two
    // columns per lane and step keep two independent fp64 divisions in flight
    double s1 = 0.0;
    long long cnt1 = 0;
    for (int i = r0 + (threadIdx.x >> 5); i < r1; i += 8) {
        const int mi = ep.mid[i];
        const int32_t* Drow = D + (size_t)i * ep.Hk;
        for (int j = ((X == Y) ? i + 1 : c0) + (threadIdx.x & 31); j < c1; j += 64) {
            const int j2 = j + 32;
            const int nij = N[upper_idx(mi, ep.mid[j], ep.Hm)];
            const int nij2 = (j2 < c1) ? N[upper_idx(mi, ep.mid[j2], ep.Hm)] : 0;
            const bool ok = !(nij == 0 || (ep.min_sites > 0 && nij < ep.min_sites));          // else: a nan entry
            const bool ok2 = !(nij2 == 0 || (ep.min_sites > 0 && nij2 < ep.min_sites));
            const double d0 = ok ? (double)Drow[j] / (double)nij : 0.0;
            const double d1 = ok2 ? (double)Drow[j2] / (double)nij2 : 0.0;
            if (ok) {
                s += d0;
                c += 1;
            }
            if (ok2) {
                s1 += d1;
                cnt1 += 1;
            }
        }
    }
    s += s1;
    c += cnt1;
    (void)nr;
    (void)nc;
    block_sum(s, c, sh_s, sh_c);
    if (threadIdx.x == 0) {
        const int nblk = P * (P + 1) / 2;
        ep.blk_s[(size_t)wb * nblk + blockIdx.x] = s;
        ep.blk_c[(size_t)wb * nblk + blockIdx.x] = c;
    }
}

// Stage 1 when the haplotypes of a sample share their missingness (mask id of plane row r = r >> 1) and every population
// starts on an even row: ONE CTA per window walks all population blocks by SAMPLE pairs (a, b).  The four haplotype
// pairs of a sample pair share n_ab, so their distances add up as (d00 + d01 + d10 + d11) / n_ab — one fp64 division per
// four pairs, exact integer numerator (the reference's four separate quotients summed differ from this by rounding only,
// ~1e-16 relative).  Fixed summation order: lane sums -> butterfly -> warps in order.
__global__ void __launch_bounds__(128) k2_popgen_epi_pairs(const __grid_constant__ PopEpiParams ep) {
    extern __shared__ __align__(16) double epi_sh[];     // [nblk][4 warps] sums, then counts
    const int P = ep.P, nblk = P * (P + 1) / 2;
    double* sh_s = epi_sh;
    long long* sh_c = reinterpret_cast<long long*>(epi_sh + (size_t)nblk * 4);
    const int wb = blockIdx.x;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int32_t* D = ep.diff + (size_t)wb * ep.Hk * ep.Hk;
    const int32_t* N = ep.n + (size_t)wb * ep.Hm * ep.Hm;
    int blk = 0;
    for (int X = 0; X < P; ++X) {
        const int a0 = ep.pop_start[X] >> 1, a1 = ep.pop_start[X + 1] >> 1;
        for (int Y = X; Y < P; ++Y, ++blk) {
            if (blk % (int)gridDim.y != (int)blockIdx.y) continue;      // few windows: the blocks of a window are dealt over gridDim.y CTAs
            const int b0 = ep.pop_start[Y] >> 1, b1 = ep.pop_start[Y + 1] >> 1;
            double s = 0.0;
            int c = 0;
            // the block's sample pairs as ONE index range over the 128 threads (full lanes, consecutive lanes on consecutive
            // b): an off-diagonal block is the na x nb rectangle; a diagonal block of n samples folds its triangle (b >= a)
            // into ceil(n / 2) rows of n + 1: row r = [row r of the triangle | row n - 1 - r]
            const int n = a1 - a0;
            const bool diag = (X == Y);
            const uint32_t width = diag ? (uint32_t)(n + 1) : (uint32_t)(b1 - b0);
            const uint32_t units = diag ? (uint32_t)((n + 1) / 2) * width : (uint32_t)n * width;
            const uint32_t magic = width > 1 ? (uint32_t)(((1ull << 32) + width - 1) / width) : 0u;
#pragma unroll 2
            for (uint32_t idx = threadIdx.x; idx < units; idx += 128) {
                uint32_t r = width > 1 ? __umulhi(idx, magic) : idx;
                int k = (int)(idx - r * width);
                if (k < 0) {                   // the rounded-up reciprocal overshoots only beyond idx * width >= 2^32
                    r -= 1;
                    k += (int)width;
                }
                int a = a0 + (int)r, b = b0 + k;
                bool use = true;
                if (diag) {
                    if (k < n - (int)r) b = a + k;
                    else {
                        const int a2 = n - 1 - (int)r;
                        use = (a2 != (int)r);          // odd n: the middle row is its own partner
                        a = a0 + a2;
                        b = a + (k - (n - (int)r));
                    }
                }
                const int nab = N[(size_t)a * ep.Hm + b];
                const int2 u = *reinterpret_cast<const int2*>(D + (size_t)(2 * a) * ep.Hk + 2 * b);
                const int2 v = *reinterpret_cast<const int2*>(D + (size_t)(2 * a + 1) * ep.Hk + 2 * b);
                const bool ok = use && nab != 0 && !(ep.min_sites > 0 && nab < ep.min_sites);      // else: nan entries
                // a == b: only the sample's own two haplotypes (2a, 2a + 1); the other three words are not pair entries
                const int num = (a == b) ? u.y : (u.x + u.y + v.x + v.y);
                const double q = (double)num / (double)(ok ? nab : 1);
                if (ok) {
                    s += q;
                    c += (a == b) ? 1 : 4;
                }
            }
#pragma unroll
            for (int d = 16; d >= 1; d >>= 1) {
                s += __shfl_xor_sync(0xffffffffu, s, d);
                c += __shfl_xor_sync(0xffffffffu, c, d);
            }
            if (lane == 0) {
                sh_s[blk * 4 + warp] = s;
                sh_c[blk * 4 + warp] = c;
            }
        }
    }
    __syncthreads();
    for (int b = threadIdx.x; b < nblk; b += 128) {
        if (b % (int)gridDim.y != (int)blockIdx.y) continue;
        ep.blk_s[(size_t)wb * nblk + b] = ((sh_s[b * 4] + sh_s[b * 4 + 1]) + sh_s[b * 4 + 2]) + sh_s[b * 4 + 3];
        ep.blk_c[(size_t)wb * nblk + b] = sh_c[b * 4] + sh_c[b * 4 + 1] + sh_c[b * 4 + 2] + sh_c[b * 4 + 3];
    }
}

// Stage 2: block sums -> pi / dxy / Fst of one window per thread (nanmean_min fractions, genomics.py:976-993).
__global__ void __launch_bounds__(128) k2_popgen_epi_final(const __grid_constant__ PopEpiParams ep, int nb) {
    const int wb = blockIdx.x * 128 + threadIdx.x;
    if (wb >= nb) return;
    const int P = ep.P;
    const int nblk = P * (P + 1) / 2;
    const double* blk_s = ep.blk_s + (size_t)wb * nblk;
    const long long* blk_c = ep.blk_c + (size_t)wb * nblk;
    const int npairs = P * (P - 1) / 2;
    double* pi_o = reinterpret_cast<double*>(ep.rec + (size_t)ep.win_idx[wb] * ep.RC + 3);
    double* dxy_o = pi_o + P;
    double* fst_o = dxy_o + npairs;
    auto bidx = [&](int X, int Y) { return X * P - X * (X - 1) / 2 + (Y - X); };
    for (int X = 0; X < P; ++X) {
        const double Nx = ep.pop_start[X + 1] - ep.pop_start[X];
        const int b = bidx(X, X);
        pi_o[X] = nanmean_min_dev(2.0 * blk_s[b], 2.0 * (double)blk_c[b], Nx * Nx, ep.min_data);
    }
    int k = 0;
    for (int X = 0; X < P; ++X)
        for (int Y = X + 1; Y < P; ++Y, ++k) {
            const double Nx = ep.pop_start[X + 1] - ep.pop_start[X], Ny = ep.pop_start[Y + 1] - ep.pop_start[Y];
            const int bxx = bidx(X, X), byy = bidx(Y, Y), bxy = bidx(X, Y);
            const double dxy = nanmean_min_dev(blk_s[bxy], (double)blk_c[bxy], Nx * Ny, ep.min_data);
            const double st = blk_s[bxx] + blk_s[byy] + blk_s[bxy];
            const double ct = (double)(blk_c[bxx] + blk_c[byy] + blk_c[bxy]);
            const double pi_t = nanmean_min_dev(2.0 * st, 2.0 * ct, (Nx + Ny) * (Nx + Ny), ep.min_data);
            const double w = 1.0 * Nx / (Nx + Ny);
            const double pi_s = w * pi_o[X] + (1 - w) * pi_o[Y];
            dxy_o[k] = dxy;
            fst_o[k] = 1 - pi_s / pi_t;
        }
}

struct IndEpiParams {
    const int32_t* diff;
    const int32_t* n;
    const int32_t* mid;
    int Hm;
    int Hk, n_ind;
    const int32_t* ind_start;   // [n_ind+1]
    int include_same;
    int min_sites;              // > 0: entries with n_ij < min_sites are nan (an earlier groupDistStats masked the
                                // cached matrix in place, genomics.py:959-961)
    double* out;                // [nb x n_ind x n_ind]
};

__global__ void __launch_bounds__(256) k2_ind_epi(const __grid_constant__ IndEpiParams ep) {
    const int wb = blockIdx.y;
    const size_t HH = (size_t)ep.Hk * ep.Hk;
    const int32_t* D = ep.diff + (size_t)wb * HH;
    const int32_t* N = ep.n + (size_t)wb * ep.Hm * ep.Hm;
    const int64_t total = (int64_t)ep.n_ind * ep.n_ind;
    double* o = ep.out + (size_t)wb * total;
    // a warp walks one output row (individual a), lanes along b: no integer division per element, coalesced stores
    const int lane = threadIdx.x & 31;
    for (int a = blockIdx.x * 8 + (threadIdx.x >> 5); a < ep.n_ind; a += gridDim.x * 8) {
        const int i0 = ep.ind_start[a], i1 = ep.ind_start[a + 1];
        for (int b = lane; b < ep.n_ind; b += 32) {
            const int j0 = ep.ind_start[b], j1 = ep.ind_start[b + 1];
            double s = 0.0;
            int c = 0;
            for (int i = i0; i < i1; ++i)
                for (int j = j0; j < j1; ++j) {
                    double d;
                    if (i == j) {
                        if (!ep.include_same || ep.min_sites > 0) continue;   // diagonal = nan (genomics.py:940; 937-938 masks it too)
                        d = 0.0;                                 // distMatrix leaves 0 on the diagonal (908)
                    } else {
                        const int nij = N[upper_idx(ep.mid[i], ep.mid[j], ep.Hm)];
                        if (nij == 0) continue;                  // np.mean of an empty array = nan
                        if (ep.min_sites > 0 && nij < ep.min_sites) continue;
                        d = (double)D[upper_idx(i, j, ep.Hk)] / (double)nij;
                    }
                    s += d;
                    c += 1;
                }
            o[(size_t)a * ep.n_ind + b] = c ? s / (double)c : nan_d();
        }
    }
}

// ---- sampleHet (genomics.py:918-929): distance between the two haplotypes of each individual ------------
struct HetParams {
    const uint32_t* planes;     // [3][Hk][NWp], rows sorted by individual
    int Hk;
    int64_t NWp;
    int64_t site_base;
    const int64_t* win_lo;      // [nb]
    const int64_t* win_hi;
    const int32_t* ind_start;   // [n_ind+1]
    int n_ind;
    int min_sites;              // in-place mask of an earlier groupDistStats (0 = none)
    double* out;                // [nb x n_ind]
};

__global__ void __launch_bounds__(128) k2_het(const __grid_constant__ HetParams hp) {
    __shared__ int sh_d[4], sh_n[4];
    const int a = blockIdx.x, wb = blockIdx.y;
    const int r0 = hp.ind_start[a], r1 = hp.ind_start[a + 1];
    double* o = hp.out + (size_t)wb * hp.n_ind + a;
    if (r1 - r0 != 2) {             // len(x) == 2 is required (the reference raises IndexError for len(x) == 1)
        if (threadIdx.x == 0) *o = nan_d();
        return;
    }
    const int64_t rel_lo = hp.win_lo[wb] - hp.site_base, rel_hi = hp.win_hi[wb] - hp.site_base;
    const int64_t w_first = rel_lo >> 5, w_last = (rel_hi - 1) >> 5;
    const uint32_t mask_first = 0xffffffffu << (rel_lo & 31);
    const uint32_t mask_last = 0xffffffffu >> (31 - (int)((rel_hi - 1) & 31));
    const size_t PS = (size_t)hp.Hk * hp.NWp;
    const uint32_t* b0i = hp.planes + (size_t)r0 * hp.NWp;
    const uint32_t* b0j = b0i + hp.NWp;
    int diff = 0, n = 0;
    for (int64_t w = w_first + threadIdx.x; w <= w_last; w += 128) {
        uint32_t m = b0i[2 * PS + w] & b0j[2 * PS + w];
        if (w == w_first) m &= mask_first;
        if (w == w_last) m &= mask_last;
        n += __popc(m);
        diff += __popc(((b0i[w] ^ b0j[w]) | (b0i[PS + w] ^ b0j[PS + w])) & m);
    }
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) {
        diff += __shfl_xor_sync(0xffffffffu, diff, d);
        n += __shfl_xor_sync(0xffffffffu, n, d);
    }
    if ((threadIdx.x & 31) == 0) {
        sh_d[threadIdx.x >> 5] = diff;
        sh_n[threadIdx.x >> 5] = n;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        diff = sh_d[0] + sh_d[1] + sh_d[2] + sh_d[3];
        n = sh_n[0] + sh_n[1] + sh_n[2] + sh_n[3];
        // `len(x)==2 & np.sum(mask) >= 1` parses as len(x) == (2 & n) >= 1: bit 1 of n must be set (924, 927)
        double v = nan_d();
        if ((n & 2) == 2 && !(hp.min_sites > 0 && n < hp.min_sites)) v = (double)diff / (double)n;
        *o = v;
    }
}

// ---- Alignment.seqNonNan (genomics.py:1038-1040): non-missing sites of each haplotype in each window ----------
__global__ void __launch_bounds__(128) k2_seq_nonnan(const uint32_t* __restrict__ vplane, int64_t NWp, int64_t site_base,
                                                     const int64_t* __restrict__ win_lo, const int64_t* __restrict__ win_hi,
                                                     int Hk, long long* __restrict__ out) {
    __shared__ int sh[4];
    const int h = blockIdx.x, wb = blockIdx.y;
    const int64_t rel_lo = win_lo[wb] - site_base, rel_hi = win_hi[wb] - site_base;
    const int64_t w_first = rel_lo >> 5, w_last = (rel_hi - 1) >> 5;
    const uint32_t mask_first = 0xffffffffu << (rel_lo & 31);
    const uint32_t mask_last = 0xffffffffu >> (31 - (int)((rel_hi - 1) & 31));
    const uint32_t* row = vplane + (size_t)h * NWp;
    int n = 0;
    for (int64_t w = w_first + threadIdx.x; w <= w_last; w += 128) {
        uint32_t m = row[w];
        if (w == w_first) m &= mask_first;
        if (w == w_last) m &= mask_last;
        n += __popc(m);
    }
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) n += __shfl_xor_sync(0xffffffffu, n, d);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = n;
    __syncthreads();
    if (threadIdx.x == 0) out[(size_t)wb * Hk + h] = (long long)sh[0] + sh[1] + sh[2] + sh[3];
}

// ---- H12stats (genomics.py:1079-1098) + distMat_to_cluster_sizes (1239-1261) ------------------------------
struct HapEpiParams {
    const int32_t* diff;        // [nb][Hk][Hk]
    const int32_t* n;           // [nb][Hm][Hm]
    const int32_t* mid;
    int Hm, Hk, P;
    const int32_t* pop_start;   // [P+1]
    int min_sites;              // in-place mask of an earlier groupDistStats (0 = none)
    int diag_nan;               // an earlier groupDistStats / indPairDists set the diagonal to nan
    double max_dist;
    double* out;                // [nb][P][3] = H1, H12, H2
};

// One CTA per (population, window). Shared memory: match bits [N][NWD] | alive [NWD] | sizes [N].
__global__ void __launch_bounds__(256) k2_hap_epi(const __grid_constant__ HapEpiParams ep) {
    extern __shared__ __align__(16) uint8_t hsm[];
    __shared__ int sh_cnt[8], sh_row[8];
    __shared__ int s_best_cnt, s_best_row;
    const int X = blockIdx.x, wb = blockIdx.y;
    const int r0 = ep.pop_start[X], N = ep.pop_start[X + 1] - r0;
    const int NWD = (N + 31) / 32;
    uint32_t* match = reinterpret_cast<uint32_t*>(hsm);
    uint32_t* alive = match + (size_t)N * NWD;
    int* sizes = reinterpret_cast<int*>(alive + NWD);
    const int32_t* D = ep.diff + (size_t)wb * ep.Hk * ep.Hk;
    const int32_t* Nn = ep.n + (size_t)wb * ep.Hm * ep.Hm;
    const int tid = threadIdx.x;
    for (int idx = tid; idx < N * NWD; idx += 256) {
        const int i = idx / NWD, wj = idx % NWD;
        uint32_t bits = 0;
        for (int b = 0; b < 32; ++b) {
            const int j = wj * 32 + b;
            if (j >= N) break;
            bool m;
            // distMatrix leaves 0 on the diagonal; a minSites mask also removes it (pairNonNan's diagonal is 0, 1043)
            if (i == j) m = !ep.diag_nan && ep.min_sites <= 0 && (0.0 <= ep.max_dist);
            else {
                const int nij = Nn[upper_idx(ep.mid[r0 + i], ep.mid[r0 + j], ep.Hm)];
                m = nij > 0 && !(ep.min_sites > 0 && nij < ep.min_sites) &&
                    ((double)D[upper_idx(r0 + i, r0 + j, ep.Hk)] / (double)nij <= ep.max_dist);
            }
            bits |= (m ? 1u : 0u) << b;
        }
        match[idx] = bits;
    }
    for (int w = tid; w < NWD; w += 256) alive[w] = (w == NWD - 1 && (N & 31)) ? ((1u << (N & 31)) - 1u) : 0xffffffffu;
    __syncthreads();
    int ncl = 0;
    while (true) {
        // row with the most matches among the rows still alive (first one on ties: np.argmax)
        int best = -1, brow = 0x7fffffff;
        for (int i = tid; i < N; i += 256) {
            if (!((alive[i >> 5] >> (i & 31)) & 1u)) continue;
            int c = 0;
            for (int w = 0; w < NWD; ++w) c += __popc(match[(size_t)i * NWD + w] & alive[w]);
            if (c > best) {         // i increases: the first maximum wins
                best = c;
                brow = i;
            }
        }
#pragma unroll
        for (int d = 16; d >= 1; d >>= 1) {
            const int oc = __shfl_xor_sync(0xffffffffu, best, d), orow = __shfl_xor_sync(0xffffffffu, brow, d);
            if (oc > best || (oc == best && orow < brow)) {
                best = oc;
                brow = orow;
            }
        }
        if ((tid & 31) == 0) {
            sh_cnt[tid >> 5] = best;
            sh_row[tid >> 5] = brow;
        }
        __syncthreads();
        if (tid == 0) {
            int bc = -1, br = 0x7fffffff;
            for (int w = 0; w < 8; ++w)
                if (sh_cnt[w] > bc || (sh_cnt[w] == bc && sh_row[w] < br)) {
                    bc = sh_cnt[w];
                    br = sh_row[w];
                }
            s_best_cnt = bc;
            s_best_row = br;
        }
        __syncthreads();
        const int bc = s_best_cnt, br = s_best_row;
        if (bc < 0) break;                       // nothing alive
        if (bc > 1) {
            if (tid == 0) sizes[ncl] = bc;
            ++ncl;
            __syncthreads();
            for (int w = tid; w < NWD; w += 256) alive[w] &= ~match[(size_t)br * NWD + w];
            __syncthreads();
        } else {
            if (tid == 0) {
                int rest = 0;
                for (int w = 0; w < NWD; ++w) rest += __popc(alive[w]);
                for (int k = 0; k < rest; ++k) sizes[ncl + k] = 1;
                s_best_cnt = rest;
            }
            __syncthreads();
            ncl += s_best_cnt;
            break;
        }
    }
    __syncthreads();
    if (tid == 0) {
        double* o = ep.out + ((size_t)wb * ep.P + X) * 3;
        long long tot = 0;
        for (int k = 0; k < ncl; ++k) tot += sizes[k];
        double H1 = 0.0, H2 = 0.0;
        for (int k = 0; k < ncl; ++k) {
            const double f = (double)sizes[k] / (double)tot;
            H1 += f * f;
            if (k >= 1) H2 += f * f;
        }
        double H12 = H1;
        if (ncl > 1) H12 = H1 + 2 * ((double)sizes[0] / (double)tot) * ((double)sizes[1] / (double)tot);
        else H2 = 0.0;
        if (ncl == 0) H1 = H12 = H2 = nan_d();
        o[0] = H1;
        o[1] = H12;
        o[2] = H2;
    }
}

// ---- `--windType cat` (distMat.py:303-314): one window = every site; pair counts add over chunks and ranks -----
// acc [2][Hk][Hk] int64 (diff, then n expanded from the unique-mask matrix) += sum over the nb chunk matrices
__global__ void __launch_bounds__(256) k2_reduce_pairs(const int32_t* __restrict__ diff, const int32_t* __restrict__ n,
                                                       const int32_t* __restrict__ mid, int Hk, int Hm, int nb,
                                                       long long* __restrict__ acc) {
    const size_t HH = (size_t)Hk * Hk, MM = (size_t)Hm * Hm;
    for (size_t idx = (size_t)blockIdx.x * 256 + threadIdx.x; idx < HH; idx += (size_t)gridDim.x * 256) {
        const int i = (int)(idx / Hk), j = (int)(idx % Hk);
        if (j < i) continue;                                 // upper triangle only (see upper_idx)
        const size_t nidx = upper_idx(mid[i], mid[j], Hm);
        long long sd = 0, sn = 0;
        for (int b = 0; b < nb; ++b) {
            sd += diff[(size_t)b * HH + idx];
            sn += n[(size_t)b * MM + nidx];
        }
        acc[idx] += sd;
        acc[HH + idx] += sn;
    }
}

struct IndEpi64Params {
    const long long* acc;       // [2][Hk][Hk]
    int Hk, n_ind;
    const int32_t* ind_start;
    int include_same;
    double* out;                // [n_ind x n_ind]
};
__global__ void __launch_bounds__(256) k2_ind_epi64(const __grid_constant__ IndEpi64Params ep) {
    const size_t HH = (size_t)ep.Hk * ep.Hk;
    const int64_t total = (int64_t)ep.n_ind * ep.n_ind;
    for (int64_t idx = (int64_t)blockIdx.x * 256 + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * 256) {
        const int a = (int)(idx / ep.n_ind), b = (int)(idx % ep.n_ind);
        double s = 0.0;
        int c = 0;
        for (int i = ep.ind_start[a]; i < ep.ind_start[a + 1]; ++i)
            for (int j = ep.ind_start[b]; j < ep.ind_start[b + 1]; ++j) {
                double d;
                if (i == j) {
                    if (!ep.include_same) continue;
                    d = 0.0;
                } else {
                    const long long nij = ep.acc[HH + upper_idx(i, j, ep.Hk)];
                    if (nij == 0) continue;
                    d = (double)ep.acc[upper_idx(i, j, ep.Hk)] / (double)nij;
                }
                s += d;
                c += 1;
            }
        ep.out[idx] = c ? s / (double)c : nan_d();
    }
}

// ---- distPaint.py (distPaint.py:26-44, 62-83): nearest reference population of every query haplotype -------------
constexpr int PAINT_WARPS = 4;         // warps per CTA; each holds its query's member distances in shared memory
constexpr int PAINT_MAX_POPS = 32;     // one lane per population
constexpr int PAINT_MAX_M = 1024;      // member entries: 8 KB of distances per warp, 32 KB per CTA

struct PaintEpiParams {
    const int32_t* diff;        // [nb][Hk][Hk]
    const int32_t* n;           // [nb][Hm][Hm]
    const int32_t* mid;
    int Hm, Hk;
    int n_query;
    const int32_t* query_row;   // [n_query] plane row of each query
    int P, M;
    const int32_t* ref_off;     // [P + 1]
    const int32_t* ref_row;     // [M] plane row of each member entry (duplicates allowed)
    int min_sites;              // >= 1
    int mode;                   // 0 rank-sum rule, 1 delta rule
    double threshold;
    int noresult;
    int32_t* out;               // [nb][n_query]
    double* means;              // [nb][n_query][P] or nullptr
    double* pvals;              // [nb][n_query][P] or nullptr
};

__device__ __forceinline__ double nan_as_zero(double v) { return v != v ? 0.0 : v; }

// np.sum of n doubles, nans read as 0 (np.nanmean's _replace_nan): numpy's pairwise summation (pairwise_sum in
// numpy/_core/src/umath/loops_utils.h.src) — sequential below 8 values, 8 strided accumulators up to 128, else split at
// n / 2 rounded down to a multiple of 8.  DEPTH bounds the splits: 5 covers PAINT_MAX_M.
template <int DEPTH>
__device__ double np_pairwise_sum(const double* a, int n) {
    if (n < 8) {
        double res = 0.0;
        for (int i = 0; i < n; ++i) res += nan_as_zero(a[i]);
        return res;
    }
    if constexpr (DEPTH > 0) {
        if (n > 128) {
            int n2 = n / 2;
            n2 -= n2 % 8;
            return np_pairwise_sum<DEPTH - 1>(a, n2) + np_pairwise_sum<DEPTH - 1>(a + n2, n - n2);
        }
    }
    double r[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) r[k] = nan_as_zero(a[k]);
    int i = 8;
    for (; i < n - (n % 8); i += 8)
#pragma unroll
        for (int k = 0; k < 8; ++k) r[k] += nan_as_zero(a[i + k]);
    double res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]));
    for (; i < n; ++i) res += nan_as_zero(a[i]);
    return res;
}

// One warp per (query, window).  The warp gathers the query's M member distances d = diff / n (nan when n < minSites; 0 for
// the query itself) into shared memory; lane p takes population p's np.nanmean; every lane then runs np.argmin (the first
// nan, else the first minimum).  Rank-sum rule: for each other population j, scipy's ranksums(x_i, x_j, "less") from
// average-tie ranks (twice the rank is an integer: 2 #less + #equal + 1), nan when either list holds a nan; p > threshold
// gives noresult.  Delta rule: lane 0 sorts the means as CPython's list.sort does for fewer than 64 items (count_run, then
// binarysort, all with <) and gives noresult when sorted[1] - sorted[0] < threshold.
__global__ void __launch_bounds__(PAINT_WARPS * 32) k2_paint_epi(const __grid_constant__ PaintEpiParams ep) {
    extern __shared__ __align__(16) double paint_sh[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int q = blockIdx.x * PAINT_WARPS + warp;
    if (q >= ep.n_query) return;                            // warp-uniform
    const int wb = blockIdx.y;
    const int P = ep.P;
    double* x = paint_sh + (size_t)warp * ep.M;
    const int32_t* D = ep.diff + (size_t)wb * ep.Hk * ep.Hk;
    const int32_t* N = ep.n + (size_t)wb * ep.Hm * ep.Hm;
    const int i = ep.query_row[q], mi = ep.mid[i];
    for (int k = lane; k < ep.M; k += 32) {
        const int j = ep.ref_row[k];
        const int nij = N[upper_idx(mi, ep.mid[j], ep.Hm)];
        double d = nan_d();
        if (nij >= ep.min_sites) d = (i == j) ? 0.0 : (double)D[upper_idx(i, j, ep.Hk)] / (double)nij;
        x[k] = d;
    }
    __syncwarp();
    double mean = nan_d();
    bool has_nan = false;
    if (lane < P) {
        const int o0 = ep.ref_off[lane], o1 = ep.ref_off[lane + 1];
        int cnt = 0;
        for (int k = o0; k < o1; ++k) cnt += (x[k] == x[k]) ? 1 : 0;
        if (cnt) mean = np_pairwise_sum<5>(x + o0, o1 - o0) / (double)cnt;
        has_nan = cnt < o1 - o0;
    }
    const unsigned full = 0xffffffffu;
    int best = 0;
    double bv = __shfl_sync(full, mean, 0);
    for (int p = 1; p < P; ++p) {
        const double v = __shfl_sync(full, mean, p);
        if (bv == bv && (v != v || v < bv)) {
            best = p;
            bv = v;
        }
    }
    int result = best;
    double pv = nan_d();                                   // lane p: p-value of the test against population p
    if (ep.mode == 1) {
        double s[PAINT_MAX_POPS];
        for (int p = 0; p < P; ++p) s[p] = __shfl_sync(full, mean, p);
        if (lane == 0) {
            int run = 1;                                   // count_run: a strictly descending run is reversed
            if (P > 1) {
                run = 2;
                if (s[1] < s[0]) {
                    while (run < P && s[run] < s[run - 1]) ++run;
                    for (int a = 0, b = run - 1; a < b; ++a, --b) {
                        const double t = s[a];
                        s[a] = s[b];
                        s[b] = t;
                    }
                } else {
                    while (run < P && !(s[run] < s[run - 1])) ++run;
                }
            }
            for (int st = run; st < P; ++st) {             // binarysort of the rest into the run
                const double pivot = s[st];
                int l = 0, r = st;
                do {
                    const int m = l + ((r - l) >> 1);
                    if (pivot < s[m]) r = m;
                    else l = m + 1;
                } while (l < r);
                for (int k = st; k > l; --k) s[k] = s[k - 1];
                s[l] = pivot;
            }
            if (s[1] - s[0] < ep.threshold) result = ep.noresult;
        }
    } else {
        const int i0 = ep.ref_off[best], n1 = ep.ref_off[best + 1] - i0;
        const bool nan_i = __shfl_sync(full, has_nan, best);
        for (int j = 0; j < P; ++j) {
            const bool nan_j = __shfl_sync(full, has_nan, j);
            if (j == best || nan_i || nan_j) continue;     // scipy propagates nan: p = nan, and nan > threshold is false
            const int j0 = ep.ref_off[j], n2 = ep.ref_off[j + 1] - j0;
            int two_s = 0;
            for (int a = lane; a < n1; a += 32) {
                const double v = x[i0 + a];
                int less = 0, eq = 0;
                for (int b = 0; b < n1; ++b) {
                    less += (x[i0 + b] < v) ? 1 : 0;
                    eq += (x[i0 + b] == v) ? 1 : 0;
                }
                for (int b = 0; b < n2; ++b) {
                    less += (x[j0 + b] < v) ? 1 : 0;
                    eq += (x[j0 + b] == v) ? 1 : 0;
                }
                two_s += 2 * less + eq + 1;
            }
#pragma unroll
            for (int d = 16; d >= 1; d >>= 1) two_s += __shfl_xor_sync(full, two_s, d);
            // ranksums: z = (s - n1 (n1 + n2 + 1) / 2.0) / sqrt(n1 n2 (n1 + n2 + 1) / 12.0), integer products as Python ints
            const double expected = (double)((long long)n1 * (n1 + n2 + 1)) / 2.0;
            const double z = (0.5 * (double)two_s - expected) / sqrt((double)((long long)n1 * n2 * (n1 + n2 + 1)) / 12.0);
            const double p = normcdf(z);
            if (p > ep.threshold) result = ep.noresult;
            if (lane == j) pv = p;
        }
    }
    const size_t row = (size_t)wb * ep.n_query + q;
    if (lane == 0) ep.out[row] = result;
    if (lane < P) {
        if (ep.means) ep.means[row * P + lane] = mean;
        if (ep.pvals) ep.pvals[row * P + lane] = pv;
    }
}

// ------------------------------------------------------------------------------------------------
// host orchestration
//
// Scratch of one call.  Each buffer keeps what it holds until the call returns, except misc4:
//   planes   the plane set: the POPC bit-planes and their mask tables (d_mid, d_rowmap), or the tensor path's valid plane,
//            site scans and mask rows (k2t.cu)
//   planes2  the tensor path's pseudo-site map and P / Q planes
//   misc     the group starts (ind_start / pop_start); pg_k2_popgen_windows keeps the batch's window indices behind them
//   misc2    the plane builders' column tables
//   misc3    the batch's window bounds d_lo | d_hi (for_each_batch)
//   misc4    short-lived scratch within one step: the POPC row hashes and their check, the Gram kernels' tile groups
//   misc5    pg_k2_popgen_windows' block sums, pg_pairdist_cat's int64 accumulator
//   pairs    the batch's pair matrices diff | n (run_pair_batch)
//   out_d    the batch's output rows, copied back to the caller's arrays
// pg_k2_popgen_windows never touches out_d or out_i: its caller keeps the record table and the path column there (k1.cu).
// ------------------------------------------------------------------------------------------------

// The operand planes of one site span: the tensor path's (k2t.cu) or the POPC kernels' three bit-planes.  The epilogues read
// the same fields of both: Hk plane rows, Hm mask rows (n_ij is computed per mask row) and each plane row's mask row, on the
// host (mid) and on the device (d_mid).  Every pointer stays valid until the call returns.
struct PlaneSet {
    int Hk = 0;
    int Hm = 0;
    std::vector<int32_t> mid;
    const int32_t* d_mid = nullptr;
    bool tensor = false;
    K2TPlanes t;                       // the tensor path's planes
    // the POPC path's planes
    int64_t site_base = 0;
    int64_t NWp = 0;
    uint32_t* planes = nullptr;        // [3][Hk][NWp]: allele bit 0, allele bit 1, valid
    const int32_t* d_rowmap = nullptr; // [Hm] mask row -> a representative plane row
};

// The POPC bit-planes of sites [lo, hi), with the plane rows grouped by identical valid plane into mask rows.
int build_popc_planes(pg_ctx* ctx, const std::vector<int32_t>& order, int64_t lo, int64_t hi, PlaneSet& ps) {
    const int Hk = (int)order.size();
    const int64_t sb = lo & ~(int64_t)(BP_SITES - 1);
    const int64_t nblk = (hi - sb + BP_SITES - 1) / BP_SITES;
    const int64_t NWp = nblk * 8 + KW + 8;     // zero tail: chunk over-reads contribute nothing
    const size_t bytes = (size_t)3 * Hk * NWp * 4;
    PG_TRY(ctx->planes.ensure(bytes + (size_t)Hk * 8));       // the planes, then the mask tables d_mid | d_rowmap
    PG_CUDA(cudaMemsetAsync(ctx->planes.p, 0, bytes, ctx->stream));
    std::vector<int32_t> c2r(ctx->pitch, -1);
    for (int r = 0; r < Hk; ++r) c2r[order[r]] = r;
    PG_TRY(ctx->misc2.ensure((size_t)ctx->pitch * 4 + 64));
    PG_CUDA(cudaMemcpyAsync(ctx->misc2.p, c2r.data(), (size_t)ctx->pitch * 4, cudaMemcpyHostToDevice, ctx->stream));
    PG_TRY(pg_smem_limit<k2_build_planes>(ctx, BP_SMEM));
    const int colblocks = (ctx->pitch + BP_COLS - 1) / BP_COLS;
    for (int64_t y0 = 0; y0 < nblk; y0 += 65535) {
        const int64_t ny = std::min<int64_t>(65535, nblk - y0);
        PG_TRY(pg_timed(ctx, "k2_planes", [&] {
            k2_build_planes<<<dim3((unsigned)colblocks, (unsigned)ny), 256, BP_SMEM, ctx->stream>>>(
                (const uint8_t*)ctx->d_geno, ctx->pitch, ctx->S, sb + y0 * BP_SITES, (const int32_t*)ctx->misc2.p,
                (uint32_t*)ctx->planes.p + y0 * 8, Hk, NWp);
        }));
    }
    ps.Hk = Hk;
    ps.site_base = sb;
    ps.NWp = NWp;
    ps.planes = (uint32_t*)ctx->planes.p;
    int32_t* d_mid = (int32_t*)(ps.planes + bytes / 4);
    int32_t* d_rowmap = d_mid + Hk;
    // group rows by identical valid plane: hash, group on the host, verify on the device
    PG_TRY(ctx->misc4.ensure((size_t)Hk * 12 + 256));
    unsigned long long* d_hash = (unsigned long long*)ctx->misc4.p;
    int32_t* d_rep = (int32_t*)(d_hash + Hk);
    int* d_flag = (int*)(d_rep + Hk);
    const uint32_t* mplane = ps.planes + (size_t)2 * Hk * NWp;
    PG_TRY(pg_timed(ctx, "k2_mask_groups", [&] { k2_hash_rows<<<Hk, 256, 0, ctx->stream>>>(mplane, NWp, d_hash); }));
    std::vector<unsigned long long> hh(Hk);
    PG_CUDA(cudaMemcpyAsync(hh.data(), d_hash, (size_t)Hk * 8, cudaMemcpyDeviceToHost, ctx->stream));
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    std::vector<int32_t> rep(Hk), mid(Hk), rowmap;
    {
        std::vector<std::pair<unsigned long long, int>> first;   // (hash, first row) — Hk is small
        for (int r = 0; r < Hk; ++r) {
            int q = -1;
            for (size_t k = 0; k < first.size(); ++k)
                if (first[k].first == hh[r]) {
                    q = (int)k;
                    break;
                }
            if (q < 0) {
                first.push_back({hh[r], r});
                q = (int)first.size() - 1;
                rowmap.push_back(r);
            }
            mid[r] = q;
            rep[r] = first[q].second;
        }
    }
    PG_CUDA(cudaMemcpyAsync(d_rep, rep.data(), (size_t)Hk * 4, cudaMemcpyHostToDevice, ctx->stream));
    PG_CUDA(cudaMemsetAsync(d_flag, 0, 4, ctx->stream));
    PG_TRY(pg_timed(ctx, "k2_mask_groups", [&] { k2_verify_rows<<<Hk, 256, 0, ctx->stream>>>(mplane, NWp, d_rep, d_flag); }));
    int flag = 0;
    PG_CUDA(cudaMemcpyAsync(&flag, d_flag, 4, cudaMemcpyDeviceToHost, ctx->stream));
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    if (flag || getenv("PG_K2_NO_MASK_SHARING")) {     // hash collision (or disabled): every row is its own group
        rowmap.resize(Hk);
        for (int r = 0; r < Hk; ++r) mid[r] = rowmap[r] = r;
    }
    ps.Hm = (int)rowmap.size();
    ps.mid = mid;
    PG_CUDA(cudaMemcpyAsync(d_mid, mid.data(), (size_t)Hk * 4, cudaMemcpyHostToDevice, ctx->stream));
    PG_CUDA(cudaMemcpyAsync(d_rowmap, rowmap.data(), (size_t)ps.Hm * 4, cudaMemcpyHostToDevice, ctx->stream));
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    ps.d_mid = d_mid;
    ps.d_rowmap = d_rowmap;
    return PG_OK;
}

// Planes for sites [lo, hi) of the haplotype columns listed in `order` (plane row r = column order[r]): the tensor path's
// unless PG_K2_POPC is set or its plane builders cannot take the width.
int build_planes(pg_ctx* ctx, const std::vector<int32_t>& order, int64_t lo, int64_t hi, PlaneSet& ps) {
    const int Hk = (int)order.size();
    PG_CHECK(Hk >= 1, "pairwise path: no haplotypes selected");
    ps.tensor = pg_k2_use_tensor() && pg_k2t_fits(ctx->pitch, Hk);
    if (!ps.tensor) return build_popc_planes(ctx, order, lo, hi, ps);
    PG_TRY(pg_k2t_build(ctx, order, lo, hi, ps.t));
    ps.Hk = Hk;
    ps.Hm = ps.t.Hm;                           // mask rows: one per row, or one per sample (see K2TPlanes)
    ps.mid.resize(Hk);
    for (int r = 0; r < Hk; ++r) ps.mid[r] = (ps.t.Hm == Hk) ? r : r / 2;
    ps.d_mid = ps.t.d_mid;
    return PG_OK;
}

// Pair matrices of a batch of nb windows (site bounds on the device) -> ctx->pairs: diff [nb][Hk^2] | n [nb][Hm^2]
int run_pair_batch(pg_ctx* ctx, const PlaneSet& ps, const int64_t* d_lo, const int64_t* d_hi, int nb, int32_t** d_diff,
                   int32_t** d_n) {
    const size_t HH = (size_t)ps.Hk * ps.Hk, MM = (size_t)ps.Hm * ps.Hm;
    PG_TRY(ctx->pairs.ensure((size_t)nb * (HH + MM) * 4 + 64));
    *d_diff = (int32_t*)ctx->pairs.p;
    *d_n = *d_diff + (size_t)nb * HH;
    if (ps.tensor) return pg_k2t_pairs(ctx, ps.t, d_lo, d_hi, nb, *d_diff, *d_n);
    PG_TRY(pg_smem_limit<k2_pair<PAIR_DIFF>>(ctx, PairGeom<PAIR_DIFF>::SMEM));
    PG_TRY(pg_smem_limit<k2_pair<PAIR_N>>(ctx, PairGeom<PAIR_N>::SMEM));
    PairParams pp;
    pp.planes = ps.planes;
    pp.Hk = ps.Hk;
    pp.NWp = ps.NWp;
    pp.site_base = ps.site_base;
    pp.win_lo = d_lo;
    pp.win_hi = d_hi;
    // diff over all haplotype rows
    pp.n_rows = ps.Hk;
    pp.row_map = nullptr;
    pp.ntile = (ps.Hk + TS - 1) / TS;
    pp.out = *d_diff;
    PG_TRY(pg_timed(ctx, "k2_pair_diff", [&] {
        k2_pair<PAIR_DIFF><<<dim3((unsigned)(pp.ntile * (pp.ntile + 1) / 2), (unsigned)nb), 256, PairGeom<PAIR_DIFF>::SMEM,
                             ctx->stream>>>(pp);
    }));
    // n over the unique valid-masks
    pp.n_rows = ps.Hm;
    pp.row_map = ps.d_rowmap;
    pp.ntile = (ps.Hm + TS - 1) / TS;
    pp.out = *d_n;
    return pg_timed(ctx, "k2_pair_n", [&] {
        k2_pair<PAIR_N><<<dim3((unsigned)(pp.ntile * (pp.ntile + 1) / 2), (unsigned)nb), 256, PairGeom<PAIR_N>::SMEM,
                          ctx->stream>>>(pp);
    });
}

// Alignment.sampleHet() rows of a batch of nb windows: [nb][n_ind] doubles
int run_het(pg_ctx* ctx, const PlaneSet& ps, const int64_t* d_lo, const int64_t* d_hi, int nb, const int32_t* d_ind_start,
            int n_ind, int min_sites, double* d_out) {
    if (ps.tensor) return pg_k2t_het(ctx, ps.t, d_lo, d_hi, nb, d_ind_start, n_ind, min_sites, d_out);
    HetParams hp;
    hp.planes = ps.planes;
    hp.Hk = ps.Hk;
    hp.NWp = ps.NWp;
    hp.site_base = ps.site_base;
    hp.win_lo = d_lo;
    hp.win_hi = d_hi;
    hp.ind_start = d_ind_start;
    hp.n_ind = n_ind;
    hp.min_sites = min_sites;
    hp.out = d_out;
    return pg_timed(ctx, "k2_het", [&] { k2_het<<<dim3((unsigned)n_ind, (unsigned)nb), 128, 0, ctx->stream>>>(hp); });
}

// non-missing sites of every plane row in a batch of nb windows: [nb][Hk] int64
int run_seq_nonnan(pg_ctx* ctx, const PlaneSet& ps, const int64_t* d_lo, const int64_t* d_hi, int nb, long long* d_out) {
    if (ps.tensor) return pg_k2t_seq_nonnan(ctx, ps.t, d_lo, d_hi, nb, d_out);
    return pg_timed(ctx, "k2_seq_nonnan", [&] {
        k2_seq_nonnan<<<dim3((unsigned)ps.Hk, (unsigned)nb), 128, 0, ctx->stream>>>(ps.planes + (size_t)2 * ps.Hk * ps.NWp,
                                                                                   ps.NWp, ps.site_base, d_lo, d_hi, ps.Hk,
                                                                                   d_out);
    });
}

// Plane rows ordered by group: the haplotypes of group 0, then of group 1, ... (each in upload order); a haplotype of group
// -1 gets no row.  start[g] = first row of group g, start[G] = rows.  `what` names a caller's map in the range check's
// message; nullptr for ctx->hap_pop, which pg_set_pops checks.
int group_rows(const pg_ctx* ctx, const int32_t* group, int G, const char* what, std::vector<int32_t>& order,
               std::vector<int32_t>& start) {
    for (int h = 0; what && h < ctx->H; ++h)
        PG_CHECK(group[h] >= -1 && group[h] < G, "%s[%d]=%d out of range", what, h, group[h]);
    start.assign(G + 1, 0);
    for (int g = 0; g < G; ++g) {
        start[g] = (int32_t)order.size();
        for (int h = 0; h < ctx->H; ++h)
            if (group[h] == g) order.push_back(h);
    }
    start[G] = (int32_t)order.size();
    return PG_OK;
}

// every haplotype, in upload order
std::vector<int32_t> all_rows(int H) {
    std::vector<int32_t> order(H);
    for (int h = 0; h < H; ++h) order[h] = h;
    return order;
}

// non-empty windows and the site span they cover
void nonempty_windows(const pg_ctx* ctx, std::vector<int64_t>& idx, int64_t& lo, int64_t& hi) {
    lo = ctx->S;
    hi = 0;
    for (int64_t w = 0; w < ctx->W; ++w)
        if (ctx->win_hi[w] > ctx->win_lo[w]) {
            idx.push_back(w);
            lo = std::min(lo, ctx->win_lo[w]);
            hi = std::max(hi, ctx->win_hi[w]);
        }
}

// Windows per batch of a caller of the pair matrices: a batch's diff and n (8 bytes per plane-row pair) and `extra` bytes
// per window fit PG_PAIR_SCRATCH_MB (default 3 GiB), and a batch is one grid dimension (at most 65535).
size_t pair_batch_size(int Hk, size_t extra) {
    const char* e = getenv("PG_PAIR_SCRATCH_MB");
    size_t mb = e ? (size_t)atoll(e) : 3072;
    if (mb < 1) mb = 1;
    return std::max<size_t>(1, std::min<size_t>((mb << 20) / ((size_t)Hk * Hk * 8 + extra), 65535));
}

// Cuts the windows `wins` (window w spans sites [lo[w], hi[w])) into batches of at most per_batch, uploads each batch's bounds
// and runs body(b0, nb, d_lo, d_hi) on windows wins[b0 .. b0 + nb).
template <class Body>
int for_each_batch(pg_ctx* ctx, const std::vector<int64_t>& wins, const int64_t* lo, const int64_t* hi, size_t per_batch,
                   Body&& body) {
    for (size_t b0 = 0; b0 < wins.size(); b0 += per_batch) {
        const size_t nb = std::min(per_batch, wins.size() - b0);
        std::vector<int64_t> blo(nb), bhi(nb);
        for (size_t k = 0; k < nb; ++k) {
            blo[k] = lo[wins[b0 + k]];
            bhi[k] = hi[wins[b0 + k]];
        }
        PG_TRY(ctx->misc3.ensure(nb * 16 + 64));
        int64_t* d_lo = (int64_t*)ctx->misc3.p;
        int64_t* d_hi = d_lo + nb;
        PG_CUDA(cudaMemcpyAsync(d_lo, blo.data(), nb * 8, cudaMemcpyHostToDevice, ctx->stream));
        PG_CUDA(cudaMemcpyAsync(d_hi, bhi.data(), nb * 8, cudaMemcpyHostToDevice, ctx->stream));
        PG_TRY(body(b0, nb, (const int64_t*)d_lo, (const int64_t*)d_hi));
    }
    return PG_OK;
}

// Copies batch rows 0 .. nb (row_bytes each) of a device buffer to the rows of windows wins[b0 .. b0 + nb) of a host array,
// one copy per run of consecutive windows, then synchronises.  staged: through pg_d2h_staged, for large rows into pageable
// memory.
int copy_rows_back(pg_ctx* ctx, const std::vector<int64_t>& wins, size_t b0, size_t nb, const void* d_src, void* h_dst,
                   size_t row_bytes, bool staged = false) {
    size_t k = 0;
    while (k < nb) {
        size_t e = k + 1;
        while (e < nb && wins[b0 + e] == wins[b0 + e - 1] + 1) ++e;
        uint8_t* dst = (uint8_t*)h_dst + (size_t)wins[b0 + k] * row_bytes;
        const uint8_t* src = (const uint8_t*)d_src + k * row_bytes;
        if (staged) PG_TRY(pg_d2h_staged(ctx, dst, src, (e - k) * row_bytes));
        else PG_CUDA(cudaMemcpyAsync(dst, src, (e - k) * row_bytes, cudaMemcpyDeviceToHost, ctx->stream));
        k = e;
    }
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    return PG_OK;
}

}  // namespace

// pi / dxy / Fst for the listed windows through the pairwise path, written straight into the device
// record table at the windows' own rows.  The bounds come from the caller: the pipelined gather resolves a batch whose
// windows the ctx may no longer hold.
int pg_k2_popgen_windows(pg_ctx* ctx, const std::vector<int64_t>& wins, const int64_t* win_lo, const int64_t* win_hi,
                         int32_t min_sites, double min_data, void* d_rec, int RC) {
    const int P = ctx->P;
    std::vector<int32_t> order, pop_start;
    PG_TRY(group_rows(ctx, ctx->hap_pop.data(), P, nullptr, order, pop_start));
    // empty windows cannot be "ragged"; every window here has at least one site
    int64_t lo = ctx->S, hi = 0;
    for (int64_t w : wins) {
        lo = std::min(lo, win_lo[w]);
        hi = std::max(hi, win_hi[w]);
    }
    PlaneSet ps;
    PG_TRY(build_planes(ctx, order, lo, hi, ps));
    const size_t per_batch = pair_batch_size(ps.Hk, 0);
    PG_TRY(ctx->misc.ensure((size_t)(P + 1) * 4 + per_batch * 8 + 128));
    PG_CUDA(cudaMemcpyAsync(ctx->misc.p, pop_start.data(), (size_t)(P + 1) * 4, cudaMemcpyHostToDevice, ctx->stream));
    int64_t* d_widx = reinterpret_cast<int64_t*>((uint8_t*)ctx->misc.p + (((size_t)(P + 1) * 4 + 63) / 64) * 64);
    return for_each_batch(ctx, wins, win_lo, win_hi, per_batch, [&](size_t b0, size_t nb, const int64_t* d_lo, const int64_t* d_hi) {
        int32_t *d_diff = nullptr, *d_n = nullptr;
        PG_TRY(run_pair_batch(ctx, ps, d_lo, d_hi, (int)nb, &d_diff, &d_n));
        PG_CUDA(cudaMemcpyAsync(d_widx, wins.data() + b0, nb * 8, cudaMemcpyHostToDevice, ctx->stream));
        PopEpiParams ep;
        ep.diff = d_diff;
        ep.n = d_n;
        ep.mid = ps.d_mid;
        ep.Hm = ps.Hm;
        ep.Hk = ps.Hk;
        ep.P = P;
        ep.pop_start = (const int32_t*)ctx->misc.p;
        ep.min_sites = min_sites;
        ep.min_data = min_data;
        ep.rec = (unsigned long long*)d_rec;
        ep.RC = RC;
        ep.win_idx = d_widx;
        const int nblk = P * (P + 1) / 2;
        PG_TRY(ctx->misc5.ensure(nb * (size_t)nblk * 16 + 64));
        ep.blk_s = (double*)ctx->misc5.p;
        ep.blk_c = (long long*)(ep.blk_s + nb * (size_t)nblk);
        // sample-pair walk: mask ids are r >> 1 (the tensor path's per-sample n rows) and populations start on even rows
        bool by_pairs = ps.tensor && ps.Hm * 2 == ps.Hk && (size_t)nblk * 64 <= 48 * 1024;
        for (int X = 0; X <= P; ++X) by_pairs = by_pairs && (pop_start[X] % 2 == 0);
        // one CTA per window when there are many windows, else the blocks of a window over several CTAs (~8 CTAs per SM)
        const unsigned nsplit = (unsigned)std::max<int64_t>(1, std::min<int64_t>(nblk, (8 * (int64_t)ctx->sm_count + (int64_t)nb - 1) / (int64_t)nb));
        // the timing label names the stage-1 kernel, so that a caller can tell which epilogue ran
        PG_TRY(pg_timed(ctx, by_pairs ? "k2_popgen_epi_pairs" : "k2_popgen_epi_blocks", [&] {
            if (by_pairs) k2_popgen_epi_pairs<<<dim3((unsigned)nb, nsplit), 128, (size_t)nblk * 64, ctx->stream>>>(ep);
            else k2_popgen_epi_blocks<<<dim3((unsigned)nblk, (unsigned)nb), 256, 0, ctx->stream>>>(ep);
            k2_popgen_epi_final<<<(unsigned)((nb + 127) / 128), 128, 0, ctx->stream>>>(ep, (int)nb);
        }));
        ctx->launches += 1;
        PG_CUDA(cudaStreamSynchronize(ctx->stream));     // host vectors and scratch are reused by the next batch
        return PG_OK;
    });
}

extern "C" int pg_pairdist(pg_ctx* ctx, int32_t n_ind, const int32_t* hap_ind, int32_t include_same_with_same,
                           int32_t min_sites, double* dist, int64_t* n_sites, int64_t* pos_sum) {
    PG_CHECK(ctx && hap_ind && dist, "pg_pairdist: null argument");
    PG_CHECK(n_ind >= 1, "pg_pairdist: n_ind must be >= 1");
    PG_CHECK(ctx->H > 0, "pg_pairdist: upload genotypes first");
    PG_CUDA(cudaSetDevice(ctx->device));
    pg_timings_reset(ctx);
    const int64_t W = ctx->W;
    if (W == 0) return PG_OK;
    std::vector<int32_t> order, ind_start;
    PG_TRY(group_rows(ctx, hap_ind, n_ind, "pg_pairdist: hap_ind", order, ind_start));
    const size_t nn = (size_t)n_ind * n_ind;
    std::vector<int64_t> wins;
    int64_t lo, hi;
    nonempty_windows(ctx, wins, lo, hi);
    for (int64_t w = 0; w < W; ++w) {
        if (n_sites) n_sites[w] = ctx->win_hi[w] - ctx->win_lo[w];
        if (ctx->win_hi[w] <= ctx->win_lo[w])
            for (size_t k = 0; k < nn; ++k) dist[(size_t)w * nn + k] = NAN;
    }
    // sites / position sums on the host side of the library: prefix sums of the positions are cheap, but the
    // positions live on the device — read them back once (4 bytes per site).
    if (pos_sum) {
        std::vector<int32_t> hp((size_t)std::max<int64_t>(ctx->S, 1));
        if (ctx->S > 0)
            PG_CUDA(cudaMemcpy(hp.data(), ctx->d_pos, (size_t)ctx->S * 4, cudaMemcpyDeviceToHost));
        std::vector<int64_t> pre((size_t)ctx->S + 1, 0);
        for (int64_t s = 0; s < ctx->S; ++s) pre[s + 1] = pre[s] + hp[s];
        for (int64_t w = 0; w < W; ++w) pos_sum[w] = pre[ctx->win_hi[w]] - pre[ctx->win_lo[w]];
    }
    if (wins.empty()) return PG_OK;
    PlaneSet ps;
    PG_TRY(build_planes(ctx, order, lo, hi, ps));
    const size_t per_batch = pair_batch_size(ps.Hk, nn * 8);
    PG_TRY(ctx->misc.ensure((size_t)(n_ind + 1) * 4 + 64));
    PG_CUDA(cudaMemcpyAsync(ctx->misc.p, ind_start.data(), (size_t)(n_ind + 1) * 4, cudaMemcpyHostToDevice, ctx->stream));
    PG_TRY(ctx->out_d.ensure(per_batch * nn * 8 + 64));
    return for_each_batch(ctx, wins, ctx->win_lo.data(), ctx->win_hi.data(), per_batch,
                          [&](size_t b0, size_t nb, const int64_t* d_lo, const int64_t* d_hi) {
        int32_t *d_diff = nullptr, *d_n = nullptr;
        PG_TRY(run_pair_batch(ctx, ps, d_lo, d_hi, (int)nb, &d_diff, &d_n));
        IndEpiParams ep;
        ep.diff = d_diff;
        ep.n = d_n;
        ep.mid = ps.d_mid;
        ep.Hm = ps.Hm;
        ep.Hk = ps.Hk;
        ep.n_ind = n_ind;
        ep.ind_start = (const int32_t*)ctx->misc.p;
        ep.include_same = include_same_with_same ? 1 : 0;
        ep.min_sites = min_sites;
        ep.out = (double*)ctx->out_d.p;
        PG_TRY(pg_timed(ctx, "k2_ind_epi", [&] {
            k2_ind_epi<<<dim3((unsigned)std::min<int>((n_ind + 7) / 8, 64), (unsigned)nb), 256, 0, ctx->stream>>>(ep);
        }));
        // n_ind^2 doubles per window, possibly into pageable memory: staged copies
        return copy_rows_back(ctx, wins, b0, nb, ctx->out_d.p, dist, nn * 8, true);
    });
}

extern "C" int pg_distpaint(pg_ctx* ctx, int32_t n_query, const int32_t* query_hap, int32_t P, const int32_t* ref_off,
                            const int32_t* ref_hap, int32_t min_sites, int32_t mode, double threshold, int32_t noresult,
                            int32_t* out, double* means, double* pvals) {
    PG_CHECK(ctx && query_hap && ref_off && ref_hap && out, "pg_distpaint: null argument");
    PG_CHECK(ctx->H > 0, "pg_distpaint: upload genotypes first");
    PG_CHECK(n_query >= 1, "pg_distpaint: n_query must be >= 1");
    PG_CHECK(P >= 1 && P <= PAINT_MAX_POPS, "pg_distpaint: P=%d populations; the epilogue takes 1 to %d (one lane each)", P,
             PAINT_MAX_POPS);
    PG_CHECK(mode == 0 || mode == 1, "pg_distpaint: mode %d is neither 0 (rank-sum rule) nor 1 (delta rule)", mode);
    PG_CHECK(mode == 0 || P >= 2, "pg_distpaint: the delta rule compares the two lowest means and needs two populations");
    PG_CHECK(min_sites >= 1, "pg_distpaint: min_sites must be >= 1");
    PG_CHECK(ref_off[0] == 0, "pg_distpaint: ref_off[0] must be 0");
    for (int p = 0; p < P; ++p)
        PG_CHECK(ref_off[p + 1] > ref_off[p], "pg_distpaint: reference population %d has no member entries", p);
    const int M = ref_off[P];
    PG_CHECK(M <= PAINT_MAX_M, "pg_distpaint: %d member entries; at most %d fit the epilogue's shared memory (8 bytes each "
             "per warp)", M, PAINT_MAX_M);
    const int H = ctx->H;
    for (int k = 0; k < M; ++k)
        PG_CHECK(ref_hap[k] >= 0 && ref_hap[k] < H, "pg_distpaint: ref_hap[%d]=%d out of range", k, ref_hap[k]);
    for (int k = 0; k < n_query; ++k)
        PG_CHECK(query_hap[k] >= 0 && query_hap[k] < H, "pg_distpaint: query_hap[%d]=%d out of range", k, query_hap[k]);
    PG_CUDA(cudaSetDevice(ctx->device));
    pg_timings_reset(ctx);
    if (ctx->W == 0) return PG_OK;
    std::vector<int64_t> wins;
    int64_t lo, hi;
    nonempty_windows(ctx, wins, lo, hi);
    if (wins.empty()) return PG_OK;
    PlaneSet ps;
    PG_TRY(build_planes(ctx, all_rows(H), lo, hi, ps));     // plane row = haplotype
    // query rows | population offsets | member rows
    PG_TRY(ctx->misc.ensure((size_t)(n_query + P + 1 + M) * 4 + 64));
    int32_t* d_query = (int32_t*)ctx->misc.p;
    int32_t* d_off = d_query + n_query;
    int32_t* d_ref = d_off + P + 1;
    PG_CUDA(cudaMemcpyAsync(d_query, query_hap, (size_t)n_query * 4, cudaMemcpyHostToDevice, ctx->stream));
    PG_CUDA(cudaMemcpyAsync(d_off, ref_off, (size_t)(P + 1) * 4, cudaMemcpyHostToDevice, ctx->stream));
    PG_CUDA(cudaMemcpyAsync(d_ref, ref_hap, (size_t)M * 4, cudaMemcpyHostToDevice, ctx->stream));
    const size_t qp = (size_t)n_query * P;
    const int n_dbl = (means ? 1 : 0) + (pvals ? 1 : 0);
    const size_t per_batch = pair_batch_size(ps.Hk, (size_t)n_query * 4 + qp * 8 * n_dbl);
    PG_TRY(ctx->out_i.ensure(per_batch * n_query * 4 + 64));
    PG_TRY(ctx->out_d.ensure(per_batch * qp * 8 * std::max(n_dbl, 1) + 64));
    const size_t smem = (size_t)PAINT_WARPS * M * 8;
    return for_each_batch(ctx, wins, ctx->win_lo.data(), ctx->win_hi.data(), per_batch,
                          [&](size_t b0, size_t nb, const int64_t* d_lo, const int64_t* d_hi) {
        int32_t *d_diff = nullptr, *d_n = nullptr;
        PG_TRY(run_pair_batch(ctx, ps, d_lo, d_hi, (int)nb, &d_diff, &d_n));
        PaintEpiParams ep;
        ep.diff = d_diff;
        ep.n = d_n;
        ep.mid = ps.d_mid;
        ep.Hm = ps.Hm;
        ep.Hk = ps.Hk;
        ep.n_query = n_query;
        ep.query_row = d_query;
        ep.P = P;
        ep.M = M;
        ep.ref_off = d_off;
        ep.ref_row = d_ref;
        ep.min_sites = min_sites;
        ep.mode = mode;
        ep.threshold = threshold;
        ep.noresult = noresult;
        ep.out = (int32_t*)ctx->out_i.p;
        ep.means = means ? (double*)ctx->out_d.p : nullptr;
        ep.pvals = pvals ? (double*)ctx->out_d.p + (means ? nb * qp : 0) : nullptr;
        PG_TRY(pg_timed(ctx, "k2_paint_epi", [&] {
            k2_paint_epi<<<dim3((unsigned)((n_query + PAINT_WARPS - 1) / PAINT_WARPS), (unsigned)nb), PAINT_WARPS * 32, smem,
                           ctx->stream>>>(ep);
        }));
        if (means) PG_TRY(copy_rows_back(ctx, wins, b0, nb, ep.means, means, qp * 8));
        if (pvals) PG_TRY(copy_rows_back(ctx, wins, b0, nb, ep.pvals, pvals, qp * 8));
        return copy_rows_back(ctx, wins, b0, nb, ep.out, out, (size_t)n_query * 4);
    });
}

extern "C" int pg_pair_counts(pg_ctx* ctx, int64_t window, int32_t* diff, int32_t* n) {
    PG_CHECK(ctx && diff && n, "pg_pair_counts: null argument");
    PG_CHECK(window >= 0 && window < ctx->W, "pg_pair_counts: window %lld out of range", (long long)window);
    PG_CUDA(cudaSetDevice(ctx->device));
    pg_timings_reset(ctx);
    const int H = ctx->H;
    const size_t HH = (size_t)H * H;
    const int64_t lo = ctx->win_lo[window], hi = ctx->win_hi[window];
    if (hi <= lo) {
        memset(diff, 0, HH * 4);
        memset(n, 0, HH * 4);
        return PG_OK;
    }
    PlaneSet ps;
    PG_TRY(build_planes(ctx, all_rows(H), lo, hi, ps));
    int32_t *d_diff = nullptr, *d_n = nullptr;
    PG_TRY(for_each_batch(ctx, std::vector<int64_t>(1, window), ctx->win_lo.data(), ctx->win_hi.data(), 1,
                          [&](size_t, size_t, const int64_t* d_lo, const int64_t* d_hi) {
        return run_pair_batch(ctx, ps, d_lo, d_hi, 1, &d_diff, &d_n);
    }));
    std::vector<int32_t> nu((size_t)ps.Hm * ps.Hm);
    PG_CUDA(cudaMemcpyAsync(diff, d_diff, HH * 4, cudaMemcpyDeviceToHost, ctx->stream));
    PG_CUDA(cudaMemcpyAsync(nu.data(), d_n, nu.size() * 4, cudaMemcpyDeviceToHost, ctx->stream));
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    for (int i = 0; i < H; ++i)
        for (int j = 0; j < H; ++j) {
            const int a = std::min(ps.mid[i], ps.mid[j]), b = std::max(ps.mid[i], ps.mid[j]);
            n[(size_t)i * H + j] = nu[(size_t)a * ps.Hm + b];
            if (j < i) diff[(size_t)i * H + j] = diff[(size_t)j * H + i];      // only the upper triangle is computed
        }
    return PG_OK;
}

// Alignment.sampleHet() (genomics.py:918-929) for every window: het [W x n_ind]
extern "C" int pg_ind_het(pg_ctx* ctx, int32_t n_ind, const int32_t* hap_ind, int32_t min_sites, double* het) {
    PG_CHECK(ctx && hap_ind && het, "pg_ind_het: null argument");
    PG_CHECK(n_ind >= 1, "pg_ind_het: n_ind must be >= 1");
    PG_CHECK(ctx->H > 0, "pg_ind_het: upload genotypes first");
    PG_CUDA(cudaSetDevice(ctx->device));
    pg_timings_reset(ctx);
    const int64_t W = ctx->W;
    if (W == 0) return PG_OK;
    std::vector<int32_t> order, ind_start;
    PG_TRY(group_rows(ctx, hap_ind, n_ind, "pg_ind_het: hap_ind", order, ind_start));
    for (size_t k = 0; k < (size_t)W * n_ind; ++k) het[k] = NAN;
    std::vector<int64_t> wins;
    int64_t lo, hi;
    nonempty_windows(ctx, wins, lo, hi);
    if (wins.empty() || order.empty()) return PG_OK;
    PlaneSet ps;
    PG_TRY(build_planes(ctx, order, lo, hi, ps));
    PG_TRY(ctx->misc.ensure((size_t)(n_ind + 1) * 4 + 64));
    PG_CUDA(cudaMemcpyAsync(ctx->misc.p, ind_start.data(), (size_t)(n_ind + 1) * 4, cudaMemcpyHostToDevice, ctx->stream));
    return for_each_batch(ctx, wins, ctx->win_lo.data(), ctx->win_hi.data(), 65535,
                          [&](size_t b0, size_t nb, const int64_t* d_lo, const int64_t* d_hi) {
        PG_TRY(ctx->out_d.ensure(nb * (size_t)n_ind * 8 + 64));
        PG_TRY(run_het(ctx, ps, d_lo, d_hi, (int)nb, (const int32_t*)ctx->misc.p, n_ind, min_sites, (double*)ctx->out_d.p));
        return copy_rows_back(ctx, wins, b0, nb, ctx->out_d.p, het, (size_t)n_ind * 8);
    });
}

// Alignment.H12stats(maxDist) (genomics.py:1079-1098) for every window and population of pg_set_pops:
// out [W x P x 3] = H1, H12, H2.  min_sites / diag_nan describe what earlier analyses of the same window did to the
// reference's cached distance matrix (popgenWindows.py:50-64): groupDistStats masks n_ij < minSites and the diagonal
// in place, indPairDists masks the diagonal.
extern "C" int pg_hapstats(pg_ctx* ctx, double max_dist, int32_t min_sites, int32_t diag_nan, double* out) {
    PG_CHECK(ctx && out, "pg_hapstats: null argument");
    PG_CHECK(ctx->P >= 1, "pg_hapstats: call pg_set_pops first");
    PG_CHECK(ctx->P <= PG_MAX_POPS, "pg_hapstats: P=%d > %d populations", ctx->P, PG_MAX_POPS);
    PG_CUDA(cudaSetDevice(ctx->device));
    pg_timings_reset(ctx);
    const int64_t W = ctx->W;
    const int P = ctx->P;
    if (W == 0) return PG_OK;
    std::vector<int32_t> order, pop_start;
    PG_TRY(group_rows(ctx, ctx->hap_pop.data(), P, nullptr, order, pop_start));
    int maxN = 0;
    for (int X = 0; X < P; ++X) {
        PG_CHECK(pop_start[X + 1] > pop_start[X], "pg_hapstats: population %d has no haplotypes", X);
        maxN = std::max(maxN, pop_start[X + 1] - pop_start[X]);
    }
    const size_t smem = (size_t)maxN * ((maxN + 31) / 32) * 4 + (size_t)((maxN + 31) / 32) * 4 + (size_t)maxN * 4 + 64;
    PG_CHECK(smem <= 200 * 1024, "pg_hapstats: a population of %d haplotypes is too large for the clustering kernel", maxN);
    for (size_t k = 0; k < (size_t)W * P * 3; ++k) out[k] = NAN;
    std::vector<int64_t> wins;
    int64_t lo, hi;
    nonempty_windows(ctx, wins, lo, hi);
    if (wins.empty()) return PG_OK;
    PlaneSet ps;
    PG_TRY(build_planes(ctx, order, lo, hi, ps));
    PG_TRY(ctx->misc.ensure((size_t)(P + 1) * 4 + 64));
    PG_CUDA(cudaMemcpyAsync(ctx->misc.p, pop_start.data(), (size_t)(P + 1) * 4, cudaMemcpyHostToDevice, ctx->stream));
    // the shared memory of k2_hap_epi follows the largest population: set on every call
    PG_CUDA(cudaFuncSetAttribute(k2_hap_epi, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    return for_each_batch(ctx, wins, ctx->win_lo.data(), ctx->win_hi.data(), pair_batch_size(ps.Hk, 0),
                          [&](size_t b0, size_t nb, const int64_t* d_lo, const int64_t* d_hi) {
        int32_t *d_diff = nullptr, *d_n = nullptr;
        PG_TRY(run_pair_batch(ctx, ps, d_lo, d_hi, (int)nb, &d_diff, &d_n));
        PG_TRY(ctx->out_d.ensure(nb * (size_t)P * 24 + 64));
        HapEpiParams ep;
        ep.diff = d_diff;
        ep.n = d_n;
        ep.mid = ps.d_mid;
        ep.Hm = ps.Hm;
        ep.Hk = ps.Hk;
        ep.P = P;
        ep.pop_start = (const int32_t*)ctx->misc.p;
        ep.min_sites = min_sites;
        ep.diag_nan = diag_nan ? 1 : 0;
        ep.max_dist = max_dist;
        ep.out = (double*)ctx->out_d.p;
        PG_TRY(pg_timed(ctx, "k2_hap_epi", [&] {
            k2_hap_epi<<<dim3((unsigned)P, (unsigned)nb), 256, smem, ctx->stream>>>(ep);
        }));
        return copy_rows_back(ctx, wins, b0, nb, ctx->out_d.p, out, (size_t)P * 24);
    });
}

// distMat.py --windType cat (distMat.py:303-314: parseGenoFile -> ONE window over every site): dist [n_ind x n_ind].
// The uploaded sites are this rank's shard of the window: they are cut into chunks (so that the pair kernel fills the
// GPU), the chunk matrices are summed as int64, and — when a communicator is set (pg_nccl_init) — ONE ncclAllReduce
// adds the ranks' matrices and site counts before the division.  *total_sites = sites over all ranks.
extern "C" int pg_pairdist_cat(pg_ctx* ctx, int32_t n_ind, const int32_t* hap_ind, int32_t include_same_with_same,
                               double* dist, int64_t* total_sites) {
    PG_CHECK(ctx && hap_ind && dist, "pg_pairdist_cat: null argument");
    PG_CHECK(n_ind >= 1, "pg_pairdist_cat: n_ind must be >= 1");
    PG_CHECK(ctx->H > 0, "pg_pairdist_cat: upload genotypes first");
    PG_CUDA(cudaSetDevice(ctx->device));
    pg_timings_reset(ctx);
    std::vector<int32_t> order, ind_start;
    PG_TRY(group_rows(ctx, hap_ind, n_ind, "pg_pairdist_cat: hap_ind", order, ind_start));
    const int Hk = (int)order.size();
    PG_CHECK(Hk >= 1, "pg_pairdist_cat: no haplotypes selected");
    const size_t HH = (size_t)Hk * Hk;
    const size_t nn = (size_t)n_ind * n_ind;
    // accumulator: diff | n | site count
    PG_TRY(ctx->misc5.ensure((2 * HH + 1) * 8 + 64));
    long long* d_acc = (long long*)ctx->misc5.p;
    PG_CUDA(cudaMemsetAsync(d_acc, 0, (2 * HH + 1) * 8, ctx->stream));
    const long long S_local = ctx->S;
    PG_CUDA(cudaMemcpyAsync(d_acc + 2 * HH, &S_local, 8, cudaMemcpyHostToDevice, ctx->stream));
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    if (ctx->S > 0) {
        PlaneSet ps;
        PG_TRY(build_planes(ctx, order, 0, ctx->S, ps));
        const int64_t CH = 32768;                                  // sites per chunk (1024 plane words)
        std::vector<int64_t> chunks, clo, chi;
        for (int64_t c = 0; c * CH < ctx->S; ++c) {
            chunks.push_back(c);
            clo.push_back(c * CH);
            chi.push_back(std::min<int64_t>(c * CH + CH, ctx->S));
        }
        PG_TRY(for_each_batch(ctx, chunks, clo.data(), chi.data(), pair_batch_size(Hk, 0),
                              [&](size_t, size_t nb, const int64_t* d_lo, const int64_t* d_hi) {
            int32_t *d_diff = nullptr, *d_n = nullptr;
            PG_TRY(run_pair_batch(ctx, ps, d_lo, d_hi, (int)nb, &d_diff, &d_n));
            PG_TRY(pg_timed(ctx, "k2_reduce_pairs", [&] {
                k2_reduce_pairs<<<(unsigned)std::min<size_t>((HH + 255) / 256, 4096), 256, 0, ctx->stream>>>(
                    d_diff, d_n, ps.d_mid, Hk, ps.Hm, (int)nb, d_acc);
            }));
            PG_CUDA(cudaStreamSynchronize(ctx->stream));           // host vectors / scratch are reused by the next batch
            return PG_OK;
        }));
    }
    if (ctx->nccl_comm && ctx->nccl_ranks > 1) PG_TRY(pg_nccl_allreduce_i64(ctx, d_acc, 2 * HH + 1));
    PG_TRY(ctx->misc.ensure((size_t)(n_ind + 1) * 4 + 64));
    PG_CUDA(cudaMemcpyAsync(ctx->misc.p, ind_start.data(), (size_t)(n_ind + 1) * 4, cudaMemcpyHostToDevice, ctx->stream));
    PG_TRY(ctx->out_d.ensure(nn * 8 + 64));
    IndEpi64Params ep;
    ep.acc = d_acc;
    ep.Hk = Hk;
    ep.n_ind = n_ind;
    ep.ind_start = (const int32_t*)ctx->misc.p;
    ep.include_same = include_same_with_same ? 1 : 0;
    ep.out = (double*)ctx->out_d.p;
    PG_TRY(pg_timed(ctx, "k2_ind_epi", [&] {
        k2_ind_epi64<<<(unsigned)std::min<size_t>((nn + 255) / 256, 1024), 256, 0, ctx->stream>>>(ep);
    }));
    long long tot = 0;
    PG_CUDA(cudaMemcpyAsync(dist, ctx->out_d.p, nn * 8, cudaMemcpyDeviceToHost, ctx->stream));
    PG_CUDA(cudaMemcpyAsync(&tot, d_acc + 2 * HH, 8, cudaMemcpyDeviceToHost, ctx->stream));
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    if (total_sites) *total_sites = tot;
    return PG_OK;
}

// Alignment.seqNonNan() per window (distMat.py:40 --minPerInd gate): out int64 [W x H], haplotypes in upload order.
extern "C" int pg_seq_nonnan(pg_ctx* ctx, int64_t* out) {
    PG_CHECK(ctx && out, "pg_seq_nonnan: null argument");
    PG_CHECK(ctx->H > 0, "pg_seq_nonnan: upload genotypes first");
    PG_CUDA(cudaSetDevice(ctx->device));
    pg_timings_reset(ctx);
    const int64_t W = ctx->W;
    const int H = ctx->H;
    if (W == 0) return PG_OK;
    memset(out, 0, (size_t)W * H * 8);
    std::vector<int64_t> wins;
    int64_t lo, hi;
    nonempty_windows(ctx, wins, lo, hi);
    if (wins.empty()) return PG_OK;
    PlaneSet ps;
    PG_TRY(build_planes(ctx, all_rows(H), lo, hi, ps));
    return for_each_batch(ctx, wins, ctx->win_lo.data(), ctx->win_hi.data(), 65535,
                          [&](size_t b0, size_t nb, const int64_t* d_lo, const int64_t* d_hi) {
        PG_TRY(ctx->out_d.ensure(nb * (size_t)H * 8 + 64));
        PG_TRY(run_seq_nonnan(ctx, ps, d_lo, d_hi, (int)nb, (long long*)ctx->out_d.p));
        return copy_rows_back(ctx, wins, b0, nb, ctx->out_d.p, out, (size_t)H * 8);
    });
}
