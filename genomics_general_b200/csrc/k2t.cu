// K2T — the pairwise path on the Hopper tensor cores (wgmma.mma_async u8 x u8 -> s32, int32 accumulators in registers).
//
// Reference semantics (genomics.py:903-916, 1042-1047, 1219-1221): for every haplotype pair of a window
//   n_ij    = #sites where both are non-missing                 = (V V^T)_ij          V  = 0/1 valid indicator
//   diff_ij = #sites where both are non-missing and different   = (P Q^T + Q P^T)_ij  over "pseudo-sites"
// Both are Gram matrices of 0/1 operands, so uint8 x uint8 -> int32 MMAs are bit-exact.
//
// Exact work reduction for diff: a site where fewer than two alleles are present among the selected haplotypes
// cannot contribute to any diff_ij.  A site with alleles a_0 < a_1 < ... < a_{m-1} present is split into m-1
// pseudo-sites k = 0..m-2 with P = [allele == a_k], Q = [allele in {a_{k+1}, ...}]; then
//   sum_k (P_i Q_j + Q_i P_j) = [both valid and different]          (each unordered allele pair is counted once).
// A biallelic site is ONE pseudo-site; monomorphic sites vanish.  Pseudo-sites are compacted (exclusive scan), so the
// diff Gram runs over ~(variable sites) columns instead of every site.
//
// Data flow (all operands stay bit-packed in HBM, 1 bit per genotype):
//   k2t_valid_class : resident one-hot bytes [S x pitch] -> valid plane (64-site chunks, chunk-major) + per-site allele
//                     presence nibble + pseudo-site count per chunk                       (one pass, HBM-bound)
//   k2t_scan / k2t_inv : exclusive scan -> cps[site] (pseudo-site prefix) + inverse map pseudo-site -> (site, P bit, Q mask)
//   k2t_build_pq    : gathers the variable sites' rows -> P / Q planes (64 pseudo-site chunks)
//   k2t_gram<NPL>   : persistent CTAs (one per SM) over (window, tile group) items: a TMA warp brings plane words into a
//                     raw ring, two consumer warpgroups expand them to 0/1 bytes in the K-major no-swizzle core-matrix
//                     layout in shared memory and issue wgmma (M=64 per warpgroup, N<=256, K=32 per instruction) on them,
//                     then write the upper triangle of the symmetric int32 matrix from their accumulator registers.
#include <stdlib.h>

#include <algorithm>

#include "pgwin_internal.h"

namespace {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    do {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(ok)
            : "r"(smem_u32(bar)), "r"(parity)
            : "memory");
    } while (!ok);
}

// ------------------------------------------------------------------------------------------------
// pass 1: valid plane + allele presence per site
// ------------------------------------------------------------------------------------------------
struct VcParams {
    const uint32_t* geno32;     // resident matrix as words, pw words per site row
    int pw, pitch;
    int64_t S;                  // sites in the matrix
    int64_t site_base;          // first site of chunk 0 (multiple of 64)
    int64_t nchunk;
    const int32_t* c2r;         // [pitch] column -> plane row (-1: unused)
    const uint32_t* cmask;      // [pw] 0xff in the bytes of used columns
    uint64_t* vplane;           // [nchunk][R]
    int R, Hk;
    uint8_t* cls;               // [nchunk*64] presence nibble (bit a: allele a present among the used haplotypes)
    int32_t* chunk_tot;         // [nchunk] pseudo-sites of the chunk
    uint64_t* vpair;            // [nchunk][R2] valid words of the even rows (nullptr: not wanted)
    int R2;
    int32_t* pair_flag;         // set to 1 when some row 2k and 2k+1 differ in a valid word
};

// one-hot bytes (bits 0,2,4,6) of two sites -> per byte: bit0 = site0 valid, bit1 = site1 valid
__device__ __forceinline__ uint32_t valid2(uint32_t w0, uint32_t w1) {
    const uint32_t z = w0 | (w1 << 1);
    const uint32_t t = z | (z >> 4);
    return (t | (t >> 2)) & 0x03030303u;
}

// eight words [4 columns x 1 byte] (one per site octet) -> per column the 64-site word (lo, hi): two 4x4 byte transposes
__device__ __forceinline__ void octets_to_words(const uint32_t (&a)[8], uint32_t (&lo)[4], uint32_t (&hi)[4]) {
    {
        const uint32_t t0 = __byte_perm(a[0], a[1], 0x5140), t1 = __byte_perm(a[2], a[3], 0x5140);
        const uint32_t t2 = __byte_perm(a[0], a[1], 0x7362), t3 = __byte_perm(a[2], a[3], 0x7362);
        lo[0] = __byte_perm(t0, t1, 0x5410);
        lo[1] = __byte_perm(t0, t1, 0x7632);
        lo[2] = __byte_perm(t2, t3, 0x5410);
        lo[3] = __byte_perm(t2, t3, 0x7632);
    }
    {
        const uint32_t t0 = __byte_perm(a[4], a[5], 0x5140), t1 = __byte_perm(a[6], a[7], 0x5140);
        const uint32_t t2 = __byte_perm(a[4], a[5], 0x7362), t3 = __byte_perm(a[6], a[7], 0x7362);
        hi[0] = __byte_perm(t0, t1, 0x5410);
        hi[1] = __byte_perm(t0, t1, 0x7632);
        hi[2] = __byte_perm(t2, t3, 0x5410);
        hi[3] = __byte_perm(t2, t3, 0x7632);
    }
}

// ALL: every column of the row is a selected haplotype or padding (padding bytes are 0 = missing): no column mask needed
template <bool ALL>
__global__ void __launch_bounds__(256, 4) k2t_valid_class(const __grid_constant__ VcParams p) {
    extern __shared__ __align__(16) uint32_t vc_st[];      // [8 octets][pw]: byte (o, c) = valid bits of 8 sites of column c
    __shared__ int s_wtot[8];
    const int tid = threadIdx.x, lane = tid & 31, o = tid >> 5;
    for (int64_t chunk = blockIdx.x; chunk < p.nchunk; chunk += gridDim.x) {
        const int64_t site0 = p.site_base + chunk * 64 + o * 8;
        uint32_t pres[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) pres[k] = 0u;
        // one lane owns 4 column words (16 haplotype bytes) of the warp's 8 sites: 8 x LDG.128 in flight per lane
        const uint4* g4 = reinterpret_cast<const uint4*>(p.geno32);
        const int pw4 = p.pw >> 2;
        for (int q = lane; q < pw4; q += 32) {
            uint4 cm = make_uint4(~0u, ~0u, ~0u, ~0u);
            if (!ALL) cm = reinterpret_cast<const uint4*>(p.cmask)[q];
            uint4 w[8];
            const uint4* rp = g4 + site0 * pw4 + q;
            if (site0 + 8 <= p.S) {      // (warp-uniform) every chunk but the last: no per-row guards
#pragma unroll
                for (int k = 0; k < 8; ++k) w[k] = __ldg(rp + (int64_t)k * pw4);
            } else {
#pragma unroll
                for (int k = 0; k < 8; ++k) w[k] = (site0 + k < p.S) ? __ldg(rp + (int64_t)k * pw4) : make_uint4(0u, 0u, 0u, 0u);
            }
#pragma unroll
            for (int k = 0; k < 8; ++k)
                pres[k] |= ALL ? (w[k].x | w[k].y | w[k].z | w[k].w)
                               : ((w[k].x & cm.x) | (w[k].y & cm.y) | (w[k].z & cm.z) | (w[k].w & cm.w));
            uint4 o4;
#define VC_WORD(C) (valid2(w[0].C, w[1].C) | (valid2(w[2].C, w[3].C) << 2) | (valid2(w[4].C, w[5].C) << 4) | (valid2(w[6].C, w[7].C) << 6))
            o4.x = VC_WORD(x);
            o4.y = VC_WORD(y);
            o4.z = VC_WORD(z);
            o4.w = VC_WORD(w);
#undef VC_WORD
            reinterpret_cast<uint4*>(vc_st + o * p.pw)[q] = o4;
        }
        uint32_t mine = 0u;
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const uint32_t v = __reduce_or_sync(0xffffffffu, pres[k]);      // REDUX.OR: one instruction per site
            if (lane == k) mine = v;
        }
        int ps = 0;
        if (lane < 8) {
            uint32_t b = mine;
            b |= b >> 16;
            b |= b >> 8;
            const uint32_t nib = (b & 1u) | ((b >> 1) & 2u) | ((b >> 2) & 4u) | ((b >> 3) & 8u);
            p.cls[chunk * 64 + o * 8 + lane] = (uint8_t)nib;
            const int cnt = __popc(nib);
            ps = cnt > 1 ? cnt - 1 : 0;
        }
#pragma unroll
        for (int d = 4; d >= 1; d >>= 1) ps += __shfl_xor_sync(0xffffffffu, ps, d);
        if (lane == 0) s_wtot[o] = ps;
        __syncthreads();
        uint64_t* s_v = reinterpret_cast<uint64_t*>(vc_st + 8 * p.pw);      // [R] this chunk's words by plane row
        // a thread turns four columns: 8 octet words [4 columns x 1 byte] -> 4 words of 64 sites (two 4x4 byte transposes)
        for (int cw = tid; cw < p.pw; cw += 256) {
            uint32_t a[8];
#pragma unroll
            for (int q = 0; q < 8; ++q) a[q] = vc_st[q * p.pw + cw];
            uint32_t lo[4], hi[4];
            octets_to_words(a, lo, hi);
            const int4 r4 = *reinterpret_cast<const int4*>(p.c2r + 4 * cw);
            const int rr[4] = {r4.x, r4.y, r4.z, r4.w};
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                if (rr[j] < 0) continue;
                const uint64_t v = (uint64_t)lo[j] | ((uint64_t)hi[j] << 32);
                p.vplane[chunk * p.R + rr[j]] = v;
                s_v[rr[j]] = v;
            }
        }
        for (int r = p.Hk + tid; r < p.R; r += 256) p.vplane[chunk * p.R + r] = 0ull;
        if (p.vpair) {
            // Missingness is usually per genotype: the two haplotypes of a sample then share their valid words, n_ij needs
            // one row per sample, and the co-valid Gram shrinks 4x.  Checked here for every word; the flag decides later.
            __syncthreads();
            bool bad = false;
            for (int k2 = tid; k2 < p.R2; k2 += 256) {
                uint64_t a = 0;
                if (2 * k2 + 1 < p.Hk) {
                    a = s_v[2 * k2];
                    bad |= (a != s_v[2 * k2 + 1]);
                }
                p.vpair[chunk * p.R2 + k2] = a;
            }
            if (bad) atomicOr(p.pair_flag, 1);
        }
        if (tid == 0) {
            int t = 0;
            for (int q = 0; q < 8; ++q) t += s_wtot[q];
            p.chunk_tot[chunk] = t;
        }
        __syncthreads();
    }
}

// exclusive scan of the chunk totals (single CTA, 4 elements per thread and iteration; 1e8 sites = 1.6 M chunks = 400 iterations)
__global__ void __launch_bounds__(1024) k2t_scan(const int32_t* __restrict__ tot, int32_t* __restrict__ off, int64_t n) {
    __shared__ int wsum[32];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    int carry = 0;
    for (int64_t base = 0; base < n; base += 4096) {
        const int64_t i = base + 4 * tid;
        int4 v = make_int4(0, 0, 0, 0);
        if (i + 3 < n) v = *reinterpret_cast<const int4*>(tot + i);
        else {
            if (i < n) v.x = tot[i];
            if (i + 1 < n) v.y = tot[i + 1];
            if (i + 2 < n) v.z = tot[i + 2];
        }
        const int mine = v.x + v.y + v.z + v.w;
        int incl = mine;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const int t = __shfl_up_sync(0xffffffffu, incl, d);
            if (lane >= d) incl += t;
        }
        if (lane == 31) wsum[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            int x = wsum[lane];
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const int t = __shfl_up_sync(0xffffffffu, x, d);
                if (lane >= d) x += t;
            }
            wsum[lane] = x;
        }
        __syncthreads();
        const int e0 = carry + (warp ? wsum[warp - 1] : 0) + incl - mine;
        if (i + 3 < n) *reinterpret_cast<int4*>(off + i) = make_int4(e0, e0 + v.x, e0 + v.x + v.y, e0 + v.x + v.y + v.z);
        else {
            if (i < n) off[i] = e0;
            if (i + 1 < n) off[i + 1] = e0 + v.x;
            if (i + 2 < n) off[i + 2] = e0 + v.x + v.y;
        }
        carry += wsum[31];
        __syncthreads();
    }
    if (tid == 0) off[n] = carry;
}

// cps[site] = pseudo-sites before the site; inv[pseudo-site] = (site relative to site_base, P shift | Q mask << 8)
__global__ void __launch_bounds__(256) k2t_inv(const uint8_t* __restrict__ cls, const int32_t* __restrict__ chunk_off,
                                               int64_t nchunk, int32_t* __restrict__ cps, uint2* __restrict__ inv) {
    const int lane = threadIdx.x & 31;
    const int64_t wid = ((int64_t)blockIdx.x * 256 + threadIdx.x) >> 5, nwarp = ((int64_t)gridDim.x * 256) >> 5;
    for (int64_t chunk = wid; chunk < nchunk; chunk += nwarp) {
        const uint32_t n0 = cls[chunk * 64 + 2 * lane], n1 = cls[chunk * 64 + 2 * lane + 1];
        const int c0 = __popc(n0) > 1 ? __popc(n0) - 1 : 0, c1 = __popc(n1) > 1 ? __popc(n1) - 1 : 0;
        const int v = c0 + c1;
        int incl = v;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const int t = __shfl_up_sync(0xffffffffu, incl, d);
            if (lane >= d) incl += t;
        }
        const int base = chunk_off[chunk] + incl - v;
        cps[chunk * 64 + 2 * lane] = base;
        cps[chunk * 64 + 2 * lane + 1] = base + c0;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            uint32_t nib = h ? n1 : n0;
            const int cnt = h ? c1 : c0;
            int j = base + (h ? c0 : 0);
            const uint32_t site_rel = (uint32_t)(chunk * 64 + 2 * lane + h);
            for (int k = 0; k < cnt; ++k, ++j) {
                const int a = __ffs(nib) - 1;          // lowest remaining allele
                nib &= nib - 1;
                uint32_t qm = 0;                        // one-hot byte mask of the remaining (higher) alleles
#pragma unroll
                for (int b = 0; b < 4; ++b)
                    if (nib & (1u << b)) qm |= 1u << (2 * b);
                inv[j] = make_uint2(site_rel, (uint32_t)(2 * a) | (qm << 8));
            }
        }
        if (chunk == nchunk - 1 && lane == 31) cps[nchunk * 64] = chunk_off[nchunk];
    }
}

// ------------------------------------------------------------------------------------------------
// pass 2: P / Q planes of the pseudo-sites
// ------------------------------------------------------------------------------------------------
struct PqParams {
    const uint32_t* geno32;
    int pw, pitch;
    int64_t site_base;
    int64_t total;              // pseudo-sites
    int64_t nchunk;             // ceil(total / 64)
    const uint2* inv;
    const int32_t* c2r;
    uint64_t* pq;               // [nchunk][2][R]
    int R, Hk;
};

__global__ void __launch_bounds__(256, 4) k2t_build_pq(const __grid_constant__ PqParams p) {
    extern __shared__ __align__(16) uint32_t pq_st[];      // [2][8][pw]
    const int tid = threadIdx.x, lane = tid & 31, o = tid >> 5;
    for (int64_t chunk = blockIdx.x; chunk < p.nchunk; chunk += gridDim.x) {
        const int64_t j0 = chunk * 64 + o * 8;
        const uint32_t* row[8];
        uint32_t psh[8], qm[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const bool ok = j0 + k < p.total;
            const uint2 e = ok ? __ldg(p.inv + j0 + k) : make_uint2(0u, 0u);
            row[k] = p.geno32 + (p.site_base + (int64_t)e.x) * p.pw;
            psh[k] = ok ? (e.y & 0xffu) : 0u;
            qm[k] = ok ? ((e.y >> 8) & 0xffu) * 0x01010101u : 0u;
            if (!ok) row[k] = nullptr;
        }
        const int pw4 = p.pw >> 2;
        for (int q = lane; q < pw4; q += 32) {
            uint4 w[8];
            if (j0 + 8 <= p.total) {       // (warp-uniform) all eight pseudo-sites exist
#pragma unroll
                for (int k = 0; k < 8; ++k) w[k] = __ldg(reinterpret_cast<const uint4*>(row[k]) + q);
            } else {
#pragma unroll
                for (int k = 0; k < 8; ++k)
                    w[k] = row[k] ? __ldg(reinterpret_cast<const uint4*>(row[k]) + q) : make_uint4(0u, 0u, 0u, 0u);
            }
            uint4 op = make_uint4(0u, 0u, 0u, 0u), oq = make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
            for (int k = 0; k < 8; ++k) {
#define PQ_WORD(C)                                         \
    {                                                      \
        op.C |= ((w[k].C >> psh[k]) & 0x01010101u) << k;   \
        uint32_t t = w[k].C & qm[k];                       \
        t |= t >> 4;                                       \
        t |= t >> 2;                                       \
        oq.C |= (t & 0x01010101u) << k;                    \
    }
                PQ_WORD(x)
                PQ_WORD(y)
                PQ_WORD(z)
                PQ_WORD(w)
#undef PQ_WORD
            }
            reinterpret_cast<uint4*>(pq_st + (0 * 8 + o) * p.pw)[q] = op;
            reinterpret_cast<uint4*>(pq_st + (1 * 8 + o) * p.pw)[q] = oq;
        }
        __syncthreads();
        for (int cw = tid; cw < p.pw; cw += 256) {      // a thread turns four columns of both planes
            uint32_t a[8], plo[4], phi[4], qlo[4], qhi[4];
#pragma unroll
            for (int q = 0; q < 8; ++q) a[q] = pq_st[q * p.pw + cw];
            octets_to_words(a, plo, phi);
#pragma unroll
            for (int q = 0; q < 8; ++q) a[q] = pq_st[(8 + q) * p.pw + cw];
            octets_to_words(a, qlo, qhi);
            const int4 r4 = *reinterpret_cast<const int4*>(p.c2r + 4 * cw);
            const int rr[4] = {r4.x, r4.y, r4.z, r4.w};
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                if (rr[j] < 0) continue;
                p.pq[(chunk * 2 + 0) * p.R + rr[j]] = (uint64_t)plo[j] | ((uint64_t)phi[j] << 32);
                p.pq[(chunk * 2 + 1) * p.R + rr[j]] = (uint64_t)qlo[j] | ((uint64_t)qhi[j] << 32);
            }
        }
        for (int r = p.Hk + tid; r < p.R; r += 256) {
            p.pq[(chunk * 2 + 0) * p.R + r] = 0ull;
            p.pq[(chunk * 2 + 1) * p.R + r] = 0ull;
        }
        __syncthreads();
    }
}

// ------------------------------------------------------------------------------------------------
// Gram kernel
// ------------------------------------------------------------------------------------------------
struct GramGroup {
    int a_row0;       // first row of the 128-row A tile
    int b_row0;       // first row of the B range
    int nb_rows;      // rows of the B range: multiple of 16, <= GRAM_BMAX
    int pad;
};
struct GramParams {
    const uint64_t* plane;      // NPL == 1: [chunk][R];  NPL == 2: [chunk][2][R]
    int R, Hk;
    int64_t site_base;          // plane coordinate of an absolute site = site - site_base
    const int64_t* win_lo;      // [nb] absolute site ranges
    const int64_t* win_hi;
    const int32_t* cps;         // NPL == 2: plane coordinate = cps[site - site_base]
    const GramGroup* groups;
    int ngroups;
    int nb;                     // windows
    int brows;                  // rows of the B region of a block: max(128, max nb_rows rounded up to 64)
    int a_sep;                  // some group's A tile lies outside its B range: blocks carry a separate 128-row A region
    int nstages;                // operand ring depth (1 or 2)
    int nraw;                   // raw plane-word ring depth
    int64_t nchunks;            // chunks of the plane (a stage of CH chunks may reach past the last one: clamped, masked to 0)
    int32_t* out;               // [nb][Hk][Hk], upper triangle (i <= j) only
};

// Warp roles of the persistent CTA (one per SM):
//   warps 0-7   two consumer warpgroups: they expand the plane words of a stage into 0/1 bytes (K-major, no-swizzle core
//               matrices) and issue wgmma on it; warpgroup w owns rows 64 w .. 64 w + 63 of the 128-row A tile and keeps its
//               64 x N int32 accumulators in registers (N <= 256: 128 registers per thread)
//   warp 8      TMA: plane words of every stage -> raw ring (1-D bulk copies completing on an mbarrier)
// The MMAs of stage k run while the consumers expand stage k + 1; one named barrier per stage hands the stage over.
constexpr int GRAM_CTHREADS = 256;
constexpr int GRAM_THREADS = GRAM_CTHREADS + 32;
constexpr int GRAM_MAX_RAW = 48;           // depth of the raw plane-word ring (TMA runs this many stages ahead)
constexpr int GRAM_BMAX = 256;             // B rows of a tile group (the largest wgmma N)
constexpr int GRAM_ACC = GRAM_BMAX / 2;    // accumulator registers per thread

// 16 bits -> 16 bytes of 0/1 (byte k = bit k): 4 bits -> 4 bytes is one IMAD + LOP3
__device__ __forceinline__ uint4 expand16(uint32_t x) {
    uint4 r;
    r.x = ((x & 0xfu) * 0x00204081u) & 0x01010101u;
    r.y = (((x >> 4) & 0xfu) * 0x00204081u) & 0x01010101u;
    r.z = (((x >> 8) & 0xfu) * 0x00204081u) & 0x01010101u;
    r.w = (((x >> 12) & 0xfu) * 0x00204081u) & 0x01010101u;
    return r;
}

// wgmma shared-memory matrix descriptor: K-major, no swizzle; core matrix = 8 rows x 16 bytes stored as 128 contiguous
// bytes; LBO = byte distance between the two K cores of a K=32 slab (128), SBO = byte distance between 8-row groups (256)
__device__ __forceinline__ uint64_t gmma_desc(uint32_t saddr) {
    return (uint64_t)((saddr & 0x3ffffu) >> 4) | ((uint64_t)(128u >> 4) << 16) | ((uint64_t)(256u >> 4) << 32);
}

// D[64 x N] (s32, registers) += A[64 x 32] (u8, shared) * B[N x 32]^T (u8, shared)
template <int N>
__device__ __forceinline__ void wgmma_u8(uint32_t (&d)[GRAM_ACC], uint64_t a, uint64_t b);
template <>
__device__ __forceinline__ void wgmma_u8<64>(uint32_t (&d)[GRAM_ACC], uint64_t a, uint64_t b) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\twgmma.mma_async.sync.aligned.m64n64k32.s32.u8.u8 {"
        "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
        "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31"
        "}, %32, %33, p;\n\t}"
        : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]),
          "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]),
          "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]),
          "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31])
        : "l"(a), "l"(b));
}
template <>
__device__ __forceinline__ void wgmma_u8<128>(uint32_t (&d)[GRAM_ACC], uint64_t a, uint64_t b) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\twgmma.mma_async.sync.aligned.m64n128k32.s32.u8.u8 {"
        "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
        "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
        "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,"
        "%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63"
        "}, %64, %65, p;\n\t}"
        : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]),
          "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]),
          "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]),
          "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]),
          "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]),
          "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]),
          "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]),
          "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63])
        : "l"(a), "l"(b));
}
template <>
__device__ __forceinline__ void wgmma_u8<192>(uint32_t (&d)[GRAM_ACC], uint64_t a, uint64_t b) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\twgmma.mma_async.sync.aligned.m64n192k32.s32.u8.u8 {"
        "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
        "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
        "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,"
        "%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,"
        "%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,"
        "%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95"
        "}, %96, %97, p;\n\t}"
        : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]),
          "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]),
          "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]),
          "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]),
          "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]),
          "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]),
          "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]),
          "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63]),
          "+r"(d[64]), "+r"(d[65]), "+r"(d[66]), "+r"(d[67]), "+r"(d[68]), "+r"(d[69]), "+r"(d[70]), "+r"(d[71]),
          "+r"(d[72]), "+r"(d[73]), "+r"(d[74]), "+r"(d[75]), "+r"(d[76]), "+r"(d[77]), "+r"(d[78]), "+r"(d[79]),
          "+r"(d[80]), "+r"(d[81]), "+r"(d[82]), "+r"(d[83]), "+r"(d[84]), "+r"(d[85]), "+r"(d[86]), "+r"(d[87]),
          "+r"(d[88]), "+r"(d[89]), "+r"(d[90]), "+r"(d[91]), "+r"(d[92]), "+r"(d[93]), "+r"(d[94]), "+r"(d[95])
        : "l"(a), "l"(b));
}
template <>
__device__ __forceinline__ void wgmma_u8<256>(uint32_t (&d)[GRAM_ACC], uint64_t a, uint64_t b) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\twgmma.mma_async.sync.aligned.m64n256k32.s32.u8.u8 {"
        "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
        "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
        "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,"
        "%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,"
        "%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,"
        "%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95,"
        "%96,%97,%98,%99,%100,%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111,"
        "%112,%113,%114,%115,%116,%117,%118,%119,%120,%121,%122,%123,%124,%125,%126,%127"
        "}, %128, %129, p;\n\t}"
        : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]),
          "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]),
          "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]),
          "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]),
          "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]),
          "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]),
          "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]),
          "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63]),
          "+r"(d[64]), "+r"(d[65]), "+r"(d[66]), "+r"(d[67]), "+r"(d[68]), "+r"(d[69]), "+r"(d[70]), "+r"(d[71]),
          "+r"(d[72]), "+r"(d[73]), "+r"(d[74]), "+r"(d[75]), "+r"(d[76]), "+r"(d[77]), "+r"(d[78]), "+r"(d[79]),
          "+r"(d[80]), "+r"(d[81]), "+r"(d[82]), "+r"(d[83]), "+r"(d[84]), "+r"(d[85]), "+r"(d[86]), "+r"(d[87]),
          "+r"(d[88]), "+r"(d[89]), "+r"(d[90]), "+r"(d[91]), "+r"(d[92]), "+r"(d[93]), "+r"(d[94]), "+r"(d[95]),
          "+r"(d[96]), "+r"(d[97]), "+r"(d[98]), "+r"(d[99]), "+r"(d[100]), "+r"(d[101]), "+r"(d[102]), "+r"(d[103]),
          "+r"(d[104]), "+r"(d[105]), "+r"(d[106]), "+r"(d[107]), "+r"(d[108]), "+r"(d[109]), "+r"(d[110]), "+r"(d[111]),
          "+r"(d[112]), "+r"(d[113]), "+r"(d[114]), "+r"(d[115]), "+r"(d[116]), "+r"(d[117]), "+r"(d[118]), "+r"(d[119]),
          "+r"(d[120]), "+r"(d[121]), "+r"(d[122]), "+r"(d[123]), "+r"(d[124]), "+r"(d[125]), "+r"(d[126]), "+r"(d[127])
        : "l"(a), "l"(b));
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
__device__ __forceinline__ void consumers_sync() { asm volatile("bar.sync 1, %0;" ::"n"(GRAM_CTHREADS) : "memory"); }

// one lane of a converged warp (the TMA warp runs its loop with all 32 lanes so that addresses stay warp-uniform)
__device__ __forceinline__ bool elect_one() {
    uint32_t pred;
    asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(pred));
    return pred != 0;
}

// work item j of this launch -> (window, group) and the chunk range of the window in plane coordinates
struct GramItem {
    GramGroup g;
    int wb;
    int64_t lo, hi, c_first;
    int nst;
};
template <int NPL, int CH>
__device__ __forceinline__ GramItem gram_item(const GramParams& gp, int64_t j) {
    constexpr int SH = 6 + (CH == 4 ? 2 : (CH == 2 ? 1 : 0));   // a stage covers CH chunks of 64 (pseudo-)sites
    GramItem it;
    it.wb = (int)(j / gp.ngroups);
    it.g = gp.groups[j - (int64_t)it.wb * gp.ngroups];
    it.lo = gp.win_lo[it.wb] - gp.site_base;
    it.hi = gp.win_hi[it.wb] - gp.site_base;
    if (NPL == 2) {
        it.lo = gp.cps[it.lo];
        it.hi = gp.cps[it.hi];
    }
    it.c_first = it.lo >> SH;                           // first STAGE of the window
    it.nst = (it.hi > it.lo) ? (int)(((it.hi - 1) >> SH) - it.c_first + 1) : 0;
    return it;
}

// the MMAs of one stage for one warpgroup: 2 CH K steps of 32 (pseudo-)sites
template <int NPL, int CH, int N>
__device__ __forceinline__ void gram_stage_mma(uint32_t (&acc)[GRAM_ACC], uint32_t st, uint32_t a_off, uint32_t b_off,
                                               uint32_t blk) {
#pragma unroll
    for (int ks = 0; ks < 2 * CH; ++ks) {
        if (NPL == 1) {
            const uint32_t bk = st + ks * blk;
            wgmma_u8<N>(acc, gmma_desc(bk + a_off), gmma_desc(bk + b_off));
        } else {
            const uint32_t bp = st + (ks * 2) * blk, bq = bp + blk;
            wgmma_u8<N>(acc, gmma_desc(bp + a_off), gmma_desc(bq + b_off));
            wgmma_u8<N>(acc, gmma_desc(bq + a_off), gmma_desc(bp + b_off));
        }
    }
}

// Shared memory: [raw ring: nraw slots of CH x NPL x RROWS plane words, filled by 1-D TMA bulk copies]
//                [operand ring: nstages stages of 2 CH K steps x NPL planes x RROWS rows x 32 bytes]
// RROWS = (128 rows of a separate A tile, only when some group needs one) + brows rows of the B range.  Rows of a block
// beyond the item's B range hold stale bytes: they only reach accumulator rows / columns that are not stored.
// CH = chunks per stage (1, 2 or 4): every per-stage hand-over (TMA wait, proxy fence, barrier, MMA issue) serves CH x 64 sites.
template <int NPL, int CH>
__global__ void __launch_bounds__(GRAM_THREADS, 1) k2t_gram(const __grid_constant__ GramParams gp) {
    static_assert(CH == 1 || CH == 2 || CH == 4, "chunks per stage");
    constexpr int GRAM_MAX_ITEMS = ((128 + GRAM_BMAX) * NPL + GRAM_CTHREADS - 1) / GRAM_CTHREADS;   // plane rows per thread
    extern __shared__ __align__(128) uint8_t gsm[];
    __shared__ __align__(8) uint64_t raw_full[GRAM_MAX_RAW], raw_empty[GRAM_MAX_RAW];
    const int tid = threadIdx.x, warp = tid >> 5;
    const int NS = gp.nstages, RD = gp.nraw;
    const int AOFF = gp.a_sep ? 128 : 0;                // rows of the separate A region in front of the B rows
    const int RROWS = AOFF + gp.brows;                  // rows of one plane in a raw slot / operand block
    const int RAW1 = NPL * RROWS * 8;                   // plane words of ONE chunk in a raw slot
    const int RAW = CH * RAW1;                          // bytes of one raw slot
    const int BLK = RROWS * 32;                         // one (K step, plane) operand block
    const int STAGE = CH * 2 * NPL * BLK;
    uint8_t* const raw_base = gsm;
    uint8_t* const op_base = gsm + (size_t)RD * RAW;

    // contiguous range of work items (window-major, groups of a window adjacent) of this CTA
    const int64_t n_items = (int64_t)gp.nb * gp.ngroups;
    const int64_t j0 = n_items * blockIdx.x / gridDim.x, j1 = n_items * (blockIdx.x + 1) / gridDim.x;

    if (tid == 0) {
        for (int s = 0; s < RD; ++s) {
            mbar_init(&raw_full[s], 1);
            mbar_init(&raw_empty[s], 1);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (__shfl_sync(0xffffffffu, warp, 0) == GRAM_CTHREADS / 32) {      // (warp-uniform, visibly so to the compiler)
        // ---------------- TMA: plane words of every stage of every item -> raw ring ----------------
        int n_done = 0, rs = 0;
        uint32_t rph = 0;
        for (int64_t j = j0; j < j1; ++j) {
            const GramItem im = gram_item<NPL, CH>(gp, j);
            const bool a_in_b = (im.g.a_row0 == im.g.b_row0);
            const int a_rows = a_in_b ? 0 : min(128, gp.R - im.g.a_row0);
            const uint32_t bytes_a = (uint32_t)a_rows * 8u, bytes_b = (uint32_t)im.g.nb_rows * 8u;
            for (int it = 0; it < im.nst; ++it) {
                if (n_done >= RD) mbar_wait(&raw_empty[rs], rph ^ 1u);
                if (elect_one()) {
                    mbar_expect_tx(&raw_full[rs], CH * NPL * (bytes_a + bytes_b));
#pragma unroll
                    for (int h = 0; h < CH; ++h) {
                        // a chunk past the end of the plane is read from the last one; its mask is 0
                        const int64_t chunk = min((im.c_first + it) * CH + h, gp.nchunks - 1);
#pragma unroll
                        for (int pl = 0; pl < NPL; ++pl) {
                            const uint64_t* src = gp.plane + (chunk * NPL + pl) * gp.R;
                            uint8_t* dst = raw_base + (size_t)rs * RAW + (size_t)h * RAW1 + (size_t)pl * RROWS * 8;
                            if (bytes_a) bulk_g2s(dst, src + im.g.a_row0, bytes_a, &raw_full[rs]);
                            bulk_g2s(dst + AOFF * 8, src + im.g.b_row0, bytes_b, &raw_full[rs]);
                        }
                    }
                }
                __syncwarp();
                ++n_done;
                if (++rs == RD) {
                    rs = 0;
                    rph ^= 1u;
                }
            }
        }
        return;
    }

    // ---------------- consumers: expand + wgmma + store ----------------
    const int wg = warp >> 2, lane = tid & 31, wq = warp & 3;
    const uint32_t op16 = smem_u32(op_base);
    int rs = 0, os = 0;                                 // raw / operand ring positions
    uint32_t rph = 0;
    uint32_t acc[GRAM_ACC];
    for (int64_t j = j0; j < j1; ++j) {
        const GramItem im = gram_item<NPL, CH>(gp, j);
        const bool a_in_b = (im.g.a_row0 == im.g.b_row0);
        // rows expanded per plane: [separate A tile (128 rows)] + B range
        const int skip_a = a_in_b ? 128 : 0;
        const int rows_tot = 128 + im.g.nb_rows - skip_a;
        const int nitems = rows_tot * NPL;
        int r_idx[GRAM_MAX_ITEMS], d_off[GRAM_MAX_ITEMS];      // raw word index (-1 none, -2 zero row) / byte offset in a block
#pragma unroll
        for (int q = 0; q < GRAM_MAX_ITEMS; ++q) {
            const int item = tid + q * GRAM_CTHREADS;
            r_idx[q] = -1;
            d_off[q] = 0;
            if (item < nitems) {
                const int pl = (NPL == 2 && item >= rows_tot) ? 1 : 0;
                const int rr = item - pl * rows_tot + skip_a;          // < 128: row of the separate A tile
                const int x = (rr < 128) ? rr : rr - 128;
                const int row = (rr < 128) ? x : AOFF + x;             // row inside the block / raw slot
                r_idx[q] = (rr < 128 && im.g.a_row0 + x >= gp.R) ? -2 : pl * RROWS + row;
                d_off[q] = pl * BLK + (row >> 3) * 256 + (row & 7) * 16;
            }
        }
        // operand offsets inside a block: this warpgroup's 64 A rows (inside the B rows for a diagonal group), the B rows
        const uint32_t a_off = (uint32_t)((a_in_b ? AOFF : 0) + 64 * wg) * 32u, b_off = (uint32_t)AOFF * 32u;
        const int nsel = __shfl_sync(0xffffffffu, (min(im.g.nb_rows, GRAM_BMAX) + 63) / 64, 0);    // wgmma N = 64 nsel
#pragma unroll
        for (int e = 0; e < GRAM_ACC; ++e) acc[e] = 0u;
        for (int it = 0; it < im.nst; ++it) {
            uint64_t mask[CH];
#pragma unroll
            for (int h = 0; h < CH; ++h) {
                const int64_t b0 = ((im.c_first + it) * CH + h) << 6;
                uint64_t m = 0ull;                                  // a chunk outside the window (CH > 1 only)
                if (b0 < im.hi && b0 + 64 > im.lo) {
                    m = ~0ull;
                    if (im.lo > b0) m &= ~0ull << (int)(im.lo - b0);
                    if (im.hi < b0 + 64) m &= ~0ull >> (int)(b0 + 64 - im.hi);
                }
                mask[h] = m;
            }
            mbar_wait(&raw_full[rs], rph);
            const uint64_t* rw = reinterpret_cast<const uint64_t*>(raw_base + (size_t)rs * RAW);
            uint64_t v[GRAM_MAX_ITEMS][CH];
#pragma unroll
            for (int q = 0; q < GRAM_MAX_ITEMS; ++q)
#pragma unroll
                for (int h = 0; h < CH; ++h) v[q][h] = (r_idx[q] >= 0) ? (rw[h * (RAW1 / 8) + r_idx[q]] & mask[h]) : 0ull;
            if (NS == 1) {                      // the only stage may still be read by the previous stage's MMAs
                wgmma_wait_all();
                consumers_sync();
            }
            uint8_t* sb = op_base + (size_t)os * STAGE;
#pragma unroll
            for (int q = 0; q < GRAM_MAX_ITEMS; ++q) {
                if (q * GRAM_CTHREADS < nitems && r_idx[q] != -1) {
#pragma unroll
                    for (int h = 0; h < CH; ++h) {
                        const uint32_t wlo = (uint32_t)v[q][h], whi = (uint32_t)(v[q][h] >> 32);
                        uint8_t* d0 = sb + (size_t)h * 2 * NPL * BLK + d_off[q];      // K steps 2h, 2h + 1
                        uint8_t* d1 = d0 + NPL * BLK;
                        *reinterpret_cast<uint4*>(d0) = expand16(wlo & 0xffffu);
                        *reinterpret_cast<uint4*>(d0 + 128) = expand16(wlo >> 16);
                        *reinterpret_cast<uint4*>(d1) = expand16(whi & 0xffffu);
                        *reinterpret_cast<uint4*>(d1 + 128) = expand16(whi >> 16);
                    }
                }
            }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> visible to the tensor core
            // this warpgroup's MMAs of the previous stage are complete; after the barrier every warpgroup's are, so the
            // other operand slot may be overwritten next, and every row of this stage has been written
            wgmma_wait_all();
            consumers_sync();
            // the loads from the raw slot were consumed by the stores above: the TMA may refill it
            if (tid == 0) mbar_arrive(&raw_empty[rs]);
            wgmma_fence();
            const uint32_t st = op16 + (uint32_t)os * (uint32_t)STAGE;
            switch (nsel) {
                case 1: gram_stage_mma<NPL, CH, 64>(acc, st, a_off, b_off, (uint32_t)BLK); break;
                case 2: gram_stage_mma<NPL, CH, 128>(acc, st, a_off, b_off, (uint32_t)BLK); break;
                case 3: gram_stage_mma<NPL, CH, 192>(acc, st, a_off, b_off, (uint32_t)BLK); break;
                default: gram_stage_mma<NPL, CH, 256>(acc, st, a_off, b_off, (uint32_t)BLK); break;
            }
            wgmma_commit();
            if (++rs == RD) {
                rs = 0;
                rph ^= 1u;
            }
            if (++os == NS) os = 0;
        }
        wgmma_wait_all();
        // ---------------- epilogue: registers -> upper triangle of the symmetric int32 matrix ----------------
        // Accumulator e of a thread: row 16 wq + lane / 4 + 8 ((e / 2) & 1) of the warpgroup's 64, column 8 (e / 4) + 2 (lane % 4)
        // + (e & 1).  Only [i][j] with i in the A tile and j in the B range is written (readers index through (min, max)).
        const int i0 = im.g.a_row0 + 64 * wg + 16 * wq + (lane >> 2);
        const bool pair_ok = (gp.Hk & 1) == 0;          // two adjacent columns are one aligned 8-byte store
#pragma unroll
        for (int e = 0; e < GRAM_ACC; e += 2) {
            const int c = 8 * (e >> 2) + 2 * (lane & 3);
            const int i = i0 + 8 * ((e >> 1) & 1), jc = im.g.b_row0 + c;
            if (c < im.g.nb_rows && i < gp.Hk && jc < gp.Hk) {
                int32_t* o = gp.out + (size_t)im.wb * gp.Hk * gp.Hk + (size_t)i * gp.Hk + jc;
                if (pair_ok) {
                    *reinterpret_cast<int2*>(o) = make_int2((int32_t)acc[e], (int32_t)acc[e + 1]);
                } else {
                    o[0] = (int32_t)acc[e];
                    if (jc + 1 < gp.Hk) o[1] = (int32_t)acc[e + 1];
                }
            }
        }
    }
}

// ---- small consumers of the planes ---------------------------------------------------------------------
__device__ __forceinline__ uint64_t chunk_mask(int64_t chunk, int64_t lo, int64_t hi) {
    uint64_t m = ~0ull;
    const int64_t b0 = chunk << 6;
    if (lo > b0) m &= ~0ull << (int)(lo - b0);
    if (hi < b0 + 64) m &= ~0ull >> (int)(b0 + 64 - hi);
    return m;
}

// Alignment.seqNonNan (genomics.py:1038-1040): thread = plane row, one CTA column per window
__global__ void __launch_bounds__(128) k2t_seq_nonnan(const uint64_t* __restrict__ vplane, int R, int Hk, int64_t site_base,
                                                      const int64_t* __restrict__ win_lo, const int64_t* __restrict__ win_hi,
                                                      long long* __restrict__ out) {
    const int r = blockIdx.x * 128 + threadIdx.x, wb = blockIdx.y;
    if (r >= Hk) return;
    const int64_t lo = win_lo[wb] - site_base, hi = win_hi[wb] - site_base;
    long long n = 0;
    if (hi > lo)
        for (int64_t c = lo >> 6; c <= (hi - 1) >> 6; ++c) n += __popcll(vplane[c * R + r] & chunk_mask(c, lo, hi));
    out[(size_t)wb * Hk + r] = n;
}

// Alignment.sampleHet (genomics.py:918-929): thread = individual (rows ind_start[a], +1)
__global__ void __launch_bounds__(128) k2t_het(const uint64_t* __restrict__ vplane, const uint64_t* __restrict__ pq,
                                               const int32_t* __restrict__ cps, int R, int64_t site_base,
                                               const int64_t* __restrict__ win_lo, const int64_t* __restrict__ win_hi,
                                               const int32_t* __restrict__ ind_start, int n_ind, int min_sites,
                                               double* __restrict__ out) {
    const int a = blockIdx.x * 128 + threadIdx.x, wb = blockIdx.y;
    if (a >= n_ind) return;
    const double nan = __longlong_as_double(0x7ff8000000000000ll);
    const int r0 = ind_start[a], r1 = ind_start[a + 1];
    double v = nan;
    if (r1 - r0 == 2) {             // len(x) == 2 is required (the reference raises IndexError for len(x) == 1)
        const int64_t lo = win_lo[wb] - site_base, hi = win_hi[wb] - site_base;
        long long n = 0, diff = 0;
        if (hi > lo) {
            for (int64_t c = lo >> 6; c <= (hi - 1) >> 6; ++c)
                n += __popcll(vplane[c * R + r0] & vplane[c * R + r0 + 1] & chunk_mask(c, lo, hi));
            const int64_t plo = cps[lo], phi = cps[hi];
            if (phi > plo)
                for (int64_t c = plo >> 6; c <= (phi - 1) >> 6; ++c) {
                    const uint64_t p0 = pq[(c * 2) * R + r0], p1 = pq[(c * 2) * R + r0 + 1];
                    const uint64_t q0 = pq[(c * 2 + 1) * R + r0], q1 = pq[(c * 2 + 1) * R + r0 + 1];
                    diff += __popcll(((p0 & q1) | (q0 & p1)) & chunk_mask(c, plo, phi));
                }
        }
        // `len(x)==2 & np.sum(mask) >= 1` parses as len(x) == (2 & n) >= 1: bit 1 of n must be set (924, 927)
        if ((n & 2) == 2 && !(min_sites > 0 && n < min_sites)) v = (double)diff / (double)n;
    }
    out[(size_t)wb * n_ind + a] = v;
}

__global__ void k2t_half(int32_t* p, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = i >> 1;
}
__global__ void k2t_iota(int32_t* p, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = i;
}

}  // namespace

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
bool pg_k2_use_tensor() { return getenv("PG_K2_POPC") == nullptr; }

// Planes for sites [lo, hi) of the haplotype columns in `order` (plane row r = column order[r]).
int pg_k2t_build(pg_ctx* ctx, const std::vector<int32_t>& order, int64_t lo, int64_t hi, K2TPlanes& ps) {
    const int Hk = (int)order.size();
    PG_CHECK(Hk >= 1, "pairwise path: no haplotypes selected");
    const int R = (Hk + 15) / 16 * 16;
    const int64_t sb = lo & ~(int64_t)63;
    const int64_t nchunk = (hi - sb + 63) / 64;
    PG_CHECK(nchunk * 64 < (int64_t)1 << 31, "pairwise path: site span too large for one call");
    const int pitch = ctx->pitch, pw = pitch / 4;
    PG_CHECK(pg_k2t_fits(pitch, Hk), "pairwise path: %d haplotype columns are too many for the plane builders", pitch);
    PG_TRY(pg_smem_limit<k2t_build_pq>(ctx, 96 * 1024));
    PG_TRY(pg_smem_limit<k2t_valid_class<true>>(ctx, 96 * 1024));
    PG_TRY(pg_smem_limit<k2t_valid_class<false>>(ctx, 96 * 1024));
    // column tables
    std::vector<int32_t> c2r(pitch, -1);
    for (int r = 0; r < Hk; ++r) c2r[order[r]] = r;
    std::vector<uint32_t> cmask(pw, 0u);
    for (int c = 0; c < pitch; ++c)
        if (c2r[c] >= 0) cmask[c / 4] |= 0xffu << (8 * (c % 4));
    PG_TRY(ctx->misc2.ensure((size_t)pitch * 4 + (size_t)pw * 4 + 256));
    int32_t* d_c2r = (int32_t*)ctx->misc2.p;
    uint32_t* d_cmask = (uint32_t*)(d_c2r + pitch);
    PG_CUDA(cudaMemcpyAsync(d_c2r, c2r.data(), (size_t)pitch * 4, cudaMemcpyHostToDevice, ctx->stream));
    PG_CUDA(cudaMemcpyAsync(d_cmask, cmask.data(), (size_t)pw * 4, cudaMemcpyHostToDevice, ctx->stream));
    // plane memory: vplane | cls | chunk_tot | chunk_off | cps | vpair | mask rows (halves) | mask rows (identity)
    const size_t span = (size_t)nchunk * 64;
    size_t off = 0;
    auto carve = [&](size_t bytes) {
        const size_t o = off;
        off += (bytes + 255) / 256 * 256;
        return o;
    };
    const bool want_pairs = (Hk % 2 == 0) && !getenv("PG_K2T_NO_PAIRS");
    const int R2 = (Hk / 2 + 15) / 16 * 16;
    const size_t o_v = carve((size_t)nchunk * R * 8), o_cls = carve(span), o_tot = carve((size_t)nchunk * 4),
                 o_off = carve((size_t)(nchunk + 2) * 4), o_cps = carve((span + 1) * 4),
                 o_vp = carve(want_pairs ? (size_t)nchunk * R2 * 8 : 0), o_mid = carve((size_t)Hk * 4),
                 o_iota = carve((size_t)Hk * 4);
    PG_TRY(ctx->planes.ensure(off));
    uint8_t* base = (uint8_t*)ctx->planes.p;
    int32_t* d_iota = (int32_t*)(base + o_iota);
    k2t_iota<<<(Hk + 255) / 256, 256, 0, ctx->stream>>>(d_iota, Hk);
    VcParams vp;
    vp.geno32 = (const uint32_t*)ctx->d_geno;
    vp.pw = pw;
    vp.pitch = pitch;
    vp.S = ctx->S;
    vp.site_base = sb;
    vp.nchunk = nchunk;
    vp.c2r = d_c2r;
    vp.cmask = d_cmask;
    vp.vplane = (uint64_t*)(base + o_v);
    vp.R = R;
    vp.Hk = Hk;
    vp.cls = base + o_cls;
    vp.chunk_tot = (int32_t*)(base + o_tot);
    int32_t* d_off = (int32_t*)(base + o_off);
    int32_t* d_cps = (int32_t*)(base + o_cps);
    vp.vpair = want_pairs ? (uint64_t*)(base + o_vp) : nullptr;
    vp.R2 = R2;
    vp.pair_flag = d_off + nchunk + 1;
    PG_CUDA(cudaMemsetAsync(vp.pair_flag, 0, 4, ctx->stream));
    const int grid1 = (int)std::min<int64_t>(nchunk, (int64_t)ctx->sm_count * 8);
    bool all_used = true;                        // unselected real columns? (padding columns hold 0 = missing and never count)
    for (int c = 0; c < ctx->H; ++c) all_used = all_used && c2r[c] >= 0;
    PG_TRY(pg_timed(ctx, "k2t_valid_class", [&] {
        if (all_used) k2t_valid_class<true><<<grid1, 256, (size_t)8 * pw * 4 + (size_t)R * 8, ctx->stream>>>(vp);
        else k2t_valid_class<false><<<grid1, 256, (size_t)8 * pw * 4 + (size_t)R * 8, ctx->stream>>>(vp);
    }));
    PG_TRY(pg_timed(ctx, "k2t_scan", [&] { k2t_scan<<<1, 1024, 0, ctx->stream>>>(vp.chunk_tot, d_off, nchunk); }));
    int32_t tf[2] = {0, 0};                       // pseudo-sites, "some sample's haplotypes differ in missingness"
    PG_CUDA(cudaMemcpyAsync(tf, d_off + nchunk, 8, cudaMemcpyDeviceToHost, ctx->stream));
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    const int32_t total = tf[0];
    const bool pairs_ok = want_pairs && tf[1] == 0;
    const int64_t nchunk_d = ((int64_t)total + 63) / 64;
    off = 0;
    const size_t o_inv = carve((size_t)std::max<int64_t>(total, 1) * 8), o_pq = carve((size_t)std::max<int64_t>(nchunk_d, 1) * 2 * R * 8);
    PG_TRY(ctx->planes2.ensure(off));
    uint8_t* base2 = (uint8_t*)ctx->planes2.p;
    const int gridi = (int)std::min<int64_t>((nchunk + 7) / 8, (int64_t)ctx->sm_count * 16);
    PG_TRY(pg_timed(ctx, "k2t_inv", [&] {
        k2t_inv<<<gridi, 256, 0, ctx->stream>>>(vp.cls, d_off, nchunk, d_cps, (uint2*)(base2 + o_inv));
    }));
    if (nchunk_d > 0) {
        PqParams pp;
        pp.geno32 = vp.geno32;
        pp.pw = pw;
        pp.pitch = pitch;
        pp.site_base = sb;
        pp.total = total;
        pp.nchunk = nchunk_d;
        pp.inv = (const uint2*)(base2 + o_inv);
        pp.c2r = d_c2r;
        pp.pq = (uint64_t*)(base2 + o_pq);
        pp.R = R;
        pp.Hk = Hk;
        const size_t smem = (size_t)16 * pw * 4;
        const int grid2 = (int)std::min<int64_t>(nchunk_d, (int64_t)ctx->sm_count * 8);
        PG_TRY(pg_timed(ctx, "k2t_build_pq", [&] { k2t_build_pq<<<grid2, 256, smem, ctx->stream>>>(pp); }));
    }
    ps.Hk = Hk;
    ps.R = R;
    ps.site_base = sb;
    ps.nchunk_v = nchunk;
    ps.vplane = vp.vplane;
    ps.cps = d_cps;
    ps.npseudo = total;
    ps.pq = (uint64_t*)(base2 + o_pq);
    // mask ids for the epilogues: row r -> r / 2 when the valid words are shared by consecutive rows
    ps.Hm = pairs_ok ? Hk / 2 : Hk;
    ps.R2 = R2;
    ps.vpair = pairs_ok ? vp.vpair : nullptr;
    if (pairs_ok) {
        int32_t* d_mid = (int32_t*)(base + o_mid);
        k2t_half<<<(Hk + 255) / 256, 256, 0, ctx->stream>>>(d_mid, Hk);
        ps.d_mid = d_mid;
    } else {
        ps.d_mid = d_iota;
    }
    return PG_OK;
}

// diff [nb][Hk^2] and n [nb][Hk^2] for nb windows (absolute site ranges on the device)
namespace {
// tile groups of an R-row Gram: one 128-row A tile x up to GRAM_BMAX B rows (the accumulators live in registers)
void gram_groups(int R, std::vector<GramGroup>& groups, int& brows, int& a_sep) {
    groups.clear();
    int nbmax = 16;
    a_sep = 0;
    for (int a0 = 0; a0 < R; a0 += 128)
        for (int c = a0; c < R; c += GRAM_BMAX) {
            GramGroup g;
            g.a_row0 = a0;
            g.b_row0 = c;
            g.nb_rows = std::min(GRAM_BMAX, R - c);
            g.pad = 0;
            nbmax = std::max(nbmax, g.nb_rows);
            if (c != a0) a_sep = 1;
            groups.push_back(g);
        }
    // the B region holds the widest wgmma N of any group, and the 128-row A tile of a diagonal group
    brows = std::max(128, (nbmax + 63) / 64 * 64);
}
}  // namespace

int pg_k2t_pairs(pg_ctx* ctx, const K2TPlanes& ps, const int64_t* d_lo, const int64_t* d_hi, int nb, int32_t* d_diff,
                 int32_t* d_n) {
    const int budget = 227 * 1024 - 1024;      // dynamic shared memory; the barriers are static
    PG_TRY((pg_smem_limit<k2t_gram<1, 1>>(ctx, budget)));
    PG_TRY((pg_smem_limit<k2t_gram<1, 2>>(ctx, budget)));
    PG_TRY((pg_smem_limit<k2t_gram<1, 4>>(ctx, budget)));
    PG_TRY((pg_smem_limit<k2t_gram<2, 1>>(ctx, budget)));
    // n_ij over the mask rows (one per sample when the haplotypes of a sample share their missingness), diff_ij over all rows
    const int Rn = ps.vpair ? ps.R2 : ps.R;
    std::vector<GramGroup> gn, gd;
    int brows_n, asep_n, brows_d, asep_d;
    gram_groups(Rn, gn, brows_n, asep_n);
    gram_groups(ps.R, gd, brows_d, asep_d);
    // the tile groups only live for this call's two launches (misc4 is short-lived scratch, see k2.cu)
    PG_TRY(ctx->misc4.ensure((gn.size() + gd.size()) * sizeof(GramGroup) + 64));
    GramGroup* d_gn = (GramGroup*)ctx->misc4.p;
    GramGroup* d_gd = d_gn + gn.size();
    PG_CUDA(cudaMemcpyAsync(d_gn, gn.data(), gn.size() * sizeof(GramGroup), cudaMemcpyHostToDevice, ctx->stream));
    PG_CUDA(cudaMemcpyAsync(d_gd, gd.data(), gd.size() * sizeof(GramGroup), cudaMemcpyHostToDevice, ctx->stream));
    GramParams gp;
    gp.site_base = ps.site_base;
    gp.win_lo = d_lo;
    gp.win_hi = d_hi;
    gp.nb = nb;
    // shared memory: two operand stages (the MMAs of one overlap the expansion of the next) + as deep a raw plane-word ring
    // as fits.  PG_K2T_NSTAGES = 1 and PG_K2T_NRAW cap both (the smallest rings stress the hand-overs).
    auto geometry = [&](int npl, int brows, int a_sep, int ch, int& nstages, int& nraw) {
        const int rrows = (a_sep ? 128 : 0) + brows;
        const int stage = ch * 2 * npl * rrows * 32, raw = ch * npl * rrows * 8;
        nstages = 2;
        if (const char* e = getenv("PG_K2T_NSTAGES")) nstages = std::max(1, std::min(nstages, atoi(e)));
        nraw = std::min(GRAM_MAX_RAW, (budget - nstages * stage) / raw);
        if (const char* e = getenv("PG_K2T_NRAW")) nraw = std::min(nraw, atoi(e));
        nraw = std::max(1, nraw);
        return (size_t)nstages * stage + (size_t)nraw * raw;
    };
    {   // persistent CTAs: one per SM, each works through a contiguous range of (window, group) items
        gp.R = Rn;
        gp.Hk = ps.Hm;
        gp.groups = d_gn;
        gp.ngroups = (int)gn.size();
        gp.brows = brows_n;
        gp.a_sep = asep_n;
        // every site counts for n_ij, so its K is the long one: the widest stage (up to 256 sites) whose two operand slots
        // leave room for at least two raw slots.  PG_K2T_CH = 1 | 2 | 4 caps it.
        int ch_n = 4;
        if (const char* e = getenv("PG_K2T_CH")) ch_n = std::min(ch_n, std::max(1, atoi(e)));
        size_t smem = geometry(1, brows_n, asep_n, ch_n, gp.nstages, gp.nraw);
        while (ch_n > 1 && (smem > (size_t)budget || gp.nraw < 2)) {
            ch_n /= 2;
            smem = geometry(1, brows_n, asep_n, ch_n, gp.nstages, gp.nraw);
        }
        PG_CHECK(smem <= (size_t)budget, "pairwise path: %d mask rows do not fit the Gram kernel's shared memory", Rn);
        gp.plane = ps.vpair ? ps.vpair : ps.vplane;
        gp.nchunks = ps.nchunk_v;
        gp.cps = nullptr;
        gp.out = d_n;
        const unsigned grid = (unsigned)std::min<int64_t>((int64_t)nb * gp.ngroups, ctx->sm_count);
        PG_TRY(pg_timed(ctx, "k2t_gram_n", [&] {
            if (ch_n == 4) k2t_gram<1, 4><<<grid, GRAM_THREADS, smem, ctx->stream>>>(gp);
            else if (ch_n == 2) k2t_gram<1, 2><<<grid, GRAM_THREADS, smem, ctx->stream>>>(gp);
            else k2t_gram<1, 1><<<grid, GRAM_THREADS, smem, ctx->stream>>>(gp);
        }));
    }
    {
        gp.R = ps.R;
        gp.Hk = ps.Hk;
        gp.groups = d_gd;
        gp.ngroups = (int)gd.size();
        gp.brows = brows_d;
        gp.a_sep = asep_d;
        const size_t smem = geometry(2, brows_d, asep_d, 1, gp.nstages, gp.nraw);
        PG_CHECK(smem <= (size_t)budget, "pairwise path: %d haplotype rows do not fit the Gram kernel's shared memory", ps.R);
        gp.plane = ps.pq;
        gp.nchunks = (ps.npseudo + 63) / 64;
        gp.cps = ps.cps;
        gp.out = d_diff;
        const unsigned grid = (unsigned)std::min<int64_t>((int64_t)nb * gp.ngroups, ctx->sm_count);
        PG_TRY(pg_timed(ctx, "k2t_gram_diff", [&] { k2t_gram<2, 1><<<grid, GRAM_THREADS, smem, ctx->stream>>>(gp); }));
    }
    return PG_OK;
}

int pg_k2t_seq_nonnan(pg_ctx* ctx, const K2TPlanes& ps, const int64_t* d_lo, const int64_t* d_hi, int nb, long long* d_out) {
    return pg_timed(ctx, "k2_seq_nonnan", [&] {
        k2t_seq_nonnan<<<dim3((unsigned)((ps.Hk + 127) / 128), (unsigned)nb), 128, 0, ctx->stream>>>(ps.vplane, ps.R, ps.Hk,
                                                                                                    ps.site_base, d_lo, d_hi, d_out);
    });
}

int pg_k2t_het(pg_ctx* ctx, const K2TPlanes& ps, const int64_t* d_lo, const int64_t* d_hi, int nb, const int32_t* d_ind_start,
               int n_ind, int min_sites, double* d_out) {
    return pg_timed(ctx, "k2_het", [&] {
        k2t_het<<<dim3((unsigned)((n_ind + 127) / 128), (unsigned)nb), 128, 0, ctx->stream>>>(
            ps.vplane, ps.pq, ps.cps, ps.R, ps.site_base, d_lo, d_hi, d_ind_start, n_ind, min_sites, d_out);
    });
}
