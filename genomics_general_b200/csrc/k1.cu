// K1 — the HBM-bound "site pass": one read of the int8 genotype matrix produces per-population allele
// counts per site and reduces them into per-window sums.
//
//   mode POPGEN : closed-form pi / dxy / Fst sums (exact when a window has no partially-missing site;
//                 otherwise the window is flagged "ragged" and routed to K2)   -- genomics.py:956-995
//   mode ABBA   : ABBA / BABA / D / fd / fdM sums                             -- genomics.py:1647-1695
//   mode COUNTS : per-site per-population A,C,G,T counts                      -- genomics.py:1049-1052
//
// Data path (DESIGN.md §K1): a persistent CTA per SM owns a contiguous range of tiles; a tile is T
// consecutive sites = one contiguous T*pitch byte range, brought into shared memory by 1-D TMA bulk copies
// (cp.async.bulk ... mbarrier::complete_tx) through a `stages`-deep ring.  One lane (or G lanes) owns one
// site row and walks it with conflict-free LDS.128; alleles are counted with SWAR byte-lane accumulators
// (8 integer ops per 4 genotypes).  Per-lane running sums are flushed per (warp, segment) into private
// slots — no atomics, deterministic — and a finalize kernel folds slots -> segments -> windows -> statistics.
#include <stdlib.h>

#include <algorithm>
#include <climits>
#include <cmath>
#include <type_traits>
#include <cub/cub.cuh>

#include "pgwin_internal.h"

namespace {

// consumer warps per CTA (+ one TMA producer warp): 8, or 12 where the register budget allows (65536 / 13 / 32 = 157)
constexpr int K1_MAX_WARPS = 12;

enum { MODE_POPGEN = 0, MODE_ABBA = 1, MODE_COUNTS = 2, MODE_POPGEN_FREQ = 3, MODE_FOURPOP = 4 };   // FREQ = POPGEN + popFreq counters

struct K1Params {
    const uint8_t* geno;
    const int32_t* pos;
    int64_t site_begin, site_end;     // sites processed by this launch
    int64_t num_tiles;
    int pitch, G, I, T, wpt, stages, tile_bytes, nw;
    // hap -> pop tables (shared-memory copies are made at kernel start)
    const int32_t* ent_chunk;
    const uint4* ent_mask;
    int n_ent;
    int ent_lo[PG_MAX_K1_POPS], ent_hi[PG_MAX_K1_POPS], full_lo[PG_MAX_K1_POPS], full_hi[PG_MAX_K1_POPS];
    int popN[PG_MAX_K1_POPS];
    // packed popgen pass: (word, mask) entries of the populations (ent_lo / ent_hi index them), words per plane
    const uint2* word_ent;
    const uint2* bit_frag;   // varied_mma's B operand: 32 lanes per K-block of 8 words (PopTables::bit_frag)
    int wd;
    // packed pass with uniform sites elided (UniformStream): geno holds only the varied rows.  Tile t covers the sites
    // [site_lo[t], site_lo[t + 1]) (at most T = Tmax of them), holds the varied rows [row0[t], row0[t + 1]) (at most row_cap = R)
    // of which n1[t] are one-plane rows, and its rows are the words [woff[t], woff[t + 1]) of geno; slots holds, at t * T,
    // the site index in the tile (slot) of each of its rows.  A stage holds the tile's rows (room for row_cap three-plane
    // rows), then their slots.  uni_gv > 0 forces the lanes per varied row (PG_K1_UNI_GV).
    const int64_t* row0;
    const int64_t* site_lo;
    const int64_t* woff;
    const int32_t* n1;
    const uint16_t* slots;
    int uni_gv;
    int row_cap;
    // segments / slots
    const int64_t* brk;
    int nseg;
    const int32_t* cta_seg_first;
    const int64_t* cta_slot_off;
    unsigned long long* part;
    // ABBA / FOURPOP: minimum non-missing count per population (exact integer form of n/N >= minData)
    int thr[4];
    int acc_limit;           // POPGEN: sites a lane may add to its 32-bit sums between flushes
    int lanepop;             // POPGEN: launch the lane-per-population variant (G == P lanes per site)
    int bytes;               // POPGEN: every population has <= 255 haplotypes -> byte-packed counts (IDP.4A statistics)
    int variant;             // FOURPOP allele choice: 0 = third of argsort (the rarer allele), 1 = polarize, 2 = fixed
    // COUNTS
    uint16_t* counts_out;
    int64_t counts_stride;   // uint16 elements per site
    int counts_pops;         // populations actually written (<= P)
};

// ---- PTX helpers: mbarrier + 1-D TMA bulk copy -------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
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

// ---- allele counting on the resident one-hot code (A 0x01, C 0x04, G 0x10, T 0x40, missing 0x00) ----------
// level 1: three words are added -> 2-bit fields hold 0..3
// level 2: split into 4-bit fields (lo = A | G<<4, hi = C | T<<4 per byte), up to 5 level-1 sums
// level 3: split into byte lanes, up to 17 level-2 flushes, then __dp4a folds the 4 byte lanes
struct Tally {
    uint32_t nlo, nhi;            // nibble fields
    uint32_t bA, bC, bG, bT;      // byte lanes
    uint32_t tA, tC, tG, tT;      // totals
    int load;                     // upper bound of what one byte lane holds
};
__device__ __forceinline__ void tally_init(Tally& t) {
    t.nlo = t.nhi = t.bA = t.bC = t.bG = t.bT = t.tA = t.tC = t.tG = t.tT = 0;
    t.load = 0;
}
__device__ __forceinline__ void add3(Tally& t, uint32_t a, uint32_t b, uint32_t c) {
    const uint32_t s = a + b + c;
    t.nlo += s & 0x33333333u;
    t.nhi += (s >> 2) & 0x33333333u;
}
__device__ __forceinline__ void nib_flush(Tally& t) {
    t.bA += t.nlo & 0x0f0f0f0fu;
    t.bG += (t.nlo >> 4) & 0x0f0f0f0fu;
    t.bC += t.nhi & 0x0f0f0f0fu;
    t.bT += (t.nhi >> 4) & 0x0f0f0f0fu;
    t.nlo = t.nhi = 0;
}
__device__ __forceinline__ void byte_flush(Tally& t) {
    t.tA = __dp4a(t.bA, 0x01010101u, t.tA);
    t.tC = __dp4a(t.bC, 0x01010101u, t.tC);
    t.tG = __dp4a(t.bG, 0x01010101u, t.tG);
    t.tT = __dp4a(t.bT, 0x01010101u, t.tT);
    t.bA = t.bC = t.bG = t.bT = 0;
    t.load = 0;
}
__device__ __forceinline__ uint4 and4(uint4 w, uint4 m) { return make_uint4(w.x & m.x, w.y & m.y, w.z & m.z, w.w & m.w); }
// 3 chunks = 12 words -> 4 level-1 sums (<= 12 per nibble), one nibble flush
__device__ __forceinline__ void add_chunks3(Tally& t, uint4 x, uint4 y, uint4 z) {
    add3(t, x.x, y.x, z.x);
    add3(t, x.y, y.y, z.y);
    add3(t, x.z, y.z, z.z);
    add3(t, x.w, y.w, z.w);
    nib_flush(t);
    t.load += 12;
    if (t.load > 240) byte_flush(t);
}
__device__ __forceinline__ void add_chunks2(Tally& t, uint4 x, uint4 y) {
    add3(t, x.x, x.y, x.z);
    add3(t, x.w, y.x, y.y);
    add3(t, y.z, y.w, 0u);
    nib_flush(t);
    t.load += 8;
    if (t.load > 240) byte_flush(t);
}
__device__ __forceinline__ void add_chunks1(Tally& t, uint4 x) {
    add3(t, x.x, x.y, x.z);
    add3(t, x.w, 0u, 0u);
    nib_flush(t);
    t.load += 4;
    if (t.load > 240) byte_flush(t);
}

// Per-lane running sums: 64-bit integers, 32-bit integers (flushed before they can overflow: K1Params::acc_limit),
// doubles.  A slot in global memory holds them as QI + QU + QD 8-byte words in that order.
template <int QI, int QU, int QD>
struct Acc {
    long long i[QI > 0 ? QI : 1];
    uint32_t u[QU > 0 ? QU : 1];
    double d[QD > 0 ? QD : 1];
};

// Warp-cooperative flush of the per-lane running sums into this warp's private slots.
template <int QI, int QU, int QD>
__device__ __forceinline__ void warp_flush(Acc<QI, QU, QD>& acc, int cur_seg, unsigned long long* part, int64_t slot_base,
                                           int seg_first, int warp, int lane, int nw) {
    constexpr int Q = QI + QU + QD;
    unsigned pending = __ballot_sync(0xffffffffu, cur_seg >= 0);
    while (pending) {
        const int leader = __ffs(pending) - 1;
        const int g = __shfl_sync(0xffffffffu, cur_seg, leader);
        const bool mine = (cur_seg == g);
        unsigned long long* dst = part + slot_base + ((int64_t)(g - seg_first) * nw + warp) * Q;
#pragma unroll
        for (int q = 0; q < QI; ++q) {
            long long v = mine ? acc.i[q] : 0ll;
#pragma unroll
            for (int d = 16; d >= 1; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
            if (lane == 0) dst[q] = (unsigned long long)((long long)dst[q] + v);
            if (mine) acc.i[q] = 0;
        }
#pragma unroll
        for (int q = 0; q < QU; ++q) {
            // 32-bit lane sums: the first butterfly step stays in 32 bits when two lanes cannot overflow... they can,
            // so widen first (33 bits after one step) — 5 steps of 64-bit adds on a once-per-segment path
            long long v = mine ? (long long)acc.u[q] : 0ll;
#pragma unroll
            for (int d = 16; d >= 1; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
            if (lane == 0) dst[QI + q] = (unsigned long long)((long long)dst[QI + q] + v);
            if (mine) acc.u[q] = 0u;
        }
#pragma unroll
        for (int q = 0; q < QD; ++q) {
            double v = mine ? acc.d[q] : 0.0;
#pragma unroll
            for (int d = 16; d >= 1; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);   // fixed butterfly order
            if (lane == 0)
                dst[QI + QU + q] =
                    (unsigned long long)__double_as_longlong(__longlong_as_double((long long)dst[QI + QU + q]) + v);
            if (mine) acc.d[q] = 0.0;
        }
        pending &= ~__ballot_sync(0xffffffffu, mine);
    }
}

__device__ __forceinline__ int find_seg(const int64_t* __restrict__ brk, int nseg, int from, int64_t site) {
    int lo = from, hi = nseg - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (__ldg(brk + mid) <= site) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// find_seg for a site at or past segment `from`'s start, galloping from there: brk[from + 1], brk[from + 3], brk[from + 7], ...
// until one lies past the site, then a binary search inside that bracket.  One load when the site lies in segment from, the
// common case of a pass that moves through its segments in order; the same result as find_seg for any jump.
__device__ __forceinline__ int next_seg(const int64_t* __restrict__ brk, int nseg, int from, int64_t site) {
    int lo = from, step = 1;
    while (lo + step < nseg && __ldg(brk + lo + step) <= site) {
        lo += step;
        step <<= 1;
    }
    return find_seg(brk, min(lo + step, nseg), lo, site);
}

// This lane's site lies in segment sg (cur_seg when it has not moved on).  Before any lane of the warp moves, the warp
// flushes the sums it holds into the segments they belong to.  Warp-uniform control flow.  sg is taken by reference:
// passed by value, it changes the instruction schedule ptxas (sm_90a) picks for 36 of the site-pass kernels.
template <class Flush>
__device__ __forceinline__ void seg_step(const int& sg, int& cur_seg, int64_t& seg_end, int& since_flush, const int64_t* brk,
                                         Flush&& flush) {
    if (__any_sync(0xffffffffu, sg != cur_seg)) {
        flush();
        since_flush = 0;
        if (sg != cur_seg) {
            cur_seg = sg;
            seg_end = __ldg(brk + sg + 1);
        }
    }
}

// the 32-bit sums must not overflow: flush them every acc_limit sites (never taken for N < ~900)
template <class Flush>
__device__ __forceinline__ void acc_limit_step(int& since_flush, int acc_limit, Flush&& flush) {
    if (++since_flush > acc_limit) {
        flush();
        since_flush = 1;
    }
}

template <int MODE, int P>
struct ModeTraits;
template <int P>
struct ModeTraits<MODE_POPGEN, P> {
    static constexpr int QI = 3, QU = P + P * (P - 1) / 2, QD = 0;
};
template <int P>
struct ModeTraits<MODE_POPGEN_FREQ, P> {
    static constexpr int QI = 3, QU = P + P * (P - 1) / 2 + P, QD = 0;   // + segregating-site counts
};
template <int P>
struct ModeTraits<MODE_ABBA, P> {
    static constexpr int QI = 3, QU = 0, QD = 6;
};
template <int P>
struct ModeTraits<MODE_COUNTS, P> {
    static constexpr int QI = 0, QU = 0, QD = 0;
};
template <int P>
struct ModeTraits<MODE_FOURPOP, P> {
    static constexpr int QI = 3, QU = 0, QD = 16;
};

// genomics.py:1409-1418, operation order of the reference's numpy expressions
__device__ __forceinline__ double f4_dev(double p1, double p2, double p3, double p4) {
    return (1 - p1) * p2 * p3 * (1 - p4) - p1 * (1 - p2) * p3 * (1 - p4);
}
__device__ __forceinline__ double f4c_dev(double p1, double p2, double p3, double p4) {
    return f4_dev(p1, p2, p3, p4) + f4_dev(1 - p1, 1 - p2, 1 - p3, 1 - p4);
}
// np.amax propagates nan
__device__ __forceinline__ double nmax(double a, double b) { return (a != a) ? a : ((b != b) ? b : (a > b ? a : b)); }

// The 16 running sums of genomics.fourPop (genomics.py:1617-1643) for one informative site: counts of the chosen allele
// k_X and non-missing haplotypes n_X of P1..P4, packed as k | n << 16.
template <class ACC>
__device__ __forceinline__ void fourpop_add(ACC& acc, uint32_t e1, uint32_t e2, uint32_t e3, uint32_t e4) {
    const double p1 = (double)(e1 & 0xffffu) / (double)(e1 >> 16);      // 0/0 = nan, as in the reference (genomics.py:597)
    const double p2 = (double)(e2 & 0xffffu) / (double)(e2 >> 16);
    const double p3 = (double)(e3 & 0xffffu) / (double)(e3 >> 16);
    const double p4 = (double)(e4 & 0xffffu) / (double)(e4 >> 16);
    const double abba = (1 - p1) * p2 * p3 * (1 - p4);
    const double baba = p1 * (1 - p2) * p3 * (1 - p4);
    const double pd = p2 * (p2 > p3 ? 1.0 : 0.0) + p3 * (p3 >= p2 ? 1.0 : 0.0);
    const bool A = p3 > p1, Bq = p3 > p2, Xq = p1 > p2, Yq = !Xq;
    const double xa = (Xq && A) ? 1.0 : 0.0, yb = (Yq && Bq) ? 1.0 : 0.0;
    const double xna = (Xq && !A) ? 1.0 : 0.0, ynb = (Yq && !Bq) ? 1.0 : 0.0;
    const double pdm1 = p3 * xa + p1 * (1.0 - xa);
    const double pdm2 = p3 * yb + p2 * (1.0 - yb);
    const double pdm3 = -p3 * xa + p3 * yb - p1 * xna + p2 * ynb;
    const double t11 = f4c_dev(p1, p3, p3, p4), t12 = f4c_dev(p4, p2, p3, p4);
    const double t21 = f4c_dev(p3, p2, p3, p4), t22 = f4c_dev(p1, p4, p3, p4);
    const double t31 = f4c_dev(p1, p2, p2, p4), t32 = f4c_dev(p1, p2, p3, p1);
    const double t41 = f4c_dev(p1, p2, p1, p4), t42 = f4c_dev(p1, p2, p3, p2);
    const double m4 = nmax(nmax(t11, t12), nmax(t21, t22));
    const double m8 = nmax(nmax(m4, nmax(t31, t32)), nmax(t41, t42));
    const double u1 = fabs(p1 - p2), u2 = fabs(p3 - p4);
    const double um = u1 * (u1 > u2 ? 1.0 : 0.0) + u2 * (u2 >= u1 ? 1.0 : 0.0);
    acc.d[0] += f4_dev(p1, p2, p3, p4);
    acc.d[1] += f4_dev(p1, p3, p3, p4);
    acc.d[2] += f4c_dev(p1, p2, p3, p4);
    acc.d[3] += t11;
    acc.d[4] += abba + baba;
    acc.d[5] += f4_dev(p1, pd, pd, p4);
    acc.d[6] += f4c_dev(p1, pd, pd, p4);
    acc.d[7] += f4_dev(pdm1, pdm2, pdm3, p4);
    acc.d[8] += f4c_dev(pdm1, pdm2, pdm3, p4);
    acc.d[9] += m4;
    acc.d[10] += m8;
    acc.d[11] += um * um;
    acc.d[12] += abba;
    acc.d[13] += baba;
    acc.d[14] += (1 - p1) * p2 * (1 - p3) * (1 - p4);
    acc.d[15] += p1 * (1 - p2) * (1 - p3) * (1 - p4);
}

// TMA producer (one elected lane of the producer warp): keeps the ring of tiles full.
template <int MODE>
__device__ __forceinline__ void k1_producer(const K1Params& prm, uint8_t* tiles, uint64_t* full, uint64_t* empty,
                                            volatile int* s_issued, int ntiles, int64_t t0) {
    for (int it = 0; it < ntiles; ++it) {
        const int stage = it % prm.stages;
        if (it >= prm.stages) mbar_wait(&empty[stage], (uint32_t)(((it / prm.stages) - 1) & 1));
        const int64_t s_lo = prm.site_begin + (t0 + it) * prm.T;
        int64_t rows = prm.site_end - s_lo;
        if (rows > prm.T) rows = prm.T;
        const uint32_t bytes = (uint32_t)(rows * prm.pitch);
        // positions of the tile ride along (rounded up to 16 bytes; the array has zeroed slack)
        const uint32_t pbytes = (MODE == MODE_COUNTS) ? 0u : (uint32_t)(((rows * 4 + 15) / 16) * 16);
        mbar_expect_tx(&full[stage], bytes + pbytes);
        const uint8_t* src = prm.geno + s_lo * prm.pitch;
        uint8_t* dst = tiles + (size_t)stage * prm.tile_bytes;
        for (uint32_t off = 0; off < bytes; off += 32768u) {
            const uint32_t n = (bytes - off) < 32768u ? (bytes - off) : 32768u;
            bulk_g2s(dst + off, src + off, n, &full[stage]);
        }
        if (pbytes) bulk_g2s(dst + (size_t)prm.T * prm.pitch, prm.pos + s_lo, pbytes, &full[stage]);
        // publish "tile `it` is armed": a consumer must not test a phase parity before its phase has
        // been armed, or try_wait.parity would alias it with the previous (already complete) phase
        __threadfence_block();
        atomicExch(const_cast<int*>(s_issued), it + 1);      // an atomic, so that racecheck sees the flag as synchronisation
    }
}

// Producer of the packed pass over the varied rows only (the whole producer warp): a stage is the tile's rows, the words
// [woff[t], woff[t + 1]) of the stream (room for row_cap three-plane rows), then the slots of its rows.  The tile's first site
// goes to s_site0[stage], and its one-plane and three-plane row counts to s_nvar[stage] (n1 | n3 << 16; R < 2^15), before the
// stage is armed, so the mbarrier's phase publishes them.  A tile is about a microsecond of HBM time, as long as a dependent
// load of its offsets, so the 32 lanes load the offsets of the next 32 tiles while the current 32 are issued.
__device__ __forceinline__ void k1_producer_uniform(const K1Params& prm, uint8_t* tiles, uint64_t* full, uint64_t* empty,
                                                    volatile int* s_issued, volatile uint32_t* s_nvar,
                                                    volatile long long* s_site0, int ntiles, int64_t t0, int lane) {
    auto ld = [&](const int64_t* a, int64_t t) { return t <= prm.num_tiles ? __ldg(a + t) : (int64_t)0; };
    auto ld_n1 = [&](int64_t t) { return t < prm.num_tiles ? __ldg(prm.n1 + t) : 0; };
    // lane l: row0, woff, site_lo and n1 of tile t0 + g + l
    int64_t cur = ld(prm.row0, t0 + lane), cur_w = ld(prm.woff, t0 + lane), cur_s = ld(prm.site_lo, t0 + lane);
    int cur_n1 = ld_n1(t0 + lane);
    for (int g = 0; g < ntiles; g += 32) {
        const int64_t nt = t0 + g + 32 + lane;
        const int64_t nxt = ld(prm.row0, nt), nxt_w = ld(prm.woff, nt), nxt_s = ld(prm.site_lo, nt);
        const int nxt_n1 = ld_n1(nt);
        const int kn = min(32, ntiles - g);
        for (int k = 0; k < kn; ++k) {
            const int64_t r0 = __shfl_sync(0xffffffffu, cur, k);
            const int64_t r1 = k < 31 ? __shfl_sync(0xffffffffu, cur, k + 1) : __shfl_sync(0xffffffffu, nxt, 0);
            const int64_t w0 = __shfl_sync(0xffffffffu, cur_w, k);
            const int64_t w1 = k < 31 ? __shfl_sync(0xffffffffu, cur_w, k + 1) : __shfl_sync(0xffffffffu, nxt_w, 0);
            const int64_t s0 = __shfl_sync(0xffffffffu, cur_s, k);
            const int n1 = __shfl_sync(0xffffffffu, cur_n1, k);
            if (lane == 0) {
                const int it = g + k;
                const int stage = it % prm.stages;
                if (it >= prm.stages) mbar_wait(&empty[stage], (uint32_t)(((it / prm.stages) - 1) & 1));
                const int64_t tile = t0 + it;
                const int nvar = (int)(r1 - r0);
                const uint32_t bytes = (uint32_t)((w1 - w0) * 4);
                const uint32_t sbytes = (uint32_t)(((nvar * 2 + 15) / 16) * 16);
                s_nvar[stage] = (uint32_t)n1 | (uint32_t)(nvar - n1) << 16;
                s_site0[stage] = s0;
                mbar_expect_tx(&full[stage], bytes + sbytes);
                const uint8_t* src = prm.geno + w0 * 4;
                uint8_t* dst = tiles + (size_t)stage * prm.tile_bytes;
                for (uint32_t off = 0; off < bytes; off += 32768u) {
                    const uint32_t n = (bytes - off) < 32768u ? (bytes - off) : 32768u;
                    bulk_g2s(dst + off, src + off, n, &full[stage]);
                }
                if (sbytes) bulk_g2s(dst + (size_t)prm.row_cap * prm.pitch, prm.slots + tile * prm.T, sbytes, &full[stage]);
                __threadfence_block();
                atomicExch(const_cast<int*>(s_issued), it + 1);
            }
            __syncwarp();
        }
        cur = nxt;
        cur_w = nxt_w;
        cur_s = nxt_s;
        cur_n1 = nxt_n1;
    }
}

// BYTES (POPGEN modes, every population <= 255 haplotypes): the four allele counts of a population travel as the
// bytes of one word, so that sum c^2 and sum c_X c_Y are ONE IDP.4A each, accumulate included.
template <int MODE, int P, int NW, bool BYTES = false>
__global__ void __launch_bounds__((NW + 1) * 32, 1) k1_site_pass(const __grid_constant__ K1Params prm) {
    constexpr int K1_THREADS = (NW + 1) * 32;
    constexpr int QI = ModeTraits<MODE, P>::QI, QU = ModeTraits<MODE, P>::QU, QD = ModeTraits<MODE, P>::QD;
    extern __shared__ __align__(128) uint8_t smem[];
    uint8_t* tiles = smem;
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + (size_t)prm.stages * prm.tile_bytes);   // [stages]
    uint64_t* empty = full + 8;                                                                  // [stages]
    volatile int* s_issued = reinterpret_cast<volatile int*>(empty + 8);   // tiles armed by the producer so far
    uint4* s_ent_mask = reinterpret_cast<uint4*>(smem + (size_t)prm.stages * prm.tile_bytes + 256);
    int32_t* s_ent_chunk = reinterpret_cast<int32_t*>(s_ent_mask + prm.n_ent);

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int b = blockIdx.x, B = gridDim.x;
    const int64_t t0 = (int64_t)b * prm.num_tiles / B, t1 = (int64_t)(b + 1) * prm.num_tiles / B;
    const int ntiles = (int)(t1 - t0);

    for (int e = tid; e < prm.n_ent; e += K1_THREADS) {
        s_ent_mask[e] = prm.ent_mask[e];
        s_ent_chunk[e] = prm.ent_chunk[e];
    }
    if (tid == 0) {
        for (int s = 0; s < prm.stages; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], (uint32_t)prm.wpt);
        }
        *s_issued = 0;
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    }
    __syncthreads();

    if (warp == NW) {
        if (lane == 0) k1_producer<MODE>(prm, tiles, full, empty, s_issued, ntiles, t0);
        return;
    }

    // ---------------- consumers: team m = warp / wpt owns tiles m, m + nteams, ... ----------------
    const int G = prm.G;
    const int spw = 32 / G;              // sites per warp per iteration
    const int gsub = lane / spw;         // which part of the row this lane walks
    const int sl = lane % spw;
    const int nteams = NW / prm.wpt;
    const int team = warp / prm.wpt, lw = warp % prm.wpt;
    const int sites_per_iter = prm.wpt * spw;

    Acc<QI, QU, QD> acc;
#pragma unroll
    for (int q = 0; q < QI; ++q) acc.i[q] = 0;
#pragma unroll
    for (int q = 0; q < QU; ++q) acc.u[q] = 0u;
    int since_flush = 0;     // sites added to the 32-bit sums since they were last flushed (warp-uniform)
#pragma unroll
    for (int q = 0; q < QD; ++q) acc.d[q] = 0.0;
    int cur_seg = -1;
    int64_t seg_end = -1;
    const int seg_first = (MODE == MODE_COUNTS) ? 0 : prm.cta_seg_first[b];
    const int64_t slot_base = (MODE == MODE_COUNTS) ? 0 : prm.cta_slot_off[b];
    auto flush = [&] { warp_flush<QI, QU, QD>(acc, cur_seg, prm.part, slot_base, seg_first, warp, lane, NW); };

    for (int it = team; it < ntiles; it += nteams) {
        const int stage = it % prm.stages;
        if (lane == 0)
            while (atomicAdd(const_cast<int*>(s_issued), 0) <= it) __nanosleep(20);
        __syncwarp();
        mbar_wait(&full[stage], (uint32_t)((it / prm.stages) & 1));
        const uint8_t* tile = tiles + (size_t)stage * prm.tile_bytes;
        const int64_t tile_site0 = prm.site_begin + (t0 + it) * prm.T;

        for (int i = 0; i < prm.I; ++i) {
            const int slot = i * sites_per_iter + lw * spw + sl;
            const int64_t site = tile_site0 + slot;
            const bool valid = site < prm.site_end;
            const bool owner = valid && (gsub == 0);
            const uint4* row = reinterpret_cast<const uint4*>(tile + (size_t)(valid ? slot : 0) * prm.pitch);
            // the tile's positions were staged behind its genotype rows by the producer
            int posv = 0;
            if (MODE != MODE_COUNTS)
                posv = owner ? reinterpret_cast<const int32_t*>(tile + (size_t)prm.T * prm.pitch)[slot] : 0;

            uint32_t n[P], c[BYTES ? 1 : P][4], cb[BYTES ? P : 1];
#pragma unroll
            for (int X = 0; X < P; ++X) {
                Tally t;
                tally_init(t);
                {   // the population's main run of fully-owned 16-byte chunks: no masks
                    int ch = prm.full_lo[X] + gsub;
                    const int hi = prm.full_hi[X];
                    for (; ch + 2 * G < hi; ch += 3 * G) add_chunks3(t, row[ch], row[ch + G], row[ch + 2 * G]);
                    if (ch + G < hi) add_chunks2(t, row[ch], row[ch + G]);
                    else if (ch < hi) add_chunks1(t, row[ch]);
                }
                {   // chunks shared with other populations / unused haplotypes / row padding: masked
                    int e = prm.ent_lo[X] + gsub;
                    const int hi = prm.ent_hi[X];
                    for (; e + G < hi; e += 2 * G)
                        add_chunks2(t, and4(row[s_ent_chunk[e]], s_ent_mask[e]), and4(row[s_ent_chunk[e + G]], s_ent_mask[e + G]));
                    if (e < hi) add_chunks1(t, and4(row[s_ent_chunk[e]], s_ent_mask[e]));
                }
                byte_flush(t);
                if (BYTES) {
                    // counts <= 255: one word per population, the G lanes of the site add their packed bytes
                    uint32_t pk = t.tA | (t.tC << 8) | (t.tG << 16) | (t.tT << 24);
                    for (int d = spw; d < 32; d <<= 1) pk += __shfl_xor_sync(0xffffffffu, pk, d);
                    cb[X] = pk;
                    n[X] = __dp4a(pk, 0x01010101u, 0u);
                } else {
                    // combine the G lanes of this site (16-bit fields: counts < 65536)
                    uint32_t p0 = t.tA | (t.tC << 16), p1 = t.tG | (t.tT << 16);
                    for (int d = spw; d < 32; d <<= 1) {
                        p0 += __shfl_xor_sync(0xffffffffu, p0, d);
                        p1 += __shfl_xor_sync(0xffffffffu, p1, d);
                    }
                    c[X][0] = p0 & 0xffffu;
                    c[X][1] = p0 >> 16;
                    c[X][2] = p1 & 0xffffu;
                    c[X][3] = p1 >> 16;
                    n[X] = c[X][0] + c[X][1] + c[X][2] + c[X][3];
                }
            }

            if (MODE == MODE_COUNTS) {
                if (owner) {
                    uint16_t* o = prm.counts_out + (site - prm.site_begin) * prm.counts_stride;
#pragma unroll
                    for (int X = 0; X < P; ++X)
                        if (X < prm.counts_pops) {
                            ushort4 v = make_ushort4((unsigned short)c[X][0], (unsigned short)c[X][1],
                                                     (unsigned short)c[X][2], (unsigned short)c[X][3]);
                            *reinterpret_cast<ushort4*>(o + X * 4) = v;
                        }
                }
                continue;
            }

            // ---- segment bookkeeping (warp-uniform control flow) ----
            int sg = cur_seg;
            if (owner && site >= seg_end) sg = find_seg(prm.brk, prm.nseg, cur_seg + 1, site);
            seg_step(sg, cur_seg, seg_end, since_flush, prm.brk, flush);

            if (MODE == MODE_POPGEN || MODE == MODE_POPGEN_FREQ) {
                bool allpres = true, allmiss = true;
#pragma unroll
                for (int X = 0; X < P; ++X) {
                    allpres = allpres && (n[X] == (uint32_t)prm.popN[X]);
                    allmiss = allmiss && (n[X] == 0u);
                }
                const bool pres = owner && allpres;
                const bool ragged = owner && !allpres && !allmiss;
                acc_limit_step(since_flush, prm.acc_limit, flush);
                acc.i[0] += pres ? 1 : 0;
                acc.i[1] += ragged ? 1 : 0;
                acc.i[2] += (long long)posv;
                if (BYTES) {
                    uint32_t cf[P];      // counts of a site that does not count are zeroed once, instead of every product
#pragma unroll
                    for (int X = 0; X < P; ++X) cf[X] = pres ? cb[X] : 0u;
#pragma unroll
                    for (int X = 0; X < P; ++X) {
                        if (MODE == MODE_POPGEN_FREQ) {
                            const uint32_t sq = __dp4a(cf[X], cb[X], 0u);
                            acc.u[X] += sq;
                            acc.u[P + P * (P - 1) / 2 + X] += (pres && sq != n[X] * n[X]) ? 1u : 0u;
                        } else {
                            acc.u[X] = __dp4a(cf[X], cb[X], acc.u[X]);
                        }
                    }
                    int kb = 0;
#pragma unroll
                    for (int X = 0; X < P; ++X)
#pragma unroll
                        for (int Y = X + 1; Y < P; ++Y) {
                            acc.u[P + kb] = __dp4a(cf[X], cb[Y], acc.u[P + kb]);
                            ++kb;
                        }
                }
                const uint32_t f = pres ? 1u : 0u;
#pragma unroll
                for (int X = 0; X < (BYTES ? 0 : P); ++X) {
                    const uint32_t sq = c[X][0] * c[X][0] + c[X][1] * c[X][1] + c[X][2] * c[X][2] + c[X][3] * c[X][3];
                    acc.u[X] += sq * f;
                    // groupFreqStats (genomics.py:1002-1028): a complete site is segregating in X iff sum c^2 < N^2
                    // (two populations share one 64-bit accumulator: 32-bit fields)
                    if (MODE == MODE_POPGEN_FREQ)
                        acc.u[P + P * (P - 1) / 2 + X] += (pres && sq != n[X] * n[X]) ? 1u : 0u;
                }
                int k = 0;
#pragma unroll
                for (int X = 0; X < (BYTES ? 0 : P); ++X)
#pragma unroll
                    for (int Y = X + 1; Y < P; ++Y) {
                        const uint32_t cr = c[X][0] * c[Y][0] + c[X][1] * c[Y][1] + c[X][2] * c[Y][2] + c[X][3] * c[Y][3];
                        acc.u[P + k] += cr * f;
                        ++k;
                    }
            }

            if (MODE == MODE_ABBA) {
                // genomics.py:1655-1662: biallelic over P1+P2+P3+O and enough data in each population
                uint32_t tot[4];
                int nall = 0;
#pragma unroll
                for (int a = 0; a < 4; ++a) {
                    tot[a] = c[0][a] + c[1][a] + c[2][a] + c[3][a];
                    nall += tot[a] > 0 ? 1 : 0;
                }
                bool good = owner && (nall == 2);
#pragma unroll
                for (int X = 0; X < 4; ++X) good = good && ((int)n[X] >= prm.thr[X]);
                acc.i[1] += good ? 1 : 0;
                acc.i[2] += (long long)posv;
                // derived allele: present overall, absent in the outgroup (1672). With two alleles overall and a
                // non-empty outgroup at most one allele qualifies, so one body serves the whole warp.
                int da = -1;
#pragma unroll
                for (int a = 0; a < 4; ++a)
                    if (tot[a] > 0 && c[3][a] == 0) da = a;
                const bool hit = good && n[3] > 0 && da >= 0;
                if (hit) {
                    const uint32_t k1 = da == 0 ? c[0][0] : (da == 1 ? c[0][1] : (da == 2 ? c[0][2] : c[0][3]));
                    const uint32_t k2 = da == 0 ? c[1][0] : (da == 1 ? c[1][1] : (da == 2 ? c[1][2] : c[1][3]));
                    const uint32_t k3 = da == 0 ? c[2][0] : (da == 1 ? c[2][1] : (da == 2 ? c[2][2] : c[2][3]));
                    // the derived allele is absent from the outgroup: p4 = 0/n4 = 0 and every (1 - p4) factor of the
                    // reference's formulas is exactly 1.0 — dropping those factors leaves the values bit-identical
                    const double p1 = (double)k1 / (double)n[0];
                    const double p2 = (double)k2 / (double)n[1];
                    const double p3 = (double)k3 / (double)n[2];
                    const double abba = (1 - p1) * p2 * p3;
                    const double baba = p1 * (1 - p2) * p3;
                    const double pd = p2 * (p2 > p3 ? 1.0 : 0.0) + p3 * (p3 >= p2 ? 1.0 : 0.0);
                    const double fd_den = (1 - p1) * pd * pd - p1 * (1 - pd) * pd;
                    const bool A = p3 > p1, Bq = p3 > p2, Xq = p1 > p2, Yq = !Xq;
                    const double xa = (Xq && A) ? 1.0 : 0.0, yb = (Yq && Bq) ? 1.0 : 0.0;
                    const double xna = (Xq && !A) ? 1.0 : 0.0, ynb = (Yq && !Bq) ? 1.0 : 0.0;
                    const double pdm1 = p3 * xa + p1 * (1.0 - xa);
                    const double pdm2 = p3 * yb + p2 * (1.0 - yb);
                    const double pdm3 = -p3 * xa + p3 * yb - p1 * xna + p2 * ynb;
                    const double fdm_den = (1 - pdm1) * pdm2 * pdm3 - pdm1 * (1 - pdm2) * pdm3;
                    acc.i[0] += 1;
                    acc.d[0] += abba;
                    acc.d[1] += baba;
                    acc.d[2] += abba - baba;
                    acc.d[3] += abba + baba;
                    acc.d[4] += fd_den;
                    acc.d[5] += fdm_den;
                }
            }

            if (MODE == MODE_FOURPOP) {
                // genomics.py:1595-1603: biallelic over P1+P2+P3+P4 and enough data in each population
                uint32_t tot[4];
                int nall = 0;
#pragma unroll
                for (int a = 0; a < 4; ++a) {
                    tot[a] = c[0][a] + c[1][a] + c[2][a] + c[3][a];
                    nall += tot[a] > 0 ? 1 : 0;
                }
                bool good = owner && (nall == 2);
#pragma unroll
                for (int X = 0; X < 4; ++X) good = good && ((int)n[X] >= prm.thr[X]);
                acc.i[1] += good ? 1 : 0;
                acc.i[2] += (long long)posv;
                int da = -1;
                if (prm.variant == 0) {
                    // np.argsort(all4freqs)[:,2] (1615): of the two alleles present, the rarer one; an exact tie is
                    // resolved by numpy's sort implementation in the reference — here the lower allele index
                    uint32_t best = 0xffffffffu;
#pragma unroll
                    for (int a = 3; a >= 0; --a)
                        if (tot[a] > 0 && tot[a] <= best) {
                            best = tot[a];
                            da = a;
                        }
                } else {
                    // polarize (1610): present overall, absent in P4 (needs data in P4: nan == 0 is False)
#pragma unroll
                    for (int a = 0; a < 4; ++a)
                        if (tot[a] > 0 && c[3][a] == 0) da = a;
                    if (n[3] == 0) da = -1;
                }
                bool hit = good && da >= 0;
                const uint32_t k1 = da == 0 ? c[0][0] : (da == 1 ? c[0][1] : (da == 2 ? c[0][2] : c[0][3]));
                const uint32_t k2 = da == 0 ? c[1][0] : (da == 1 ? c[1][1] : (da == 2 ? c[1][2] : c[1][3]));
                const uint32_t k3 = da == 0 ? c[2][0] : (da == 1 ? c[2][1] : (da == 2 ? c[2][2] : c[2][3]));
                const uint32_t k4 = da == 0 ? c[3][0] : (da == 1 ? c[3][1] : (da == 2 ? c[3][2] : c[3][3]));
                if (prm.variant == 2)       // fixed (1611-1614): frequency exactly 0 or 1 in P1, P2, P3 (nan fails both)
                    hit = hit && n[0] > 0 && n[1] > 0 && n[2] > 0 && (k1 == 0 || k1 == n[0]) && (k2 == 0 || k2 == n[1]) &&
                          (k3 == 0 || k3 == n[2]);
                const uint32_t e1 = k1 | (n[0] << 16), e2 = k2 | (n[1] << 16), e3 = k3 | (n[2] << 16), e4 = k4 | (n[3] << 16);
                acc.i[0] += hit ? 1 : 0;
                if (hit) fourpop_add(acc, e1, e2, e3, e4);
            }
        }

        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[stage]);   // this warp is done with the stage's bytes
    }
    if (MODE != MODE_COUNTS) flush();
}


// ---- lane-per-population variant for LONG rows (popgen modes, byte-packed counts) ----------------------------------
// P lanes share one site and lane X walks population X's chunks alone: no per-population cross-lane combine, every
// lane holds ONE packed count word, and the pair products are spread over the lanes — lane X accumulates
// sum c_X^2 and sum c_X c_{X+d} for d = 1 .. P/2 (partner words arrive by shuffle) — so a lane carries 1 + P/2 32-bit
// sums instead of P + P(P-1)/2.  The slot layout in global memory is the same as k1_site_pass's.
template <int QI, int QU>
__device__ __forceinline__ void warp_flush_lp(long long (&ai)[QI], uint32_t (&au)[QU], int cur_seg, unsigned long long* part,
                                              int64_t slot_base, int seg_first, int warp, int lane, int nw, int Q, int spw,
                                              int X, const int* s_q) {
    unsigned pending = __ballot_sync(0xffffffffu, cur_seg >= 0);
    while (pending) {
        const int leader = __ffs(pending) - 1;
        const int g = __shfl_sync(0xffffffffu, cur_seg, leader);
        const bool mine = (cur_seg == g);
        unsigned long long* dst = part + slot_base + ((int64_t)(g - seg_first) * nw + warp) * Q;
        const bool head = (lane % spw) == 0;
#pragma unroll
        for (int q = 0; q < QI; ++q) {      // site bookkeeping lives in the lanes of population 0
            long long v = (mine && X == 0) ? ai[q] : 0ll;
            for (int d = spw >> 1; d >= 1; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
            if (lane == 0) dst[q] = (unsigned long long)((long long)dst[q] + v);
            if (mine) ai[q] = 0;
        }
#pragma unroll
        for (int q = 0; q < QU; ++q) {      // lanes of the same population are neighbours: butterfly inside the group
            long long v = mine ? (long long)au[q] : 0ll;
            for (int d = spw >> 1; d >= 1; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
            const int slot = s_q[X * QU + q];
            if (head && slot >= 0) dst[slot] = (unsigned long long)((long long)dst[slot] + v);
            if (mine) au[q] = 0u;
        }
        pending &= ~__ballot_sync(0xffffffffu, mine);
    }
}

template <int MODE, int P, int NW>
__global__ void __launch_bounds__((NW + 1) * 32, 1) k1_site_pass_lp(const __grid_constant__ K1Params prm) {
    static_assert(MODE == MODE_POPGEN || MODE == MODE_POPGEN_FREQ || MODE == MODE_COUNTS, "lane-per-population: popgen / counts");
    constexpr int K1_THREADS = (NW + 1) * 32;
    constexpr int HP = P / 2;
    constexpr int QU = 1 + HP + (MODE == MODE_POPGEN_FREQ ? 1 : 0);      // sq, cross d = 1..P/2, (segregating sites)
    constexpr int spw = 32 / P;                                            // sites per warp per step
    const int Q = 3 + P + P * (P - 1) / 2 + (MODE == MODE_POPGEN_FREQ ? P : 0);
    extern __shared__ __align__(128) uint8_t smem[];
    uint8_t* tiles = smem;
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + (size_t)prm.stages * prm.tile_bytes);
    uint64_t* empty = full + 8;
    volatile int* s_issued = reinterpret_cast<volatile int*>(empty + 8);
    uint4* s_ent_mask = reinterpret_cast<uint4*>(smem + (size_t)prm.stages * prm.tile_bytes + 256);
    int32_t* s_ent_chunk = reinterpret_cast<int32_t*>(s_ent_mask + prm.n_ent);
    int* s_pop = s_ent_chunk + prm.n_ent;            // [5][P]: full_lo, full_hi, ent_lo, ent_hi, popN
    int* s_q = s_pop + 5 * P;                        // [P][QU]: slot word of each lane-local sum (-1 = unused)

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int b = blockIdx.x, B = gridDim.x;
    const int64_t t0 = (int64_t)b * prm.num_tiles / B, t1 = (int64_t)(b + 1) * prm.num_tiles / B;
    const int ntiles = (int)(t1 - t0);

    for (int e = tid; e < prm.n_ent; e += K1_THREADS) {
        s_ent_mask[e] = prm.ent_mask[e];
        s_ent_chunk[e] = prm.ent_chunk[e];
    }
    if (tid < P) {
        s_pop[0 * P + tid] = prm.full_lo[tid];
        s_pop[1 * P + tid] = prm.full_hi[tid];
        s_pop[2 * P + tid] = prm.ent_lo[tid];
        s_pop[3 * P + tid] = prm.ent_hi[tid];
        s_pop[4 * P + tid] = prm.popN[tid];
        // slot words (layout of k1_site_pass): [3 ints][P sq][pairs (x<y) in order][P segregating]
        const int x = tid;
        s_q[x * QU + 0] = 3 + x;
        for (int d = 1; d <= HP; ++d) {
            int slot = -1;
            if (d < HP || x < HP) {
                const int y = (x + d) % P;
                const int lo = x < y ? x : y, hi = x < y ? y : x;
                int kp = 0;
                for (int xx = 0; xx < lo; ++xx) kp += P - 1 - xx;
                kp += hi - lo - 1;
                slot = 3 + P + kp;
            }
            s_q[x * QU + d] = slot;
        }
        if (MODE == MODE_POPGEN_FREQ) s_q[x * QU + 1 + HP] = 3 + P + P * (P - 1) / 2 + x;
    }
    if (tid == 0) {
        for (int st = 0; st < prm.stages; ++st) {
            mbar_init(&full[st], 1);
            mbar_init(&empty[st], (uint32_t)prm.wpt);
        }
        *s_issued = 0;
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    }
    __syncthreads();

    if (warp == NW) {
        if (lane == 0) k1_producer<MODE>(prm, tiles, full, empty, s_issued, ntiles, t0);
        return;
    }

    const int X = lane / spw;                // this lane's population
    const int sl = lane % spw;               // its site within the warp's step
    unsigned site_lanes = 0;                 // the P lanes that share this lane's site
#pragma unroll
    for (int k = 0; k < P; ++k) site_lanes |= 1u << (sl + k * spw);
    const int nteams = NW / prm.wpt;
    const int team = warp / prm.wpt, lw = warp % prm.wpt;
    const int sites_per_iter = prm.wpt * spw;
    const int f_lo = s_pop[0 * P + X], f_hi = s_pop[1 * P + X], e_lo = s_pop[2 * P + X], e_hi = s_pop[3 * P + X];
    const uint32_t myN = (uint32_t)s_pop[4 * P + X];

    long long ai[3] = {0, 0, 0};
    uint32_t au[QU];
#pragma unroll
    for (int q = 0; q < QU; ++q) au[q] = 0u;
    int since_flush = 0;
    int cur_seg = -1;
    int64_t seg_end = -1;
    const int seg_first = (MODE == MODE_COUNTS) ? 0 : prm.cta_seg_first[b];
    const int64_t slot_base = (MODE == MODE_COUNTS) ? 0 : prm.cta_slot_off[b];
    auto flush = [&] { warp_flush_lp<3, QU>(ai, au, cur_seg, prm.part, slot_base, seg_first, warp, lane, NW, Q, spw, X, s_q); };

    for (int it = team; it < ntiles; it += nteams) {
        const int stage = it % prm.stages;
        if (lane == 0)
            while (atomicAdd(const_cast<int*>(s_issued), 0) <= it) __nanosleep(20);
        __syncwarp();
        mbar_wait(&full[stage], (uint32_t)((it / prm.stages) & 1));
        const uint8_t* tile = tiles + (size_t)stage * prm.tile_bytes;
        const int64_t tile_site0 = prm.site_begin + (t0 + it) * prm.T;

        for (int i = 0; i < prm.I; ++i) {
            const int slot = i * sites_per_iter + lw * spw + sl;
            const int64_t site = tile_site0 + slot;
            const bool valid = site < prm.site_end;
            const bool owner = valid && (X == 0);
            const uint4* row = reinterpret_cast<const uint4*>(tile + (size_t)(valid ? slot : 0) * prm.pitch);
            int posv = 0;
            if (MODE != MODE_COUNTS)
                posv = owner ? reinterpret_cast<const int32_t*>(tile + (size_t)prm.T * prm.pitch)[slot] : 0;

            Tally t;
            tally_init(t);
            {
                int ch = f_lo;
                for (; ch + 2 < f_hi; ch += 3) add_chunks3(t, row[ch], row[ch + 1], row[ch + 2]);
                if (ch + 1 < f_hi) add_chunks2(t, row[ch], row[ch + 1]);
                else if (ch < f_hi) add_chunks1(t, row[ch]);
            }
            {
                int e = e_lo;
                for (; e + 1 < e_hi; e += 2)
                    add_chunks2(t, and4(row[s_ent_chunk[e]], s_ent_mask[e]), and4(row[s_ent_chunk[e + 1]], s_ent_mask[e + 1]));
                if (e < e_hi) add_chunks1(t, and4(row[s_ent_chunk[e]], s_ent_mask[e]));
            }
            byte_flush(t);
            if (MODE == MODE_COUNTS) {       // every lane writes its own population's four counts
                if (valid && X < prm.counts_pops)
                    *reinterpret_cast<ushort4*>(prm.counts_out + (site - prm.site_begin) * prm.counts_stride + X * 4) =
                        make_ushort4((unsigned short)t.tA, (unsigned short)t.tC, (unsigned short)t.tG, (unsigned short)t.tT);
                continue;
            }
            const uint32_t cb = t.tA | (t.tC << 8) | (t.tG << 16) | (t.tT << 24);
            const uint32_t n = __dp4a(cb, 0x01010101u, 0u);

            // ---- segment bookkeeping: the site's owner lane looks it up, its P lanes share it ----
            int sg = cur_seg;
            if (owner && site >= seg_end) sg = find_seg(prm.brk, prm.nseg, cur_seg + 1, site);
            sg = __shfl_sync(0xffffffffu, sg, sl);                   // lane sl is population 0 of this site
            if (!valid) sg = cur_seg;
            seg_step(sg, cur_seg, seg_end, since_flush, prm.brk, flush);
            acc_limit_step(since_flush, prm.acc_limit, flush);

            const unsigned bf = __ballot_sync(0xffffffffu, valid && n == myN);
            const unsigned bz = __ballot_sync(0xffffffffu, valid && n == 0u);
            const bool allpres = (bf & site_lanes) == site_lanes;
            const bool allmiss = (bz & site_lanes) == site_lanes;
            const bool pres = valid && allpres;
            ai[0] += (owner && allpres) ? 1 : 0;
            ai[1] += (owner && !allpres && !allmiss) ? 1 : 0;
            ai[2] += (long long)posv;
            const uint32_t cf = pres ? cb : 0u;
            if (MODE == MODE_POPGEN_FREQ) {
                const uint32_t sq = __dp4a(cf, cb, 0u);
                au[0] += sq;
                au[1 + HP] += (pres && sq != n * n) ? 1u : 0u;
            } else {
                au[0] = __dp4a(cf, cb, au[0]);
            }
#pragma unroll
            for (int d = 1; d <= HP; ++d) {
                int px = X + d;
                if (px >= P) px -= P;
                const uint32_t cbp = __shfl_sync(0xffffffffu, cb, px * spw + sl);
                if (d < HP || X < HP) au[d] = __dp4a(cf, cbp, au[d]);
            }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[stage]);
    }
    if (MODE != MODE_COUNTS) flush();
}

// ---- bit-sliced popgen pass on the packed companion (ctx.cu pg_pack_rows) ------------------------------------------
// A site row is three planes of wd words: valid bits V, low code bits B0, high code bits B1 (A 0, C 1, G 2, T 3).  Population
// X is the (word, mask) entries [ent_lo[X], ent_hi[X]) of prm.word_ent; one entry adds
//   n = popc(M), c1 = popc(M & B0), c2 = popc(M & B1), c3 = popc(M & B0 & B1)      with M = V & mask
// and the allele counts are T = c3, C = c1 - c3, G = c2 - c3, A = n - c1 - c2 + c3.  The per-site sums and the slot layout
// are k1_site_pass's (MODE_POPGEN / MODE_POPGEN_FREQ), so k1_finalize folds the same integers into bit-identical records.
// Tiles and the ring are k1_site_pass's too, over rows of prm.pitch = packed bytes.  Rows start on 16-byte boundaries, so
// the 32 lanes of a warp reading the same word of their own rows meet in at most 8 banks: each lane starts its walk over a
// population's entries at an offset taken from its site index, which spreads the reads over the banks.
// UNI: the tiles hold only the varied rows (k1_producer_uniform) and the slot of each (its site's index in the tile;
// Tmax <= 32768).  A complete biallelic row (PG_CLS_VARIED2*: every haplotype called, two alleles) is one plane of wd words,
// "carries the higher of the two codes"; any other varied row is the three planes.  A tile stores its one-plane rows, then its
// three-plane rows, each kind word-major: word x of its row j at word x * n + j of the kind's run (n rows of the kind), so
// that the lanes reading the same word of consecutive rows read consecutive words, in distinct banks whatever the pitch.  A
// team takes the one-plane rows in blocks of 32, counted on the tensor cores (varied_mma, a row per lane; or gram_counts and
// the Gram of GRAM), then the three-plane rows Gv lanes per row: the plan's lanes per site (1 at C2 and C5, where more
// measured slower; 2 for rows of 1 KiB and more; PG_K1_UNI_GV forces 1 .. 32 for the tests), in blocks of 32 / Gv rows; block
// k of either kind goes to warp (k + tile) % wpt, the three-plane blocks numbered on from the one-plane ones.  The uniform
// sites and every site's position are not streamed: k1_finalize adds them from per-site prefix sums (UniformStream::pre).

// this lane's entries of population X: the first one, then steps of G (wrapping inside the population), as many as
// walk[X] >> 16 (first | count << 16: the table holds < 6144 entries).  The G lanes of a site (gsub = 0 .. G - 1) share the
// start offset, so that together they visit every entry once; sl (the site's index in the warp) spreads the banks.
template <int P>
__device__ __forceinline__ void packed_walk(const K1Params& prm, int G, int gsub, int sl, uint32_t (&walk)[P]) {
#pragma unroll
    for (int X = 0; X < P; ++X) {
        const int n = prm.ent_hi[X] - prm.ent_lo[X];
        const int cnt = gsub < n ? (n - gsub + G - 1) / G : 0;
        const int first = prm.ent_lo[X] + (n > 0 ? (((sl >> 2) & 7) + gsub) % n : 0);
        walk[X] = (uint32_t)first | ((uint32_t)cnt << 16);
    }
}

// the allele counts of one packed row, combined over the 32 / spw lanes that share it; walk[X] as packed_walk sets it
// A row's counts per population: n(X) haplotypes present and c(X, a) of allele a.  ArrCounts holds the five numbers;
// PkCounts holds the two 16-bit-field words they come from and derives them where they are used, which can keep 3 * P fewer
// registers live between the walk and the sums.
template <int P>
struct ArrCounts {
    uint32_t nn[P], cc[P][4];
    __device__ __forceinline__ void set(int X, uint32_t p0, uint32_t p1) {
        const uint32_t m = p0 & 0xffffu, n1 = p0 >> 16, n2 = p1 & 0xffffu, n3 = p1 >> 16;
        nn[X] = m;
        cc[X][0] = m - n1 - n2 + n3;
        cc[X][1] = n1 - n3;
        cc[X][2] = n2 - n3;
        cc[X][3] = n3;
    }
    __device__ __forceinline__ uint32_t n(int X) const { return nn[X]; }
    __device__ __forceinline__ uint32_t c(int X, int a) const { return cc[X][a]; }
};
template <int P>
struct PkCounts {
    uint32_t p0[P], p1[P];
    __device__ __forceinline__ void set(int X, uint32_t a, uint32_t b) {
        p0[X] = a;
        p1[X] = b;
    }
    __device__ __forceinline__ uint32_t n(int X) const { return p0[X] & 0xffffu; }
    __device__ __forceinline__ uint32_t c(int X, int a) const {
        const uint32_t n1 = p0[X] >> 16, n2 = p1[X] & 0xffffu, n3 = p1[X] >> 16;
        return a == 0 ? (p0[X] & 0xffffu) - n1 - n2 + n3 : (a == 1 ? n1 - n3 : (a == 2 ? n2 - n3 : n3));
    }
};

template <int P, class W, class CT>
__device__ __forceinline__ void packed_counts(const K1Params& prm, const uint2* s_ent, const uint32_t* row, const W& walk,
                                              int G, int spw, CT& ct) {
    const int wd = prm.wd;
#pragma unroll
    for (int X = 0; X < P; ++X) {
        uint32_t a = 0u, a1 = 0u, a2 = 0u, a3 = 0u;
        const int lo = prm.ent_lo[X], span = prm.ent_hi[X] - lo;
        int e = (int)(walk[X] & 0xffffu);
        const int cnt = (int)(walk[X] >> 16);
        for (int k = 0; k < cnt; ++k) {
            const uint2 em = s_ent[e];
            const uint32_t m = row[em.x] & em.y;
            const uint32_t b0 = row[wd + em.x], b1 = row[2 * wd + em.x];
            a += __popc(m);
            a1 += __popc(m & b0);
            a2 += __popc(m & b1);
            a3 += __popc(m & b0 & b1);
            e += G;
            if (e >= lo + span) e -= span;
        }
        // combine the G lanes of this site (16-bit fields: counts < 65536)
        uint32_t p0 = a | (a1 << 16), p1 = a2 | (a3 << 16);
        for (int d = spw; d < 32; d <<= 1) {
            p0 += __shfl_xor_sync(0xffffffffu, p0, d);
            p1 += __shfl_xor_sync(0xffffffffu, p1, d);
        }
        ct.set(X, p0, p1);
    }
}

// packed_counts for a varied row stored word-major (word x at row[x * nvar]).  Lane gsub of the row's Gv lanes takes entries
// gsub, gsub + Gv, ... of each population.  ONE (Gv = 1): every lane walks all the entries in the same order, so the entry
// index is warp-uniform, an entry's load is a broadcast and the lanes' row words are consecutive words.
template <int P, bool ONE, class CT>
__device__ __forceinline__ void varied_counts(const K1Params& prm, const uint2* s_ent, const uint32_t* row, int nvar, int Gv,
                                              int gsub, int spv, CT& ct) {
    const int pn = prm.wd * nvar;     // words from one plane to the next
#pragma unroll
    for (int X = 0; X < P; ++X) {
        uint32_t a = 0u, a1 = 0u, a2 = 0u, a3 = 0u;
        // not unrolled: unrolled, the walks of the two variants made the kernel four times longer and slower at C2
#pragma unroll 1
        for (int e = prm.ent_lo[X] + (ONE ? 0 : gsub); e < prm.ent_hi[X]; e += (ONE ? 1 : Gv)) {
            const uint2 em = s_ent[e];
            const uint32_t* w = row + em.x * nvar;
            const uint32_t m = w[0] & em.y;
            const uint32_t b0 = w[pn], b1 = w[2 * pn];
            a += __popc(m);
            a1 += __popc(m & b0);
            a2 += __popc(m & b1);
            a3 += __popc(m & b0 & b1);
        }
        uint32_t p0 = a | (a1 << 16), p1 = a2 | (a3 << 16);
        for (int d = spv; !ONE && d < 32; d <<= 1) {
            p0 += __shfl_xor_sync(0xffffffffu, p0, d);
            p1 += __shfl_xor_sync(0xffffffffu, p1, d);
        }
        ct.set(X, p0, p1);
    }
}

// A complete biallelic row's counts: every haplotype of population X is present, k(X) of them carry the higher code.
template <int P>
struct BitCounts {
    uint32_t k[P];
    const int* N;
    __device__ __forceinline__ void set(int X, uint32_t kx) { k[X] = kx; }
    __device__ __forceinline__ uint32_t n(int X) const { return (uint32_t)N[X]; }
    __device__ __forceinline__ uint32_t c(int X, int a) const { return a == 0 ? (uint32_t)N[X] - k[X] : (a == 1 ? k[X] : 0u); }
};

// d += popc-sums of (A AND B) over 256 haplotypes, 16 rows x 8 populations (BMMA.168256.AND.POPC on sm_90a)
__device__ __forceinline__ void bmma_and_popc(int (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint2 b) {
    asm("mma.sync.aligned.m16n8k256.row.col.s32.b1.b1.s32.and.popc {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
        "{%0, %1, %2, %3};"
        : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3])
        : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b.x), "r"(b.y));
}

// the row of its block of 32 one-plane rows whose counts a lane gets from varied_mma
__device__ __forceinline__ int mma_row(int lane) { return (lane >> 2) + 8 * (lane & 3); }

// The counts of the one-plane rows [r, r + 32) (word x of row j at rows[x * n1 + j]) on the tensor cores: k(X) is the binary
// matrix product of the rows' bits and the populations' member bits, 16 rows x 8 populations x 256 haplotypes per mma.  The
// block is two m16 tiles (rows r .. r + 15, r + 16 .. r + 31) over K-blocks of 8 words.  Lane (g, t) = (lane / 4, lane % 4)
// holds words 8 kb + t and 8 kb + 4 + t of a tile's rows g and g + 8 (A) and, in s_bf[32 kb + lane], of population g's
// members (B, build_word_tables: zero past wd words, past H, for no population and for g >= the padded populations, so that a
// row's bits past H count for nothing).  Words past wd are not read: they lie outside the one-plane rows.  Rows past n1 read
// row n1 - 1 instead, so every load stays in the tile's one-plane rows; their counts are dropped (add_row's owner).  Lane
// (g, t) ends with populations 2t, 2t + 1 of the block's rows g + 8q (q = 0 .. 3), as 16-bit pairs (counts < 65536), and
// takes those of its own row g + 8t (mma_row) in four exchanges: in exchange j it sends pair q = t ^ j to lane ^ j, and gets
// populations 2 (t ^ j), 2 (t ^ j) + 1 of its row.
template <int P>
__device__ __forceinline__ void varied_mma(const uint2* s_bf, const uint32_t* rows, int n1, int wd, int r, int lane,
                                           BitCounts<P>& ct) {
    static_assert(P <= 4, "one-plane rows: up to 4 (padded) populations");
    const int g = lane >> 2, t = lane & 3;
    const int j0 = min(r + g, n1 - 1), j1 = min(r + g + 8, n1 - 1), j2 = min(r + g + 16, n1 - 1), j3 = min(r + g + 24, n1 - 1);
    int d0[4] = {0, 0, 0, 0}, d1[4] = {0, 0, 0, 0};
    const uint32_t* w = rows + t * n1;    // word 8 kb + t of the rows; word 8 kb + 4 + t at w + 4 n1
    for (int kb = 0; kb * 8 < wd; ++kb, w += 8 * n1) {
        const bool lo = kb * 8 + t < wd, hi = kb * 8 + 4 + t < wd;
        const uint32_t* v = w + 4 * n1;
        const uint2 b = s_bf[kb * 32 + lane];
        bmma_and_popc(d0, lo ? w[j0] : 0u, lo ? w[j1] : 0u, hi ? v[j0] : 0u, hi ? v[j1] : 0u, b);
        bmma_and_popc(d1, lo ? w[j2] : 0u, lo ? w[j3] : 0u, hi ? v[j2] : 0u, hi ? v[j3] : 0u, b);
    }
    const uint32_t pk[4] = {(uint32_t)d0[0] | (uint32_t)d0[1] << 16, (uint32_t)d0[2] | (uint32_t)d0[3] << 16,
                            (uint32_t)d1[0] | (uint32_t)d1[1] << 16, (uint32_t)d1[2] | (uint32_t)d1[3] << 16};
    uint32_t k01 = 0u, k23 = 0u;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int q = t ^ j;
        const uint32_t v = __shfl_xor_sync(0xffffffffu, (q & 2) ? ((q & 1) ? pk[3] : pk[2]) : ((q & 1) ? pk[1] : pk[0]), j);
        if (q == 0) k01 = v;
        if (q == 1) k23 = v;
    }
    ct.set(0, k01 & 0xffffu);
    ct.set(1, k01 >> 16);
    if constexpr (P > 2) {
        ct.set(2, k23 & 0xffffu);
        ct.set(3, k23 >> 16);
    }
}

// The counts of the one-plane rows [r, r + 32) as bytes (every population has at most 255 haplotypes), populations as M and
// rows as N: k(X) is the binary product of the populations' member bits (A: s_bf[32 kb + lane] holds population g's words
// 8 kb + t and 8 kb + 4 + t, A rows 8 .. 15 are zero) and the bits of 8 rows (B), in four n-tiles of 8 rows.  Lane (g, t)
// loads words 8 kb + t and 8 kb + 4 + t of row r + 8 j + g of n-tile j, zero past n1, and ends with k(g) of the block's rows
// 8 j + 2 t and 8 j + 2 t + 1: rows 2 t, 2 t + 1, 8 + 2 t, 9 + 2 t in the bytes of k0, the same rows + 16 in k1 (gram_row).
__device__ __forceinline__ void gram_counts(const uint2* s_bf, const uint32_t* rows, int n1, int wd, int r, int lane,
                                            uint32_t& k0, uint32_t& k1) {
    const int g = lane >> 2, t = lane & 3, j = r + g;
    const bool v0 = j < n1, v1 = j + 8 < n1, v2 = j + 16 < n1, v3 = j + 24 < n1;
    int d[4][4] = {{0, 0, 0, 0}, {0, 0, 0, 0}, {0, 0, 0, 0}, {0, 0, 0, 0}};
    const uint32_t* w = rows + t * n1 + j;    // word 8 kb + t of row j; word 8 kb + 4 + t at w + 4 n1
    for (int kb = 0; kb * 8 < wd; ++kb, w += 8 * n1) {
        const bool lo = kb * 8 + t < wd, hi = kb * 8 + 4 + t < wd;
        const uint32_t* v = w + 4 * n1;
        const uint2 a = s_bf[kb * 32 + lane];
        bmma_and_popc(d[0], a.x, 0u, a.y, 0u, make_uint2(lo && v0 ? w[0] : 0u, hi && v0 ? v[0] : 0u));
        bmma_and_popc(d[1], a.x, 0u, a.y, 0u, make_uint2(lo && v1 ? w[8] : 0u, hi && v1 ? v[8] : 0u));
        bmma_and_popc(d[2], a.x, 0u, a.y, 0u, make_uint2(lo && v2 ? w[16] : 0u, hi && v2 ? v[16] : 0u));
        bmma_and_popc(d[3], a.x, 0u, a.y, 0u, make_uint2(lo && v3 ? w[24] : 0u, hi && v3 ? v[24] : 0u));
    }
    k0 = (uint32_t)d[0][0] | (uint32_t)d[0][1] << 8 | (uint32_t)d[1][0] << 16 | (uint32_t)d[1][1] << 24;
    k1 = (uint32_t)d[2][0] | (uint32_t)d[2][1] << 8 | (uint32_t)d[3][0] << 16 | (uint32_t)d[3][1] << 24;
}

// the bytes of gram_counts' k0 (half = 0) or k1 (half = 1) in lane t whose rows are in the row mask m (bit i: row i of the block)
__device__ __forceinline__ uint32_t gram_bytes(uint32_t m, int t, int half) {
    const uint32_t x = m >> (2 * t + 16 * half);
    const uint32_t b = (x & 3u) | ((x >> 6) & 0xcu);           // rows 2t, 2t + 1, 8 + 2t, 9 + 2t
    return ((b * 0x00204081u) & 0x01010101u) * 0xffu;          // bit i to byte i
}

// d[0..1] += row g, columns 2t, 2t + 1 of the s32 product of A (16 x 32 bytes) and B (32 x 8 bytes), A rows 8 .. 15 zero
// (IMMA.16832.U8.U8 on sm_90a)
__device__ __forceinline__ void imma_u8(int (&d)[2], uint32_t a0, uint32_t a2, uint32_t b0, uint32_t b1) {
    int z0, z1;
    asm("mma.sync.aligned.m16n8k32.row.col.s32.u8.u8.s32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %10, %10};"
        : "+r"(d[0]), "+r"(d[1]), "=r"(z0), "=r"(z1)
        : "r"(a0), "r"(0u), "r"(a2), "r"(0u), "r"(b0), "r"(b1), "r"(0));
}

// whether the site (of the lane that owns it) has every haplotype of every population, or some but not all of them
template <int P, class CT>
__device__ __forceinline__ void packed_class(const K1Params& prm, bool owner, const CT& ct, bool& pres, bool& ragged) {
    bool allpres = true, allmiss = true;
#pragma unroll
    for (int X = 0; X < P; ++X) {
        allpres = allpres && (ct.n(X) == (uint32_t)prm.popN[X]);
        allmiss = allmiss && (ct.n(X) == 0u);
    }
    pres = owner && allpres;
    ragged = owner && !allpres && !allmiss;
}

// one site's sums but its position
template <int MODE, int P, class ACC, class CT>
__device__ __forceinline__ void packed_add(ACC& acc, bool pres, bool ragged, const CT& ct) {
    acc.i[0] += pres ? 1 : 0;
    acc.i[1] += ragged ? 1 : 0;
    const uint32_t f = pres ? 1u : 0u;
#pragma unroll
    for (int X = 0; X < P; ++X) {
        const uint32_t sq = ct.c(X, 0) * ct.c(X, 0) + ct.c(X, 1) * ct.c(X, 1) + ct.c(X, 2) * ct.c(X, 2) + ct.c(X, 3) * ct.c(X, 3);
        acc.u[X] += sq * f;
        if (MODE == MODE_POPGEN_FREQ) acc.u[P + P * (P - 1) / 2 + X] += (pres && sq != ct.n(X) * ct.n(X)) ? 1u : 0u;
    }
    int k = 0;
#pragma unroll
    for (int X = 0; X < P; ++X)
#pragma unroll
        for (int Y = X + 1; Y < P; ++Y) {
            const uint32_t cr = ct.c(X, 0) * ct.c(Y, 0) + ct.c(X, 1) * ct.c(Y, 1) + ct.c(X, 2) * ct.c(Y, 2) + ct.c(X, 3) * ct.c(Y, 3);
            acc.u[P + k] += cr * f;
            ++k;
        }
}

// GRAM (UNI, P < 8, every population <= 255 haplotypes: K1Params::bytes): the one-plane rows are not added row by row.  A
// complete biallelic row has every haplotype present and none ragged, and its counts are c(X, 0) = N_X - k_X, c(X, 1) = k_X,
// so a run of n such rows in one segment adds
//   sum c_Xa^2 = n N_X^2 - 2 N_X sum k_X + 2 sum k_X^2,   sum c_Xa c_Ya = n N_X N_Y - N_X sum k_Y - N_Y sum k_X + 2 sum k_X k_Y,
// exact integers, equal to what the rows add one by one.  The warp keeps the Gram D = K^T K of its rows' byte counts in the
// tensor cores' s32 accumulator (gram_counts, then one IMMA per block of 32 rows), with a column of ones per valid row
// (lane g = 4 of the operand) for sum k_X and n, and folds D into its slot (gram_flush) when the rows move to another
// segment or before an entry could overflow.
template <int MODE, int P, int NW, bool UNI = false, bool GRAM = false>
__global__ void __launch_bounds__((NW + 1) * 32, 1) k1_site_pass_packed(const __grid_constant__ K1Params prm) {
    static_assert(MODE == MODE_POPGEN || MODE == MODE_POPGEN_FREQ, "packed site pass: popgen modes");
    static_assert(!GRAM || (UNI && P <= 4), "the Gram of the one-plane rows: varied-row stream, up to 4 (padded) populations");
    constexpr int K1_THREADS = (NW + 1) * 32;
    constexpr int QI = ModeTraits<MODE, P>::QI, QU = ModeTraits<MODE, P>::QU;
    extern __shared__ __align__(128) uint8_t smem[];
    uint8_t* tiles = smem;
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + (size_t)prm.stages * prm.tile_bytes);   // [stages]
    uint64_t* empty = full + 8;                                                                  // [stages]
    volatile int* s_issued = reinterpret_cast<volatile int*>(empty + 8);
    volatile uint32_t* s_nvar = reinterpret_cast<volatile uint32_t*>(s_issued + 8);   // UNI: n1 | n3 << 16 [stages]
    volatile long long* s_site0 = reinterpret_cast<volatile long long*>(s_issued + 16);   // UNI: first site [stages]
    uint2* s_ent = reinterpret_cast<uint2*>(smem + (size_t)prm.stages * prm.tile_bytes + 256);
    uint2* s_bf = s_ent + prm.n_ent;                                  // UNI, P < 8: varied_mma's B operand

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int b = blockIdx.x, B = gridDim.x;
    const int64_t t0 = (int64_t)b * prm.num_tiles / B, t1 = (int64_t)(b + 1) * prm.num_tiles / B;
    const int ntiles = (int)(t1 - t0);

    for (int e = tid; e < prm.n_ent; e += K1_THREADS) s_ent[e] = prm.word_ent[e];
    if constexpr (UNI && P < 8)
        for (int e = tid; e < (prm.wd + 7) / 8 * 32; e += K1_THREADS) s_bf[e] = prm.bit_frag[e];
    const int Gv = prm.uni_gv > 0 ? prm.uni_gv : prm.G;                    // UNI: lanes per varied row, the plan's per site
    if (tid == 0) {
        for (int s = 0; s < prm.stages; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], (uint32_t)prm.wpt);
        }
        *s_issued = 0;
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    }
    __syncthreads();

    if (warp == NW) {
        if (UNI) k1_producer_uniform(prm, tiles, full, empty, s_issued, s_nvar, s_site0, ntiles, t0, lane);
        else if (lane == 0) k1_producer<MODE>(prm, tiles, full, empty, s_issued, ntiles, t0);
        return;
    }

    const int nteams = NW / prm.wpt;
    const int team = warp / prm.wpt, lw = warp % prm.wpt;

    Acc<QI, QU, 0> acc;
#pragma unroll
    for (int q = 0; q < QI; ++q) acc.i[q] = 0;
#pragma unroll
    for (int q = 0; q < QU; ++q) acc.u[q] = 0u;
    int since_flush = 0;
    int cur_seg = -1;
    int64_t seg_end = -1;
    const int seg_first = prm.cta_seg_first[b];
    const int64_t slot_base = prm.cta_slot_off[b];

    if constexpr (!UNI) {
        const int G = prm.G;
        const int spw = 32 / G;
        const int gsub = lane / spw;
        const int sl = lane % spw;
        const int sites_per_iter = prm.wpt * spw;
        uint32_t walk[P];
        packed_walk<P>(prm, G, gsub, sl, walk);

        for (int it = team; it < ntiles; it += nteams) {
            const int stage = it % prm.stages;
            if (lane == 0)
                while (atomicAdd(const_cast<int*>(s_issued), 0) <= it) __nanosleep(20);
            __syncwarp();
            mbar_wait(&full[stage], (uint32_t)((it / prm.stages) & 1));
            const uint8_t* tile = tiles + (size_t)stage * prm.tile_bytes;
            const int64_t tile_site0 = prm.site_begin + (t0 + it) * prm.T;

            for (int i = 0; i < prm.I; ++i) {
                const int slot = i * sites_per_iter + lw * spw + sl;
                const int64_t site = tile_site0 + slot;
                const bool valid = site < prm.site_end;
                const bool owner = valid && (gsub == 0);
                const uint32_t* row = reinterpret_cast<const uint32_t*>(tile + (size_t)(valid ? slot : 0) * prm.pitch);
                const int posv = owner ? reinterpret_cast<const int32_t*>(tile + (size_t)prm.T * prm.pitch)[slot] : 0;

                ArrCounts<P> ct;
                packed_counts<P>(prm, s_ent, row, walk, G, spw, ct);

                // ---- segment bookkeeping: seg_step and acc_limit_step written out.  Calling them (flush as a lambda) here
                // changes the instruction schedule ptxas (sm_90a) picks for six of the packed kernels ----
                int sg = cur_seg;
                if (owner && site >= seg_end) sg = find_seg(prm.brk, prm.nseg, cur_seg + 1, site);
                if (__any_sync(0xffffffffu, sg != cur_seg)) {
                    warp_flush<QI, QU, 0>(acc, cur_seg, prm.part, slot_base, seg_first, warp, lane, NW);
                    since_flush = 0;
                    if (sg != cur_seg) {
                        cur_seg = sg;
                        seg_end = __ldg(prm.brk + sg + 1);
                    }
                }
                bool pres, ragged;
                packed_class<P>(prm, owner, ct, pres, ragged);
                if (++since_flush > prm.acc_limit) {      // the 32-bit sums must not overflow
                    warp_flush<QI, QU, 0>(acc, cur_seg, prm.part, slot_base, seg_first, warp, lane, NW);
                    since_flush = 1;
                }
                acc.i[2] += (long long)posv;
                packed_add<MODE, P>(acc, pres, ragged, ct);
            }

            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[stage]);
        }
    } else {
        const int spv = 32 / Gv, gsub = lane / spv, sl = lane % spv, wpt = prm.wpt;
        // One row's sums, its segment first.  A lane's rows come in site order within each kind, so only the three-plane
        // rows (back) may lie before the lane's segment: the one-plane rows of the same tile may have moved it on.
        auto add_row = [&](int64_t site, bool owner, const auto& ct, bool back) {
            int sg = cur_seg;
            if (owner && site >= seg_end) sg = next_seg(prm.brk, prm.nseg, cur_seg + 1, site);
            else if (back && owner && site < __ldg(prm.brk + cur_seg)) sg = find_seg(prm.brk, cur_seg, 0, site);
            if (__any_sync(0xffffffffu, sg != cur_seg)) {
                warp_flush<QI, QU, 0>(acc, cur_seg, prm.part, slot_base, seg_first, warp, lane, NW);
                since_flush = 0;
                // A lane that owns no row here (a row's other lanes, lanes past the block) would keep an old segment
                // and flush the warp once more when it next owns one.  Its sums are zero now, so it takes the warp's last
                // segment, which no later row of it lies before but for a three-plane row, which searches back.
                const int last = __reduce_max_sync(0xffffffffu, sg);
                const int to = owner ? sg : last;
                if (to != cur_seg) {
                    cur_seg = to;
                    seg_end = __ldg(prm.brk + to + 1);
                }
            }
            bool pres, ragged;
            packed_class<P>(prm, owner, ct, pres, ragged);
            if (++since_flush > prm.acc_limit) {      // the 32-bit sums must not overflow
                warp_flush<QI, QU, 0>(acc, cur_seg, prm.part, slot_base, seg_first, warp, lane, NW);
                since_flush = 1;
            }
            packed_add<MODE, P>(acc, pres, ragged, ct);
        };

        // GRAM: the Gram's own segment (warp-uniform; the warp's one-plane rows come in site order), D[g][2t], D[g][2t + 1]
        // in lane (g, t), the rows it holds, and per lane the rows with 0 < k_g < N_g (popFreq's segregating sites)
        int gseg = -1, grows = 0;
        int64_t gseg_end = -1;
        int gd[2] = {0, 0};
        uint32_t gfreq = 0u;
        const uint32_t gN4 = (lane >> 2) < P ? (uint32_t)prm.popN[min(lane >> 2, P - 1)] * 0x01010101u : 0u;
        // the entries of D are below 2^31 while the rows number at most 2^31 / maxN^2 (acc_limit is 2^32 / maxN^2)
        const int glimit = max(prm.acc_limit / 2, 32);
        // lane q < QU adds slot word QI + q: the sums of population X = Y (q < P), of the pair X < Y (then), or X's segregating
        // sites; lane 31 adds the complete sites (word 0)
        auto gram_flush = [&]() {
            if (grows == 0) return;
            __syncwarp();       // the lanes' read-modify-writes after warp_flush's, of the same slot
            int X = 0, Y = 0;
            long long NX = 0, NY = 0;
            int k = P;
#pragma unroll
            for (int x = 0; x < P; ++x) {
                if (lane == x || lane == P + P * (P - 1) / 2 + x) X = Y = x;
#pragma unroll
                for (int y = x + 1; y < P; ++y, ++k)
                    if (lane == k) {
                        X = x;
                        Y = y;
                    }
            }
#pragma unroll
            for (int x = 0; x < P; ++x) {
                if (X == x) NX = prm.popN[x];
                if (Y == x) NY = prm.popN[x];
            }
            const int src = 4 * X + (Y >> 1);                                          // D[X][Y]
            const int d0 = __shfl_sync(0xffffffffu, gd[0], src), d1 = __shfl_sync(0xffffffffu, gd[1], src);
            const long long SX = __shfl_sync(0xffffffffu, gd[0], 4 * X + 2);           // D[X][4] = sum k_X
            const long long SY = __shfl_sync(0xffffffffu, gd[0], 4 * Y + 2);
            const long long n = __shfl_sync(0xffffffffu, gd[0], 18);                   // D[4][4] = rows
            uint32_t f = gfreq;
            f += __shfl_xor_sync(0xffffffffu, f, 1);
            f += __shfl_xor_sync(0xffffffffu, f, 2);
            f = __shfl_sync(0xffffffffu, f, 4 * X);
            unsigned long long* dst = prm.part + slot_base + ((int64_t)(gseg - seg_first) * NW + warp) * (QI + QU);
            if (lane < P + P * (P - 1) / 2)
                dst[QI + lane] += (unsigned long long)(n * NX * NY - NX * SY - NY * SX + 2ll * ((Y & 1) ? d1 : d0));
            else if (lane < QU)
                dst[QI + lane] += (unsigned long long)f;
            else if (lane == 31)
                dst[0] += (unsigned long long)n;
            __syncwarp();
            gd[0] = gd[1] = 0;
            gfreq = 0u;
            grows = 0;
        };
        // the rows of the block in the row mask m (of the Gram's segment) into the Gram
        auto gram_add = [&](uint32_t k0, uint32_t k1, uint32_t m) {
            if (grows + __popc(m) > glimit) gram_flush();
            grows += __popc(m);
            const int t = lane & 3;
            if ((lane >> 2) == 4) k0 = k1 = 0x01010101u;     // operand row / column 4: a one per row
            k0 &= gram_bytes(m, t, 0);
            k1 &= gram_bytes(m, t, 1);
            imma_u8(gd, k0, k1, k0, k1);
            if (MODE == MODE_POPGEN_FREQ)
                gfreq += __popc((__vsetgtu4(k0, 0u) & __vsetltu4(k0, gN4)) | (__vsetgtu4(k1, 0u) & __vsetltu4(k1, gN4)) << 1);
        };

        for (int it = team; it < ntiles; it += nteams) {
            const int stage = it % prm.stages;
            if (lane == 0)
                while (atomicAdd(const_cast<int*>(s_issued), 0) <= it) __nanosleep(20);
            __syncwarp();
            mbar_wait(&full[stage], (uint32_t)((it / prm.stages) & 1));
            const uint8_t* tile = tiles + (size_t)stage * prm.tile_bytes;
            const int64_t tile_site0 = s_site0[stage];
            const uint32_t sizes = s_nvar[stage];
            const int n1 = (int)(sizes & 0xffffu), n3 = (int)(sizes >> 16);
            const uint16_t* s_slot = reinterpret_cast<const uint16_t*>(tile + (size_t)prm.row_cap * prm.pitch);
            // block k of the tile goes to warp (k + rot) % wpt: the one-plane rows' blocks of 32 first, then the three-plane
            // rows' blocks of spv
            const int rot = (int)((t0 + it) % wpt), nb1 = (n1 + 31) / 32;

            // ---- one-plane rows, a row per lane (none at 8 populations: uniform_prepare streams three planes there) ----
            if constexpr (GRAM) {
                for (int r = ((lw - rot + wpt) % wpt) * 32; r < n1; r += wpt * 32) {
                    uint32_t k0, k1;
                    gram_counts(s_bf, reinterpret_cast<const uint32_t*>(tile), n1, prm.wd, r, lane, k0, k1);
                    const int nv = min(32, n1 - r);
                    uint32_t pending = nv == 32 ? 0xffffffffu : (1u << nv) - 1u;
                    if (tile_site0 + s_slot[r + nv - 1] < gseg_end) {
                        gram_add(k0, k1, pending);      // the whole block lies in the Gram's segment
                        continue;
                    }
                    // the block's rows segment by segment
                    const int64_t site = tile_site0 + s_slot[r + min(lane, nv - 1)];
                    while (pending) {
                        const int64_t first = __shfl_sync(0xffffffffu, site, __ffs(pending) - 1);
                        if (first >= gseg_end) {
                            gram_flush();
                            gseg = next_seg(prm.brk, prm.nseg, gseg + 1, first);
                            gseg_end = __ldg(prm.brk + gseg + 1);
                        }
                        const uint32_t in = pending & __ballot_sync(0xffffffffu, site < gseg_end);
                        gram_add(k0, k1, in);
                        pending &= ~in;
                    }
                }
            } else if constexpr (P < 8) {
                for (int r = ((lw - rot + wpt) % wpt) * 32; r < n1; r += wpt * 32) {
                    const int rw = r + mma_row(lane);
                    BitCounts<P> ct;
                    ct.N = prm.popN;
                    varied_mma<P>(s_bf, reinterpret_cast<const uint32_t*>(tile), n1, prm.wd, r, lane, ct);
                    add_row(tile_site0 + (rw < n1 ? s_slot[rw] : 0), rw < n1, ct, false);
                }
            }

            // ---- three-plane rows, behind the one-plane rows' words rounded up to 16 bytes ----
            const uint32_t* rows3 = reinterpret_cast<const uint32_t*>(tile) + ((n1 * prm.wd + 3) & ~3);
            for (int r = ((lw - rot - nb1 % wpt + 2 * wpt) % wpt) * spv; r < n3; r += wpt * spv) {
                const int rw = r + sl;
                const bool valid = rw < n3;
                const bool owner = valid && (gsub == 0);
                const uint32_t* row = rows3 + (valid ? rw : r);
                // with 8 populations the counts are expanded once; with fewer they stay two words per population (the
                // choices with the fewest spills, ptxas sm_90a)
                std::conditional_t<P == 8, ArrCounts<P>, PkCounts<P>> ct;
                if (P < 8 && Gv == 1) varied_counts<P, true>(prm, s_ent, row, n3, 1, 0, 32, ct);
                else varied_counts<P, false>(prm, s_ent, row, n3, Gv, gsub, spv, ct);
                add_row(tile_site0 + (valid ? s_slot[n1 + rw] : 0), owner, ct, true);
            }

            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[stage]);
        }
        if constexpr (GRAM) gram_flush();
    }
    warp_flush<QI, QU, 0>(acc, cur_seg, prm.part, slot_base, seg_first, warp, lane, NW);
}

// ---- finalize: slots -> segments -> windows -> statistics ------------------------------------------
struct FinParams {
    const unsigned long long* part;
    const int32_t* seg_cta_lo;     // [nseg] first CTA touching the segment
    const int32_t* seg_cta_hi;     // [nseg] last CTA (inclusive)
    const int32_t* cta_seg_first;  // [ctas]
    const int64_t* cta_slot_off;   // [ctas]
    const int32_t* win_seg_lo;     // [W]
    const int32_t* win_seg_hi;     // [W]
    const int64_t* win_lo;
    const int64_t* win_hi;
    int64_t W;
    int Q, QI, nw;
    int P;                         // real population count
    int Ppad;                      // template P used by the site pass
    int popN[PG_MAX_K1_POPS];
    double harm_a[PG_MAX_K1_POPS], harm_a2[PG_MAX_K1_POPS];
    int min_sites;
    double min_data;
    int force_path;
    int with_freq;                 // the site pass carried the popFreq counters
    int bookkeeping_only;          // P > 8: the site pass saw one collapsed population; statistics come from K2
    // popgen over the varied-row stream: exclusive per-site prefixes of the positions and of the uniform non-missing sites
    // (nullptr: the site pass added every site itself), S sites
    const int64_t* pre_pos;
    const int64_t* pre_uni;
    int64_t S;
    // outputs: fixed-width 8-byte records per window
    //   popgen: [sites(i64) pos_sum(i64) path(i64) pi[P] dxy[npairs] fst[npairs]]
    //   abba  : [sites(i64) pos_sum(i64) ABBA BABA D fd fdM sitesUsed]
    unsigned long long* rec;
    int RC;
    int32_t* path;                 // [W] popgen routing, also counted in *n_pairwise
    int* n_pairwise;
};

__device__ __forceinline__ unsigned long long d2u(double x) { return (unsigned long long)__double_as_longlong(x); }

__device__ __forceinline__ double nan_d() { return __longlong_as_double(0x7ff8000000000000ll); }

// mean over the off-diagonal entries of an N x N block whose pairs all have n_ij = Lp
__device__ __forceinline__ double cf_pi(long long N, long long Lp, long long sumsq, bool all_nan, double min_data) {
    if (N <= 0) return nan_d();
    const double size = (double)(N * N);
    const double nan_cnt = all_nan ? size : (double)N;
    if (1.0 - (1.0 * nan_cnt / size) < min_data) return nan_d();      // nanmean_min, genomics.py:88-90
    if (all_nan) return nan_d();
    const double num = (double)(N * N * Lp - sumsq);
    const double den = (double)((N * N - N) * Lp);
    return num / den;
}

template <int MODE>
__global__ void __launch_bounds__(64) k1_finalize(const __grid_constant__ FinParams fp) {
    __shared__ unsigned long long sums[64];
    const int q = threadIdx.x;
    for (int64_t w = blockIdx.x; w < fp.W; w += gridDim.x) {
        __syncthreads();
        if (q < fp.Q) {
            long long si = 0;
            double sd = 0.0;
            for (int g = fp.win_seg_lo[w]; g < fp.win_seg_hi[w]; ++g) {
                for (int b = fp.seg_cta_lo[g]; b <= fp.seg_cta_hi[g]; ++b) {
                    const unsigned long long* src =
                        fp.part + fp.cta_slot_off[b] + (int64_t)(g - fp.cta_seg_first[b]) * fp.nw * fp.Q;
                    for (int wp = 0; wp < fp.nw; ++wp) {
                        const unsigned long long v = src[wp * fp.Q + q];
                        if (q < fp.QI) si += (long long)v; else sd += __longlong_as_double((long long)v);
                    }
                }
            }
            if (MODE == MODE_POPGEN && fp.pre_uni) {
                // the window's positions, and what its uniform non-missing sites add: 1 to the complete sites, and per
                // site N_X^2 to sum c_Xa^2 and N_X N_Y to sum c_Xa c_Ya (population X = Y, then the pairs X < Y in order)
                const int64_t lo = min(max(fp.win_lo[w], (int64_t)0), fp.S), hi = min(max(fp.win_hi[w], lo), fp.S);
                const long long u = fp.pre_uni[hi] - fp.pre_uni[lo];
                const int Pp = fp.Ppad;
                if (q == 0) si += u;
                else if (q == 2) si += fp.pre_pos[hi] - fp.pre_pos[lo];
                else if (q >= 3 && q < 3 + Pp + Pp * (Pp - 1) / 2) {
                    int X = q - 3, Y = X;
                    if (X >= Pp) {
                        int k = X - Pp, left = Pp - 1;
                        for (X = 0; k >= left; ++X, --left) k -= left;
                        Y = X + 1 + k;
                    }
                    si += u * (long long)fp.popN[X] * (long long)fp.popN[Y];
                }
            }
            sums[q] = (q < fp.QI) ? (unsigned long long)si : (unsigned long long)__double_as_longlong(sd);
        }
        __syncthreads();
        if (q != 0) continue;
        const long long sites = fp.win_hi[w] - fp.win_lo[w];
        unsigned long long* rec = fp.rec + (size_t)w * fp.RC;
        rec[0] = (unsigned long long)sites;
        rec[1] = sums[2];
        if (MODE == MODE_POPGEN) {
            const int P = fp.P, Pp = fp.Ppad;
            const int npairs = P * (P - 1) / 2;
            double* pi_o = reinterpret_cast<double*>(rec + 3);
            double* dxy_o = pi_o + P;
            double* fst_o = dxy_o + npairs;
            const long long Lp = (long long)sums[0];
            const bool ragged = (long long)sums[1] > 0;
            if (fp.bookkeeping_only) {
                const int path = sites < fp.min_sites ? 0 : 2;
                fp.path[w] = path;
                rec[2] = (unsigned long long)path;
                if (path == 2) atomicAdd(fp.n_pairwise, 1);
                for (int k = 3; k < fp.RC; ++k) rec[k] = d2u(nan_d());
                continue;
            }
            {   // popFreq columns (valid for every window: they only use sites complete in all haplotypes)
                double* fq = fst_o + npairs;           // [l, S[P], thetaPi[P], thetaW[P], TajD[P]]
                fq[0] = fp.with_freq ? (double)Lp : nan_d();
                const int npp = Pp * (Pp - 1) / 2;
                for (int x = 0; x < P; ++x) {
                    double Sx = nan_d(), tpi = nan_d(), tw = nan_d(), tD = nan_d();
                    if (Lp >= 1 && fp.with_freq) {
                        const long long N = fp.popN[x];
                        // a population of one haplotype: the reference's site pi is 0 / 0 = nan, which its sitePi != 0
                        // counts (genomics.py:1016-1017), so every complete site is segregating there and thetaW = S / 0
                        const long long seg = N == 1 ? (long long)Lp : (long long)sums[3 + Pp + npp + x];
                        const long long pairs = (N * N * Lp - (long long)sums[3 + x]) / 2;   // sum over sites of sum_{a<b} c_a c_b
                        Sx = (double)seg;
                        tpi = (double)pairs / (.5 * (double)N * (double)(N - 1));
                        const double a = fp.harm_a[x], a2 = fp.harm_a2[x];   // sum 1/i, sum 1/i^2 for i < N (host, same order)
                        tw = (double)seg / a;
                        // TajimaD (genomics.py:619-632)
                        const double n_ = (double)N;
                        const double b1 = (n_ + 1.) / (3 * (n_ - 1));
                        const double b2 = (2. * (n_ * n_ + n_ + 3)) / (9 * n_ * (n_ - 1));
                        const double c1 = b1 - (1. / a);
                        const double c2 = b2 - ((n_ + 2) / (a * n_)) + a2 / (a * a);
                        const double e1 = c1 / a;
                        const double e2 = c2 / (a * a + a2);
                        const double d = tpi - tw;
                        tD = d / sqrt(e1 * Sx + e2 * Sx * (Sx - 1));
                    }
                    fq[1 + x] = Sx;
                    fq[1 + P + x] = tpi;
                    fq[1 + 2 * P + x] = tw;
                    fq[1 + 3 * P + x] = tD;
                }
            }
            int path = 1;
            if (sites < fp.min_sites) path = 0;
            else if (ragged || fp.force_path == 2) path = 2;
            fp.path[w] = path;
            rec[2] = (unsigned long long)path;
            if (path == 2) atomicAdd(fp.n_pairwise, 1);
            if (path != 1) {
                for (int x = 0; x < P; ++x) pi_o[x] = nan_d();
                for (int k = 0; k < npairs; ++k) dxy_o[k] = fst_o[k] = nan_d();
                continue;
            }
            const bool all_nan = (Lp == 0) || (fp.min_sites > 0 && Lp < fp.min_sites);
            double piv[PG_MAX_K1_POPS];
            for (int x = 0; x < P; ++x) {
                piv[x] = cf_pi(fp.popN[x], Lp, (long long)sums[3 + x], all_nan, fp.min_data);
                pi_o[x] = piv[x];
            }
            int k = 0;
            for (int x = 0; x < P; ++x)
                for (int y = x + 1; y < P; ++y) {
                    // index of (x,y) in the padded pair enumeration of the site pass
                    int kp = 0;
                    for (int xx = 0; xx < x; ++xx) kp += Pp - 1 - xx;
                    kp += y - x - 1;
                    const long long cross = (long long)sums[3 + Pp + kp];
                    const long long Nx = fp.popN[x], Ny = fp.popN[y];
                    double dxy = nan_d();
                    {
                        const double size = (double)(Nx * Ny);
                        const double nan_cnt = all_nan ? size : 0.0;
                        const bool frac_bad = (1.0 - (1.0 * nan_cnt / size) < fp.min_data);
                        if (!frac_bad && !all_nan) dxy = (double)(Nx * Ny * Lp - cross) / (double)(Nx * Ny * Lp);
                    }
                    const long long sq_t = (long long)sums[3 + x] + (long long)sums[3 + y] + 2 * cross;
                    const double pi_t = cf_pi(Nx + Ny, Lp, sq_t, all_nan, fp.min_data);
                    const double wgt = 1.0 * (double)Nx / (double)(Nx + Ny);
                    const double pi_s = wgt * piv[x] + (1 - wgt) * piv[y];
                    dxy_o[k] = dxy;
                    fst_o[k] = 1 - pi_s / pi_t;
                    ++k;
                }
        } else if (MODE == MODE_FOURPOP) {
            // genomics.py:1623-1643: [fhom, fhom', D, fd, fd', fdm, fdm', fdh, fdh2, fh, ABBA, BABA, ABAA, BAAA, sitesUsed]
            const long long used = (long long)sums[0], n_good = (long long)sums[1];
            double* o = reinterpret_cast<double*>(rec + 2);
            if (n_good < 1) {
                for (int k = 0; k < 14; ++k) o[k] = nan_d();
                o[14] = 0.0;
                continue;
            }
            double d[16];
            for (int k = 0; k < 16; ++k) d[k] = __longlong_as_double((long long)sums[3 + k]);
            o[0] = d[0] * 1. / d[1];
            o[1] = d[2] * 1. / d[3];
            o[2] = d[0] * 1. / d[4];
            o[3] = d[0] * 1. / d[5];
            o[4] = d[2] * 1. / d[6];
            o[5] = d[0] * 1. / d[7];
            o[6] = d[2] * 1. / d[8];
            o[7] = d[2] * 1. / d[9];
            o[8] = d[2] * 1. / d[10];
            o[9] = d[2] * 1. / d[11];
            o[10] = d[12];
            o[11] = d[13];
            o[12] = d[14];
            o[13] = d[15];
            o[14] = (double)used;
        } else {   // MODE_ABBA
            const long long used = (long long)sums[0], n_good = (long long)sums[1];
            double* o = reinterpret_cast<double*>(rec + 2);
            if (n_good < 1) {   // genomics.py:1694-1695: every value nan, sitesUsed included
                for (int k = 0; k < 6; ++k) o[k] = nan_d();
                continue;
            }
            const double s_abba = __longlong_as_double((long long)sums[3]), s_baba = __longlong_as_double((long long)sums[4]);
            const double s_f4 = __longlong_as_double((long long)sums[5]), s_ab = __longlong_as_double((long long)sums[6]);
            const double s_fd = __longlong_as_double((long long)sums[7]), s_fdm = __longlong_as_double((long long)sums[8]);
            o[0] = s_abba;
            o[1] = s_baba;
            o[2] = s_f4 * 1.0 / s_ab;
            o[3] = s_f4 * 1.0 / s_fd;
            o[4] = s_f4 * 1.0 / s_fdm;
            o[5] = (double)used;
        }
    }
}

// ---- host side ---------------------------------------------------------------------------------
struct PopTables {
    std::vector<int32_t> ent_chunk;
    std::vector<uint32_t> ent_mask;   // 4 words per entry
    std::vector<uint32_t> word_ent;   // packed pass: (word, mask) per entry, instead of ent_chunk / ent_mask
    std::vector<uint32_t> bit_frag;   // packed pass: varied_mma's B operand, 2 words per lane and K-block
    int ent_lo[PG_MAX_K1_POPS], ent_hi[PG_MAX_K1_POPS], full_lo[PG_MAX_K1_POPS], full_hi[PG_MAX_K1_POPS];
    int popN[PG_MAX_K1_POPS];
};

// The packed pass's form of the tables: population X is entries [ent_lo[X], ent_hi[X]) of word_ent, one per 32-haplotype
// word it has a member in, with the mask of its members.  bit_frag holds the same masks in the order of an mma B operand
// (varied_mma): for K-block kb (words 8 kb .. 8 kb + 7) and lane 4 X + t, population X's masks of words 8 kb + t and
// 8 kb + 4 + t, zero past wd words and for lanes 4 X + t with X >= Ppad.
void build_word_tables(const std::vector<int32_t>& hap_pop_local, int H, int Ppad, PopTables& t) {
    t.ent_chunk.clear();
    t.ent_mask.clear();
    t.word_ent.clear();
    for (int X = 0; X < PG_MAX_K1_POPS; ++X) t.ent_lo[X] = t.ent_hi[X] = t.full_lo[X] = t.full_hi[X] = t.popN[X] = 0;
    const int wd = (H + 31) / 32;
    t.bit_frag.assign((size_t)(wd + 7) / 8 * 64, 0u);
    for (int X = 0; X < Ppad; ++X) {
        std::vector<uint32_t> m(wd, 0u);
        for (int h = 0; h < H; ++h)
            if (hap_pop_local[h] == X) {
                m[h / 32] |= 1u << (h % 32);
                ++t.popN[X];
            }
        t.ent_lo[X] = (int)t.word_ent.size() / 2;
        for (int w = 0; w < wd; ++w) {
            if (m[w]) {
                t.word_ent.push_back((uint32_t)w);
                t.word_ent.push_back(m[w]);
            }
            t.bit_frag[((size_t)(w / 8) * 32 + 4 * X + w % 4) * 2 + (w % 8) / 4] = m[w];
        }
        t.ent_hi[X] = (int)t.word_ent.size() / 2;
    }
}

// hap_pop_local[h] in [0, Ppad) or -1
void build_tables(const std::vector<int32_t>& hap_pop_local, int H, int chunks, int Ppad, PopTables& t) {
    t.ent_chunk.clear();
    t.ent_mask.clear();
    for (int X = 0; X < PG_MAX_K1_POPS; ++X) t.ent_lo[X] = t.ent_hi[X] = t.full_lo[X] = t.full_hi[X] = t.popN[X] = 0;
    for (int X = 0; X < Ppad; ++X) {
        std::vector<uint16_t> cm(chunks, 0);
        int N = 0;
        for (int h = 0; h < H; ++h)
            if (hap_pop_local[h] == X) {
                cm[h / 16] |= (uint16_t)(1u << (h % 16));
                ++N;
            }
        t.popN[X] = N;
        // longest run of completely-owned chunks
        int best_lo = 0, best_hi = 0, run_lo = -1;
        for (int cidx = 0; cidx <= chunks; ++cidx) {
            const bool fullc = cidx < chunks && cm[cidx] == 0xffff;
            if (fullc && run_lo < 0) run_lo = cidx;
            if (!fullc && run_lo >= 0) {
                if (cidx - run_lo > best_hi - best_lo) {
                    best_lo = run_lo;
                    best_hi = cidx;
                }
                run_lo = -1;
            }
        }
        t.full_lo[X] = best_lo;
        t.full_hi[X] = best_hi;
        t.ent_lo[X] = (int)t.ent_chunk.size();
        for (int cidx = 0; cidx < chunks; ++cidx) {
            if (cm[cidx] == 0) continue;
            if (cidx >= best_lo && cidx < best_hi) continue;
            t.ent_chunk.push_back(cidx);
            for (int wd = 0; wd < 4; ++wd) {
                uint32_t m = 0;
                for (int by = 0; by < 4; ++by)
                    if (cm[cidx] & (1u << (wd * 4 + by))) m |= 0xffu << (8 * by);
                t.ent_mask.push_back(m);
            }
        }
        t.ent_hi[X] = (int)t.ent_chunk.size();
    }
}

// shared memory of the mask tables (+ the per-population tables of the lane-per-population variant)
int table_bytes_of(const PopTables& t) { return (int)t.ent_chunk.size() * 20 + (int)t.word_ent.size() * 4 + 64 + 512; }

int check_plan(const K1Plan& pl) {
    PG_CHECK((pl.T % 4) == 0, "rows of %d bytes are too long for the site-pass kernel", pl.pitch);
    PG_CHECK(pg_k1_plan_ok(pl), "invalid site-pass geometry G=%d wpt=%d I=%d stages=%d smem=%d", pl.G, pl.wpt, pl.I, pl.stages,
             pl.smem_bytes);
    return PG_OK;
}

// consumer warps per CTA.  The general kernels: 12 (+ the producer = 416 threads, 128 registers each) for rows below 1 KiB; 8
// (up to 168 registers, no spills) for longer rows, where the 8-population instantiations need the registers
// (tools/k1_sweep2.py compares the two).  The lane-per-population kernel: 12.  PG_K1_NW = 8 or 12 overrides either.
int k1_nw_for(int pitch, bool lanepop) {
    const char* e = getenv("PG_K1_NW");
    const int v = (e && *e) ? atoi(e) : ((lanepop || pitch < 1024) ? 12 : 8);
    return lanepop ? (v == 8 ? 8 : 12) : (v == 12 ? 12 : 8);
}

// Whether every population's counts fit a byte, so that the popgen byte pass packs them four to a word (PG_K1_NO_BYTES: never).
bool byte_counts(int maxN) { return maxN <= 255 && !getenv("PG_K1_NO_BYTES"); }

// Whether a byte-pass launch over S sites runs the lane-per-population kernel (k1_site_pass_lp, G = Pp lanes per site), and
// with how many consumer warps.  Long rows of a full group of 4 or 8 populations prefer it, but its plan stops fitting
// earlier than the general one (T = 8 sites at G = 4), so it is taken only where it runs.  The two callers differ in
// narrow_counts alone: the popgen instantiations keep byte-packed counts, so popgen passes byte_counts() of its largest
// population; the per-site counts fit their 16 bits in any case, so the counts launch passes true.  PG_K1_LANEPOP decides for
// any row length and group wherever the kernel exists (tests).
struct WarpChoice {
    bool lanepop;
    int nw;
};
WarpChoice choose_warps(const pg_ctx* ctx, int64_t S, int Pp, bool full_group, int table_bytes, bool narrow_counts) {
    bool lp = (Pp == 4 || Pp == 8) && narrow_counts;
    if (const char* e = getenv("PG_K1_LANEPOP")) lp = lp && atoi(e) != 0;
    else
        lp = lp && full_group && ctx->pitch >= 1024 &&
             pg_k1_plan_ok(pg_make_k1_plan(S, ctx->H, ctx->sm_count, table_bytes, k1_nw_for(ctx->pitch, true), Pp));
    return {lp, k1_nw_for(ctx->pitch, lp)};
}

// Where a launch's CTAs keep their sums, as device tables: CTA b's slots start at word cta_slot_off[b] with the segment
// cta_seg_first[b], and segment g is touched by the CTAs seg_cta_lo[g] .. seg_cta_hi[g].  The site pass reads the first two
// and k1_finalize all four, so both take them from the launch that runs (arm_slots, fill_fin).
struct SlotTables {
    int32_t *cta_seg_first = nullptr, *seg_cta_lo = nullptr, *seg_cta_hi = nullptr;
    int64_t* cta_slot_off = nullptr;
    int64_t words = 0;   // 8-byte words of all slots
};

struct K1Launch {
    K1Plan plan;
    K1Params prm;
    SlotTables slots;
};

int seg_of(const std::vector<int64_t>& brk, int64_t site) {
    // brk[g] <= site < brk[g+1]
    return (int)(std::upper_bound(brk.begin(), brk.end(), site) - brk.begin()) - 1;
}

// device layout of the uploaded tables inside K1Cache::tables:
//   [ent_mask (16B each)] [ent_chunk] [word_ent (8B each)] [bit_frag (8B each)] [brk] [the launch's SlotTables] [win_seg_lo]
//   [win_seg_hi] [win_lo] [win_hi]
struct DevTables {
    uint4* ent_mask;
    int32_t* ent_chunk;
    uint2* word_ent;
    uint2* bit_frag;
    int64_t* brk;
    int32_t* win_seg_lo;
    int32_t* win_seg_hi;
    int64_t* win_lo;
    int64_t* win_hi;
};

size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

template <typename T>
int push(pg_ctx* ctx, uint8_t* base, size_t& off, const T* src, size_t n, T** out) {
    off = align_up(off, 16);
    *out = reinterpret_cast<T*>(base + off);
    if (n) PG_CUDA(cudaMemcpyAsync(base + off, src, n * sizeof(T), cudaMemcpyHostToDevice, ctx->stream));
    off += n * sizeof(T);
    return PG_OK;
}

// ---- the packed rows of the varied sites only (DESIGN.md "Uniform sites") -------------------------------------------
// Derived from the companion and its site classes (ctx->d_site_cls) for one data generation, row budget R, tile bound Tmax
// and row kinds (bits: complete biallelic rows as one plane).  Tiles are cut by a budget of varied rows: group k holds the
// varied rows of ranks [k R, (k + 1) R) and runs from the site of rank k R (site 0 for k = 0) to the next group's; a group of
// more than Tmax sites is split into pieces of Tmax (the slots are 16 bits).  So a tile has at most R varied rows and at most
// Tmax sites, and tile t covers the sites [site_lo[t], site_lo[t + 1]).  Per tile: the index of its first varied row (row0,
// int64 [tiles + 1]), its one-plane rows (n1, int32 [tiles]), its first word in the stream (woff, int64 [tiles + 1]: a tile's
// one-plane rows take n1 wd words rounded up to 4, its three-plane rows a packed row's words each), the slot (index in the
// tile) of each of its rows at t * Tmax; and the rows (k1_uni_rows).  bound holds the first site of each CTA's tiles (B + 1).
// pre holds the exclusive prefixes, over the S + 1 site bounds, of the positions and of the uniform non-missing sites, which
// k1_finalize adds to each window in place of walking those sites.
struct UniformStream {
    uint64_t gen = 0;         // ctx->data_gen it describes (0: none)
    uint64_t serial = 0;      // counts the builds (the slot tables follow it)
    int R = 0, Tmax = 0, ctas = 0;
    bool forced = false, bits = false, wb = false;
    bool in_use = false;      // false: too few uniform sites to pay off, or no memory; the packed pass streams every row
    int64_t varied = 0;
    int64_t nt = 0;           // tiles
    const int64_t* woff = nullptr;   // in words
    std::vector<int64_t> bound;
    PgBuf cnt, row0, slots, src, rows, scan, site_lo, groups, info, words, n1, pre, wts, scan2;
    void release() {
        for (PgBuf* b : {&cnt, &row0, &slots, &src, &rows, &scan, &site_lo, &groups, &info, &words, &n1, &pre, &wts, &scan2})
            b->release();
        gen = 0;
    }
};

// whether a site of class c is streamed as one plane (bits: complete biallelic rows are)
__device__ __forceinline__ bool uni_one_plane(uint32_t c, bool bits) { return bits && pg_cls_biallelic(c); }

// varied sites per tile: tile t is [site_lo[t], site_lo[t + 1]), or the T sites from t * T when site_lo is null.  With wcnt,
// also the tile's one-plane rows (n1) and the stream words of its rows (wcnt): wd words per one-plane row, rounded up to 4,
// and pw per three-plane row.
__global__ void __launch_bounds__(256) k1_uni_count(const uint8_t* __restrict__ cls, int64_t S, const int64_t* __restrict__ site_lo,
                                                    int T, int64_t* __restrict__ cnt, int64_t* __restrict__ wcnt = nullptr,
                                                    int32_t* __restrict__ n1 = nullptr, int wd = 0, int pw = 0, bool bits = false) {
    __shared__ int s_n, s_n1;
    if (threadIdx.x == 0) s_n = s_n1 = 0;
    __syncthreads();
    const int64_t s0 = site_lo ? site_lo[blockIdx.x] : (int64_t)blockIdx.x * T;
    const int64_t len = site_lo ? site_lo[blockIdx.x + 1] - s0 : (S - s0 < T ? S - s0 : (int64_t)T);
    int n = 0, m = 0;
    for (int j = threadIdx.x; j < len; j += blockDim.x) {
        const uint32_t c = cls[s0 + j];
        if (pg_cls_varied(c)) ++n;
        if (uni_one_plane(c, bits)) ++m;
    }
    n = __reduce_add_sync(0xffffffffu, n);
    m = __reduce_add_sync(0xffffffffu, m);
    if ((threadIdx.x & 31) == 0) {
        atomicAdd(&s_n, n);
        atomicAdd(&s_n1, m);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        cnt[blockIdx.x] = s_n;
        if (wcnt) {
            n1[blockIdx.x] = s_n1;
            wcnt[blockIdx.x] = (int64_t)((s_n1 * wd + 3) & ~3) + (int64_t)(s_n - s_n1) * pw;
        }
    }
}

// The source site of each varied row of tile blockIdx.x (tiles as in k1_uni_count), in site order.  With slots (tiles of
// site_lo), in the tile's row order instead: its one-plane rows, then its three-plane rows, each kind in site order, with
// the slot of each; the block then copies the rows from the companion (ppw words per row) into the stream from word
// woff[t], word-major: word x of one-plane row j (its plane B0 or B1, as the class says) to word x * n1 + j, then word x of
// three-plane row j to word x * n3 + j of the run that starts at the one-plane rows' words rounded up to 4.
__global__ void __launch_bounds__(256) k1_uni_rows(const uint8_t* __restrict__ cls, int64_t S, const int64_t* __restrict__ site_lo,
                                                   int T, const int64_t* __restrict__ row0, int64_t* __restrict__ src,
                                                   uint16_t* __restrict__ slots = nullptr, const int32_t* __restrict__ n1 = nullptr,
                                                   const int64_t* __restrict__ woff = nullptr, const uint32_t* __restrict__ packed = nullptr,
                                                   int ppw = 0, int wd = 0, bool bits = false, uint32_t* __restrict__ rows = nullptr) {
    typedef cub::BlockScan<int, 256> Scan;
    __shared__ typename Scan::TempStorage tmp;
    const int64_t t = blockIdx.x, r0 = row0[t];
    const int64_t s0 = site_lo ? site_lo[t] : t * T;
    const int64_t len = site_lo ? site_lo[t + 1] - s0 : (S - s0 < T ? S - s0 : (int64_t)T);
    const int m1 = slots ? n1[t] : 0;
    int base1 = 0, base3 = 0;
    for (int j0 = 0; j0 < len; j0 += 256) {
        const int j = j0 + threadIdx.x;
        const int64_t s = s0 + j;
        const uint32_t k = j < len ? cls[s] : (uint32_t)PG_CLS_MISSING;
        // a row of either kind counts in the low half, a three-plane row in the high half too (< 256 each)
        const int one = slots && uni_one_plane(k, bits) ? 1 : 0, var = pg_cls_varied(k) ? 1 : 0;
        int rank, total;
        Scan(tmp).ExclusiveSum(var | (var - one) << 16, rank, total);
        __syncthreads();
        if (var) {
            const int r3 = rank >> 16, r1 = (rank & 0xffff) - r3;
            const int idx = !slots ? base1 + (rank & 0xffff) : (one ? base1 + r1 : m1 + base3 + r3);
            if (slots) slots[t * T + idx] = (uint16_t)j;
            src[r0 + idx] = s;
        }
        base1 += slots ? (total & 0xffff) - (total >> 16) : (total & 0xffff);
        base3 += total >> 16;
    }
    if (!rows) return;
    __syncthreads();                          // the block's src entries, read back below
    const int nvar = (int)(row0[t + 1] - r0), m3 = nvar - m1;
    uint32_t* dst = rows + woff[t];
    // a thread per row: the words a warp writes are consecutive, and each thread's reads stay in its row's sectors (a warp
    // per row, its lanes over the words, took the C2 rebuild from 0.68 to 1.03 ms and C5's from 1.6 to 4.3, H100)
    for (int j = threadIdx.x; j < m1; j += blockDim.x) {
        const int64_t site = src[r0 + j];
        const uint32_t* w = packed + site * ppw + (cls[site] == PG_CLS_VARIED2_B1 ? 2 : 1) * wd;
        for (int x = 0; x < wd; ++x) dst[(int64_t)x * m1 + j] = w[x];
    }
    dst += (m1 * wd + 3) & ~3;
    const int lane = threadIdx.x & 31, chunks = ppw / 4;
    for (int c = threadIdx.x >> 5; c < chunks; c += blockDim.x >> 5)
        for (int j = lane; j < m3; j += 32) {
            const uint4 v = reinterpret_cast<const uint4*>(packed)[src[r0 + m1 + j] * chunks + c];
            uint32_t* d = dst + (int64_t)4 * c * m3 + j;
            d[0] = v.x;
            d[m3] = v.y;
            d[2 * m3] = v.z;
            d[3 * m3] = v.w;
        }
}

// the uniform non-missing sites, as 0 / 1 per site for the prefix scan
struct UniformSite {
    __host__ __device__ int64_t operator()(uint8_t c) const { return c >= PG_CLS_A && c <= PG_CLS_T ? 1 : 0; }
};
struct Widen {
    __host__ __device__ int64_t operator()(int32_t v) const { return v; }
};

// group k's first site (the site of varied rank k R, or of rank first[k] for a budget of words; 0 for k = 0) and end (the next
// group's first site; S for the last)
__device__ __forceinline__ void uni_group(const int64_t* src, int R, int64_t S, int64_t ng, int64_t k, int64_t& lo, int64_t& hi,
                                          const int64_t* first) {
    lo = k == 0 ? 0 : src[first ? first[k] : k * R];
    hi = k + 1 < ng ? src[first ? first[k + 1] : (k + 1) * R] : S;
}
// the words of each varied row (src: its site, in site order), and 0 behind the last, for the scan of their first words
__global__ void k1_uni_w(const uint8_t* cls, const int64_t* src, int64_t varied, int wd, int pw, bool bits, int64_t* w) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r <= varied; r += (int64_t)gridDim.x * blockDim.x)
        w[r] = r < varied ? (uni_one_plane(cls[src[r]], bits) ? wd : pw) : 0;
}
// group g of a budget of Bw words: the rows whose first word cw lies in [g Bw, (g + 1) Bw) (consecutive, as no row exceeds Bw
// words); first[g] = its first row's rank
__global__ void k1_uni_first(const int64_t* cw, int64_t varied, int64_t Bw, int64_t* first) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < varied; r += (int64_t)gridDim.x * blockDim.x) {
        const int64_t g = cw[r] / Bw;
        if (r == 0 || cw[r - 1] / Bw != g) first[g] = r;
    }
}

// pieces of at most tmax sites per group
__global__ void __launch_bounds__(256) k1_uni_groups(const int64_t* __restrict__ src, int R, int64_t S, int tmax, int64_t ng,
                                                     int64_t* __restrict__ pieces, const int64_t* first) {
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= ng) return;
    int64_t lo, hi;
    uni_group(src, R, S, ng, k, lo, hi, first);
    const int64_t n = (hi - lo + tmax - 1) / tmax;
    pieces[k] = n > 1 ? n : 1;
}

// site_lo of every tile from the groups' first pieces (base, the exclusive scan of the pieces: base[ng] = tiles); the entries
// from the last tile on up to nt_max hold S (empty tiles)
__global__ void __launch_bounds__(256) k1_uni_tiles(const int64_t* __restrict__ src, int R, int64_t S, int tmax, int64_t ng,
                                                    const int64_t* __restrict__ base, int64_t nt_max, int64_t* __restrict__ site_lo,
                                                    const int64_t* first) {
    const int64_t nt = base[ng];
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i <= (ng > nt_max ? ng : nt_max);
         i += (int64_t)gridDim.x * blockDim.x) {
        if (i < ng) {
            int64_t lo, hi;
            uni_group(src, R, S, ng, i, lo, hi, first);
            for (int64_t b = base[i], j = 0; b + j < base[i + 1]; ++j) site_lo[b + j] = lo + j * tmax;
        }
        if (i >= nt && i <= nt_max) site_lo[i] = S;
    }
}

// info[0] = tiles, info[1 + b] = the first site of CTA b's tiles for b = 0 .. B (B = min(ctas, tiles) CTAs, tiles b * nt / B
// on)
__global__ void __launch_bounds__(256) k1_uni_bounds(const int64_t* __restrict__ base, int64_t ng, const int64_t* __restrict__ site_lo,
                                                     int ctas, int64_t* __restrict__ info) {
    const int64_t nt = base[ng];
    const int64_t B = nt < ctas ? (nt > 1 ? nt : 1) : ctas;
    for (int64_t b = threadIdx.x; b <= B; b += blockDim.x) info[1 + b] = site_lo[b * nt / B];
    if (threadIdx.x == 0) info[0] = nt;
}

// The packed popgen pass over the varied rows only: the stream, its geometry, the slot tables of its CTA ranges and the
// launch of k1_site_pass_packed<..., true> made of them.  uni_geometry sets the geometry on every call (its hooks);
// uniform_prepare rebuilds the stream when the data or the geometry changed; uniform_slots rebuilds the slot tables and the
// launch when the windows (epoch), the stream (serial), the slot width or the ring changed.
struct UniformPass {
    K1Plan plan;              // the cache's plan (its G, wpt and warps serve the stream)
    int table_bytes = 0;      // shared-memory bytes of the stream kernel's tables (plan's, and varied_mma's B operand)
    int R = 0, Tmax = 0, stages = 0, stage_bytes = 0;   // row budget, tile bound, and ring (uni_geometry)
    // complete biallelic rows as one plane: below 8 (padded) populations.  At 8 the one-plane walk that preceded varied_mma
    // was slower than the three-plane one (C5, H100 80GB HBM3, 700 W: 0.963 against 0.884 ms) and spilled more, so there
    // every varied row is streamed as three planes and the kernel has no one-plane rows
    bool one_plane = true;
    int wd = 0;                     // words per plane
    bool bits = false, words = false;   // this call: one-plane rows; tiles by a budget of row words (uni_geometry)
    int row_cap = 0, cap_rows = 0;      // three-plane rows a stage has room for; rows a tile may hold
    UniformStream us;
    PgBuf slot_buf;
    uint64_t slots_epoch = 0, slots_serial = 0;
    int slots_Q = 0;
    K1Launch L;
    bool last = false;        // the last popgen launch was L
    int32_t launched[3] = {0, 0, 0};   // of L's last launch: CTAs, consumer warps per CTA, 1 for the Gram kernel
    void release() {
        us.release();
        slot_buf.release();
    }
};

// Everything a windowed launch needs, cached per configuration (data shape, populations, windows): a repeated
// statistics call on the same configuration only clears the slots and launches two kernels.
struct K1Cache {
    bool valid = false;
    bool lanepop = false;
    bool packed = false;      // the launch reads the packed companion (k1_site_pass_packed)
    uint64_t epoch = 0;
    int mode = -1;
    int sel[4] = {-1, -1, -1, -1};
    K1Launch L;
    DevTables dt;
    PopTables pt;
    PgBuf tables;
    UniformPass up;           // packed (popgen cache only)
};

// The one-hot rows' launch plan for this population map, or the error that refuses such rows.
int byte_plan(pg_ctx* ctx, const std::vector<int32_t>& hap_pop_local, int Ppad, int nw, int force_G, PopTables& pt,
              K1Plan& plan) {
    build_tables(hap_pop_local, ctx->H, ctx->pitch / 16, Ppad, pt);
    const int table_bytes = table_bytes_of(pt);
    PG_CHECK(table_bytes <= 48 * 1024, "population layout needs %d bytes of mask tables (limit 48 KiB)", table_bytes);
    plan = pg_make_k1_plan(ctx->S, ctx->H, ctx->sm_count, table_bytes, nw, force_G);
    PG_CHECK(plan.stages >= 2, "rows of %d haplotypes are too long for the site-pass kernel (pitch %d bytes)", ctx->H,
             plan.pitch);
    return check_plan(plan);
}

// The slots of a launch whose CTA b adds the sites [bound[b], bound[b + 1]): each CTA gets nw slots of Q words per segment it
// touches (cta_seg_first, cta_slot_off), and each segment the range of CTAs that touch it (seg_cta_lo / _hi), for k1_finalize.
// On the host, until push_slots has uploaded them.
struct HostSlots {
    std::vector<int32_t> cta_seg_first, seg_cta_lo, seg_cta_hi;
    std::vector<int64_t> cta_slot_off;
    int64_t words = 0;
    size_t bytes() const { return cta_seg_first.size() * 12 + seg_cta_lo.size() * 8 + 4 * 16; }   // on the device (push)
};

void slot_tables(const std::vector<int64_t>& brk, const std::vector<int64_t>& bound, int nw, int Q, HostSlots& L) {
    const int B = (int)bound.size() - 1;
    const int nseg = (int)brk.size() - 1;
    L.cta_seg_first.assign(B, 0);
    L.cta_slot_off.assign(B, 0);
    L.seg_cta_lo.assign(std::max(nseg, 1), 0);
    L.seg_cta_hi.assign(std::max(nseg, 1), -1);
    std::vector<int> cta_seg_last(B, -1);
    int64_t off = 0;
    for (int b = 0; b < B; ++b) {
        const int64_t s0 = bound[b], s1 = bound[b + 1];
        L.cta_slot_off[b] = off;
        if (s1 <= s0) continue;
        const int g0 = seg_of(brk, s0), g1 = seg_of(brk, s1 - 1);
        L.cta_seg_first[b] = g0;
        cta_seg_last[b] = g1;
        off += (int64_t)(g1 - g0 + 1) * nw * Q;
    }
    for (int g = 0; g < nseg; ++g) {
        L.seg_cta_lo[g] = B;
        L.seg_cta_hi[g] = -1;
    }
    for (int b = 0; b < B; ++b) {
        if (cta_seg_last[b] < 0) continue;
        for (int g = L.cta_seg_first[b]; g <= cta_seg_last[b]; ++g) {
            L.seg_cta_lo[g] = std::min(L.seg_cta_lo[g], b);
            L.seg_cta_hi[g] = std::max(L.seg_cta_hi[g], b);
        }
    }
    L.words = off;
}

// Uploads h behind base + o; the caller synchronises before h goes away.
int push_slots(pg_ctx* ctx, uint8_t* base, size_t& o, const HostSlots& h, SlotTables& st) {
    PG_TRY(push(ctx, base, o, h.cta_seg_first.data(), h.cta_seg_first.size(), &st.cta_seg_first));
    PG_TRY(push(ctx, base, o, h.cta_slot_off.data(), h.cta_slot_off.size(), &st.cta_slot_off));
    PG_TRY(push(ctx, base, o, h.seg_cta_lo.data(), h.seg_cta_lo.size(), &st.seg_cta_lo));
    PG_TRY(push(ctx, base, o, h.seg_cta_hi.data(), h.seg_cta_hi.size(), &st.seg_cta_hi));
    st.words = h.words;
    return PG_OK;
}

// The fields of a launch's parameters that follow from its plan and the population tables (dt: the tables on the device;
// packed: the companion's rows and (word, mask) entries instead of the one-hot rows and chunk masks).  The rest is zero and
// its caller's: the site range; segments and slots of a windowed launch; counts_* of a counts launch.
void fill_params(K1Params& p, const pg_ctx* ctx, const K1Plan& pl, const PopTables& pt, const DevTables& dt, bool packed) {
    memset(&p, 0, sizeof(p));
    p.geno = packed ? (const uint8_t*)ctx->d_packed : (const uint8_t*)ctx->d_geno;
    p.pos = ctx->d_pos;
    p.num_tiles = pl.num_tiles;
    p.pitch = pl.pitch;
    p.G = pl.G;
    p.I = pl.I;
    p.T = pl.T;
    p.wpt = pl.wpt;
    p.nw = pl.nw;
    p.stages = pl.stages;
    p.tile_bytes = pl.tile_bytes;
    p.ent_chunk = dt.ent_chunk;
    p.ent_mask = dt.ent_mask;
    p.word_ent = dt.word_ent;
    p.bit_frag = dt.bit_frag;
    p.wd = (ctx->H + 31) / 32;
    p.n_ent = packed ? (int)pt.word_ent.size() / 2 : (int)pt.ent_chunk.size();
    for (int X = 0; X < PG_MAX_K1_POPS; ++X) {
        p.ent_lo[X] = pt.ent_lo[X];
        p.ent_hi[X] = pt.ent_hi[X];
        p.full_lo[X] = pt.full_lo[X];
        p.full_hi[X] = pt.full_hi[X];
        p.popN[X] = pt.popN[X];
    }
}

// packed: plan and tables for the packed companion's rows (k1_site_pass_packed) instead of the one-hot rows
int prepare_windowed(pg_ctx* ctx, K1Cache& c, const std::vector<int32_t>& hap_pop_local, int Ppad, int Q, int nw, int force_G,
                     bool packed) {
    K1Launch& L = c.L;
    DevTables& dt = c.dt;
    PopTables& pt = c.pt;
    PG_TRY(pg_build_segments(ctx));
    if (packed) {
        build_word_tables(hap_pop_local, ctx->H, Ppad, pt);
        const int table_bytes = table_bytes_of(pt);
        PG_CHECK(table_bytes <= 48 * 1024, "population layout needs %d bytes of mask tables (limit 48 KiB)", table_bytes);
        L.plan = pg_make_k1_plan_rows(ctx->S, ctx->packed_pitch, ctx->sm_count, table_bytes, nw, force_G);
        PG_CHECK(L.plan.stages >= 2, "rows of %d haplotypes are too long for the packed site pass (%d bytes)", ctx->H,
                 L.plan.pitch);
        PG_TRY(check_plan(L.plan));
    } else {
        PG_TRY(byte_plan(ctx, hap_pop_local, Ppad, nw, force_G, pt, L.plan));
    }
    for (int X = 0; X < Ppad; ++X) PG_CHECK(pt.popN[X] <= 65535, "a population has more than 65535 haplotypes");
    const K1Plan& pl = L.plan;
    const int B = pl.ctas;
    std::vector<int64_t> bound(B + 1);
    for (int b = 0; b <= B; ++b) bound[b] = std::min<int64_t>((int64_t)b * pl.num_tiles / B * pl.T, ctx->S);
    HostSlots hs;
    slot_tables(ctx->brk, bound, nw, Q, hs);
    size_t bytes = 4096 + pt.ent_mask.size() * 4 + pt.ent_chunk.size() * 4 + pt.word_ent.size() * 4 + pt.bit_frag.size() * 4 +
                   ctx->brk.size() * 8 + hs.bytes() + (size_t)ctx->W * 24 + 14 * 16;
    PG_TRY(c.tables.ensure(bytes));
    uint8_t* base = (uint8_t*)c.tables.p;
    size_t o = 0;
    uint32_t* d_mask_words = nullptr;
    PG_TRY(push(ctx, base, o, pt.ent_mask.data(), pt.ent_mask.size(), &d_mask_words));
    dt.ent_mask = reinterpret_cast<uint4*>(d_mask_words);
    PG_TRY(push(ctx, base, o, pt.ent_chunk.data(), pt.ent_chunk.size(), &dt.ent_chunk));
    uint32_t* d_word_ent = nullptr;
    PG_TRY(push(ctx, base, o, pt.word_ent.data(), pt.word_ent.size(), &d_word_ent));
    dt.word_ent = reinterpret_cast<uint2*>(d_word_ent);
    uint32_t* d_bit_frag = nullptr;
    PG_TRY(push(ctx, base, o, pt.bit_frag.data(), pt.bit_frag.size(), &d_bit_frag));
    dt.bit_frag = reinterpret_cast<uint2*>(d_bit_frag);
    PG_TRY(push(ctx, base, o, ctx->brk.data(), ctx->brk.size(), &dt.brk));
    PG_TRY(push_slots(ctx, base, o, hs, L.slots));
    PG_TRY(push(ctx, base, o, ctx->win_seg_lo.data(), ctx->win_seg_lo.size(), &dt.win_seg_lo));
    PG_TRY(push(ctx, base, o, ctx->win_seg_hi.data(), ctx->win_seg_hi.size(), &dt.win_seg_hi));
    PG_TRY(push(ctx, base, o, ctx->win_lo.data(), ctx->win_lo.size(), &dt.win_lo));
    PG_TRY(push(ctx, base, o, ctx->win_hi.data(), ctx->win_hi.size(), &dt.win_hi));
    PG_CHECK(o <= c.tables.cap, "internal: table buffer overflow");
    // the host vectors must outlive the async copies
    PG_CUDA(cudaStreamSynchronize(ctx->stream));

    K1Params& p = L.prm;
    fill_params(p, ctx, pl, pt, dt, packed);
    p.site_begin = 0;
    p.site_end = ctx->S;
    p.brk = dt.brk;
    p.nseg = (int)ctx->brk.size() - 1;
    p.cta_seg_first = L.slots.cta_seg_first;
    p.cta_slot_off = L.slots.cta_slot_off;
    return PG_OK;
}

// per-call part of the launch that runs: its slots zeroed, and the addresses that an upload of the same shape may have moved
// (rows: what the launch streams)
int arm_slots(pg_ctx* ctx, K1Launch& L, const void* rows) {
    const size_t bytes = (size_t)std::max<int64_t>(L.slots.words, 1) * 8;
    PG_TRY(ctx->part.ensure(bytes));
    PG_CUDA(cudaMemsetAsync(ctx->part.p, 0, bytes, ctx->stream));
    L.prm.part = (unsigned long long*)ctx->part.p;
    L.prm.geno = (const uint8_t*)rows;
    L.prm.pos = ctx->d_pos;
    return PG_OK;
}

// One site-pass kernel on the launch's grid, NW consumer warps and the producer warp per CTA.
template <auto Kern, int NW>
int launch_kernel(pg_ctx* ctx, const K1Launch& L, const char* name) {
    PG_TRY(pg_smem_limit<Kern>(ctx, 227 * 1024));
    const int ti = pg_time_begin(ctx, name);
    Kern<<<L.plan.ctas, (NW + 1) * 32, L.plan.smem_bytes, ctx->stream>>>(L.prm);
    pg_time_end(ctx, ti);
    PG_CUDA(cudaGetLastError());
    return PG_OK;
}

// The byte pass: the lane-per-population kernel, the byte-packed counts or the general kernel, as the launch says.
template <int MODE, int P>
int launch_site_pass(pg_ctx* ctx, const K1Launch& L, const char* name) {
    constexpr bool POPGEN_MODE = (MODE == MODE_POPGEN || MODE == MODE_POPGEN_FREQ);
    const bool w12 = L.prm.nw == 12;
    if constexpr ((POPGEN_MODE || MODE == MODE_COUNTS) && (P == 4 || P == 8)) {
        if (L.prm.lanepop)
            return w12 ? launch_kernel<k1_site_pass_lp<MODE, P, 12>, 12>(ctx, L, name)
                       : launch_kernel<k1_site_pass_lp<MODE, P, 8>, 8>(ctx, L, name);
    }
    if constexpr (POPGEN_MODE) {
        if (L.prm.bytes)
            return w12 ? launch_kernel<k1_site_pass<MODE, P, 12, true>, 12>(ctx, L, name)
                       : launch_kernel<k1_site_pass<MODE, P, 8, true>, 8>(ctx, L, name);
    }
    return w12 ? launch_kernel<k1_site_pass<MODE, P, 12, false>, 12>(ctx, L, name)
               : launch_kernel<k1_site_pass<MODE, P, 8, false>, 8>(ctx, L, name);
}

// The varied-row stream with one-plane rows and byte counts sums its one-plane rows as a Gram (k1_site_pass_packed's GRAM).
// launched (may be null) receives the grid, the consumer warps and whether the Gram kernel runs.
template <int MODE, int P, bool UNI>
int launch_site_pass_packed(pg_ctx* ctx, const K1Launch& L, const char* name, int32_t* launched = nullptr) {
    if (launched) {
        launched[0] = L.plan.ctas;
        launched[1] = L.prm.nw;
        launched[2] = UNI && P < 8 && L.prm.bytes ? 1 : 0;
    }
    if constexpr (UNI && P < 8) {
        if (L.prm.bytes)
            return L.prm.nw == 12 ? launch_kernel<k1_site_pass_packed<MODE, P, 12, true, true>, 12>(ctx, L, name)
                                  : launch_kernel<k1_site_pass_packed<MODE, P, 8, true, true>, 8>(ctx, L, name);
    }
    return L.prm.nw == 12 ? launch_kernel<k1_site_pass_packed<MODE, P, 12, UNI>, 12>(ctx, L, name)
                          : launch_kernel<k1_site_pass_packed<MODE, P, 8, UNI>, 8>(ctx, L, name);
}

// f(P) with the padded population count (2, 4 or 8) as a compile-time constant
template <typename F>
int with_pops(int Pp, F&& f) {
    if (Pp == 2) return f(std::integral_constant<int, 2>());
    if (Pp == 4) return f(std::integral_constant<int, 4>());
    return f(std::integral_constant<int, 8>());
}

// f(MODE, P) for the popgen pass, with or without the popFreq counters
template <typename F>
int with_popgen_mode(bool with_freq, int Pp, F&& f) {
    return with_pops(Pp, [&](auto P) {
        return with_freq ? f(std::integral_constant<int, MODE_POPGEN_FREQ>(), P) : f(std::integral_constant<int, MODE_POPGEN>(), P);
    });
}

// Streaming only the varied rows costs (1 - u) * (pitch + 2) bytes per site (row, slot; a third of the row for a complete
// biallelic site) against 4 + pitch, for a uniform fraction u, plus a rebuild whenever the data change.
// tools/packed_site_pass.py --sweep timed the two passes across u at the C2 shape when the stream still carried 6 bytes of
// position and code per site (H100 80GB HBM3, 700 W): 0.48 against 0.55 ms at u = 20 %, 0.52 against 0.55 at 10 %, 0.553
// against 0.555 at 5 %, 0.57 against 0.555 at 1 %.  The stream is kept from u >= 1/8 on, where its gain is clear of the
// run-to-run spread.
constexpr double UNI_MIN_FRACTION = 0.125;

// One-plane rows of wd words a budget of R three-plane rows (of pitch bytes) holds, less 3 words of padding
int uni_word_rows(int R, int pitch, int wd) { return (R * (pitch / 4) - 3) / wd; }

// Bytes of a stage of the stream's ring: row_cap three-plane rows, then a slot per row (cap_rows of them).
int uni_stage_bytes(int row_cap, int cap_rows, int pitch) {
    return (int)align_up((size_t)row_cap * pitch + align_up((size_t)cap_rows * 2, 16), 128);
}

// The stream's geometry for the plan u.plan: a tile bound of Tmax = 512 sites (PG_K1_UNI_TMAX, a multiple of 8 up to 32768), and a
// budget of R varied rows per tile, one per lane of a team at the plan's lanes per site, halved (down to one warp's lanes)
// while the ring would hold fewer than 2 stages (PG_K1_UNI_R sets R).  The ring: as many such stages as fit
// (pg_k1_ring_stages).  tools/packed_site_pass.py --sweep (H100 80GB HBM3, 700 W): C2 (4 warps per team, 160-byte rows)
// R = 32 / 64 / 128 / 256 0.50 / 0.30 / 0.22 / 0.23 ms; C5 (2 warps, 608-byte rows) R = 32 / 64 / 128 1.40 / 1.09 / 1.62 ms
// (8, 5 and 2 stages): rows that fill the lanes matter more than stages beyond the teams' count.  Tmax = 256 / 512 / 2048:
// C2 0.30 / 0.22 / 0.24 ms.
// With one-plane rows (bits) and R not set, tiles are cut by a budget of row words instead: the words of R three-plane rows,
// so a tile holds up to about 3R one-plane rows (cap_rows).  A row belongs to the tile its first word falls in, so the last
// one may run past the budget by a row: the stage has room for R + 1 rows (row_cap).  H100 80GB HBM3, 700 W,
// tools/packed_site_pass.py: C2 0.120 ms against 0.156 with R rows (5,000-site windows 0.145 against 0.176), with Tmax 2048 (the
// R-row budget at Tmax 2048: 0.156, 0.176).  PG_K1_UNI_R sets a budget of R rows of either kind, as before.
void uni_geometry(UniformPass& u) {
    const K1Plan& pl = u.plan;
    const char* eb = getenv("PG_K1_UNI_BITS");
    u.bits = u.one_plane && !(eb && *eb && atoi(eb) == 0);
    const char* er = getenv("PG_K1_UNI_R");
    u.words = u.bits && !(er && *er);
    int Tmax = u.words ? 2048 : 512;
    if (const char* e = getenv("PG_K1_UNI_TMAX")) Tmax = std::max(8, std::min(32768, (atoi(e) + 7) / 8 * 8));
    const int lanes = 32 / std::max(1, pl.G);
    int R = lanes * pl.wpt;
    auto stage = [&](int r) {
        const bool w = u.words && r >= 2;     // from 2 rows on the budget holds a three-plane row whole
        u.row_cap = w ? r + 1 : r;
        u.cap_rows = w ? uni_word_rows(r, pl.pitch, u.wd) : r;
        return uni_stage_bytes(u.row_cap, u.cap_rows, pl.pitch);
    };
    if (er && *er) {
        R = std::max(1, std::min(0x7fff, atoi(er)));
    } else {
        while (R > lanes && pg_k1_ring_stages(stage(R), u.table_bytes) < 2) R /= 2;
    }
    u.words = u.words && R >= 2;
    u.R = R;
    u.Tmax = Tmax;
    u.stage_bytes = stage(R);
    u.stages = pl.stages >= 2 ? pg_k1_ring_stages(u.stage_bytes, u.table_bytes) : 0;
}

// The stream's CTAs: one per SM, or PG_K1_UNI_CTAS (1 .. SMs), which lets the tests put many rows of one segment on a few
// warps.  It sets both the tile ranges (k1_uni_bounds) and the grid, so that the slot tables and the kernel's t0 agree.
int uni_ctas(const pg_ctx* ctx) {
    const char* e = getenv("PG_K1_UNI_CTAS");
    return (e && *e) ? std::max(1, std::min(ctx->sm_count, atoi(e))) : ctx->sm_count;
}

// (Re)builds u.us for the current data and geometry when they changed: two host synchronisations per rebuild (the count of
// varied rows, which sizes the buffers; the count of tiles with the CTAs' first sites, which size the launch and its slots),
// nothing on a call over unchanged data.  PG_K1_UNIFORM_FORCE keeps the stream whatever the uniform fraction (tests on missing
// data); PG_K1_UNI_BITS=0 streams every varied row as three planes (the tests and tools/packed_site_pass.py compare the two),
// as the stream does at 8 populations (UniformPass::one_plane).
int uniform_prepare(pg_ctx* ctx, UniformPass& u) {
    UniformStream& us = u.us;
    const bool forced = getenv("PG_K1_UNIFORM_FORCE") != nullptr;
    const bool bits = u.bits, wb = u.words;
    const int R = u.R, Tmax = u.Tmax, ctas = uni_ctas(ctx);
    if (us.gen == ctx->data_gen && us.R == R && us.Tmax == Tmax && us.forced == forced && us.bits == bits && us.wb == wb &&
        us.ctas == ctas)
        return PG_OK;
    us.wb = wb;
    us.ctas = ctas;
    us.gen = ctx->data_gen;
    us.R = R;
    us.Tmax = Tmax;
    us.forced = forced;
    us.bits = bits;
    us.in_use = false;
    us.varied = ctx->S;
    us.serial += 1;
    if (u.stages < 2) return PG_OK;
    const int64_t S = ctx->S;
    constexpr int CH = 2048;                  // the chunks of the first pass (varied counts, then each varied row's site)
    const int64_t nc = (S + CH - 1) / CH;
    const int ppw = ctx->packed_pitch / 4, wd = u.wd;
    const int64_t Bw = (int64_t)u.cap_rows * wd;   // words budget: a multiple of the one-plane rows' words
    // groups + S / Tmax bound the pieces
    const int64_t nt_max = S / Tmax + 1 + (wb ? S * ppw / Bw + 2 : (S + R - 1) / R) + 1;
    const int64_t nscan = std::max(nc, nt_max) + 1;
    PG_TRY(us.cnt.ensure((size_t)nscan * 8));
    PG_TRY(us.row0.ensure((size_t)nscan * 8));
    int64_t* d_cnt = (int64_t*)us.cnt.p;
    int64_t* d_row0 = (int64_t*)us.row0.p;
    size_t scan_bytes = 0, pre_bytes = 0;
    PG_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, d_cnt, d_row0, nscan, ctx->stream));
    const auto uni_in = cub::TransformInputIterator<int64_t, UniformSite, const uint8_t*>(ctx->d_site_cls, UniformSite());
    const auto pos_in = cub::TransformInputIterator<int64_t, Widen, const int32_t*>(ctx->d_pos, Widen());
    PG_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, pre_bytes, uni_in, d_row0, S + 1, ctx->stream));
    PG_TRY(us.scan.ensure(std::max(scan_bytes, pre_bytes)));
    int ti = pg_time_begin(ctx, "k1_uniform");
    PG_CUDA(cudaMemsetAsync(d_cnt + nc, 0, 8, ctx->stream));
    k1_uni_count<<<(unsigned)nc, 256, 0, ctx->stream>>>(ctx->d_site_cls, S, nullptr, CH, d_cnt);
    PG_CUDA(cudaGetLastError());
    PG_CUDA(cub::DeviceScan::ExclusiveSum(us.scan.p, scan_bytes, d_cnt, d_row0, nc + 1, ctx->stream));
    pg_time_end(ctx, ti);
    int64_t varied = 0;
    PG_CUDA(cudaMemcpyAsync(&varied, d_row0 + nc, 8, cudaMemcpyDeviceToHost, ctx->stream));
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    us.varied = varied;
    if (!forced && (double)(S - varied) < UNI_MIN_FRACTION * (double)S) return PG_OK;
    // the group count, exact for a budget of rows, a bound for a budget of words (set below)
    int64_t ng = varied > 0 ? (wb ? varied * ppw / Bw + 2 : (varied + R - 1) / R) : 1;
    if (us.slots.ensure((size_t)nt_max * Tmax * 2) != PG_OK || us.src.ensure((size_t)std::max<int64_t>(varied, 1) * 8) != PG_OK ||
        us.rows.ensure((size_t)std::max<int64_t>(varied, 1) * ctx->packed_pitch + (size_t)nt_max * 16) != PG_OK ||
        us.site_lo.ensure((size_t)(nt_max + 1) * 8) != PG_OK || us.groups.ensure((size_t)(ng + 1) * 8 * 2) != PG_OK ||
        us.info.ensure((size_t)(ctx->sm_count + 2) * 8) != PG_OK || us.words.ensure((size_t)(nt_max + 1) * 8 * 2) != PG_OK ||
        us.n1.ensure((size_t)(nt_max + 1) * 4) != PG_OK || us.pre.ensure((size_t)(S + 1) * 8 * 2) != PG_OK ||
        (wb && us.wts.ensure((size_t)(varied + 1) * 8 * 2 + (size_t)(ng + 1) * 8) != PG_OK)) {
        cudaGetLastError();                   // no memory for the stream: the packed pass streams every row
        for (PgBuf* b : {&us.rows, &us.src, &us.slots, &us.pre}) b->release();
        return PG_OK;
    }
    int64_t* d_src = (int64_t*)us.src.p;
    int64_t* d_pieces = (int64_t*)us.groups.p;
    int64_t* d_base = d_pieces + ng + 1;
    int64_t* d_site_lo = (int64_t*)us.site_lo.p;
    int64_t* d_info = (int64_t*)us.info.p;
    int64_t* d_wcnt = (int64_t*)us.words.p;
    int64_t* d_woff = d_wcnt + nt_max + 1;
    us.woff = d_woff;
    int32_t* d_n1 = (int32_t*)us.n1.p;
    int64_t* d_pre = (int64_t*)us.pre.p;
    ti = pg_time_begin(ctx, "k1_uniform");
    // each varied row's site, then the groups of R rows, their pieces, the tiles' first sites, first rows, one-plane rows and
    // first words, their slots and rows; the per-site prefixes
    k1_uni_rows<<<(unsigned)nc, 256, 0, ctx->stream>>>(ctx->d_site_cls, S, nullptr, CH, d_row0, d_src);
    PG_CUDA(cudaGetLastError());
    // a budget of words: each row's first word (cw), the first row of each group, and (a third synchronisation) the count
    int64_t* d_first = nullptr;
    if (wb && varied > 0) {
        int64_t* w = (int64_t*)us.wts.p;
        int64_t* cw = w + varied + 1;
        d_first = cw + varied + 1;
        k1_uni_w<<<ctx->sm_count * 8, 256, 0, ctx->stream>>>(ctx->d_site_cls, d_src, varied, wd, ppw, bits, w);
        PG_CUDA(cudaGetLastError());
        size_t tb = 0;
        PG_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tb, w, cw, varied + 1, ctx->stream));
        PG_TRY(us.scan2.ensure(tb));
        PG_CUDA(cub::DeviceScan::ExclusiveSum(us.scan2.p, tb, w, cw, varied + 1, ctx->stream));
        k1_uni_first<<<ctx->sm_count * 8, 256, 0, ctx->stream>>>(cw, varied, Bw, d_first);
        PG_CUDA(cudaGetLastError());
        int64_t last = 0;
        PG_CUDA(cudaMemcpyAsync(&last, cw + varied - 1, 8, cudaMemcpyDeviceToHost, ctx->stream));
        PG_CUDA(cudaStreamSynchronize(ctx->stream));
        ng = last / Bw + 1;
    } else if (wb) {
        ng = 1;
    }
    PG_CUDA(cudaMemsetAsync(d_pieces + ng, 0, 8, ctx->stream));
    k1_uni_groups<<<(unsigned)((ng + 255) / 256), 256, 0, ctx->stream>>>(d_src, R, S, Tmax, ng, d_pieces, d_first);
    PG_CUDA(cudaGetLastError());
    PG_CUDA(cub::DeviceScan::ExclusiveSum(us.scan.p, scan_bytes, d_pieces, d_base, ng + 1, ctx->stream));
    const int64_t nfill = std::max(ng, nt_max) + 1;
    k1_uni_tiles<<<(unsigned)std::min<int64_t>((nfill + 255) / 256, (int64_t)ctx->sm_count * 16), 256, 0, ctx->stream>>>(
        d_src, R, S, Tmax, ng, d_base, nt_max, d_site_lo, d_first);
    PG_CUDA(cudaGetLastError());
    PG_CUDA(cudaMemsetAsync(d_cnt + nt_max, 0, 8, ctx->stream));
    PG_CUDA(cudaMemsetAsync(d_wcnt + nt_max, 0, 8, ctx->stream));
    k1_uni_count<<<(unsigned)nt_max, 256, 0, ctx->stream>>>(ctx->d_site_cls, S, d_site_lo, Tmax, d_cnt, d_wcnt, d_n1, wd, ppw,
                                                           bits);
    PG_CUDA(cudaGetLastError());
    PG_CUDA(cub::DeviceScan::ExclusiveSum(us.scan.p, scan_bytes, d_cnt, d_row0, nt_max + 1, ctx->stream));
    PG_CUDA(cub::DeviceScan::ExclusiveSum(us.scan.p, scan_bytes, d_wcnt, d_woff, nt_max + 1, ctx->stream));
    k1_uni_rows<<<(unsigned)nt_max, 256, 0, ctx->stream>>>(ctx->d_site_cls, S, d_site_lo, Tmax, d_row0, d_src,
                                                          (uint16_t*)us.slots.p, d_n1, d_woff, ctx->d_packed, ppw, wd, bits,
                                                          (uint32_t*)us.rows.p);
    PG_CUDA(cudaGetLastError());
    k1_uni_bounds<<<1, 256, 0, ctx->stream>>>(d_base, ng, d_site_lo, ctas, d_info);
    PG_CUDA(cudaGetLastError());
    PG_CUDA(cub::DeviceScan::ExclusiveSum(us.scan.p, pre_bytes, uni_in, d_pre, S + 1, ctx->stream));
    PG_CUDA(cub::DeviceScan::ExclusiveSum(us.scan.p, pre_bytes, pos_in, d_pre + S + 1, S + 1, ctx->stream));
    pg_time_end(ctx, ti);
    std::vector<int64_t> info(ctx->sm_count + 2);
    PG_CUDA(cudaMemcpyAsync(info.data(), d_info, info.size() * 8, cudaMemcpyDeviceToHost, ctx->stream));
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    us.nt = info[0];
    const int B = (int)std::max<int64_t>(1, std::min<int64_t>(ctas, us.nt));
    us.bound.assign(info.begin() + 1, info.begin() + 2 + B);
    us.in_use = true;
    return PG_OK;
}

// The slot tables of the stream's CTA ranges and the launch that uses them (L: the cache's packed launch, whose tables and
// segments it shares), rebuilt when the windows (epoch), the stream, the slot width or the ring (PG_K1_STAGES) changed.
// Tiles of at most R varied rows and Tmax sites, a stage sized for such a tile: at 70 % uniform sites it is less than half a
// fixed tile's bytes, so the ring has more stages than teams and a team's next tile is in flight while it works on this one.
// Its CTAs own the stream's tile ranges and add into slots of their own.
int uniform_slots(pg_ctx* ctx, UniformPass& u, const K1Launch& L, int Q) {
    if (u.slots_epoch == ctx->epoch && u.slots_serial == u.us.serial && u.slots_Q == Q && u.L.plan.stages == u.stages)
        return PG_OK;
    HostSlots hs;
    slot_tables(ctx->brk, u.us.bound, L.prm.nw, Q, hs);
    PG_TRY(u.slot_buf.ensure(hs.bytes()));
    size_t o = 0;
    PG_TRY(push_slots(ctx, (uint8_t*)u.slot_buf.p, o, hs, u.L.slots));
    PG_CHECK(o <= u.slot_buf.cap, "internal: slot table buffer overflow");
    PG_CUDA(cudaStreamSynchronize(ctx->stream));     // the host vectors must outlive the copies
    K1Plan& pl = u.L.plan;
    pl = u.plan;
    pl.T = u.Tmax;
    pl.num_tiles = u.us.nt;
    pl.ctas = (int)u.us.bound.size() - 1;
    pl.tile_bytes = u.stage_bytes;
    pl.stages = u.stages;
    pl.smem_bytes = pl.stages * pl.tile_bytes + 256 + u.table_bytes;
    K1Params& p = u.L.prm;
    p = L.prm;
    p.T = pl.T;
    p.num_tiles = pl.num_tiles;
    p.stages = pl.stages;
    p.tile_bytes = pl.tile_bytes;
    p.row_cap = u.row_cap;
    p.cta_seg_first = u.L.slots.cta_seg_first;
    p.cta_slot_off = u.L.slots.cta_slot_off;
    p.row0 = (const int64_t*)u.us.row0.p;
    p.site_lo = (const int64_t*)u.us.site_lo.p;
    p.woff = u.us.woff;
    p.n1 = (const int32_t*)u.us.n1.p;
    p.slots = (const uint16_t*)u.us.slots.p;
    u.slots_epoch = ctx->epoch;
    u.slots_serial = u.us.serial;
    u.slots_Q = Q;
    return PG_OK;
}

int pad_pops(int P) { return P <= 2 ? 2 : (P <= 4 ? 4 : 8); }

K1Cache* cache_of(pg_ctx* ctx, int slot) {
    if (!ctx->k1_cache[slot]) ctx->k1_cache[slot] = new K1Cache();
    return static_cast<K1Cache*>(ctx->k1_cache[slot]);
}

// slots: those of the launch that filled ctx->part
void fill_fin(FinParams& fp, pg_ctx* ctx, const K1Cache& c, const SlotTables& slots, int Q, int QI) {
    memset(&fp, 0, sizeof(fp));
    fp.part = (const unsigned long long*)ctx->part.p;
    fp.seg_cta_lo = slots.seg_cta_lo;
    fp.seg_cta_hi = slots.seg_cta_hi;
    fp.cta_seg_first = slots.cta_seg_first;
    fp.cta_slot_off = slots.cta_slot_off;
    fp.win_seg_lo = c.dt.win_seg_lo;
    fp.win_seg_hi = c.dt.win_seg_hi;
    fp.win_lo = c.dt.win_lo;
    fp.win_hi = c.dt.win_hi;
    fp.W = ctx->W;
    fp.Q = Q;
    fp.QI = QI;
    fp.nw = c.L.prm.nw;
    for (int X = 0; X < PG_MAX_K1_POPS; ++X) {
        fp.popN[X] = c.pt.popN[X];
        double a = 0.0, a2 = 0.0;                       // TajimaD's python sums (genomics.py:621-623), same order
        for (int i = 1; i < c.pt.popN[X]; ++i) {
            a += 1. / (double)i;
            a2 += 1. / ((double)i * (double)i);
        }
        fp.harm_a[X] = a;
        fp.harm_a2[X] = a2;
    }
}

template <int MODE>
int launch_finalize(pg_ctx* ctx, const FinParams& fp) {
    const int ti = pg_time_begin(ctx, "k1_finalize");
    k1_finalize<MODE><<<(unsigned)std::min<int64_t>(fp.W, 65535), 64, 0, ctx->stream>>>(fp);
    pg_time_end(ctx, ti);
    PG_CUDA(cudaGetLastError());
    return PG_OK;
}

unsigned long long nan_bits() {
    const double qn = NAN;
    unsigned long long u;
    memcpy(&u, &qn, 8);
    return u;
}

// The matrix has no sites: every window's record is `one`.  On the ctx stream, so that work queued behind it (the pipelined
// gather's read-back) sees the records.
int put_empty_records(pg_ctx* ctx, const std::vector<unsigned long long>& one, void* d_rec) {
    std::vector<unsigned long long> h;
    h.reserve((size_t)ctx->W * one.size());
    for (int64_t w = 0; w < ctx->W; ++w) h.insert(h.end(), one.begin(), one.end());
    PG_CUDA(cudaMemcpyAsync(d_rec, h.data(), h.size() * 8, cudaMemcpyHostToDevice, ctx->stream));
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    return PG_OK;
}

// smallest n with (double)n / N >= minData, N + 1 when there is none: the reference's test of a population's non-missing
// count, exact in integers (genomics.py:1657-1660 for ABBABABA, 1597-1600 for fourPop)
int min_count(int N, double min_data) {
    for (int n = 0; n <= N; ++n)
        if ((double)n * 1.0 / (double)N >= min_data) return n;
    return N + 1;
}

// Site pass + finalize of a statistic over four selected populations (cache `slot`, Q words per slot), enqueued on the ctx
// stream without synchronising: records of RC words [sites, pos_sum, statistics ...] are left in the DEVICE buffer d_rec.
// With no sites the words [2, nan_end) of a record are NaN and the others 0.  launch(L) runs the site pass; `who` heads the
// error messages.
template <int FIN_MODE, typename Launch>
int fourpop_enqueue(pg_ctx* ctx, const char* who, int slot, int Q, int RC, int nan_end, const int* sel, double min_data,
                    int variant, void* d_rec, Launch launch) {
    PG_CHECK(ctx->P >= 1, "%s: call pg_set_pops first", who);
    for (int k = 0; k < 4; ++k) {
        PG_CHECK(sel[k] >= 0 && sel[k] < ctx->P, "%s: population index %d out of range", who, sel[k]);
        for (int j = 0; j < k; ++j) PG_CHECK(sel[j] != sel[k], "%s: populations must be distinct", who);
    }
    PG_CUDA(cudaSetDevice(ctx->device));
    pg_timings_reset(ctx);
    if (ctx->W == 0) return PG_OK;
    if (ctx->S == 0) {
        std::vector<unsigned long long> one(RC, 0ull);
        std::fill(one.begin() + 2, one.begin() + nan_end, nan_bits());
        return put_empty_records(ctx, one, d_rec);
    }
    K1Cache& c = *cache_of(ctx, slot);
    if (!c.valid || c.epoch != ctx->epoch || memcmp(c.sel, sel, 4 * sizeof(int)) != 0) {
        c.valid = false;
        std::vector<int32_t> local(ctx->H, -1);
        for (int h = 0; h < ctx->H; ++h)
            for (int k = 0; k < 4; ++k)
                if (ctx->hap_pop[h] == sel[k]) local[h] = k;
        PG_TRY(prepare_windowed(ctx, c, local, 4, Q, k1_nw_for(ctx->pitch, false), /*force_G=*/0, /*packed=*/false));
        for (int k = 0; k < 4; ++k) PG_CHECK(c.pt.popN[k] >= 1, "%s: population %d has no haplotypes", who, sel[k]);
        memcpy(c.sel, sel, 4 * sizeof(int));
        c.epoch = ctx->epoch;
        c.valid = true;
    }
    for (int k = 0; k < 4; ++k) c.L.prm.thr[k] = min_count(c.pt.popN[k], min_data);
    c.L.prm.variant = variant;
    PG_TRY(arm_slots(ctx, c.L, ctx->d_geno));
    PG_TRY(launch(c.L));
    FinParams fp;
    fill_fin(fp, ctx, c, c.L.slots, Q, 3);
    fp.P = 4;
    fp.Ppad = 4;
    fp.rec = (unsigned long long*)d_rec;
    fp.RC = RC;
    return launch_finalize<FIN_MODE>(ctx, fp);
}

// Enqueue, read the records back and split them: [sites, pos_sum, RC - 3 statistics, sitesUsed]
template <typename Enqueue>
int fourpop_read(pg_ctx* ctx, int RC, Enqueue enqueue, double* out, double* sites_used, int64_t* n_sites, int64_t* pos_sum) {
    const int64_t W = ctx->W;
    PG_CUDA(cudaSetDevice(ctx->device));
    PG_TRY(ctx->out_d.ensure((size_t)std::max<int64_t>(W, 1) * RC * 8 + 64));
    PG_TRY(enqueue(ctx->out_d.p));
    if (W == 0) return PG_OK;
    void* hp = nullptr;
    PG_TRY(pg_pinned(ctx, (size_t)W * RC * 8 + 64, &hp));
    const unsigned long long* hrec = (const unsigned long long*)hp;
    PG_CUDA(cudaMemcpyAsync(hp, ctx->out_d.p, (size_t)W * RC * 8, cudaMemcpyDeviceToHost, ctx->stream));
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    const int n = RC - 3;
    for (int64_t w = 0; w < W; ++w) {
        const unsigned long long* r = hrec + (size_t)w * RC;
        n_sites[w] = (int64_t)r[0];
        pos_sum[w] = (int64_t)r[1];
        memcpy(out + (size_t)w * n, r + 2, (size_t)n * 8);
        memcpy(sites_used + w, r + 2 + n, 8);
    }
    return PG_OK;
}

}  // namespace

void pg_k1_cache_free(pg_ctx* ctx) {
    for (int k = 0; k < 3; ++k)
        if (ctx->k1_cache[k]) {
            K1Cache* c = static_cast<K1Cache*>(ctx->k1_cache[k]);
            c->tables.release();
            c->up.release();
            delete c;
            ctx->k1_cache[k] = nullptr;
        }
}

// ================================================================================================
// pg_popgen
// ================================================================================================
// Enqueue the site pass + finalize on the ctx stream WITHOUT synchronising; *h_count (pinned) holds the number of
// windows routed to the pairwise path once the stream has been synchronised (nullptr when nothing was launched).  A null
// h_count (a caller that reads the routing off the records' path column) skips that counter's read-back.
int pg_popgen_enqueue(pg_ctx* ctx, int32_t min_sites, double min_data, int32_t force_path, void* d_rec, int** h_count) {
    PG_CHECK(ctx && d_rec, "pg_popgen_device: null argument");
    if (h_count) *h_count = nullptr;
    PG_CHECK(ctx->P >= 1, "pg_popgen: call pg_set_pops first");
    PG_CHECK(force_path == 0 || force_path == 2, "pg_popgen: force_path must be 0 or 2");
    PG_CHECK(ctx->P <= PG_MAX_POPS, "pg_popgen: P=%d > %d populations", ctx->P, PG_MAX_POPS);
    PG_CUDA(cudaSetDevice(ctx->device));
    pg_timings_reset(ctx);
    const int P = ctx->P;
    // More populations than the site pass keeps in registers: it still does the bookkeeping (sites, position sums,
    // failed / ragged windows) with all used haplotypes collapsed into one population, and every window that passes
    // minSites goes through the pairwise path, whose epilogue handles up to PG_MAX_POPS populations.
    const bool many = P > PG_MAX_K1_POPS;
    const int npairs = P * (P - 1) / 2;
    const int RC = 3 + P + 2 * npairs + 1 + 4 * P;
    const int64_t W = ctx->W;
    if (W == 0) return PG_OK;
    if (ctx->S == 0) {
        std::vector<unsigned long long> one(RC, nan_bits());
        one[0] = one[1] = 0;
        one[2] = (0 < min_sites) ? 0 : 1;
        return put_empty_records(ctx, one, d_rec);
    }
    const int Pp = many ? 2 : pad_pops(P);
    const bool wf = ctx->want_freq && !many;
    const int Q = 3 + Pp + Pp * (Pp - 1) / 2 + (wf ? Pp : 0);
    // The bit-sliced pass over the packed companion moves 3/8 of the one-hot bytes and is the faster one at every shape;
    // the byte pass runs when the context has no companion, and PG_K1_BYTE_PASS selects it for the tests that compare the two.
    const bool packed = ctx->d_packed != nullptr && !getenv("PG_K1_BYTE_PASS");
    K1Cache& c = *cache_of(ctx, 0);
    UniformPass& u = c.up;
    if (!c.valid || c.epoch != ctx->epoch || c.packed != packed) {
        c.valid = false;
        int maxN = 0;
        for (int x = 0; x < P; ++x) {
            int N = 0;
            for (int h = 0; h < ctx->H; ++h) N += ctx->hap_pop[h] == x;
            PG_CHECK(N >= 1, "pg_popgen: population %d has no haplotypes", x);
            maxN = std::max(maxN, N);
        }
        std::vector<int32_t> collapsed;
        if (many) {
            collapsed.assign(ctx->hap_pop.begin(), ctx->hap_pop.end());
            for (int32_t& v : collapsed) v = v >= 0 ? 0 : -1;
        }
        const std::vector<int32_t>& pop_map = many ? collapsed : ctx->hap_pop;
        PopTables pt;
        if (packed) {
            // the rows the byte pass refuses are refused here too, so that whether a call runs never depends on the
            // companion having found memory
            K1Plan bp;
            PG_TRY(byte_plan(ctx, pop_map, Pp, k1_nw_for(ctx->pitch, false), 0, pt, bp));
            c.lanepop = false;
            const int nw = k1_nw_for(ctx->packed_pitch, false);
            PG_TRY(prepare_windowed(ctx, c, pop_map, Pp, Q, nw, /*force_G=*/0, /*packed=*/true));
            u.one_plane = Pp < 8;
            // the stream's kernel also keeps varied_mma's B operand in shared memory, where it has one-plane rows
            u.table_bytes = table_bytes_of(c.pt) + (u.one_plane ? (int)c.pt.bit_frag.size() * 4 : 0);
            u.plan = c.L.plan;
            u.wd = (ctx->H + 31) / 32;
            u.slots_epoch = 0;                                  // u.L follows c.L
        } else {
            // long rows, 4 or 8 real populations of <= 255 haplotypes: one lane per population (k1_site_pass_lp)
            build_tables(pop_map, ctx->H, ctx->pitch / 16, Pp, pt);
            const WarpChoice wc = choose_warps(ctx, ctx->S, Pp, Pp == P, table_bytes_of(pt), byte_counts(maxN));
            c.lanepop = wc.lanepop;
            PG_TRY(prepare_windowed(ctx, c, pop_map, Pp, Q, wc.nw, wc.lanepop ? Pp : 0, /*packed=*/false));
        }
        c.packed = packed;
        c.epoch = ctx->epoch;
        c.valid = true;
    }
    // The packed pass streams only the varied rows when enough sites are uniform (uniform_prepare); PG_K1_NO_UNIFORM keeps
    // every row streamed, for the tests that compare the two.
    const bool uni = c.packed && ctx->d_site_cls && !getenv("PG_K1_NO_UNIFORM");
    if (c.packed) uni_geometry(u);
    if (uni) PG_TRY(uniform_prepare(ctx, u));
    u.last = uni && u.us.in_use;
    if (u.last) PG_TRY(uniform_slots(ctx, u, c.L, Q));
    K1Launch& L = u.last ? u.L : c.L;
    {
        long long maxN = 1;
        for (int X = 0; X < Pp; ++X) maxN = std::max<long long>(maxN, c.pt.popN[X]);
        L.prm.acc_limit = (int)std::max<long long>(1, std::min<long long>(0xffffffffll / (maxN * maxN), 1 << 30));
        if (const char* e = getenv("PG_K1_ACC_LIMIT")) L.prm.acc_limit = std::max(1, atoi(e));   // test hook: force early flushes
        L.prm.bytes = byte_counts((int)maxN) ? 1 : 0;
        L.prm.lanepop = c.lanepop ? 1 : 0;
        const char* gv = getenv("PG_K1_UNI_GV");           // test hook: lanes per varied row (1, 2, 4, ... 32)
        L.prm.uni_gv = u.last && gv && *gv ? atoi(gv) : 0;
        PG_CHECK(L.prm.uni_gv >= 0 && L.prm.uni_gv <= 32 && (L.prm.uni_gv & (L.prm.uni_gv - 1)) == 0,
                 "PG_K1_UNI_GV must be a power of two up to 32");
    }
    PG_TRY(arm_slots(ctx, L, u.last ? u.us.rows.p : c.packed ? (const void*)ctx->d_packed : ctx->d_geno));
    PG_TRY(with_popgen_mode(wf, Pp, [&](auto M, auto PP) {
        constexpr int MODE = decltype(M)::value, PT = decltype(PP)::value;
        if (u.last) return launch_site_pass_packed<MODE, PT, true>(ctx, L, "k1_popgen", u.launched);
        if (c.packed) return launch_site_pass_packed<MODE, PT, false>(ctx, L, "k1_popgen");
        return launch_site_pass<MODE, PT>(ctx, L, "k1_popgen");
    }));

    PG_TRY(ctx->out_i.ensure((size_t)W * 4 + 128));
    int* d_cnt = (int*)ctx->out_i.p;
    int32_t* d_path = (int32_t*)ctx->out_i.p + 16;
    PG_CUDA(cudaMemsetAsync(d_cnt, 0, 4, ctx->stream));
    FinParams fp;
    fill_fin(fp, ctx, c, L.slots, Q, Q);
    fp.P = P;
    fp.Ppad = Pp;
    fp.min_sites = min_sites;
    fp.min_data = min_data;
    fp.force_path = many ? 2 : force_path;
    fp.bookkeeping_only = many ? 1 : 0;
    fp.with_freq = wf ? 1 : 0;
    if (u.last) {
        fp.pre_uni = (const int64_t*)u.us.pre.p;
        fp.pre_pos = fp.pre_uni + ctx->S + 1;
        fp.S = ctx->S;
    }
    fp.rec = (unsigned long long*)d_rec;
    fp.RC = RC;
    fp.path = d_path;
    fp.n_pairwise = d_cnt;
    PG_TRY(launch_finalize<MODE_POPGEN>(ctx, fp));
    if (!h_count) return PG_OK;
    void* hp = nullptr;
    PG_TRY(pg_pinned(ctx, (size_t)W * 4 + 256, &hp));
    int* h_cnt = (int*)hp;
    *h_cnt = 0;
    PG_CUDA(cudaMemcpyAsync(h_cnt, d_cnt, 4, cudaMemcpyDeviceToHost, ctx->stream));
    *h_count = h_cnt;
    return PG_OK;
}

extern "C" int pg_debug_uniform(pg_ctx* ctx, int32_t* in_use, int64_t* varied_sites) {
    PG_CHECK(ctx && in_use && varied_sites, "pg_debug_uniform: null argument");
    const K1Cache* c = static_cast<const K1Cache*>(ctx->k1_cache[0]);
    const bool read = c && c->up.last;
    *in_use = read ? 1 : 0;
    *varied_sites = (c && c->up.us.gen == ctx->data_gen) ? c->up.us.varied : ctx->S;
    return PG_OK;
}

extern "C" int pg_debug_uniform_tile(pg_ctx* ctx, int32_t* out) {
    PG_CHECK(ctx && out, "pg_debug_uniform_tile: null argument");
    const K1Cache* c = static_cast<const K1Cache*>(ctx->k1_cache[0]);
    const bool planned = c && c->valid && c->packed;
    out[0] = planned ? c->up.Tmax : 0;
    out[1] = planned ? c->up.plan.wpt : 0;
    return PG_OK;
}

extern "C" int pg_debug_uniform_ring(pg_ctx* ctx, int32_t* out) {
    PG_CHECK(ctx && out, "pg_debug_uniform_ring: null argument");
    const K1Cache* c = static_cast<const K1Cache*>(ctx->k1_cache[0]);
    const bool read = c && c->up.last;
    out[0] = read ? c->up.cap_rows : 0;
    out[1] = read ? c->up.stages : 0;
    out[2] = read ? c->up.stage_bytes : 0;
    return PG_OK;
}

extern "C" int pg_debug_uniform_launch(pg_ctx* ctx, int32_t* out) {
    PG_CHECK(ctx && out, "pg_debug_uniform_launch: null argument");
    const K1Cache* c = static_cast<const K1Cache*>(ctx->k1_cache[0]);
    const bool read = c && c->up.last;
    for (int k = 0; k < 3; ++k) out[k] = read ? c->up.launched[k] : 0;
    return PG_OK;
}

extern "C" int pg_debug_uniform_tiles(pg_ctx* ctx, int64_t cap, int64_t* site_lo, int64_t* row0, int64_t* ntiles,
                                      int32_t* geometry) {
    PG_CHECK(ctx && ntiles && geometry, "pg_debug_uniform_tiles: null argument");
    const K1Cache* c = static_cast<const K1Cache*>(ctx->k1_cache[0]);
    const bool read = c && c->up.last;
    const UniformStream* us = read ? &c->up.us : nullptr;
    *ntiles = read ? us->nt : 0;
    geometry[0] = read ? c->up.cap_rows : 0;
    geometry[1] = read ? c->up.Tmax : 0;
    if (!read || cap < us->nt + 1) return PG_OK;
    PG_CHECK(site_lo && row0, "pg_debug_uniform_tiles: null table");
    PG_CUDA(cudaSetDevice(ctx->device));
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    PG_CUDA(cudaMemcpy(site_lo, us->site_lo.p, (size_t)(us->nt + 1) * 8, cudaMemcpyDeviceToHost));
    PG_CUDA(cudaMemcpy(row0, us->row0.p, (size_t)(us->nt + 1) * 8, cudaMemcpyDeviceToHost));
    return PG_OK;
}

extern "C" int pg_debug_uniform_rows(pg_ctx* ctx, int64_t* one_plane_rows, int64_t* words) {
    PG_CHECK(ctx && one_plane_rows && words, "pg_debug_uniform_rows: null argument");
    const K1Cache* c = static_cast<const K1Cache*>(ctx->k1_cache[0]);
    const bool read = c && c->up.last;
    *one_plane_rows = *words = 0;
    if (!read) return PG_OK;
    const UniformStream& us = c->up.us;
    PG_CUDA(cudaSetDevice(ctx->device));
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    std::vector<int32_t> n1((size_t)us.nt);
    PG_CUDA(cudaMemcpy(n1.data(), us.n1.p, n1.size() * 4, cudaMemcpyDeviceToHost));
    PG_CUDA(cudaMemcpy(words, us.woff + us.nt, 8, cudaMemcpyDeviceToHost));
    for (int32_t v : n1) *one_plane_rows += v;
    return PG_OK;
}

// After the stream has been synchronised: run the pairwise path for the windows the finalize kernel routed to it
// (their rows of d_rec are overwritten in place).
int pg_popgen_resolve(pg_ctx* ctx, int32_t min_sites, double min_data, void* d_rec, int nk2) {
    if (nk2 <= 0) return PG_OK;
    const int P = ctx->P;
    const int RC = 3 + P + 2 * (P * (P - 1) / 2) + 1 + 4 * P;
    const int64_t W = ctx->W;
    const int32_t* d_path = (const int32_t*)ctx->out_i.p + 16;
    std::vector<int32_t> h_path((size_t)W);
    PG_CUDA(cudaMemcpyAsync(h_path.data(), d_path, (size_t)W * 4, cudaMemcpyDeviceToHost, ctx->stream));
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    std::vector<int64_t> k2_windows;
    k2_windows.reserve((size_t)nk2);
    for (int64_t w = 0; w < W; ++w)
        if (h_path[w] == 2) k2_windows.push_back(w);
    return pg_k2_popgen_windows(ctx, k2_windows, ctx->win_lo.data(), ctx->win_hi.data(), min_sites, min_data, d_rec, RC);
}

// Device-record variant: d_rec is a DEVICE buffer of W * (4 + 5P + 2*npairs) 8-byte words.
extern "C" int pg_popgen_device(pg_ctx* ctx, int32_t min_sites, double min_data, int32_t force_path, void* d_rec,
                                int64_t* n_pairwise) {
    if (n_pairwise) *n_pairwise = 0;
    int* h_cnt = nullptr;
    PG_TRY(pg_popgen_enqueue(ctx, min_sites, min_data, force_path, d_rec, &h_cnt));
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    const int nk2 = h_cnt ? *h_cnt : 0;
    if (n_pairwise) *n_pairwise = nk2;
    return pg_popgen_resolve(ctx, min_sites, min_data, d_rec, nk2);
}


extern "C" int pg_popgen(pg_ctx* ctx, int32_t min_sites, double min_data, int32_t force_path, double* pi, double* dxy,
                         double* fst, int64_t* n_sites, int64_t* pos_sum, int32_t* path) {
    PG_CHECK(ctx && pi && dxy && fst && n_sites && pos_sum && path, "pg_popgen: null argument");
    PG_CHECK(ctx->P >= 1, "pg_popgen: call pg_set_pops first");
    PG_CHECK(ctx->P <= PG_MAX_POPS, "pg_popgen: P=%d > %d populations", ctx->P, PG_MAX_POPS);
    const int P = ctx->P;
    const int npairs = P * (P - 1) / 2;
    const int RC = 3 + P + 2 * npairs + 1 + 4 * P;
    const int64_t W = ctx->W;
    if (W == 0) {
        pg_timings_reset(ctx);
        return PG_OK;
    }
    PG_CUDA(cudaSetDevice(ctx->device));
    PG_TRY(ctx->out_d.ensure((size_t)W * RC * 8 + 64));
    // site pass -> finalize -> D2H of the record table into pinned staging, ONE host synchronisation; only when the
    // finalize kernel routed windows to the pairwise path are those rows recomputed and the table read again
    void* hp = nullptr;
    PG_TRY(pg_pinned(ctx, (size_t)W * RC * 8 + 64 + 256, &hp));     // (+ the routed-window counter of the enqueue step)
    int* h_cnt = nullptr;
    PG_TRY(pg_popgen_enqueue(ctx, min_sites, min_data, force_path, ctx->out_d.p, &h_cnt));
    hp = (uint8_t*)hp + 256;
    const unsigned long long* hrec = (const unsigned long long*)hp;
    PG_CUDA(cudaMemcpyAsync(hp, ctx->out_d.p, (size_t)W * RC * 8, cudaMemcpyDeviceToHost, ctx->stream));
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    const int nk2 = h_cnt ? *h_cnt : 0;
    if (nk2 > 0) {
        PG_TRY(pg_popgen_resolve(ctx, min_sites, min_data, ctx->out_d.p, nk2));
        PG_CUDA(cudaMemcpyAsync(hp, ctx->out_d.p, (size_t)W * RC * 8, cudaMemcpyDeviceToHost, ctx->stream));
        PG_CUDA(cudaStreamSynchronize(ctx->stream));
    }
    if (ctx->want_freq) ctx->h_rec.assign(hrec, hrec + (size_t)W * RC);     // kept for pg_popgen_freqstats
    else ctx->h_rec.clear();
    for (int64_t w = 0; w < W; ++w) {
        const unsigned long long* r = hrec + (size_t)w * RC;
        n_sites[w] = (int64_t)r[0];
        pos_sum[w] = (int64_t)r[1];
        path[w] = (int32_t)r[2];
        memcpy(pi + (size_t)w * P, r + 3, (size_t)P * 8);
        if (npairs) {
            memcpy(dxy + (size_t)w * npairs, r + 3 + P, (size_t)npairs * 8);
            memcpy(fst + (size_t)w * npairs, r + 3 + P + npairs, (size_t)npairs * 8);
        }
    }
    return PG_OK;
}

extern "C" int pg_set_freqstats(pg_ctx* ctx, int32_t enable) {
    PG_CHECK(ctx != nullptr, "pg_set_freqstats: null ctx");
    const bool e = enable != 0;
    if (e != ctx->want_freq) {
        ctx->want_freq = e;
        ctx->epoch += 1;              // the slot layout of the site pass changes
        ctx->h_rec.clear();
    }
    return PG_OK;
}

// popFreq columns of the records produced by the most recent pg_popgen on this ctx
extern "C" int pg_popgen_freqstats(pg_ctx* ctx, double* l, double* S, double* theta_pi, double* theta_w, double* taj_d) {
    PG_CHECK(ctx && l && S && theta_pi && theta_w && taj_d, "pg_popgen_freqstats: null argument");
    const int P = ctx->P;
    const int npairs = P * (P - 1) / 2;
    const int RC = 3 + P + 2 * npairs + 1 + 4 * P;
    const int64_t W = ctx->W;
    PG_CHECK(ctx->want_freq, "pg_popgen_freqstats: enable the popFreq counters first (pg_set_freqstats(ctx, 1))");
    PG_CHECK(ctx->h_rec.size() == (size_t)W * RC, "pg_popgen_freqstats: call pg_popgen first (same pops / windows)");
    for (int64_t w = 0; w < W; ++w) {
        const double* f = reinterpret_cast<const double*>(ctx->h_rec.data() + (size_t)w * RC + 3 + P + 2 * npairs);
        l[w] = f[0];
        memcpy(S + (size_t)w * P, f + 1, (size_t)P * 8);
        memcpy(theta_pi + (size_t)w * P, f + 1 + P, (size_t)P * 8);
        memcpy(theta_w + (size_t)w * P, f + 1 + 2 * P, (size_t)P * 8);
        memcpy(taj_d + (size_t)w * P, f + 1 + 3 * P, (size_t)P * 8);
    }
    return PG_OK;
}

// ================================================================================================
// pg_abbababa
// ================================================================================================
// Enqueue site pass + finalize of the ABBA-BABA statistics on the ctx stream; records [W x 8] 8-byte words
// [sites, pos_sum, ABBA, BABA, D, fd, fdM, sitesUsed] are left in the DEVICE buffer d_rec.  No synchronisation.
int pg_abba_enqueue(pg_ctx* ctx, const int* sel, double min_data, void* d_rec) {
    return fourpop_enqueue<MODE_ABBA>(ctx, "pg_abbababa", 1, 9, 8, 8, sel, min_data, 0, d_rec, [&](const K1Launch& L) {
        return launch_site_pass<MODE_ABBA, 4>(ctx, L, "k1_abba");
    });
}

extern "C" int pg_abbababa(pg_ctx* ctx, int32_t p1, int32_t p2, int32_t p3, int32_t o, double min_data, double* out,
                           double* sites_used, int64_t* n_sites, int64_t* pos_sum) {
    PG_CHECK(ctx && out && sites_used && n_sites && pos_sum, "pg_abbababa: null argument");
    const int sel[4] = {p1, p2, p3, o};
    return fourpop_read(ctx, 8, [&](void* d_rec) { return pg_abba_enqueue(ctx, sel, min_data, d_rec); }, out, sites_used,
                        n_sites, pos_sum);
}

// ================================================================================================
// pg_fourpop
// ================================================================================================
// Enqueue site pass + finalize of genomics.fourPop; records [W x 17] words [sites, pos_sum, 14 statistics, sitesUsed]
// are left in the DEVICE buffer d_rec.  No synchronisation.
int pg_fourpop_enqueue(pg_ctx* ctx, const int* sel, double min_data, int mode, void* d_rec) {
    PG_CHECK(mode >= 0 && mode <= 2, "pg_fourpop: mode must be 0 (default), 1 (polarize) or 2 (fixed)");
    // sitesUsed of a record without sites is 0.0, not NaN
    return fourpop_enqueue<MODE_FOURPOP>(ctx, "pg_fourpop", 2, 19, 17, 16, sel, min_data, mode, d_rec, [&](const K1Launch& L) {
        return launch_site_pass<MODE_FOURPOP, 4>(ctx, L, "k1_fourpop");
    });
}

extern "C" int pg_fourpop(pg_ctx* ctx, int32_t p1, int32_t p2, int32_t p3, int32_t p4, double min_data, int32_t mode,
                          double* out, double* sites_used, int64_t* n_sites, int64_t* pos_sum) {
    PG_CHECK(ctx && out && sites_used && n_sites && pos_sum, "pg_fourpop: null argument");
    const int sel[4] = {p1, p2, p3, p4};
    return fourpop_read(ctx, 17, [&](void* d_rec) { return pg_fourpop_enqueue(ctx, sel, min_data, mode, d_rec); }, out,
                        sites_used, n_sites, pos_sum);
}

// ================================================================================================
// pg_site_counts / pg_site_target_freqs
// ================================================================================================
namespace {
// Many small populations (freq.py --indFreqs: one population per individual): one thread per (site, population) gathers
// the population's few haplotype bytes — ONE pass over the rows instead of P/8 site passes.
__global__ void __launch_bounds__(256) k1_counts_gather(const uint8_t* __restrict__ geno, int pitch, int64_t site0, int64_t n,
                                                        int P, const int32_t* __restrict__ pop_off,
                                                        const int32_t* __restrict__ pop_cols, uint16_t* __restrict__ out) {
    const int64_t total = n * P;
    for (int64_t idx = (int64_t)blockIdx.x * 256 + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * 256) {
        const int64_t s = idx / P;
        const int X = (int)(idx % P);
        const uint8_t* row = geno + (site0 + s) * pitch;
        unsigned a = 0, c = 0, g = 0, t = 0;
        for (int k = pop_off[X]; k < pop_off[X + 1]; ++k) {
            const unsigned b = row[pop_cols[k]];            // one-hot: A 0x01, C 0x04, G 0x10, T 0x40
            a += b & 1u;
            c += (b >> 2) & 1u;
            g += (b >> 4) & 1u;
            t += (b >> 6) & 1u;
        }
        reinterpret_cast<ushort4*>(out)[idx] = make_ushort4((unsigned short)a, (unsigned short)c, (unsigned short)g, (unsigned short)t);
    }
}

// per-site counts of `cnt` sites starting at `first` -> ctx->misc as uint16 [cnt x P x 4]
int site_counts_slab(pg_ctx* ctx, int64_t first, int64_t cnt) {
    const int P = ctx->P;
    const int64_t stride = (int64_t)P * 4;
    if (P > 16 && !getenv("PG_COUNTS_NO_GATHER")) {
        std::vector<int32_t> off(P + 1, 0), cols;
        cols.reserve((size_t)ctx->H);
        for (int X = 0; X < P; ++X) {
            off[X] = (int32_t)cols.size();
            for (int h = 0; h < ctx->H; ++h)
                if (ctx->hap_pop[h] == X) cols.push_back(h);
        }
        off[P] = (int32_t)cols.size();
        PG_TRY(ctx->tables.ensure((size_t)(P + 1) * 4 + cols.size() * 4 + 256));
        uint8_t* base = (uint8_t*)ctx->tables.p;
        size_t o = 0;
        int32_t *d_off = nullptr, *d_cols = nullptr;
        PG_TRY(push(ctx, base, o, off.data(), off.size(), &d_off));
        PG_TRY(push(ctx, base, o, cols.data(), cols.size(), &d_cols));
        const int ti = pg_time_begin(ctx, "k1_counts");
        k1_counts_gather<<<(unsigned)std::min<int64_t>((cnt * P + 255) / 256, (int64_t)ctx->sm_count * 32), 256, 0, ctx->stream>>>(
            (const uint8_t*)ctx->d_geno, ctx->pitch, first, cnt, P, d_off, d_cols, (uint16_t*)ctx->misc.p);
        pg_time_end(ctx, ti);
        PG_CUDA(cudaGetLastError());
        PG_CUDA(cudaStreamSynchronize(ctx->stream));       // host vectors behind the async copies
        return PG_OK;
    }
    for (int p0 = 0; p0 < P; p0 += PG_MAX_K1_POPS) {
        const int pc = std::min(PG_MAX_K1_POPS, P - p0);
        const int Pp = pad_pops(pc);
        std::vector<int32_t> local(ctx->H, -1);
        for (int h = 0; h < ctx->H; ++h)
            if (ctx->hap_pop[h] >= p0 && ctx->hap_pop[h] < p0 + pc) local[h] = ctx->hap_pop[h] - p0;
        PopTables pt;
        build_tables(local, ctx->H, ctx->pitch / 16, Pp, pt);
        const int table_bytes = table_bytes_of(pt);
        PG_CHECK(table_bytes <= 48 * 1024, "population layout needs too many mask entries");
        K1Launch L;
        // long rows, a full group of 4 or 8 populations: one lane per population
        const WarpChoice wc = choose_warps(ctx, cnt, Pp, Pp == pc, table_bytes, true);
        L.plan = pg_make_k1_plan(cnt, ctx->H, ctx->sm_count, table_bytes, wc.nw, wc.lanepop ? Pp : 0);
        PG_CHECK(L.plan.stages >= 2, "rows of %d haplotypes are too long for the site-pass kernel", ctx->H);
        PG_TRY(check_plan(L.plan));
        PG_TRY(ctx->tables.ensure(pt.ent_chunk.size() * 20 + 4096));
        uint8_t* base = (uint8_t*)ctx->tables.p;
        size_t o = 0;
        DevTables dt = {};
        uint32_t* d_mask_words = nullptr;
        PG_TRY(push(ctx, base, o, pt.ent_mask.data(), pt.ent_mask.size(), &d_mask_words));
        dt.ent_mask = reinterpret_cast<uint4*>(d_mask_words);
        PG_TRY(push(ctx, base, o, pt.ent_chunk.data(), pt.ent_chunk.size(), &dt.ent_chunk));
        K1Params& p = L.prm;
        fill_params(p, ctx, L.plan, pt, dt, /*packed=*/false);
        p.site_begin = first;
        p.site_end = first + cnt;
        p.counts_out = (uint16_t*)ctx->misc.p + (size_t)p0 * 4;
        p.counts_stride = stride;
        p.counts_pops = pc;
        p.lanepop = wc.lanepop ? 1 : 0;
        PG_TRY(with_pops(Pp, [&](auto PP) { return launch_site_pass<MODE_COUNTS, decltype(PP)::value>(ctx, L, "k1_counts"); }));
        // the table buffer (and the host vectors behind the async copies) are reused by the next group
        PG_CUDA(cudaStreamSynchronize(ctx->stream));
    }
    return PG_OK;
}

// freq.py --target (freq.py:62-92): one thread per site turns the per-population counts into the frequency (or
// count) of the target allele.  target 1 = derived (last population is the outgroup; derivedAllele, genomics.py:636-659),
// 2 = minor (minorAllele, 663-668; an exact tie, random in the reference, takes the lower allele and is flagged).
__global__ void __launch_bounds__(256) k1_target_freqs(const uint16_t* __restrict__ counts, int64_t n, int P, int target,
                                                       double min_data, int as_counts, double* __restrict__ out,
                                                       uint8_t* __restrict__ tie) {
    const int64_t s = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (s >= n) return;
    const ushort4* c = reinterpret_cast<const ushort4*>(counts) + s * P;
    unsigned in[4] = {0, 0, 0, 0}, outg[4] = {0, 0, 0, 0};
    for (int X = 0; X < P; ++X) {
        const ushort4 v = c[X];
        unsigned* dst = (target == 1 && X == P - 1) ? outg : in;
        dst[0] += v.x;
        dst[1] += v.y;
        dst[2] += v.z;
        dst[3] += v.w;
    }
    int tgt = -1;
    bool tied = false;
    if (target == 1) {
        int n_in = 0, n_out = 0, oa = -1;
        for (int a = 0; a < 4; ++a) {
            n_in += in[a] > 0;
            if (outg[a] > 0) {
                ++n_out;
                oa = a;
            }
        }
        if (n_out == 1 && n_in == 2 && in[oa] > 0)
            for (int a = 0; a < 4; ++a)
                if (in[a] > 0 && a != oa) tgt = a;
    } else {
        int a0 = -1, a1 = -1, na = 0;
        for (int a = 0; a < 4; ++a)
            if (in[a] > 0) {
                if (na == 0) a0 = a; else a1 = a;
                ++na;
            }
        if (na == 2) {
            tied = in[a0] == in[a1];
            tgt = in[a1] < in[a0] ? a1 : a0;
        }
    }
    if (tie) tie[s] = tied ? 1 : 0;
    const double none = as_counts ? 0.0 : __longlong_as_double(0x7ff8000000000000ll);
    for (int X = 0; X < P; ++X) {
        const ushort4 v = c[X];
        const unsigned nk = (unsigned)v.x + v.y + v.z + v.w;
        double r = none;
        if (tgt >= 0 && (double)nk >= min_data) {            // siteNonNan() >= minData compares a COUNT (freq.py:79)
            const unsigned k = tgt == 0 ? v.x : (tgt == 1 ? v.y : (tgt == 2 ? v.z : v.w));
            if (as_counts) r = (double)k;
            else if (nk > 0) r = (double)k / (double)nk;     // nan when the population has no data (genomics.py:597)
        }
        out[s * P + X] = r;
    }
}
}  // namespace

extern "C" int pg_site_counts(pg_ctx* ctx, int64_t site0, int64_t n, uint16_t* counts) {
    PG_CHECK(ctx && counts, "pg_site_counts: null argument");
    PG_CHECK(ctx->P >= 1, "pg_site_counts: call pg_set_pops first");
    PG_CHECK(site0 >= 0 && n >= 0 && site0 + n <= ctx->S, "pg_site_counts: range outside the uploaded sites");
    PG_CUDA(cudaSetDevice(ctx->device));
    pg_timings_reset(ctx);
    if (n == 0) return PG_OK;
    const int64_t stride = (int64_t)ctx->P * 4;
    // bounded device output buffer: process the range in slabs
    const int64_t slab = std::max<int64_t>(1, std::min<int64_t>(n, (int64_t)(1ll << 30) / (stride * 2)));
    PG_TRY(ctx->misc.ensure((size_t)slab * stride * 2 + 64));
    for (int64_t s = 0; s < n; s += slab) {
        const int64_t cnt = std::min(slab, n - s);
        PG_TRY(site_counts_slab(ctx, site0 + s, cnt));
        PG_TRY(pg_d2h_staged(ctx, counts + (size_t)s * stride, ctx->misc.p, (size_t)cnt * stride * 2));
    }
    return PG_OK;
}

extern "C" int pg_site_target_freqs(pg_ctx* ctx, int64_t site0, int64_t n, int32_t target, double min_data,
                                    int32_t as_counts, double* out, uint8_t* tie) {
    PG_CHECK(ctx && out, "pg_site_target_freqs: null argument");
    PG_CHECK(ctx->P >= 1, "pg_site_target_freqs: call pg_set_pops first");
    PG_CHECK(target == 1 || target == 2, "pg_site_target_freqs: target must be 1 (derived) or 2 (minor)");
    PG_CHECK(target != 1 || ctx->P >= 2, "pg_site_target_freqs: derived needs an outgroup population (the last one)");
    PG_CHECK(site0 >= 0 && n >= 0 && site0 + n <= ctx->S, "pg_site_target_freqs: range outside the uploaded sites");
    PG_CUDA(cudaSetDevice(ctx->device));
    pg_timings_reset(ctx);
    if (n == 0) return PG_OK;
    const int P = ctx->P;
    const int64_t stride = (int64_t)P * 4;
    const int64_t slab = std::max<int64_t>(1, std::min<int64_t>(n, (int64_t)(1ll << 28) / (stride * 2)));
    PG_TRY(ctx->misc.ensure((size_t)slab * stride * 2 + 64));
    PG_TRY(ctx->out_d.ensure((size_t)slab * P * 8 + (size_t)slab + 64));
    double* d_out = (double*)ctx->out_d.p;
    uint8_t* d_tie = (uint8_t*)(d_out + (size_t)slab * P);
    for (int64_t s = 0; s < n; s += slab) {
        const int64_t cnt = std::min(slab, n - s);
        PG_TRY(site_counts_slab(ctx, site0 + s, cnt));
        const int ti = pg_time_begin(ctx, "k1_target_freqs");
        k1_target_freqs<<<(unsigned)((cnt + 255) / 256), 256, 0, ctx->stream>>>((const uint16_t*)ctx->misc.p, cnt, P, target,
                                                                              min_data, as_counts ? 1 : 0, d_out, d_tie);
        pg_time_end(ctx, ti);
        PG_CUDA(cudaGetLastError());
        PG_TRY(pg_d2h_staged(ctx, out + (size_t)s * P, d_out, (size_t)cnt * P * 8));
        if (tie) PG_TRY(pg_d2h_staged(ctx, tie + s, d_tie, (size_t)cnt));
    }
    return PG_OK;
}

// ================================================================================================
// pg_sfs — sfs.py's per-site loop for --inputType genotypes (sfs.py:430-470, getTargetCounts 68-92, SparseFS 94-125)
// ================================================================================================
namespace {
// One non-empty cell of a sparse spectrum (or one site before the reduction): its count and the first site that hit it.
struct SfsRun {
    long long count, first;
};

struct SfsParams {
    const uint16_t* counts;     // [n x P x 4] of this slab
    int64_t n, site0;           // sites of the slab, absolute index of its first site
    int P, n_in, outgroup;      // in-group = populations 0 .. n_in-1; outgroup = population index or -1
    int popN[PG_MAX_POPS];      // haplotypes per population: an in-group population must be complete (sfs.py:449)
    int dims[PG_MAX_POPS];      // radix of each population in the histograms (largest possible count + 1)
    int require_complete;       // genotype input only
    const int32_t* targets;     // targetCounts input: [n x P] counts of the target allele, no allele logic at all
    const uint8_t* mask;        // [S] absolute, or nullptr
    int n_groups;
    const int32_t* group_off;   // [n_groups+1] into group_pops
    const int32_t* group_pops;
    const long long* hist_off;  // [n_groups] first cell of each group's dense histogram
    unsigned long long* hist;
    long long* first;           // first site (absolute) that hit the cell
    unsigned long long* n_counted;
    // sparse path (k1_sfs_keys): the slab's counted sites are packed; entry j of spectrum g is at g * key_stride + j
    unsigned long long* keys;   // dense flat index of the cell
    SfsRun* runs;               // {1, absolute site}
    int64_t key_stride;
};

// sfs.py's per-site test (430-474), shared by the dense and the sparse path: is site s of the slab counted, and which
// allele is its target.  target = -1: a targetCounts row (sfs.py:472-474), whose table already holds the counts.
__device__ __forceinline__ bool sfs_site_target(const SfsParams& sp, int64_t s, int& target) {
    const int64_t site = sp.site0 + s;
    if (sp.mask && !sp.mask[site]) return false;
    target = -1;
    if (sp.targets) return true;
    const ushort4* c = reinterpret_cast<const ushort4*>(sp.counts) + s * sp.P;
    unsigned tot[4] = {0, 0, 0, 0};
    for (int X = 0; X < sp.n_in; ++X) {
        const ushort4 v = c[X];
        if (sp.require_complete && (int)v.x + v.y + v.z + v.w != sp.popN[X]) return false;   // every in-group haplotype called (449)
        tot[0] += v.x;
        tot[1] += v.y;
        tot[2] += v.z;
        tot[3] += v.w;
    }
    if (sp.outgroup >= 0) {
        const ushort4 o = c[sp.outgroup];
        const unsigned oc[4] = {o.x, o.y, o.z, o.w};
        int n_all = 0, n_out = 0;
        for (int a = 0; a < 4; ++a) {
            n_all += (tot[a] > 0 || oc[a] > 0) ? 1 : 0;
            n_out += oc[a] > 0 ? 1 : 0;
        }
        if (n_all < 1 || n_all > 2) return false;                    // 79
        // `outgroupMono & nOutAlleles != 1` is (outgroupMono & nOutAlleles) != 1: the count must be odd, i.e. 1 (84)
        if (n_out == 0 || (n_out & 1) != 1) return false;
        for (int a = 3; a >= 0; --a)
            if (tot[a] > 0 && oc[a] == 0) target = a;               // first in-group allele the outgroup lacks (86)
        if (target < 0)
            for (int a = 3; a >= 0; --a)
                if (tot[a] == 0) target = a;                         // invariant: first absent allele (87), count 0
        return target >= 0;
    }
    int n_all = 0;
    for (int a = 0; a < 4; ++a) n_all += tot[a] > 0 ? 1 : 0;
    if (n_all < 1 || n_all > 2) return false;
    // totalBaseCounts.argsort()[-2] (90): second in a stable ascending order = with two alleles the rarer one, the
    // lower allele on an exact tie; with one allele an absent allele (count 0 everywhere)
    int best = -1, second = -1;                                      // positions [-1] and [-2] of the stable argsort
    for (int a = 0; a < 4; ++a) {
        if (best < 0 || tot[a] >= tot[best]) {
            second = best;
            best = a;
        } else if (second < 0 || tot[a] >= tot[second]) second = a;
    }
    target = second;
    return true;
}

// Row-major mixed-radix index of the site's cell in spectrum g: the dense histogram's flat index, and the sparse key.
__device__ __forceinline__ long long sfs_cell(const SfsParams& sp, int64_t s, int target, int g) {
    long long idx = 0;
    if (target < 0) {
        const int32_t* t = sp.targets + s * sp.P;
        for (int k = sp.group_off[g]; k < sp.group_off[g + 1]; ++k) idx = idx * sp.dims[sp.group_pops[k]] + t[sp.group_pops[k]];
        return idx;
    }
    const ushort4* c = reinterpret_cast<const ushort4*>(sp.counts) + s * sp.P;
    for (int k = sp.group_off[g]; k < sp.group_off[g + 1]; ++k) {
        const int X = sp.group_pops[k];
        const ushort4 v = c[X];
        const unsigned t = target == 0 ? v.x : (target == 1 ? v.y : (target == 2 ? v.z : v.w));
        idx = idx * sp.dims[X] + t;
    }
    return idx;
}

__global__ void __launch_bounds__(256) k1_sfs(const __grid_constant__ SfsParams sp) {
    const int64_t s = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (s >= sp.n) return;
    int target;
    if (!sfs_site_target(sp, s, target)) return;
    const int64_t site = sp.site0 + s;
    atomicAdd(sp.n_counted, 1ull);
    for (int g = 0; g < sp.n_groups; ++g) {
        const long long idx = sfs_cell(sp, s, target, g);
        atomicAdd(sp.hist + sp.hist_off[g] + idx, 1ull);
        atomicMin(sp.first + sp.hist_off[g] + idx, (long long)site);
    }
}

// Sparse path: every counted site of the slab writes its cell of every spectrum as a (key, {1, site}) entry.  The
// entries are packed by a warp-aggregated counter (n_counted, zeroed per slab), so their order within the slab is that of
// the atomics; the reduction that follows sums counts and takes the minimum site, which no order changes.
__global__ void __launch_bounds__(256) k1_sfs_keys(const __grid_constant__ SfsParams sp) {
    const int64_t s = (int64_t)blockIdx.x * 256 + threadIdx.x;
    int target = -1;
    const bool ok = s < sp.n && sfs_site_target(sp, s, target);
    const unsigned m = __ballot_sync(0xffffffffu, ok);
    if (m == 0) return;
    const int lane = threadIdx.x & 31, leader = __ffs(m) - 1;
    unsigned long long base = 0;
    if (lane == leader) base = atomicAdd(sp.n_counted, (unsigned long long)__popc(m));
    base = __shfl_sync(0xffffffffu, base, leader);
    if (!ok) return;
    const int64_t j = (int64_t)base + __popc(m & ((1u << lane) - 1u));
    const long long site = sp.site0 + s;
    for (int g = 0; g < sp.n_groups; ++g) {
        sp.keys[g * sp.key_stride + j] = (unsigned long long)sfs_cell(sp, s, target, g);
        sp.runs[g * sp.key_stride + j] = SfsRun{1, site};
    }
}

struct SfsRunMerge {
    __device__ __forceinline__ SfsRun operator()(const SfsRun& a, const SfsRun& b) const {
        return SfsRun{a.count + b.count, a.first < b.first ? a.first : b.first};
    }
};

__global__ void sfs_runs_split(const SfsRun* __restrict__ runs, int64_t n, long long* __restrict__ count,
                               long long* __restrict__ first) {
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= n) return;
    const SfsRun r = runs[i];
    count[i] = r.count;
    first[i] = r.first;
}
}  // namespace

extern "C" int pg_sfs(pg_ctx* ctx, int32_t n_in, int32_t outgroup, int32_t n_groups, const int32_t* group_off,
                      const int32_t* group_pops, const uint8_t* site_mask, int64_t* hist, int64_t* first, int64_t* n_counted) {
    PG_CHECK(ctx && group_off && group_pops && hist && first, "pg_sfs: null argument");
    PG_CHECK(ctx->P >= 1 && ctx->P <= PG_MAX_POPS, "pg_sfs: call pg_set_pops first (at most %d populations)", PG_MAX_POPS);
    PG_CHECK(n_in >= 1 && n_in <= ctx->P, "pg_sfs: n_in out of range");
    PG_CHECK(outgroup == -1 || (outgroup >= n_in && outgroup < ctx->P), "pg_sfs: the outgroup must be a population after the in-group");
    PG_CHECK(n_groups >= 1, "pg_sfs: no spectra requested");
    PG_CUDA(cudaSetDevice(ctx->device));
    pg_timings_reset(ctx);
    const int P = ctx->P;
    std::vector<int> popN(P, 0);
    for (int h = 0; h < ctx->H; ++h)
        if (ctx->hap_pop[h] >= 0) popN[ctx->hap_pop[h]] += 1;
    std::vector<long long> hist_off(n_groups, 0);
    long long cells = 0;
    for (int g = 0; g < n_groups; ++g) {
        hist_off[g] = cells;
        long long sz = 1;
        PG_CHECK(group_off[g + 1] > group_off[g], "pg_sfs: spectrum %d has no population", g);
        for (int k = group_off[g]; k < group_off[g + 1]; ++k) {
            PG_CHECK(group_pops[k] >= 0 && group_pops[k] < n_in, "pg_sfs: spectrum %d uses a population outside the in-group", g);
            sz *= (long long)popN[group_pops[k]] + 1;
            PG_CHECK(sz <= (1ll << 28), "pg_sfs: spectrum %d is too large for a dense histogram", g);
        }
        cells += sz;
        PG_CHECK(cells <= (1ll << 28), "pg_sfs: the spectra need more than 2^28 cells");
    }
    if (n_counted) *n_counted = 0;
    const int n_gp = group_off[n_groups];
    // device buffers: histograms | first | tables | counter
    PG_TRY(ctx->pairs.ensure((size_t)cells * 16 + 64));
    unsigned long long* d_hist = (unsigned long long*)ctx->pairs.p;
    long long* d_first = (long long*)(d_hist + cells);
    PG_CUDA(cudaMemsetAsync(d_hist, 0, (size_t)cells * 8, ctx->stream));
    PG_CUDA(cudaMemsetAsync(d_first, 0x7f, (size_t)cells * 8, ctx->stream));
    PG_TRY(ctx->misc2.ensure((size_t)(n_groups + 1) * 4 + (size_t)n_gp * 4 + (size_t)n_groups * 8 + 64 + 64));
    uint8_t* tb = (uint8_t*)ctx->misc2.p;
    size_t o = 0;
    int32_t* d_goff = nullptr;
    int32_t* d_gpops = nullptr;
    long long* d_hoff = nullptr;
    PG_TRY(push(ctx, tb, o, group_off, (size_t)n_groups + 1, &d_goff));
    PG_TRY(push(ctx, tb, o, group_pops, (size_t)n_gp, &d_gpops));
    PG_TRY(push(ctx, tb, o, hist_off.data(), (size_t)n_groups, &d_hoff));
    PG_TRY(ctx->out_i.ensure(64));
    unsigned long long* d_cnt = (unsigned long long*)ctx->out_i.p;
    PG_CUDA(cudaMemsetAsync(d_cnt, 0, 8, ctx->stream));
    uint8_t* d_mask = nullptr;
    if (site_mask && ctx->S > 0) {
        PG_TRY(ctx->misc3.ensure((size_t)ctx->S + 64));
        d_mask = (uint8_t*)ctx->misc3.p;
        PG_CUDA(cudaMemcpyAsync(d_mask, site_mask, (size_t)ctx->S, cudaMemcpyHostToDevice, ctx->stream));
    }
    PG_CUDA(cudaStreamSynchronize(ctx->stream));       // host tables behind the async copies
    const int64_t stride = (int64_t)P * 4;
    const int64_t slab = std::max<int64_t>(1, std::min<int64_t>(std::max<int64_t>(ctx->S, 1), (int64_t)(1ll << 28) / (stride * 2)));
    PG_TRY(ctx->misc.ensure((size_t)slab * stride * 2 + 64));
    for (int64_t s0 = 0; s0 < ctx->S; s0 += slab) {
        const int64_t cnt = std::min(slab, ctx->S - s0);
        PG_TRY(site_counts_slab(ctx, s0, cnt));
        SfsParams sp;
        memset(&sp, 0, sizeof(sp));
        sp.counts = (const uint16_t*)ctx->misc.p;
        sp.n = cnt;
        sp.site0 = s0;
        sp.P = P;
        sp.n_in = n_in;
        sp.outgroup = outgroup;
        for (int X = 0; X < P; ++X) {
            sp.popN[X] = popN[X];
            sp.dims[X] = popN[X] + 1;
        }
        sp.require_complete = 1;
        sp.mask = d_mask;
        sp.n_groups = n_groups;
        sp.group_off = d_goff;
        sp.group_pops = d_gpops;
        sp.hist_off = d_hoff;
        sp.hist = d_hist;
        sp.first = d_first;
        sp.n_counted = d_cnt;
        const int ti = pg_time_begin(ctx, "k1_sfs");
        k1_sfs<<<(unsigned)((cnt + 255) / 256), 256, 0, ctx->stream>>>(sp);
        pg_time_end(ctx, ti);
        PG_CUDA(cudaGetLastError());
    }
    unsigned long long h_cnt = 0;
    PG_CUDA(cudaMemcpyAsync(hist, d_hist, (size_t)cells * 8, cudaMemcpyDeviceToHost, ctx->stream));
    PG_CUDA(cudaMemcpyAsync(first, d_first, (size_t)cells * 8, cudaMemcpyDeviceToHost, ctx->stream));
    PG_CUDA(cudaMemcpyAsync(&h_cnt, d_cnt, 8, cudaMemcpyDeviceToHost, ctx->stream));
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    for (long long k = 0; k < cells; ++k)
        if (hist[k] == 0) first[k] = -1;
    if (n_counted) *n_counted = (int64_t)h_cnt;
    return PG_OK;
}

// The same spectra from TABLES of counts on the host (sfs.py --inputType baseCounts | targetCounts, sfs.py:456-474): no
// genotype matrix, no completeness test.  kind 0: table = uint16 [n x P x 4] base counts per population (freq.py's
// default output); kind 1: table = int32 [n x P] counts of the target allele.  dims[X] = largest count of population X + 1.
extern "C" int pg_sfs_tables(pg_ctx* ctx, int32_t kind, const void* table, int64_t n, int32_t P, const int32_t* dims,
                             int32_t n_in, int32_t outgroup, int32_t n_groups, const int32_t* group_off,
                             const int32_t* group_pops, const uint8_t* site_mask, int64_t* hist, int64_t* first,
                             int64_t* n_counted) {
    PG_CHECK(ctx && (table || n == 0) && dims && group_off && group_pops && hist && first, "pg_sfs_tables: null argument");
    PG_CHECK(kind == 0 || kind == 1, "pg_sfs_tables: kind must be 0 (base counts) or 1 (target counts)");
    PG_CHECK(P >= 1 && P <= PG_MAX_POPS, "pg_sfs_tables: at most %d populations", PG_MAX_POPS);
    PG_CHECK(n_in >= 1 && n_in <= P && n >= 0, "pg_sfs_tables: bad shape");
    PG_CHECK(outgroup == -1 || (kind == 0 && outgroup >= n_in && outgroup < P), "pg_sfs_tables: bad outgroup");
    PG_CHECK(n_groups >= 1, "pg_sfs_tables: no spectra requested");
    PG_CUDA(cudaSetDevice(ctx->device));
    pg_timings_reset(ctx);
    std::vector<long long> hist_off(n_groups, 0);
    long long cells = 0;
    for (int g = 0; g < n_groups; ++g) {
        hist_off[g] = cells;
        long long sz = 1;
        PG_CHECK(group_off[g + 1] > group_off[g], "pg_sfs_tables: spectrum %d has no population", g);
        for (int k = group_off[g]; k < group_off[g + 1]; ++k) {
            PG_CHECK(group_pops[k] >= 0 && group_pops[k] < n_in, "pg_sfs_tables: spectrum %d uses a population outside the in-group", g);
            PG_CHECK(dims[group_pops[k]] >= 1, "pg_sfs_tables: dims must be >= 1");
            sz *= (long long)dims[group_pops[k]];
            PG_CHECK(sz <= (1ll << 28), "pg_sfs_tables: spectrum %d is too large for a dense histogram", g);
        }
        cells += sz;
        PG_CHECK(cells <= (1ll << 28), "pg_sfs_tables: the spectra need more than 2^28 cells");
    }
    if (n_counted) *n_counted = 0;
    const int n_gp = group_off[n_groups];
    PG_TRY(ctx->pairs.ensure((size_t)cells * 16 + 64));
    unsigned long long* d_hist = (unsigned long long*)ctx->pairs.p;
    long long* d_first = (long long*)(d_hist + cells);
    PG_CUDA(cudaMemsetAsync(d_hist, 0, (size_t)cells * 8, ctx->stream));
    PG_CUDA(cudaMemsetAsync(d_first, 0x7f, (size_t)cells * 8, ctx->stream));
    PG_TRY(ctx->misc2.ensure((size_t)(n_groups + 1) * 4 + (size_t)n_gp * 4 + (size_t)n_groups * 8 + 128));
    uint8_t* tb = (uint8_t*)ctx->misc2.p;
    size_t o = 0;
    int32_t* d_goff = nullptr;
    int32_t* d_gpops = nullptr;
    long long* d_hoff = nullptr;
    PG_TRY(push(ctx, tb, o, group_off, (size_t)n_groups + 1, &d_goff));
    PG_TRY(push(ctx, tb, o, group_pops, (size_t)n_gp, &d_gpops));
    PG_TRY(push(ctx, tb, o, hist_off.data(), (size_t)n_groups, &d_hoff));
    PG_TRY(ctx->out_i.ensure(64));
    unsigned long long* d_cnt = (unsigned long long*)ctx->out_i.p;
    PG_CUDA(cudaMemsetAsync(d_cnt, 0, 8, ctx->stream));
    uint8_t* d_mask = nullptr;
    if (site_mask && n > 0) {
        PG_TRY(ctx->misc3.ensure((size_t)n + 64));
        d_mask = (uint8_t*)ctx->misc3.p;
        PG_CUDA(cudaMemcpyAsync(d_mask, site_mask, (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
    }
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    const size_t row_bytes = kind == 0 ? (size_t)P * 8 : (size_t)P * 4;
    const int64_t slab = std::max<int64_t>(1, std::min<int64_t>(std::max<int64_t>(n, 1), (int64_t)(((size_t)256 << 20) / row_bytes)));
    PG_TRY(ctx->misc.ensure((size_t)slab * row_bytes + 64));
    for (int64_t s0 = 0; s0 < n; s0 += slab) {
        const int64_t cnt = std::min(slab, n - s0);
        PG_CUDA(cudaMemcpyAsync(ctx->misc.p, (const uint8_t*)table + (size_t)s0 * row_bytes, (size_t)cnt * row_bytes,
                                cudaMemcpyHostToDevice, ctx->stream));
        SfsParams sp;
        memset(&sp, 0, sizeof(sp));
        sp.counts = kind == 0 ? (const uint16_t*)ctx->misc.p : nullptr;
        sp.targets = kind == 1 ? (const int32_t*)ctx->misc.p : nullptr;
        sp.n = cnt;
        sp.site0 = s0;
        sp.P = P;
        sp.n_in = n_in;
        sp.outgroup = outgroup;
        for (int X = 0; X < P; ++X) sp.dims[X] = dims[X];
        sp.require_complete = 0;
        sp.mask = d_mask;
        sp.n_groups = n_groups;
        sp.group_off = d_goff;
        sp.group_pops = d_gpops;
        sp.hist_off = d_hoff;
        sp.hist = d_hist;
        sp.first = d_first;
        sp.n_counted = d_cnt;
        const int ti = pg_time_begin(ctx, "k1_sfs");
        k1_sfs<<<(unsigned)((cnt + 255) / 256), 256, 0, ctx->stream>>>(sp);
        pg_time_end(ctx, ti);
        PG_CUDA(cudaGetLastError());
        PG_CUDA(cudaStreamSynchronize(ctx->stream));           // the staging buffer is reused by the next slab
    }
    unsigned long long h_cnt = 0;
    PG_CUDA(cudaMemcpyAsync(hist, d_hist, (size_t)cells * 8, cudaMemcpyDeviceToHost, ctx->stream));
    PG_CUDA(cudaMemcpyAsync(first, d_first, (size_t)cells * 8, cudaMemcpyDeviceToHost, ctx->stream));
    PG_CUDA(cudaMemcpyAsync(&h_cnt, d_cnt, 8, cudaMemcpyDeviceToHost, ctx->stream));
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    for (long long k = 0; k < cells; ++k)
        if (hist[k] == 0) first[k] = -1;
    if (n_counted) *n_counted = (int64_t)h_cnt;
    return PG_OK;
}

// ================================================================================================
// Sparse spectra — sfs.py's SparseFS (94-125) without a dense histogram: pg_sfs_sparse / pg_sfs_tables_sparse / _fetch
// ================================================================================================
// Per slab, k1_sfs_keys packs one (cell, {1, site}) entry per counted site and spectrum.  Each spectrum's entries are
// appended to the runs it has so far, radix-sorted on the bits its cell count needs and reduced by cell (counts summed,
// the smallest site kept), so after every slab a spectrum holds at most one run per non-empty cell, cells ascending.
namespace {
// bits of the largest cell index of a spectrum of `cells` cells: the radix sort's end_bit
int sfs_key_bits(long long cells) {
    int b = 1;
    while (b < 63 && (1ll << b) < cells) ++b;
    return b;
}

// Π dims of every spectrum, refused when one does not fit in 63 bits (the cell index is an int64)
int sfs_sparse_cells(const char* who, int32_t n_groups, const int32_t* group_off, const int32_t* group_pops, int32_t n_in,
                     const int32_t* dims, std::vector<long long>& cells) {
    cells.assign(n_groups, 1);
    for (int g = 0; g < n_groups; ++g) {
        PG_CHECK(group_off[g + 1] > group_off[g], "%s: spectrum %d has no population", who, g);
        long long sz = 1;
        for (int k = group_off[g]; k < group_off[g + 1]; ++k) {
            PG_CHECK(group_pops[k] >= 0 && group_pops[k] < n_in, "%s: spectrum %d uses a population outside the in-group", who, g);
            const long long d = dims[group_pops[k]];
            PG_CHECK(d >= 1, "%s: dims must be >= 1", who);
            PG_CHECK(sz <= LLONG_MAX / d, "%s: spectrum %d has more than 2^63 - 1 cells (the product of its populations' "
                     "largest counts + 1); its cell index does not fit in 64 bits", who, g);
            sz *= d;
        }
        cells[g] = sz;
    }
    return PG_OK;
}

// Sites per slab: the dense path's slab, cut so that the entries of all spectra stay at most 2^25 (24 bytes each, about
// 0.8 GB); PG_SFS_SPARSE_SLAB caps it further (tests put slab seams into small inputs with it).
int64_t sfs_sparse_slab(int64_t dense_slab, int n_groups) {
    int64_t slab = std::max<int64_t>(1, std::min<int64_t>(dense_slab, ((int64_t)1 << 25) / n_groups));
    if (const char* e = getenv("PG_SFS_SPARSE_SLAB")) slab = std::max<int64_t>(1, std::min<int64_t>(slab, atoll(e)));
    return slab;
}

// The pass shared by genotypes and tables.  `sp` carries everything but the slab fields; load(s0, cnt) puts the slab's
// rows where sp.counts / sp.targets point.
template <typename Load>
int sfs_sparse_pass(pg_ctx* ctx, SfsParams sp, int64_t n_sites, int64_t slab, const std::vector<long long>& cells, Load load,
                    int64_t* nnz, int64_t* n_counted) {
    const int G = sp.n_groups;
    std::vector<int64_t> len(G, 0), off(G, 0);                      // runs of each spectrum in sfs_acc_*[cur], group-major
    int cur = 0;
    int64_t total = 0, counted = 0;
    const size_t slab_keys = align_up((size_t)slab * G * 8, 16);
    PG_TRY(ctx->sfs_slab.ensure(slab_keys + (size_t)slab * G * sizeof(SfsRun) + 64));
    unsigned long long* d_keys = (unsigned long long*)ctx->sfs_slab.p;
    SfsRun* d_runs = (SfsRun*)((uint8_t*)ctx->sfs_slab.p + slab_keys);
    PG_TRY(ctx->out_i.ensure(64));
    unsigned long long* d_cnt = (unsigned long long*)ctx->out_i.p;
    int* d_nruns = (int*)(d_cnt + 1);
    for (int64_t s0 = 0; s0 < n_sites; s0 += slab) {
        const int64_t cnt = std::min(slab, n_sites - s0);
        PG_TRY(load(s0, cnt));
        PG_CUDA(cudaMemsetAsync(d_cnt, 0, 8, ctx->stream));
        sp.n = cnt;
        sp.site0 = s0;
        sp.keys = d_keys;
        sp.runs = d_runs;
        sp.key_stride = slab;
        sp.n_counted = d_cnt;
        const int ti = pg_time_begin(ctx, "k1_sfs_keys");
        k1_sfs_keys<<<(unsigned)((cnt + 255) / 256), 256, 0, ctx->stream>>>(sp);
        pg_time_end(ctx, ti);
        PG_CUDA(cudaGetLastError());
        unsigned long long h_m = 0;
        PG_CUDA(cudaMemcpyAsync(&h_m, d_cnt, 8, cudaMemcpyDeviceToHost, ctx->stream));
        PG_CUDA(cudaStreamSynchronize(ctx->stream));                 // also frees the slab's rows for the next load
        const int64_t m = (int64_t)h_m;
        counted += m;
        if (m == 0) continue;
        const int nxt = cur ^ 1;
        PG_TRY(ctx->sfs_acc_k[nxt].ensure((size_t)(total + m * G) * 8 + 64));
        PG_TRY(ctx->sfs_acc_r[nxt].ensure((size_t)(total + m * G) * sizeof(SfsRun) + 64));
        unsigned long long* out_k = (unsigned long long*)ctx->sfs_acc_k[nxt].p;
        SfsRun* out_r = (SfsRun*)ctx->sfs_acc_r[nxt].p;
        int64_t o = 0;
        for (int g = 0; g < G; ++g) {
            const int64_t n = len[g] + m;
            PG_CHECK(n < INT_MAX, "pg_sfs_sparse: spectrum %d holds more than 2^31 entries in one merge", g);
            const size_t part_k = align_up((size_t)n * 8, 16), part = part_k + (size_t)n * sizeof(SfsRun);
            PG_TRY(ctx->sfs_merge.ensure(2 * part + 64));
            uint8_t* mb = (uint8_t*)ctx->sfs_merge.p;
            unsigned long long *a_k = (unsigned long long*)mb, *b_k = (unsigned long long*)(mb + part);
            SfsRun *a_r = (SfsRun*)(mb + part_k), *b_r = (SfsRun*)(mb + part + part_k);
            const unsigned long long* in_k = d_keys + (size_t)g * slab;
            const SfsRun* in_r = d_runs + (size_t)g * slab;
            if (len[g] > 0) {                                        // the runs so far, then this slab's entries
                const unsigned long long* acc_k = (const unsigned long long*)ctx->sfs_acc_k[cur].p + off[g];
                const SfsRun* acc_r = (const SfsRun*)ctx->sfs_acc_r[cur].p + off[g];
                PG_CUDA(cudaMemcpyAsync(a_k, acc_k, (size_t)len[g] * 8, cudaMemcpyDeviceToDevice, ctx->stream));
                PG_CUDA(cudaMemcpyAsync(a_k + len[g], in_k, (size_t)m * 8, cudaMemcpyDeviceToDevice, ctx->stream));
                PG_CUDA(cudaMemcpyAsync(a_r, acc_r, (size_t)len[g] * sizeof(SfsRun), cudaMemcpyDeviceToDevice, ctx->stream));
                PG_CUDA(cudaMemcpyAsync(a_r + len[g], in_r, (size_t)m * sizeof(SfsRun), cudaMemcpyDeviceToDevice, ctx->stream));
                in_k = a_k;
                in_r = a_r;
            }
            const int bits = sfs_key_bits(cells[g]);
            size_t t_sort = 0, t_red = 0;
            PG_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, t_sort, in_k, b_k, in_r, b_r, (int)n, 0, bits, ctx->stream));
            PG_CUDA(cub::DeviceReduce::ReduceByKey(nullptr, t_red, b_k, out_k + o, b_r, out_r + o, d_nruns, SfsRunMerge(),
                                                   (int)n, ctx->stream));
            PG_TRY(ctx->sfs_cub.ensure(std::max(t_sort, t_red) + 64));
            int ti2 = pg_time_begin(ctx, "sfs_sort");
            PG_CUDA(cub::DeviceRadixSort::SortPairs(ctx->sfs_cub.p, t_sort, in_k, b_k, in_r, b_r, (int)n, 0, bits, ctx->stream));
            pg_time_end(ctx, ti2);
            ti2 = pg_time_begin(ctx, "sfs_reduce");
            PG_CUDA(cub::DeviceReduce::ReduceByKey(ctx->sfs_cub.p, t_red, b_k, out_k + o, b_r, out_r + o, d_nruns, SfsRunMerge(),
                                                   (int)n, ctx->stream));
            pg_time_end(ctx, ti2);
            int h_runs = 0;
            PG_CUDA(cudaMemcpyAsync(&h_runs, d_nruns, 4, cudaMemcpyDeviceToHost, ctx->stream));
            PG_CUDA(cudaStreamSynchronize(ctx->stream));             // scratch may be regrown for the next spectrum
            off[g] = o;
            len[g] = h_runs;
            o += h_runs;
        }
        total = o;
        cur = nxt;
    }
    for (int g = 0; g < G; ++g) nnz[g] = len[g];
    if (n_counted) *n_counted = counted;
    ctx->sfs_cur = cur;
    ctx->sfs_total = total;
    return PG_OK;
}

// group tables and site mask on the device, as pg_sfs / pg_sfs_tables put them
int sfs_sparse_tables(pg_ctx* ctx, int32_t n_groups, const int32_t* group_off, const int32_t* group_pops,
                      const uint8_t* site_mask, int64_t n_mask, SfsParams& sp) {
    const int n_gp = group_off[n_groups];
    PG_TRY(ctx->misc2.ensure((size_t)(n_groups + 1) * 4 + (size_t)n_gp * 4 + 128));
    uint8_t* tb = (uint8_t*)ctx->misc2.p;
    size_t o = 0;
    int32_t* d_goff = nullptr;
    int32_t* d_gpops = nullptr;
    PG_TRY(push(ctx, tb, o, group_off, (size_t)n_groups + 1, &d_goff));
    PG_TRY(push(ctx, tb, o, group_pops, (size_t)n_gp, &d_gpops));
    sp.n_groups = n_groups;
    sp.group_off = d_goff;
    sp.group_pops = d_gpops;
    sp.mask = nullptr;
    if (site_mask && n_mask > 0) {
        PG_TRY(ctx->misc3.ensure((size_t)n_mask + 64));
        sp.mask = (uint8_t*)ctx->misc3.p;
        PG_CUDA(cudaMemcpyAsync(ctx->misc3.p, site_mask, (size_t)n_mask, cudaMemcpyHostToDevice, ctx->stream));
    }
    PG_CUDA(cudaStreamSynchronize(ctx->stream));                     // host tables behind the async copies
    return PG_OK;
}
}  // namespace

extern "C" int pg_sfs_sparse(pg_ctx* ctx, int32_t n_in, int32_t outgroup, int32_t n_groups, const int32_t* group_off,
                             const int32_t* group_pops, const uint8_t* site_mask, int64_t* nnz, int64_t* n_counted) {
    PG_CHECK(ctx && group_off && group_pops && nnz, "pg_sfs_sparse: null argument");
    ctx->sfs_total = -1;
    PG_CHECK(ctx->P >= 1 && ctx->P <= PG_MAX_POPS, "pg_sfs_sparse: call pg_set_pops first (at most %d populations)", PG_MAX_POPS);
    PG_CHECK(n_in >= 1 && n_in <= ctx->P, "pg_sfs_sparse: n_in out of range");
    PG_CHECK(outgroup == -1 || (outgroup >= n_in && outgroup < ctx->P),
             "pg_sfs_sparse: the outgroup must be a population after the in-group");
    PG_CHECK(n_groups >= 1, "pg_sfs_sparse: no spectra requested");
    const int P = ctx->P;
    std::vector<int> popN(P, 0), dims(P, 0);
    for (int h = 0; h < ctx->H; ++h)
        if (ctx->hap_pop[h] >= 0) popN[ctx->hap_pop[h]] += 1;
    for (int X = 0; X < P; ++X) dims[X] = popN[X] + 1;
    std::vector<long long> cells;
    PG_TRY(sfs_sparse_cells("pg_sfs_sparse", n_groups, group_off, group_pops, n_in, dims.data(), cells));
    PG_CUDA(cudaSetDevice(ctx->device));
    pg_timings_reset(ctx);
    SfsParams sp;
    memset(&sp, 0, sizeof(sp));
    PG_TRY(sfs_sparse_tables(ctx, n_groups, group_off, group_pops, site_mask, ctx->S, sp));
    sp.P = P;
    sp.n_in = n_in;
    sp.outgroup = outgroup;
    for (int X = 0; X < P; ++X) {
        sp.popN[X] = popN[X];
        sp.dims[X] = dims[X];
    }
    sp.require_complete = 1;
    const int64_t stride = (int64_t)P * 4;
    const int64_t slab = sfs_sparse_slab((int64_t)(1ll << 28) / (stride * 2), n_groups);
    PG_TRY(ctx->misc.ensure((size_t)std::min<int64_t>(slab, std::max<int64_t>(ctx->S, 1)) * stride * 2 + 64));
    sp.counts = (const uint16_t*)ctx->misc.p;
    return sfs_sparse_pass(ctx, sp, ctx->S, slab, cells, [&](int64_t s0, int64_t cnt) { return site_counts_slab(ctx, s0, cnt); },
                           nnz, n_counted);
}

extern "C" int pg_sfs_tables_sparse(pg_ctx* ctx, int32_t kind, const void* table, int64_t n, int32_t P, const int32_t* dims,
                                    int32_t n_in, int32_t outgroup, int32_t n_groups, const int32_t* group_off,
                                    const int32_t* group_pops, const uint8_t* site_mask, int64_t* nnz, int64_t* n_counted) {
    PG_CHECK(ctx && (table || n == 0) && dims && group_off && group_pops && nnz, "pg_sfs_tables_sparse: null argument");
    ctx->sfs_total = -1;
    PG_CHECK(kind == 0 || kind == 1, "pg_sfs_tables_sparse: kind must be 0 (base counts) or 1 (target counts)");
    PG_CHECK(P >= 1 && P <= PG_MAX_POPS, "pg_sfs_tables_sparse: at most %d populations", PG_MAX_POPS);
    PG_CHECK(n_in >= 1 && n_in <= P && n >= 0, "pg_sfs_tables_sparse: bad shape");
    PG_CHECK(outgroup == -1 || (kind == 0 && outgroup >= n_in && outgroup < P), "pg_sfs_tables_sparse: bad outgroup");
    PG_CHECK(n_groups >= 1, "pg_sfs_tables_sparse: no spectra requested");
    std::vector<long long> cells;
    PG_TRY(sfs_sparse_cells("pg_sfs_tables_sparse", n_groups, group_off, group_pops, n_in, dims, cells));
    PG_CUDA(cudaSetDevice(ctx->device));
    pg_timings_reset(ctx);
    SfsParams sp;
    memset(&sp, 0, sizeof(sp));
    PG_TRY(sfs_sparse_tables(ctx, n_groups, group_off, group_pops, site_mask, n, sp));
    const size_t row_bytes = kind == 0 ? (size_t)P * 8 : (size_t)P * 4;
    const int64_t slab = sfs_sparse_slab((int64_t)(((size_t)256 << 20) / row_bytes), n_groups);
    PG_TRY(ctx->misc.ensure((size_t)std::min<int64_t>(slab, std::max<int64_t>(n, 1)) * row_bytes + 64));
    sp.counts = kind == 0 ? (const uint16_t*)ctx->misc.p : nullptr;
    sp.targets = kind == 1 ? (const int32_t*)ctx->misc.p : nullptr;
    sp.P = P;
    sp.n_in = n_in;
    sp.outgroup = outgroup;
    for (int X = 0; X < P; ++X) sp.dims[X] = dims[X];
    sp.require_complete = 0;
    auto load = [&](int64_t s0, int64_t cnt) {
        PG_CUDA(cudaMemcpyAsync(ctx->misc.p, (const uint8_t*)table + (size_t)s0 * row_bytes, (size_t)cnt * row_bytes,
                                cudaMemcpyHostToDevice, ctx->stream));
        return PG_OK;
    };
    return sfs_sparse_pass(ctx, sp, n, slab, cells, load, nnz, n_counted);
}

extern "C" int pg_sfs_sparse_fetch(pg_ctx* ctx, int64_t total, int64_t* cell, int64_t* count, int64_t* first) {
    PG_CHECK(ctx, "pg_sfs_sparse_fetch: null argument");
    PG_CHECK(ctx->sfs_total >= 0, "pg_sfs_sparse_fetch: no sparse spectra pending (already fetched, or the pass failed)");
    PG_CHECK(total == ctx->sfs_total, "pg_sfs_sparse_fetch: %lld entries requested, the pending spectra hold %lld",
             (long long)total, (long long)ctx->sfs_total);
    PG_CHECK(total == 0 || (cell && count && first), "pg_sfs_sparse_fetch: null argument");
    PG_CUDA(cudaSetDevice(ctx->device));
    ctx->sfs_total = -1;                                             // fetched once
    if (total == 0) return PG_OK;
    const int cur = ctx->sfs_cur;
    PG_TRY(ctx->sfs_merge.ensure((size_t)total * 16 + 64));
    long long* d_count = (long long*)ctx->sfs_merge.p;
    long long* d_first = d_count + total;
    sfs_runs_split<<<(unsigned)((total + 255) / 256), 256, 0, ctx->stream>>>((const SfsRun*)ctx->sfs_acc_r[cur].p, total,
                                                                            d_count, d_first);
    PG_CUDA(cudaGetLastError());
    PG_TRY(pg_d2h_staged(ctx, cell, ctx->sfs_acc_k[cur].p, (size_t)total * 8));
    PG_TRY(pg_d2h_staged(ctx, count, d_count, (size_t)total * 8));
    PG_TRY(pg_d2h_staged(ctx, first, d_first, (size_t)total * 8));
    return PG_OK;
}
