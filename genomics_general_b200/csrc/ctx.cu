// libpgwin.so — context, data movement, synthetic data, windows/segments, timing.
// C-ABI: include/pgwin.h.  No CPU fallback anywhere: every compute entry needs a CUDA device.
#include <stdarg.h>
#include <stdlib.h>

#include <algorithm>
#include <thread>

#include "pgwin_internal.h"

static thread_local char g_err[1024] = "";

void pg_set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

extern "C" const char* pg_last_error(void) { return g_err; }
extern "C" int pg_version(void) { return 110; }

extern "C" int pg_device_count(int* n) {
    PG_CHECK(n != nullptr, "pg_device_count: null argument");
    *n = 0;
    PG_CUDA(cudaGetDeviceCount(n));
    return PG_OK;
}

int PgBuf::ensure(size_t bytes) {
    if (bytes <= cap && p) return PG_OK;
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
    size_t want = bytes + bytes / 8 + 256;
    PG_CUDA(cudaMalloc(&p, want));
    cap = want;
    return PG_OK;
}
void PgBuf::release() {
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
}

extern "C" int pg_ctx_create(int device, pg_ctx** out) {
    PG_CHECK(out != nullptr, "pg_ctx_create: null out pointer");
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n <= 0) {
        pg_set_error("pg_ctx_create: no CUDA device available (%s); libpgwin has no CPU fallback",
                     e == cudaSuccess ? "device count is 0" : cudaGetErrorString(e));
        return PG_ERR;
    }
    PG_CHECK(device >= 0 && device < n, "pg_ctx_create: device %d out of range (have %d)", device, n);
    PG_CUDA(cudaSetDevice(device));
    cudaDeviceProp prop;
    PG_CUDA(cudaGetDeviceProperties(&prop, device));
    PG_CHECK(prop.major == 9 && prop.minor == 0, "pg_ctx_create: device %d is sm_%d%d; libpgwin is built for sm_90a only",
             device, prop.major, prop.minor);
    pg_ctx* ctx = new pg_ctx();
    ctx->device = device;
    ctx->sm_count = prop.multiProcessorCount;
    PG_CUDA(cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking));
    *out = ctx;
    return PG_OK;
}

extern "C" int pg_ctx_destroy(pg_ctx* ctx) {
    if (!ctx) return PG_OK;
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    pg_k1_cache_free(ctx);
    pg_filter_free(ctx);
    pg_vcf_free(ctx);
    pg_seq_free(ctx);
    pg_g2v_free(ctx);
    pg_s2g_free(ctx);
    pg_ws_free(ctx);
    pg_merge_free(ctx);
    pg_nccl_finalize(ctx);
    ctx->gather.release();
    ctx->gather_flag.release();
    if (ctx->d_geno) cudaFree(ctx->d_geno);
    if (ctx->d_packed) cudaFree(ctx->d_packed);
    if (ctx->d_site_cls) cudaFree(ctx->d_site_cls);
    if (ctx->d_pos) cudaFree(ctx->d_pos);
    PgBuf* bufs[] = {&ctx->tables, &ctx->part, &ctx->segmeta, &ctx->winmeta, &ctx->out_d, &ctx->out_i,
                     &ctx->planes, &ctx->planes2, &ctx->pairs, &ctx->misc, &ctx->misc2, &ctx->misc3, &ctx->misc4, &ctx->misc5, &ctx->text, &ctx->starts, &ctx->meta,
                     &ctx->sfs_acc_k[0], &ctx->sfs_acc_k[1], &ctx->sfs_acc_r[0], &ctx->sfs_acc_r[1], &ctx->sfs_slab,
                     &ctx->sfs_merge, &ctx->sfs_cub, &ctx->flt_aux, &ctx->flt_tab,
                     &ctx->flt_stats, &ctx->flt_rows, &ctx->flt_off, &ctx->flt_out, &ctx->flt_cub};
    for (PgBuf* b : bufs) b->release();
    for (cudaEvent_t ev : ctx->event_pool) cudaEventDestroy(ev);
    ctx->stage[0].release();
    ctx->stage[1].release();
    if (ctx->copy_stream) {
        for (int k = 0; k < 2; ++k) {
            cudaEventDestroy(ctx->stage_full[k]);
            cudaEventDestroy(ctx->stage_free[k]);
        }
        cudaStreamDestroy(ctx->copy_stream);
    }
    if (ctx->h_pinned) cudaFreeHost(ctx->h_pinned);
    for (int k = 0; k < 2; ++k) {
        ctx->gslot[k].release();
        if (ctx->gslot_host[k]) cudaFreeHost(ctx->gslot_host[k]);
        if (ctx->g_rec[k]) cudaEventDestroy(ctx->g_rec[k]);
        if (ctx->g_done[k]) cudaEventDestroy(ctx->g_done[k]);
    }
    if (ctx->gather_stream) cudaStreamDestroy(ctx->gather_stream);
    for (int k = 0; k < 2; ++k)
        if (ctx->h_text[k]) {
            cudaFreeHost(ctx->h_text[k]);
            cudaEventDestroy(ctx->h_text_free[k]);
        }
    cudaStreamDestroy(ctx->stream);
    delete ctx;
    return PG_OK;
}

extern "C" int pg_host_alloc(void** ptr, size_t bytes) {
    PG_CHECK(ptr != nullptr, "pg_host_alloc: null pointer");
    PG_CUDA(cudaHostAlloc(ptr, bytes, cudaHostAllocDefault));
    return PG_OK;
}
extern "C" int pg_host_free(void* ptr) {
    if (ptr) PG_CUDA(cudaFreeHost(ptr));
    return PG_OK;
}

int pg_pinned(pg_ctx* ctx, size_t bytes, void** out) {
    if (bytes > ctx->h_pinned_cap) {
        if (ctx->h_pinned) cudaFreeHost(ctx->h_pinned);
        ctx->h_pinned = nullptr;
        ctx->h_pinned_cap = 0;
        size_t want = bytes + bytes / 4 + 4096;
        PG_CUDA(cudaHostAlloc(&ctx->h_pinned, want, cudaHostAllocDefault));
        ctx->h_pinned_cap = want;
    }
    *out = ctx->h_pinned;
    return PG_OK;
}

// Large device -> PAGEABLE host copy (the 800 MB of distMat matrices): a cudaMemcpy into pageable memory is staged by the
// driver at a few GB/s.  Here the copy engine fills two pinned 64 MB buffers in turn while host threads move the previous
// one to its destination.  Synchronous: dst is complete on return (work queued on the ctx stream before is waited for).
int pg_d2h_staged(pg_ctx* ctx, void* dst, const void* src, size_t bytes) {
    if (bytes == 0) return PG_OK;
    const size_t slab = (size_t)64 << 20;
    bool pinned = false;                                       // a caller buffer from pg_host_alloc: the copy engine writes it directly
    {
        cudaPointerAttributes at;
        if (cudaPointerGetAttributes(&at, dst) == cudaSuccess) pinned = (at.type == cudaMemoryTypeHost);
        else cudaGetLastError();
    }
    if (pinned || bytes < ((size_t)8 << 20)) {
        PG_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, ctx->stream));
        PG_CUDA(cudaStreamSynchronize(ctx->stream));
        return PG_OK;
    }
    if (!ctx->h_text[0]) {
        for (int k = 0; k < 2; ++k) {
            PG_CUDA(cudaHostAlloc(&ctx->h_text[k], slab, cudaHostAllocDefault));
            PG_CUDA(cudaEventCreateWithFlags(&ctx->h_text_free[k], cudaEventDisableTiming));
        }
    }
    const int n_threads = std::max(1, std::min(16, (int)std::thread::hardware_concurrency() / 2));
    auto drain = [&](int b, size_t off, size_t n) {
        std::vector<std::thread> th;
        auto work = [&](int t) {
            const size_t a = n * (size_t)t / (size_t)n_threads, e = n * (size_t)(t + 1) / (size_t)n_threads;
            memcpy((char*)dst + off + a, (const char*)ctx->h_text[b] + a, e - a);
        };
        for (int t = 1; t < n_threads; ++t) th.emplace_back(work, t);
        work(0);
        for (auto& x : th) x.join();
    };
    size_t prev_off = 0, prev_n = 0;
    int k = 0;
    for (size_t off = 0; off < bytes; off += slab, ++k) {
        const size_t n = std::min(slab, bytes - off);
        const int b = k & 1;
        PG_CUDA(cudaMemcpyAsync(ctx->h_text[b], (const char*)src + off, n, cudaMemcpyDeviceToHost, ctx->stream));
        PG_CUDA(cudaEventRecord(ctx->h_text_free[b], ctx->stream));
        if (k > 0) {                                           // the previous slab: wait for its copy, move it out
            PG_CUDA(cudaEventSynchronize(ctx->h_text_free[b ^ 1]));
            drain(b ^ 1, prev_off, prev_n);
        }
        prev_off = off;
        prev_n = n;
    }
    PG_CUDA(cudaEventSynchronize(ctx->h_text_free[(k - 1) & 1]));
    drain((k - 1) & 1, prev_off, prev_n);
    return PG_OK;
}

// ------------------------------------------------------------------------------------------------
// timing: CUDA events on the launching stream around every kernel
// ------------------------------------------------------------------------------------------------
void pg_timings_reset(pg_ctx* ctx) {
    ctx->timings.clear();
    ctx->events_used = 0;
}
static cudaEvent_t next_event(pg_ctx* ctx) {
    if (ctx->events_used == ctx->event_pool.size()) {
        cudaEvent_t ev;
        cudaEventCreate(&ev);
        ctx->event_pool.push_back(ev);
    }
    return ctx->event_pool[ctx->events_used++];
}
int pg_time_begin(pg_ctx* ctx, const char* name) {
    PgTiming t;
    memset(&t, 0, sizeof(t));
    strncpy(t.name, name, sizeof(t.name) - 1);
    t.start = next_event(ctx);
    t.stop = next_event(ctx);
    t.launches = 1;
    cudaEventRecord(t.start, ctx->stream);
    ctx->timings.push_back(t);
    ctx->launches += 1;
    return (int)ctx->timings.size() - 1;
}
void pg_time_end(pg_ctx* ctx, int idx) { cudaEventRecord(ctx->timings[idx].stop, ctx->stream); }

extern "C" int pg_last_timings(pg_ctx* ctx, int32_t cap, char (*names)[32], float* ms, int32_t* launches,
                               int32_t* count) {
    PG_CHECK(ctx && count, "pg_last_timings: null argument");
    PG_CUDA(cudaSetDevice(ctx->device));
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    // aggregate by name, in order of first appearance
    std::vector<std::string> order;
    std::vector<float> tot;
    std::vector<int> cnt;
    for (const PgTiming& t : ctx->timings) {
        float m = 0.f;
        PG_CUDA(cudaEventElapsedTime(&m, t.start, t.stop));
        size_t k = 0;
        for (; k < order.size(); ++k)
            if (order[k] == t.name) break;
        if (k == order.size()) {
            order.push_back(t.name);
            tot.push_back(0.f);
            cnt.push_back(0);
        }
        tot[k] += m;
        cnt[k] += t.launches;
    }
    int n = (int)std::min<size_t>(order.size(), (size_t)std::max(cap, 0));
    for (int k = 0; k < n; ++k) {
        if (names) {
            memset(names[k], 0, 32);
            strncpy(names[k], order[k].c_str(), 31);
        }
        if (ms) ms[k] = tot[k];
        if (launches) launches[k] = cnt[k];
    }
    *count = n;
    return PG_OK;
}

extern "C" int pg_launch_count(pg_ctx* ctx, int64_t* n) {
    PG_CHECK(ctx && n, "pg_launch_count: null argument");
    *n = ctx->launches;
    return PG_OK;
}

// ------------------------------------------------------------------------------------------------
// K1 launch geometry (host only; exported through pg_debug_k1_plan for the CPU test-suite)
// ------------------------------------------------------------------------------------------------
int pg_pitch_for(int H) {
    int chunks = (H + 15) / 16;
    if (chunks < 1) chunks = 1;
    if ((chunks & 1) == 0) chunks += 1;   // odd chunk count: lane-per-row LDS.128 is bank-conflict-free
    return chunks * 16;
}

static int env_int(const char* name, int dflt) {
    const char* e = getenv(name);
    return (e && *e) ? atoi(e) : dflt;
}

// Tile geometry: 8 consumer warps per CTA are split into teams of `wpt` warps; one team owns one tile
// (T consecutive sites) at a time, so up to 8/wpt tiles are being consumed while `stages` tiles sit in the
// TMA ring.  G lanes share one site row when a row is too long for one lane's tile share.
K1Plan pg_make_k1_plan(int64_t S, int H, int sm_count, int table_bytes, int nw, int force_G) {
    return pg_make_k1_plan_rows(S, pg_pitch_for(H), sm_count, table_bytes, nw, force_G);
}

// stages of tile_bytes each in the per-CTA dynamic shared memory we allow ourselves, at most 8 (PG_K1_STAGES lowers it)
int pg_k1_ring_stages(int tile_bytes, int table_bytes) {
    const int smem_cap = 227 * 1024 - 2048 - table_bytes;
    int stages = smem_cap / tile_bytes;
    if (stages > 8) stages = 8;
    return std::min(stages, std::max(2, env_int("PG_K1_STAGES", stages)));
}

K1Plan pg_make_k1_plan_rows(int64_t S, int pitch, int sm_count, int table_bytes, int nw, int force_G) {
    K1Plan p;
    memset(&p, 0, sizeof(p));
    p.pitch = pitch;
    p.chunks = p.pitch / 16;
    const int tile_target = env_int("PG_K1_TILE_KB", 64) * 1024;
    int G = 1, wpt = 1, I = 1;
    // lanes per site: keep one lane's walk below ~64 chunks (long rows are shared by G lanes; PG_K1_G overrides),
    // and a 32/G-site slab inside the tile target
    while (G < 32 && (p.chunks / G > 64 || (32 / G) * p.pitch > tile_target)) G *= 2;
    if (force_G > 0) G = force_G;           // lane-per-population variant: G = number of populations
    // warps per tile: the largest team (dividing the consumer-warp count) whose tile still fits the target
    const int wpt_max = (nw % 8 == 0) ? 8 : 4;
    while (wpt < wpt_max && (32 * (wpt * 2) / G) * p.pitch <= tile_target) wpt *= 2;
    // a tile holds a multiple of 4 sites (the positions ride behind the rows in 16-byte pieces): with 16 or 32 lanes per
    // site that takes a team of G / 8 warps, even when 4 rows exceed the tile target (pitches above 16 KiB, i.e. more
    // than 16,368 haplotypes)
    while (wpt < wpt_max && (32 * wpt / G) % 4 != 0) wpt *= 2;
    if (wpt == wpt_max && G == 1) {
        I = tile_target / (32 * wpt * p.pitch);
        if (I < 1) I = 1;
        if (I > 8) I = 8;
    }
    if (force_G <= 0) G = env_int("PG_K1_G", G);
    wpt = env_int("PG_K1_WPT", wpt);
    I = env_int("PG_K1_I", I);
    p.G = G;
    p.I = I;
    p.wpt = wpt;
    p.nw = nw;
    p.T = (32 * wpt / G) * I;
    // genotype rows + the tile's positions
    p.tile_bytes = ((p.T * p.pitch + p.T * 4 + 127) / 128) * 128;
    p.stages = pg_k1_ring_stages(p.tile_bytes, table_bytes);   // < 2 means the row is too long for this kernel
    p.smem_bytes = p.stages * p.tile_bytes + 256 + table_bytes;
    p.num_tiles = (S + p.T - 1) / p.T;
    int64_t ctas = sm_count;
    if (ctas > p.num_tiles) ctas = p.num_tiles;
    if (ctas < 1) ctas = 1;
    p.ctas = (int)ctas;
    return p;
}

// The geometry the site-pass kernels run: whole 16-byte position pieces per tile (T % 4 == 0), power-of-two G, teams that
// divide the consumer warps, a ring of 2..8 stages inside the shared memory.
int pg_k1_plan_ok(const K1Plan& p) {
    const bool pow2G = p.G >= 1 && p.G <= 32 && (p.G & (p.G - 1)) == 0;
    const bool okw = (p.wpt == 1 || p.wpt == 2 || p.wpt == 4 || p.wpt == 8) && p.nw > 0 && (p.nw % p.wpt) == 0;
    return (p.T % 4) == 0 && pow2G && okw && p.I >= 1 && p.stages >= 2 && p.stages <= 8 && p.smem_bytes <= 227 * 1024;
}

extern "C" int pg_debug_k1_plan(int64_t S, int32_t H, int32_t* pitch, int32_t* lanes_per_site, int32_t* tile_sites,
                                int32_t* stages, int32_t* smem_bytes) {
    PG_CHECK(S >= 0 && H > 0, "pg_debug_k1_plan: bad shape");
    K1Plan p = pg_make_k1_plan(S, H, 132, 4096);     // H100 SXM: 132 SMs (the fields reported do not depend on it)
    if (pitch) *pitch = p.pitch;
    if (lanes_per_site) *lanes_per_site = p.G;
    if (tile_sites) *tile_sites = p.T;
    if (stages) *stages = p.stages;
    if (smem_bytes) *smem_bytes = p.smem_bytes;
    return PG_OK;
}

extern "C" int pg_debug_k1_plan_ex(int64_t S, int32_t H, int32_t nw, int32_t force_G, int32_t table_bytes, int32_t* out) {
    PG_CHECK(S >= 0 && H > 0 && (nw == 8 || nw == 12) && force_G >= 0 && table_bytes >= 0 && out,
             "pg_debug_k1_plan_ex: bad arguments");
    K1Plan p = pg_make_k1_plan(S, H, 132, table_bytes, nw, force_G);
    const int vals[9] = {p.pitch, p.G, p.wpt, p.I, p.T, p.stages, p.smem_bytes, p.ctas, pg_k1_plan_ok(p)};
    memcpy(out, vals, sizeof(vals));
    return PG_OK;
}

// ------------------------------------------------------------------------------------------------
// upload / download
// ------------------------------------------------------------------------------------------------
// Resident device code (DESIGN.md "HBM layout"): still ONE byte per genotype, but one-hot with 2-bit
// spacing so that three bytes can be added before any field overflows:
//     A = 0x01, C = 0x04, G = 0x10, T = 0x40, missing = 0x00
// The C-ABI keeps the reference's codes (A0 C1 G2 T3, bit7 = missing); upload transcodes in place on the
// device right behind the H2D copy, download decodes.
__device__ __forceinline__ uint32_t encode4(uint32_t w) {
    const uint32_t v = ~(w >> 7) & 0x01010101u;        // valid flag per byte
    const uint32_t a0 = w & v, a1 = (w >> 1) & v;
    const uint32_t A = v & ~a0 & ~a1, Cc = a0 & ~a1, Gg = a1 & ~a0, T = a0 & a1;
    return A | (Cc << 2) | (Gg << 4) | (T << 6);
}
__device__ __forceinline__ uint32_t decode4(uint32_t c) {
    const uint32_t lo = ((c >> 2) | (c >> 6)) & 0x01010101u;      // C or T
    const uint32_t hi = ((c >> 4) | (c >> 6)) & 0x01010101u;      // G or T
    const uint32_t any = (c | (c >> 2) | (c >> 4) | (c >> 6)) & 0x01010101u;
    const uint32_t miss = (any ^ 0x01010101u) * 0xffu;            // 0xFF in missing bytes
    return (lo | (hi << 1)) | miss;
}

// rows [row0, row0+n) of the pitched matrix; only the H data bytes of a row are touched
__global__ void k_transcode(uint8_t* geno, int64_t row0, int64_t n, int pitch, int H, int decode) {
    const int wpr = (H + 3) / 4;
    const int64_t total = n * wpr;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = idx / wpr;
        const int wi = (int)(idx % wpr);
        uint32_t* p = reinterpret_cast<uint32_t*>(geno + (row0 + r) * pitch) + wi;
        const uint32_t w = *p;
        uint32_t x = decode ? decode4(w) : encode4(w);
        const int rem = H - wi * 4;
        if (rem < 4) {
            const uint32_t keep = 0xffffffffu << (8 * rem);       // padding bytes stay as they are
            x = (x & ~keep) | (w & keep);
        }
        *p = x;
    }
}

extern "C" int pg_alloc_sites(pg_ctx* ctx, int64_t S, int32_t H) {
    PG_CHECK(ctx != nullptr, "pg_alloc_sites: null ctx");
    PG_CHECK(S >= 0 && H > 0, "pg_alloc_sites: bad shape S=%lld H=%d", (long long)S, H);
    PG_CUDA(cudaSetDevice(ctx->device));
    const int pitch = pg_pitch_for(H);
    // over-allocate one tile of slack rows so that 16-byte vector reads past the end stay in bounds
    size_t need = (size_t)(S + 64) * pitch + 4096;
    if (need > ctx->geno_cap) {
        if (ctx->d_geno) cudaFree(ctx->d_geno);
        ctx->d_geno = nullptr;
        ctx->geno_cap = 0;
        PG_CUDA(cudaMalloc((void**)&ctx->d_geno, need));
        ctx->geno_cap = need;
    }
    size_t pneed = (size_t)(S + 64) * sizeof(int32_t);
    if (pneed > ctx->pos_cap) {
        if (ctx->d_pos) cudaFree(ctx->d_pos);
        ctx->d_pos = nullptr;
        ctx->pos_cap = 0;
        PG_CUDA(cudaMalloc((void**)&ctx->d_pos, pneed));
        ctx->pos_cap = pneed;
    }
    const int ppitch = pg_packed_pitch_for(H);
    const size_t kneed = (size_t)(S + 64) * ppitch + 4096;
    if (kneed > ctx->packed_cap) {
        if (ctx->d_packed) cudaFree(ctx->d_packed);
        ctx->d_packed = nullptr;
        ctx->packed_cap = 0;
        if (cudaMalloc((void**)&ctx->d_packed, kneed) == cudaSuccess) ctx->packed_cap = kneed;
        else {                                 // no companion: the popgen site pass reads the one-hot bytes
            ctx->d_packed = nullptr;
            cudaGetLastError();
        }
    }
    const size_t cneed = (size_t)(S + 64);
    if (!ctx->d_packed || cneed > ctx->cls_cap) {
        if (ctx->d_site_cls) cudaFree(ctx->d_site_cls);
        ctx->d_site_cls = nullptr;
        ctx->cls_cap = 0;
        if (ctx->d_packed) {
            if (cudaMalloc((void**)&ctx->d_site_cls, cneed) == cudaSuccess) ctx->cls_cap = cneed;
            else {                             // no classes: the popgen pass streams every packed row
                ctx->d_site_cls = nullptr;
                cudaGetLastError();
            }
        }
    }
    const bool same_shape = (ctx->S == S && ctx->H == H && ctx->pitch == pitch);
    ctx->S = S;
    ctx->H = H;
    ctx->pitch = pitch;
    ctx->packed_pitch = ppitch;
    if (!same_shape) ctx->epoch += 1;          // same shape: cached launch plans stay valid
    ctx->data_gen += 1;                        // (synth_fill and the text ingest come through here too)
    PG_CUDA(cudaMemsetAsync(ctx->d_pos, 0, pneed, ctx->stream));
    // every byte starts as "missing" (0x00): row padding and the slack rows never count
    PG_CUDA(cudaMemsetAsync(ctx->d_geno, 0, need, ctx->stream));
    if (ctx->d_packed) PG_CUDA(cudaMemsetAsync(ctx->d_packed, 0, kneed, ctx->stream));
    if (ctx->d_site_cls) PG_CUDA(cudaMemsetAsync(ctx->d_site_cls, 0, cneed, ctx->stream));
    // windows/pops stay; segments depend on S only
    if (!same_shape) ctx->brk.clear();
    return PG_OK;
}

// Grows the resident matrix by n sites appended after the current ones (multi-GPU command lines: the few sites of the
// next rank's byte range that this rank's last windows reach into).  The matrix is re-allocated when its capacity is short.
extern "C" int pg_append_sites(pg_ctx* ctx, int64_t n, const int8_t* geno, const int32_t* pos) {
    PG_CHECK(ctx && (n == 0 || geno), "pg_append_sites: null argument");
    PG_CHECK(n >= 0 && ctx->H > 0, "pg_append_sites: no matrix to append to");
    if (n == 0) return PG_OK;
    PG_CUDA(cudaSetDevice(ctx->device));
    const int64_t S0 = ctx->S, S1 = S0 + n;
    const size_t need = (size_t)(S1 + 64) * ctx->pitch + 4096;
    if (need > ctx->geno_cap) {
        int8_t* fresh = nullptr;
        PG_CUDA(cudaMalloc((void**)&fresh, need));
        PG_CUDA(cudaMemsetAsync(fresh, 0, need, ctx->stream));
        PG_CUDA(cudaMemcpyAsync(fresh, ctx->d_geno, (size_t)S0 * ctx->pitch, cudaMemcpyDeviceToDevice, ctx->stream));
        PG_CUDA(cudaStreamSynchronize(ctx->stream));
        cudaFree(ctx->d_geno);
        ctx->d_geno = fresh;
        ctx->geno_cap = need;
    }
    const size_t pneed = (size_t)(S1 + 64) * sizeof(int32_t);
    if (pneed > ctx->pos_cap) {
        int32_t* fresh = nullptr;
        PG_CUDA(cudaMalloc((void**)&fresh, pneed));
        PG_CUDA(cudaMemsetAsync(fresh, 0, pneed, ctx->stream));
        PG_CUDA(cudaMemcpyAsync(fresh, ctx->d_pos, (size_t)S0 * sizeof(int32_t), cudaMemcpyDeviceToDevice, ctx->stream));
        PG_CUDA(cudaStreamSynchronize(ctx->stream));
        cudaFree(ctx->d_pos);
        ctx->d_pos = fresh;
        ctx->pos_cap = pneed;
    }
    const size_t kneed = (size_t)(S1 + 64) * ctx->packed_pitch + 4096;
    if (ctx->d_packed && kneed > ctx->packed_cap) {   // the companion grows with the matrix, or is dropped
        uint32_t* fresh = nullptr;
        if (cudaMalloc((void**)&fresh, kneed) == cudaSuccess) {
            PG_CUDA(cudaMemsetAsync(fresh, 0, kneed, ctx->stream));
            PG_CUDA(cudaMemcpyAsync(fresh, ctx->d_packed, (size_t)S0 * ctx->packed_pitch, cudaMemcpyDeviceToDevice,
                                    ctx->stream));
            PG_CUDA(cudaStreamSynchronize(ctx->stream));
            cudaFree(ctx->d_packed);
            ctx->d_packed = fresh;
            ctx->packed_cap = kneed;
        } else {
            cudaGetLastError();
            PG_CUDA(cudaStreamSynchronize(ctx->stream));
            cudaFree(ctx->d_packed);
            ctx->d_packed = nullptr;
            ctx->packed_cap = 0;
        }
    }
    const size_t cneed = (size_t)(S1 + 64);
    if (ctx->d_site_cls && (!ctx->d_packed || cneed > ctx->cls_cap)) {   // the classes grow with the companion, or are dropped
        uint8_t* fresh = nullptr;
        if (ctx->d_packed && cudaMalloc((void**)&fresh, cneed) == cudaSuccess) {
            PG_CUDA(cudaMemsetAsync(fresh, 0, cneed, ctx->stream));
            PG_CUDA(cudaMemcpyAsync(fresh, ctx->d_site_cls, (size_t)S0, cudaMemcpyDeviceToDevice, ctx->stream));
            PG_CUDA(cudaStreamSynchronize(ctx->stream));
            cudaFree(ctx->d_site_cls);
            ctx->d_site_cls = fresh;
            ctx->cls_cap = cneed;
        } else {
            cudaGetLastError();
            PG_CUDA(cudaStreamSynchronize(ctx->stream));
            cudaFree(ctx->d_site_cls);
            ctx->d_site_cls = nullptr;
            ctx->cls_cap = 0;
        }
    }
    ctx->S = S1;
    ctx->epoch += 1;
    ctx->data_gen += 1;
    ctx->brk.clear();
    ctx->ingest_sites = -1;
    return pg_upload_range(ctx, S0, n, geno, pos);
}

// dense staging rows [n x H] (reference codes) -> resident pitched rows (one-hot code)
__global__ void k_ingest(const uint8_t* __restrict__ stage, uint8_t* __restrict__ geno, int64_t row0, int64_t n,
                         int pitch, int H) {
    const int wpr = (H + 3) / 4;
    const int64_t total = n * wpr;
    const bool aligned = (H & 3) == 0;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = idx / wpr;
        const int wi = (int)(idx % wpr);
        const uint8_t* src = stage + r * H + (int64_t)wi * 4;
        uint32_t w;
        if (aligned) w = *reinterpret_cast<const uint32_t*>(src);
        else {
            const int rem = H - wi * 4;
            w = 0xffffffffu;                                   // bytes past the row end: missing
            w = (w & ~0xffu) | src[0];
            if (rem > 1) w = (w & ~0xff00u) | ((uint32_t)src[1] << 8);
            if (rem > 2) w = (w & ~0xff0000u) | ((uint32_t)src[2] << 16);
            if (rem > 3) w = (w & ~0xff000000u) | ((uint32_t)src[3] << 24);
        }
        reinterpret_cast<uint32_t*>(geno + (row0 + r) * pitch)[wi] = encode4(w);   // padding bytes encode to 0x00
    }
}

// Packed companion: a row is three planes of wd = ceil(H / 32) words — valid bits, then the low and the high bit of the
// allele code (A 0, C 1, G 2, T 3) — haplotype h at bit h % 32 of word h / 32, padded to 16 bytes.  A site is one contiguous
// row, so the site pass streams it like the one-hot rows, at 3/8 of their bytes.
int pg_packed_pitch_for(int H) {
    const int wd = (H + 31) / 32;
    return (3 * wd * 4 + 15) / 16 * 16;
}

// One warp per row, 32 words (1024 haplotypes) at a time: lane j loads bytes 4j..4j+3 of each 128-haplotype group (coalesced,
// the groups' loads in flight together), each 32-haplotype word is three ballots, and lane w % 32 keeps word w of the three
// planes for coalesced stores.  The resident bytes of the H haplotypes are one-hot or 0 by construction (encode4 / k_ingest,
// k_synth, k_parse_lines), so "valid" is byte != 0 and the code bits are "C or T" (0x44) and "G or T" (0x50).  Bytes past H
// are ignored: an append inside the capacity of an earlier, wider matrix leaves them as that matrix wrote them.
// With cls, the warp also writes the row's class (PG_CLS_*) from the same ballots: a word is uniform when its valid bits and
// each code plane are all clear or all set over the word's haplotypes below H.
__global__ void __launch_bounds__(256) k_pack_rows(const uint8_t* __restrict__ geno, uint32_t* __restrict__ packed,
                                                   uint8_t* __restrict__ cls, int64_t row0, int64_t n, int pitch, int H, int ppw,
                                                   int wd) {
    const unsigned full = 0xffffffffu;
    const int lane = threadIdx.x & 31;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = row0 + (((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5); r < row0 + n; r += nwarps) {
        const uint8_t* src = geno + r * pitch;
        uint32_t* dst = packed + r * ppw;
        // warp-uniform: some haplotype valid / missing, some valid code bit 0 (1) set / clear; alleles present (bit a: code a)
        bool any_v = false, any_m = false, any_b0 = false, any_nb0 = false, any_b1 = false, any_nb1 = false;
        uint32_t present = 0u;
        for (int w0 = 0; w0 < wd; w0 += 32) {
            const int ng = min(8, (wd - w0 + 3) / 4);       // 128-haplotype groups in this stretch (warp-uniform)
            uint32_t v[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int off = w0 * 32 + j * 128 + lane * 4;
                v[j] = (j < ng && off < pitch) ? *reinterpret_cast<const uint32_t*>(src + off) : 0u;
            }
            uint32_t V = 0u, B0 = 0u, B1 = 0u;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                if (j >= ng) break;
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    // haplotype 32 (w0 + 4 j + k) + lane is byte (lane & 3) of the word lane 8 k + lane / 4 loaded
                    const uint32_t byte = (__shfl_sync(full, v[j], k * 8 + (lane >> 2)) >> (8 * (lane & 3))) & 0xffu;
                    const uint32_t b = 32 * (w0 + 4 * j + k) + lane < H ? byte : 0u;
                    const uint32_t bv = __ballot_sync(full, b != 0u);
                    const uint32_t b0 = __ballot_sync(full, (b & 0x44u) != 0u);
                    const uint32_t b1 = __ballot_sync(full, (b & 0x50u) != 0u);
                    const int nh = min(32, max(0, H - 32 * (w0 + 4 * j + k)));     // haplotypes of this word below H
                    const uint32_t in = nh == 32 ? full : (1u << nh) - 1u;
                    any_v |= bv != 0u;
                    any_m |= bv != in;
                    any_b0 |= b0 != 0u;
                    any_nb0 |= (bv & ~b0) != 0u;
                    any_b1 |= b1 != 0u;
                    any_nb1 |= (bv & ~b1) != 0u;
                    present |= ((bv & ~b0 & ~b1) != 0u ? 1u : 0u) | ((bv & b0 & ~b1) != 0u ? 2u : 0u) |
                               ((bv & ~b0 & b1) != 0u ? 4u : 0u) | ((bv & b0 & b1) != 0u ? 8u : 0u);
                    if (lane == 4 * j + k) {
                        V = bv;
                        B0 = b0;
                        B1 = b1;
                    }
                }
            }
            const int w = w0 + lane;
            if (w < wd) {
                dst[w] = V;
                dst[wd + w] = B0;
                dst[2 * wd + w] = B1;
            }
        }
        if (cls && lane == 0) {
            uint8_t c = PG_CLS_VARIED;
            if (!any_v) c = PG_CLS_MISSING;
            else if (!any_m && !(any_b0 && any_nb0) && !(any_b1 && any_nb1))
                c = (uint8_t)(PG_CLS_A + (any_b0 ? 1 : 0) + (any_b1 ? 2 : 0));
            else if (!any_m && __popc(present) == 2)
                c = (any_b1 && any_nb1) ? PG_CLS_VARIED2_B1 : PG_CLS_VARIED2;
            cls[r] = c;
        }
    }
}

int pg_pack_rows(pg_ctx* ctx, int64_t s0, int64_t n) {
    if (!ctx->d_packed || n <= 0) return PG_OK;
    const int wd = (ctx->H + 31) / 32;
    const int blocks = (int)std::max<int64_t>(1, std::min<int64_t>((n + 7) / 8, (int64_t)ctx->sm_count * 16));
    k_pack_rows<<<blocks, 256, 0, ctx->stream>>>((const uint8_t*)ctx->d_geno, ctx->d_packed, ctx->d_site_cls, s0, n,
                                                 ctx->pitch, ctx->H, ctx->packed_pitch / 4, wd);
    PG_CUDA(cudaGetLastError());
    ctx->launches += 1;
    return PG_OK;
}

extern "C" int pg_debug_packed(pg_ctx* ctx, int64_t site0, int64_t n, int32_t* row_words, uint32_t* out) {
    PG_CHECK(ctx && row_words, "pg_debug_packed: null argument");
    PG_CHECK(site0 >= 0 && n >= 0 && site0 + n <= ctx->S, "pg_debug_packed: range outside S");
    *row_words = ctx->d_packed ? ctx->packed_pitch / 4 : 0;
    if (!ctx->d_packed || !out || n == 0) return PG_OK;
    PG_CUDA(cudaSetDevice(ctx->device));
    PG_CUDA(cudaMemcpyAsync(out, (const uint8_t*)ctx->d_packed + site0 * ctx->packed_pitch, (size_t)n * ctx->packed_pitch,
                            cudaMemcpyDeviceToHost, ctx->stream));
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    return PG_OK;
}

// the class bytes (PG_CLS_*) of sites [site0, site0 + n); *avail = 0 when the context keeps none
extern "C" int pg_debug_site_cls(pg_ctx* ctx, int64_t site0, int64_t n, int32_t* avail, uint8_t* out) {
    PG_CHECK(ctx && avail, "pg_debug_site_cls: null argument");
    PG_CHECK(site0 >= 0 && n >= 0 && site0 + n <= ctx->S, "pg_debug_site_cls: range outside S");
    *avail = ctx->d_site_cls ? 1 : 0;
    if (!ctx->d_site_cls || !out || n == 0) return PG_OK;
    PG_CUDA(cudaSetDevice(ctx->device));
    PG_CUDA(cudaMemcpyAsync(out, ctx->d_site_cls + site0, (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    return PG_OK;
}

extern "C" int pg_upload_range(pg_ctx* ctx, int64_t site0, int64_t n, const int8_t* geno, const int32_t* pos) {
    PG_CHECK(ctx && geno, "pg_upload_range: null argument");
    PG_CHECK(site0 >= 0 && n >= 0 && site0 + n <= ctx->S, "pg_upload_range: range [%lld,+%lld) outside S=%lld",
             (long long)site0, (long long)n, (long long)ctx->S);
    PG_CUDA(cudaSetDevice(ctx->device));
    if (n == 0) return PG_OK;
    ctx->data_gen += 1;
    if (!ctx->copy_stream) {
        PG_CUDA(cudaStreamCreateWithFlags(&ctx->copy_stream, cudaStreamNonBlocking));
        for (int k = 0; k < 2; ++k) {
            PG_CUDA(cudaEventCreateWithFlags(&ctx->stage_full[k], cudaEventDisableTiming));
            PG_CUDA(cudaEventCreateWithFlags(&ctx->stage_free[k], cudaEventDisableTiming));
        }
    }
    // dense 1-D H2D copies (full PCIe rate) into two staging buffers on the copy stream; the ingest kernel
    // (transcode + re-pitch) runs behind each copy on the compute stream.
    const size_t stage_bytes = (size_t)128 << 20;
    const int64_t rows_per = std::max<int64_t>(1, (int64_t)(stage_bytes / (size_t)ctx->H));
    PG_TRY(ctx->stage[0].ensure((size_t)rows_per * ctx->H + 16));
    PG_TRY(ctx->stage[1].ensure((size_t)rows_per * ctx->H + 16));
    // the copy stream must not overtake work already queued on the compute stream that reads the staging buffers
    int k = 0;
    for (int64_t s = 0; s < n; s += rows_per, ++k) {
        const int64_t cnt = std::min(rows_per, n - s);
        const int b = k & 1;
        if (k >= 2) PG_CUDA(cudaStreamWaitEvent(ctx->copy_stream, ctx->stage_free[b], 0));
        PG_CUDA(cudaMemcpyAsync(ctx->stage[b].p, geno + (size_t)s * ctx->H, (size_t)cnt * ctx->H,
                                cudaMemcpyHostToDevice, ctx->copy_stream));
        PG_CUDA(cudaEventRecord(ctx->stage_full[b], ctx->copy_stream));
        PG_CUDA(cudaStreamWaitEvent(ctx->stream, ctx->stage_full[b], 0));
        k_ingest<<<ctx->sm_count * 8, 256, 0, ctx->stream>>>((const uint8_t*)ctx->stage[b].p, (uint8_t*)ctx->d_geno,
                                                              site0 + s, cnt, ctx->pitch, ctx->H);
        PG_CUDA(cudaGetLastError());
        ctx->launches += 1;
        PG_CUDA(cudaEventRecord(ctx->stage_free[b], ctx->stream));
        PG_TRY(pg_pack_rows(ctx, site0 + s, cnt));      // under the next slab's H2D copy
    }
    if (pos) {
        PG_CUDA(cudaMemcpyAsync(ctx->d_pos + site0, pos, (size_t)n * sizeof(int32_t), cudaMemcpyHostToDevice,
                                ctx->copy_stream));
        PG_CUDA(cudaEventRecord(ctx->stage_full[0], ctx->copy_stream));
        PG_CUDA(cudaStreamWaitEvent(ctx->stream, ctx->stage_full[0], 0));
    }
    // the caller's buffers may be reused as soon as this returns
    PG_CUDA(cudaStreamSynchronize(ctx->copy_stream));
    // staging buffers are reused by the next call: their last readers must be done before the next H2D lands
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    return PG_OK;
}

extern "C" int pg_upload(pg_ctx* ctx, const int8_t* geno, int64_t S, int32_t H, const int32_t* pos) {
    PG_TRY(pg_alloc_sites(ctx, S, H));
    return pg_upload_range(ctx, 0, S, geno, pos);
}

extern "C" int pg_download(pg_ctx* ctx, int64_t site0, int64_t n, int8_t* geno, int32_t* pos) {
    PG_CHECK(ctx != nullptr, "pg_download: null ctx");
    PG_CHECK(site0 >= 0 && n >= 0 && site0 + n <= ctx->S, "pg_download: range outside S");
    PG_CUDA(cudaSetDevice(ctx->device));
    if (n == 0) return PG_OK;
    if (geno) {
        // decode into a scratch copy so that the resident matrix is never modified
        PG_TRY(ctx->misc.ensure((size_t)n * ctx->pitch + 64));
        PG_CUDA(cudaMemcpyAsync(ctx->misc.p, ctx->d_geno + site0 * ctx->pitch, (size_t)n * ctx->pitch,
                                cudaMemcpyDeviceToDevice, ctx->stream));
        k_transcode<<<ctx->sm_count * 8, 256, 0, ctx->stream>>>((uint8_t*)ctx->misc.p, 0, n, ctx->pitch, ctx->H, 1);
        PG_CUDA(cudaGetLastError());
        PG_CUDA(cudaMemcpy2DAsync(geno, ctx->H, ctx->misc.p, ctx->pitch, ctx->H, (size_t)n, cudaMemcpyDeviceToHost,
                                  ctx->stream));
    }
    if (pos)
        PG_CUDA(cudaMemcpyAsync(pos, ctx->d_pos + site0, (size_t)n * sizeof(int32_t), cudaMemcpyDeviceToHost,
                                ctx->stream));
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    return PG_OK;
}

// ------------------------------------------------------------------------------------------------
// synthetic data: device twin of genomics_general_b200/synth.py (bit-identical integer hashing)
// ------------------------------------------------------------------------------------------------
__host__ __device__ __forceinline__ uint64_t mix64(uint64_t x) {
    x ^= x >> 30;
    x *= 0xBF58476D1CE4E5B9ull;
    x ^= x >> 27;
    x *= 0x94D049BB133111EBull;
    x ^= x >> 31;
    return x;
}

struct SynthParams {
    int64_t S;
    int H, pitch, n_pops, samples_per_pop, ploidy, spacing;
    uint64_t seed, thr_var, thr_out0, thr_third, thr_miss;
};

__global__ void k_synth(int8_t* __restrict__ geno, int32_t* __restrict__ pos, SynthParams sp) {
    const uint64_t GOLD = 0x9E3779B97F4A7C15ull, K_STREAM = 0xD1B54A32D192ED03ull, K_HAP = 0xA24BAED4963EE407ull,
                   K_SAMPLE = 0x9FB21C651E98DF25ull;
    const int hpp = sp.samples_per_pop * sp.ploidy;
    for (int64_t site = blockIdx.x; site < sp.S; site += gridDim.x) {
        const uint64_t base = mix64(sp.seed * GOLD + (uint64_t)site);
        auto draw = [&](int k) { return mix64(base + (uint64_t)k * K_STREAM + 1ull); };
        const uint64_t d0 = draw(0);
        const int ref = (int)(d0 >> 62);
        const int alt = (ref + 1 + (int)((d0 >> 40) % 3ull)) % 4;
        const bool variable = (draw(1) >> 32) < sp.thr_var;
        const bool out0 = (draw(2) >> 32) < sp.thr_out0;
        const bool third_site = variable && ((draw(3) >> 32) < sp.thr_third);
        const int third_pop = (int)((draw(4) >> 40) % (uint64_t)sp.n_pops);
        int third = 0;
        for (int cand = 3; cand >= 0; --cand)
            if (ref != cand && alt != cand) third = cand;
        if (threadIdx.x == 0) {
            const uint64_t h = mix64(sp.seed * GOLD + (uint64_t)site + 0x5851F42D4C957F2Dull);
            pos[site] = (int32_t)((uint64_t)site * (uint64_t)sp.spacing + 1ull + ((h >> 33) % (uint64_t)sp.spacing));
        }
        for (int hap = threadIdx.x; hap < sp.H; hap += blockDim.x) {
            const int pop = hap / hpp;
            uint64_t freq = draw(8 + pop) >> 32;
            if (!variable) freq = 0;
            if (out0 && pop == sp.n_pops - 1) freq = 0;
            const uint64_t hh = mix64(base ^ (((uint64_t)hap + 1ull) * K_HAP));
            const bool is_alt = (hh >> 32) < freq;
            int g = is_alt ? alt : ref;
            if (is_alt && third_site && pop == third_pop && (((hh >> 8) & 1ull) == 1ull)) g = third;
            if (sp.thr_miss > 0) {
                const int samp = hap / sp.ploidy;
                const uint64_t mm = mix64(base + ((uint64_t)samp + 1ull) * K_SAMPLE);
                if ((mm >> 32) < sp.thr_miss) g = -1;
            }
            geno[site * sp.pitch + hap] = (int8_t)(g < 0 ? 0 : (1 << (2 * g)));   // resident one-hot code
        }
    }
}

extern "C" int pg_synth_fill(pg_ctx* ctx, int64_t S, int32_t n_pops, int32_t samples_per_pop, int32_t ploidy,
                             uint64_t seed, uint64_t thr_var, uint64_t thr_out0, uint64_t thr_third,
                             uint64_t thr_miss, int32_t spacing) {
    PG_CHECK(ctx != nullptr, "pg_synth_fill: null ctx");
    PG_CHECK(n_pops > 0 && samples_per_pop > 0 && ploidy > 0 && spacing > 0, "pg_synth_fill: bad parameters");
    const int H = n_pops * samples_per_pop * ploidy;
    PG_TRY(pg_alloc_sites(ctx, S, H));
    if (S == 0) return PG_OK;
    SynthParams sp;
    sp.S = S;
    sp.H = H;
    sp.pitch = ctx->pitch;
    sp.n_pops = n_pops;
    sp.samples_per_pop = samples_per_pop;
    sp.ploidy = ploidy;
    sp.spacing = spacing;
    sp.seed = seed;
    sp.thr_var = thr_var;
    sp.thr_out0 = thr_out0;
    sp.thr_third = thr_third;
    sp.thr_miss = thr_miss;
    int blocks = (int)std::min<int64_t>(S, (int64_t)ctx->sm_count * 16);
    k_synth<<<blocks, 128, 0, ctx->stream>>>(ctx->d_geno, ctx->d_pos, sp);
    PG_CUDA(cudaGetLastError());
    PG_TRY(pg_pack_rows(ctx, 0, S));
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    return PG_OK;
}

// ------------------------------------------------------------------------------------------------
// populations / windows / segments
// ------------------------------------------------------------------------------------------------
extern "C" int pg_set_pops(pg_ctx* ctx, int32_t P, const int32_t* hap_pop) {
    PG_CHECK(ctx && hap_pop, "pg_set_pops: null argument");
    PG_CHECK(ctx->H > 0, "pg_set_pops: upload genotypes first");
    // the windowed statistics take at most PG_MAX_POPS populations (checked there); per-site counts / target
    // frequencies (freq.py --indFreqs: one population per individual) take any number
    PG_CHECK(P >= 1 && P <= 65535, "pg_set_pops: P=%d outside [1,65535]", P);
    ctx->hap_pop.assign(hap_pop, hap_pop + ctx->H);
    for (int h = 0; h < ctx->H; ++h)
        PG_CHECK(hap_pop[h] >= -1 && hap_pop[h] < P, "pg_set_pops: hap_pop[%d]=%d outside [-1,%d)", h, hap_pop[h], P);
    ctx->P = P;
    ctx->epoch += 1;
    ctx->data_gen += 1;
    return PG_OK;
}

extern "C" int pg_set_windows(pg_ctx* ctx, int64_t W, const int64_t* lo, const int64_t* hi) {
    PG_CHECK(ctx != nullptr && W >= 0, "pg_set_windows: bad argument");
    PG_CHECK(W == 0 || (lo && hi), "pg_set_windows: null ranges");
    for (int64_t w = 0; w < W; ++w)
        PG_CHECK(lo[w] >= 0 && lo[w] <= hi[w] && hi[w] <= ctx->S,
                 "pg_set_windows: window %lld = [%lld,%lld) is not a valid range of [0,%lld)", (long long)w,
                 (long long)lo[w], (long long)hi[w], (long long)ctx->S);
    ctx->W = W;
    ctx->win_lo.assign(lo, lo + W);
    ctx->win_hi.assign(hi, hi + W);
    ctx->brk.clear();
    ctx->epoch += 1;
    return PG_OK;
}

// Segments: maximal site intervals between consecutive window boundaries.  Every window is a contiguous
// run of segments, so one pass over the sites serves overlapping windows too.
int pg_build_segments(pg_ctx* ctx) {
    if (!ctx->brk.empty()) return PG_OK;
    std::vector<int64_t>& b = ctx->brk;
    b.reserve((size_t)ctx->W * 2 + 2);
    b.push_back(0);
    b.push_back(ctx->S);
    for (int64_t w = 0; w < ctx->W; ++w) {
        if (ctx->win_lo[w] == ctx->win_hi[w]) continue;   // empty windows own no segment
        b.push_back(ctx->win_lo[w]);
        b.push_back(ctx->win_hi[w]);
    }
    std::sort(b.begin(), b.end());
    b.erase(std::unique(b.begin(), b.end()), b.end());
    PG_CHECK(b.size() - 1 < (size_t)0x7fffffff, "too many segments");
    ctx->win_seg_lo.resize((size_t)ctx->W);
    ctx->win_seg_hi.resize((size_t)ctx->W);
    for (int64_t w = 0; w < ctx->W; ++w) {
        if (ctx->win_lo[w] == ctx->win_hi[w]) {
            ctx->win_seg_lo[w] = ctx->win_seg_hi[w] = 0;
            continue;
        }
        ctx->win_seg_lo[w] = (int32_t)(std::lower_bound(b.begin(), b.end(), ctx->win_lo[w]) - b.begin());
        ctx->win_seg_hi[w] = (int32_t)(std::lower_bound(b.begin(), b.end(), ctx->win_hi[w]) - b.begin());
    }
    return PG_OK;
}
