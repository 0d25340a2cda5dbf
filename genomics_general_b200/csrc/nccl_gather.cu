// Native NCCL all-gather of the per-window records (SURVEY.md §8e: "one ncclAllGather of fixed-width per-window
// records").  NCCL is resolved at run time with dlopen/dlsym: inside a torchrun process this binds to the libnccl
// that PyTorch already loaded, otherwise to the system library — the engine itself links neither.
//
// The all-gather is enqueued on the ctx stream directly behind k1_finalize, in place in the gather buffer
// (rank r's records live at offset r * w_max * RC), followed by one D2H of the whole table: the host synchronises
// once per call.  Windows that need the pairwise path (rare in the resident-matrix benchmark, the rule with
// missing data) are computed afterwards into the same slot and the gather is repeated.
#include <dlfcn.h>

#include <vector>

#include "pgwin_internal.h"

namespace {

struct NcclUniqueId {
    char internal[128];
};
typedef void* NcclComm;
typedef int (*fn_get_id)(NcclUniqueId*);
typedef int (*fn_init_rank)(NcclComm*, int, NcclUniqueId, int);
typedef int (*fn_all_gather)(const void*, void*, size_t, int, NcclComm, cudaStream_t);
typedef int (*fn_all_reduce)(const void*, void*, size_t, int, int, NcclComm, cudaStream_t);
typedef int (*fn_destroy)(NcclComm);
typedef const char* (*fn_errstr)(int);

struct NcclApi {
    void* handle = nullptr;
    fn_get_id get_id = nullptr;
    fn_init_rank init_rank = nullptr;
    fn_all_gather all_gather = nullptr;
    fn_all_reduce all_reduce = nullptr;
    fn_destroy destroy = nullptr;
    fn_errstr errstr = nullptr;
};
NcclApi g_nccl;

int load_nccl() {
    if (g_nccl.handle) return PG_OK;
    const char* names[] = {"libnccl.so.2", "libnccl.so"};
    void* h = nullptr;
    for (const char* n : names) {
        h = dlopen(n, RTLD_NOW | RTLD_GLOBAL | RTLD_NOLOAD);     // already in the process (PyTorch's copy)?
        if (h) break;
    }
    if (!h)
        for (const char* n : names) {
            h = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
            if (h) break;
        }
    PG_CHECK(h != nullptr, "NCCL is not available: %s", dlerror());
    g_nccl.get_id = (fn_get_id)dlsym(h, "ncclGetUniqueId");
    g_nccl.init_rank = (fn_init_rank)dlsym(h, "ncclCommInitRank");
    g_nccl.all_gather = (fn_all_gather)dlsym(h, "ncclAllGather");
    g_nccl.all_reduce = (fn_all_reduce)dlsym(h, "ncclAllReduce");
    g_nccl.destroy = (fn_destroy)dlsym(h, "ncclCommDestroy");
    g_nccl.errstr = (fn_errstr)dlsym(h, "ncclGetErrorString");
    PG_CHECK(g_nccl.get_id && g_nccl.init_rank && g_nccl.all_gather && g_nccl.all_reduce && g_nccl.destroy,
             "NCCL symbols missing");
    g_nccl.handle = h;
    return PG_OK;
}

#define PG_NCCL(call)                                                                                   \
    do {                                                                                                \
        int _r = (call);                                                                                \
        if (_r != 0) {                                                                                  \
            pg_set_error("%s failed: %s", #call, g_nccl.errstr ? g_nccl.errstr(_r) : "NCCL error");     \
            return PG_ERR;                                                                              \
        }                                                                                               \
    } while (0)

constexpr int NCCL_UINT64 = 5;   // ncclUint64 in every NCCL 2.x
constexpr int NCCL_INT64 = 4;    // ncclInt64
constexpr int NCCL_SUM = 0;      // ncclSum

}  // namespace

extern "C" int pg_nccl_unique_id(void* id128) {
    PG_CHECK(id128 != nullptr, "pg_nccl_unique_id: null argument");
    PG_TRY(load_nccl());
    NcclUniqueId id;
    PG_NCCL(g_nccl.get_id(&id));
    memcpy(id128, id.internal, 128);
    return PG_OK;
}

extern "C" int pg_nccl_init(pg_ctx* ctx, int32_t nranks, int32_t rank, const void* id128) {
    PG_CHECK(ctx && id128 && nranks >= 1 && rank >= 0 && rank < nranks, "pg_nccl_init: bad argument");
    PG_TRY(load_nccl());
    PG_CUDA(cudaSetDevice(ctx->device));
    if (ctx->nccl_comm) {
        g_nccl.destroy((NcclComm)ctx->nccl_comm);
        ctx->nccl_comm = nullptr;
    }
    NcclUniqueId id;
    memcpy(id.internal, id128, 128);
    NcclComm comm = nullptr;
    PG_NCCL(g_nccl.init_rank(&comm, nranks, id, rank));
    ctx->nccl_comm = comm;
    ctx->nccl_ranks = nranks;
    ctx->nccl_rank = rank;
    return PG_OK;
}

extern "C" int pg_nccl_finalize(pg_ctx* ctx) {
    if (ctx && ctx->nccl_comm && g_nccl.destroy) {
        cudaSetDevice(ctx->device);
        cudaStreamSynchronize(ctx->stream);
        g_nccl.destroy((NcclComm)ctx->nccl_comm);
        ctx->nccl_comm = nullptr;
    }
    return PG_OK;
}

// In-place integer sum over the ranks, enqueued on the ctx stream (the one exchange of `--windType cat`: each rank
// holds a shard of the SITES of the single window, the pair matrices add up; SURVEY.md §8e).
int pg_nccl_allreduce_i64(pg_ctx* ctx, void* d_buf, size_t count) {
    PG_CHECK(ctx->nccl_comm != nullptr, "all-reduce: call pg_nccl_init first");
    PG_NCCL(g_nccl.all_reduce(d_buf, d_buf, count, NCCL_INT64, NCCL_SUM, (NcclComm)ctx->nccl_comm, ctx->stream));
    ctx->launches += 1;
    return PG_OK;
}

// statistics of this rank's windows + all-gather of every rank's records into h_table
// (host, nranks * w_max * RC 8-byte words; rows beyond a rank's own window count are zero).
extern "C" int pg_popgen_allgather(pg_ctx* ctx, int32_t min_sites, double min_data, int32_t force_path, int64_t w_max,
                                   void* h_table, int64_t* n_pairwise) {
    PG_CHECK(ctx && h_table, "pg_popgen_allgather: null argument");
    PG_CHECK(ctx->nccl_comm != nullptr, "pg_popgen_allgather: call pg_nccl_init first");
    PG_CHECK(w_max >= ctx->W && w_max >= 1, "pg_popgen_allgather: w_max (%lld) is smaller than this rank's window count (%lld)",
             (long long)w_max, (long long)ctx->W);
    PG_CUDA(cudaSetDevice(ctx->device));
    const int P = ctx->P;
    const int RC = 4 + 5 * P + 2 * (P * (P - 1) / 2);
    const size_t slot_words = (size_t)w_max * RC;
    const size_t total_words = slot_words * (size_t)ctx->nccl_ranks;
    PG_TRY(ctx->gather.ensure(total_words * 8));
    unsigned long long* base = (unsigned long long*)ctx->gather.p;
    unsigned long long* mine = base + slot_words * (size_t)ctx->nccl_rank;
    // the finalize writes every word of rows < W and the all-gather every other rank's part; rows W..w_max-1 may hold an
    // earlier call's records (more windows, or another record layout of the same buffer)
    PG_CUDA(cudaMemsetAsync(mine + (size_t)ctx->W * RC, 0, (size_t)(w_max - ctx->W) * RC * 8, ctx->stream));
    // enqueue: site pass -> finalize -> all-gather -> D2H of the table; ONE host synchronisation
    int* h_cnt = nullptr;
    PG_TRY(pg_popgen_enqueue(ctx, min_sites, min_data, force_path, mine, &h_cnt));
    PG_NCCL(g_nccl.all_gather(mine, base, slot_words, NCCL_UINT64, (NcclComm)ctx->nccl_comm, ctx->stream));
    ctx->launches += 1;
    PG_CUDA(cudaMemcpyAsync(h_table, base, total_words * 8, cudaMemcpyDeviceToHost, ctx->stream));
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    const int nk2 = h_cnt ? *h_cnt : 0;
    if (n_pairwise) *n_pairwise = nk2;
    // Windows routed to the pairwise path: every rank must take part in the second gather, so the decision is
    // collective — the path column of the gathered table tells each rank whether ANY rank has such windows.
    bool any = false;
    {
        const unsigned long long* tab = (const unsigned long long*)h_table;
        for (size_t r = 0; r < (size_t)ctx->nccl_ranks * (size_t)w_max && !any; ++r) any = (tab[r * RC + 2] == 2ull);
    }
    if (any) {
        PG_TRY(pg_popgen_resolve(ctx, min_sites, min_data, mine, nk2));
        PG_NCCL(g_nccl.all_gather(mine, base, slot_words, NCCL_UINT64, (NcclComm)ctx->nccl_comm, ctx->stream));
        ctx->launches += 1;
        PG_CUDA(cudaMemcpyAsync(h_table, base, total_words * 8, cudaMemcpyDeviceToHost, ctx->stream));
        PG_CUDA(cudaStreamSynchronize(ctx->stream));
    }
    return PG_OK;
}

// Pipelined form of pg_popgen_allgather: `begin` enqueues the site pass + finalize of one batch on the ctx stream and the
// exchange (ncclAllGather, when a communicator is set) + the read-back of the table on a SIDE stream; `end` waits for that
// batch's table.  With two slots the exchange and the D2H of batch k run under the site pass of batch k+1:
//     begin(0); begin(1); end(0); begin(0); end(1); ...
// Windows that need the pairwise path are resolved in `end` (synchronously, then gathered again).
extern "C" int pg_popgen_gather_begin(pg_ctx* ctx, int32_t min_sites, double min_data, int64_t w_max, int32_t slot) {
    PG_CHECK(ctx && (slot == 0 || slot == 1), "pg_popgen_gather_begin: bad argument");
    PG_CHECK(w_max >= ctx->W && w_max >= 1, "pg_popgen_gather_begin: w_max (%lld) is smaller than this rank's window count (%lld)",
             (long long)w_max, (long long)ctx->W);
    PG_CUDA(cudaSetDevice(ctx->device));
    const int ranks = ctx->nccl_comm ? ctx->nccl_ranks : 1, rank = ctx->nccl_comm ? ctx->nccl_rank : 0;
    const int P = ctx->P;
    const int RC = 4 + 5 * P + 2 * (P * (P - 1) / 2);
    const size_t slot_words = (size_t)w_max * RC, total_words = slot_words * (size_t)ranks;
    if (!ctx->gather_stream) {
        PG_CUDA(cudaStreamCreateWithFlags(&ctx->gather_stream, cudaStreamNonBlocking));
        for (int k = 0; k < 2; ++k) {
            PG_CUDA(cudaEventCreateWithFlags(&ctx->g_rec[k], cudaEventDisableTiming));
            PG_CUDA(cudaEventCreateWithFlags(&ctx->g_done[k], cudaEventDisableTiming));
        }
    }
    if (ctx->gslot_words[slot] != total_words || ctx->gslot[slot].cap < total_words * 8) {
        PG_TRY(ctx->gslot[slot].ensure(total_words * 8));
        PG_CUDA(cudaMemsetAsync(ctx->gslot[slot].p, 0, total_words * 8, ctx->stream));
        ctx->gslot_words[slot] = total_words;
    }
    if (ctx->gslot_host_cap[slot] < total_words * 8) {
        if (ctx->gslot_host[slot]) cudaFreeHost(ctx->gslot_host[slot]);
        ctx->gslot_host[slot] = nullptr;
        PG_CUDA(cudaHostAlloc(&ctx->gslot_host[slot], total_words * 8, cudaHostAllocDefault));
        ctx->gslot_host_cap[slot] = total_words * 8;
    }
    ctx->gslot_wmax[slot] = w_max;
    ctx->gslot_min_sites[slot] = min_sites;
    ctx->gslot_min_data[slot] = min_data;
    // `end` may run after the windows, the matrix or the populations have changed for the next batch
    ctx->gslot_W[slot] = ctx->W;
    ctx->gslot_RC[slot] = RC;
    ctx->gslot_lo[slot] = ctx->win_lo;
    ctx->gslot_hi[slot] = ctx->win_hi;
    ctx->gslot_gen[slot] = ctx->data_gen;
    unsigned long long* base = (unsigned long long*)ctx->gslot[slot].p;
    unsigned long long* mine = base + slot_words * (size_t)rank;
    // the finalize writes rows < W only: rows of an earlier batch with more windows must not reach the table
    PG_CUDA(cudaMemsetAsync(mine + (size_t)ctx->W * RC, 0, (size_t)(w_max - ctx->W) * RC * 8, ctx->stream));
    // `end` reads the routed windows off the gathered path column: no counter read-back
    PG_TRY(pg_popgen_enqueue(ctx, min_sites, min_data, 0, mine, nullptr));
    PG_CUDA(cudaEventRecord(ctx->g_rec[slot], ctx->stream));
    PG_CUDA(cudaStreamWaitEvent(ctx->gather_stream, ctx->g_rec[slot], 0));
    if (ranks > 1) {
        PG_NCCL(g_nccl.all_gather(mine, base, slot_words, NCCL_UINT64, (NcclComm)ctx->nccl_comm, ctx->gather_stream));
        ctx->launches += 1;
    }
    PG_CUDA(cudaMemcpyAsync(ctx->gslot_host[slot], base, total_words * 8, cudaMemcpyDeviceToHost, ctx->gather_stream));
    PG_CUDA(cudaEventRecord(ctx->g_done[slot], ctx->gather_stream));
    return PG_OK;
}

// *h_table: the slot's pinned table (nranks * w_max records, rank order; valid until the slot's next `begin`).
extern "C" int pg_popgen_gather_end(pg_ctx* ctx, int32_t slot, const void** h_table, int64_t* n_pairwise) {
    PG_CHECK(ctx && h_table && (slot == 0 || slot == 1) && ctx->gslot_host[slot], "pg_popgen_gather_end: no batch in this slot");
    PG_CUDA(cudaSetDevice(ctx->device));
    PG_CUDA(cudaEventSynchronize(ctx->g_done[slot]));
    const int ranks = ctx->nccl_comm ? ctx->nccl_ranks : 1, rank = ctx->nccl_comm ? ctx->nccl_rank : 0;
    // the batch as it was at `begin`: the ctx may already hold the next batch's windows, populations or data
    const int RC = ctx->gslot_RC[slot];
    const int64_t w_max = ctx->gslot_wmax[slot], W = ctx->gslot_W[slot];
    const size_t slot_words = (size_t)w_max * RC, total_words = slot_words * (size_t)ranks;
    const unsigned long long* tab = (const unsigned long long*)ctx->gslot_host[slot];
    // windows routed to the pairwise path: a collective decision read off the gathered path column (rows past a rank's
    // window count are zero); this rank's own windows are read off its rows of the slot's table
    bool any = false;
    std::vector<int64_t> k2_windows;
    for (size_t r = 0; r < (size_t)ranks * (size_t)w_max; ++r) {
        const bool k2 = tab[r * RC + 2] == 2ull;
        any = any || k2;
        if (k2 && r / (size_t)w_max == (size_t)rank && (int64_t)(r % (size_t)w_max) < W)
            k2_windows.push_back((int64_t)(r % (size_t)w_max));
    }
    if (n_pairwise) *n_pairwise = (int64_t)k2_windows.size();
    if (any) {
        const long long refuse = (!k2_windows.empty() && ctx->gslot_gen[slot] != ctx->data_gen) ? 1 : 0;
        long long refusals = refuse;
        if (ctx->nccl_comm) {      // collective: a rank refusing alone would leave the others waiting in the second gather
            PG_TRY(ctx->gather_flag.ensure(8));
            PG_CUDA(cudaMemcpyAsync(ctx->gather_flag.p, &refuse, 8, cudaMemcpyHostToDevice, ctx->stream));
            PG_TRY(pg_nccl_allreduce_i64(ctx, ctx->gather_flag.p, 1));
            PG_CUDA(cudaMemcpyAsync(&refusals, ctx->gather_flag.p, 8, cudaMemcpyDeviceToHost, ctx->stream));
            PG_CUDA(cudaStreamSynchronize(ctx->stream));
        }
        PG_CHECK(!refuse, "pg_popgen_gather_end: the genotype matrix or the populations changed after this slot's "
                 "pg_popgen_gather_begin; its %lld pairwise windows cannot be computed from the batch's data "
                 "(call end before changing them)", (long long)k2_windows.size());
        PG_CHECK(refusals == 0, "pg_popgen_gather_end: %lld other rank(s) refused this slot: their genotype matrix or "
                 "populations changed after pg_popgen_gather_begin", refusals);
        unsigned long long* base = (unsigned long long*)ctx->gslot[slot].p;
        unsigned long long* mine = base + slot_words * (size_t)rank;
        PG_CUDA(cudaStreamSynchronize(ctx->gather_stream));
        if (!k2_windows.empty())
            PG_TRY(pg_k2_popgen_windows(ctx, k2_windows, ctx->gslot_lo[slot].data(), ctx->gslot_hi[slot].data(),
                                        ctx->gslot_min_sites[slot], ctx->gslot_min_data[slot], mine, RC));
        if (ranks > 1) {
            PG_NCCL(g_nccl.all_gather(mine, base, slot_words, NCCL_UINT64, (NcclComm)ctx->nccl_comm, ctx->stream));
            ctx->launches += 1;
        }
        PG_CUDA(cudaMemcpyAsync(ctx->gslot_host[slot], base, total_words * 8, cudaMemcpyDeviceToHost, ctx->stream));
        PG_CUDA(cudaStreamSynchronize(ctx->stream));
    }
    *h_table = ctx->gslot_host[slot];
    return PG_OK;
}

namespace {
// this rank's records (rc words per window, written by `enqueue` into its slot of the gather buffer) + all-gather + D2H
template <typename F>
int gather_fixed_records(pg_ctx* ctx, int rc, int64_t w_max, void* h_table, const char* what, F enqueue) {
    PG_CHECK(ctx && h_table, "%s: null argument", what);
    PG_CHECK(ctx->nccl_comm != nullptr, "%s: call pg_nccl_init first", what);
    PG_CHECK(w_max >= ctx->W && w_max >= 1, "%s: w_max (%lld) is smaller than this rank's window count (%lld)", what,
             (long long)w_max, (long long)ctx->W);
    PG_CUDA(cudaSetDevice(ctx->device));
    const size_t slot_words = (size_t)w_max * rc;
    const size_t total_words = slot_words * (size_t)ctx->nccl_ranks;
    PG_TRY(ctx->gather.ensure(total_words * 8));
    unsigned long long* base = (unsigned long long*)ctx->gather.p;
    unsigned long long* mine = base + slot_words * (size_t)ctx->nccl_rank;
    PG_CUDA(cudaMemsetAsync(mine, 0, slot_words * 8, ctx->stream));
    PG_TRY(enqueue(mine));
    PG_NCCL(g_nccl.all_gather(mine, base, slot_words, NCCL_UINT64, (NcclComm)ctx->nccl_comm, ctx->stream));
    ctx->launches += 1;
    PG_CUDA(cudaMemcpyAsync(h_table, base, total_words * 8, cudaMemcpyDeviceToHost, ctx->stream));
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    return PG_OK;
}
}  // namespace

// ABBA-BABA statistics of this rank's windows + ONE ncclAllGather of every rank's records (config 3: ABBABABAwindows
// window-sharded over the GPUs).  h_table: nranks * w_max * 8 words [sites, pos_sum, ABBA, BABA, D, fd, fdM, sitesUsed].
extern "C" int pg_abbababa_allgather(pg_ctx* ctx, int32_t p1, int32_t p2, int32_t p3, int32_t o, double min_data,
                                     int64_t w_max, void* h_table) {
    const int sel[4] = {p1, p2, p3, o};
    return gather_fixed_records(ctx, 8, w_max, h_table, "pg_abbababa_allgather",
                                [&](void* d_rec) { return pg_abba_enqueue(ctx, sel, min_data, d_rec); });
}

// The same for genomics.fourPop: 17 words per window [sites, pos_sum, 14 statistics (pg_fourpop order), sitesUsed].
extern "C" int pg_fourpop_allgather(pg_ctx* ctx, int32_t p1, int32_t p2, int32_t p3, int32_t p4, double min_data,
                                    int32_t mode, int64_t w_max, void* h_table) {
    const int sel[4] = {p1, p2, p3, p4};
    return gather_fixed_records(ctx, 17, w_max, h_table, "pg_fourpop_allgather",
                                [&](void* d_rec) { return pg_fourpop_enqueue(ctx, sel, min_data, mode, d_rec); });
}
