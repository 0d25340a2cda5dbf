// The FASTA loader shared by genoToVCF's reference (geno2vcf.cu) and seqToGeno's input (seq2geno.cu): genomics.parseFasta
// (genomics.py:2256-2261) after universal newlines.
//
//   pg_fa_load  : the text goes to HBM, k_fa_marks flags the '>' bytes and a CUB select gives the record starts (the starts
//                 of parseFasta's pieces), which the host reads back with pg_fa_starts and names from their header pieces;
//   pg_fa_index : k_fa_keep flags the sequence bytes (after a record's first newline, not '\n', '\r' or ' ') and counts them
//                 per record, and a CUB select compacts them into one resident buffer, with {rec_off, rec_len} per record.
#include <algorithm>
#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>

#include "pgwin_internal.h"

namespace {

// flags of the '>' bytes, and their count
__global__ void k_fa_marks(const uint8_t* __restrict__ t, size_t n, uint8_t* __restrict__ flags,
                           unsigned long long* __restrict__ count) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const bool gt = t[i] == '>';
        flags[i] = gt;
        const unsigned act = __activemask();
        const unsigned b = __ballot_sync(act, gt);
        if (b && (threadIdx.x & 31) == __ffs(act) - 1) atomicAdd(count, (unsigned long long)__popc(b));
    }
}

// flags of the bytes of a record's sequence ([lo[k], hi[k]) without '\n', '\r' and ' ': genomics.parseFasta after universal
// newlines), and their count per record.  FA_BYTES consecutive bytes per thread.
constexpr int FA_BYTES = 16;
__global__ void k_fa_keep(const uint8_t* __restrict__ t, size_t n, const int64_t* __restrict__ lo,
                          const int64_t* __restrict__ hi, int64_t n_rec, uint8_t* __restrict__ flags,
                          unsigned long long* __restrict__ count) {
    const size_t nb = (n + FA_BYTES - 1) / FA_BYTES;
    for (size_t blk0 = (size_t)blockIdx.x * blockDim.x; blk0 < nb; blk0 += (size_t)gridDim.x * blockDim.x) {
        const size_t blk = blk0 + threadIdx.x;          // warp-uniform loop: every lane takes part in the reduction below
        long long k = -1;
        unsigned kept = 0;
        if (blk < nb) {
            const size_t i0 = blk * FA_BYTES;
            if (lo[0] <= (int64_t)i0) {                 // the last record with lo <= i0
                int64_t a = 0, b = n_rec - 1;
                while (a < b) {
                    const int64_t mid = (a + b + 1) >> 1;
                    if (lo[mid] <= (int64_t)i0) a = mid;
                    else b = mid - 1;
                }
                k = a;
            }
            for (size_t i = i0; i < i0 + FA_BYTES && i < n; ++i) {
                if (k + 1 < n_rec && lo[k + 1] <= (int64_t)i) {     // a record starts inside the run: flush the count
                    if (kept) atomicAdd(count + k, (unsigned long long)kept);
                    kept = 0;
                    ++k;
                }
                const unsigned c = t[i];
                const bool keep = k >= 0 && (int64_t)i < hi[k] && c != '\n' && c != '\r' && c != ' ';
                flags[i] = keep;
                kept += keep;
            }
        }
        // one atomic per warp and record: the lanes that end in the same record add up their counts first
        const unsigned same = __match_any_sync(0xffffffffu, k);
        const unsigned sum = __reduce_add_sync(same, kept);
        if ((int)(threadIdx.x & 31) == __ffs(same) - 1 && k >= 0 && sum) atomicAdd(count + k, (unsigned long long)sum);
    }
}

std::string label(const char* tag, const char* what) { return std::string(tag) + what; }

}  // namespace

void PgFasta::release() {
    PgBuf* bufs[] = {&fa, &flags, &seq, &rec, &scratch, &cub};
    for (PgBuf* b : bufs) b->release();
    fa_len = 0;
    n_rec = 0;
    indexed = false;
}

int pg_fa_load(pg_ctx* ctx, PgFasta& fs, const char* text, size_t len, const char* tag, int64_t* n_rec) {
    *n_rec = 0;
    fs.indexed = false;
    fs.n_rec = 0;
    fs.fa_len = len;
    PG_TRY(fs.fa.ensure(len + 64));
    PG_TRY(fs.flags.ensure(len + 64));
    PG_TRY(fs.scratch.ensure(64));
    unsigned long long* d_n = (unsigned long long*)fs.scratch.p;
    PG_CUDA(cudaMemsetAsync(d_n, 0, 8, ctx->stream));
    if (len == 0) return PG_OK;
    {
        const int ti = pg_time_begin(ctx, label(tag, "_fa_h2d").c_str());
        PG_CUDA(cudaMemcpyAsync(fs.fa.p, text, len, cudaMemcpyHostToDevice, ctx->stream));
        pg_time_end(ctx, ti);
    }
    const std::string marks = label(tag, "_fa_marks");
    const unsigned grid = (unsigned)std::min<size_t>((len + 255) / 256, (size_t)ctx->sm_count * 32);
    PG_TRY(pg_timed(ctx, marks.c_str(), [&] {
        k_fa_marks<<<grid, 256, 0, ctx->stream>>>((const uint8_t*)fs.fa.p, len, (uint8_t*)fs.flags.p, d_n);
    }));
    unsigned long long cnt = 0;
    PG_CUDA(cudaMemcpyAsync(&cnt, d_n, 8, cudaMemcpyDeviceToHost, ctx->stream));
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    fs.n_rec = (int64_t)cnt;
    if (cnt) {                                          // the record starts: offsets of the flagged bytes, into fs.rec
        PG_TRY(fs.rec.ensure((size_t)cnt * 16 + 64));
        thrust::counting_iterator<int64_t> idx(0);
        size_t tmp = 0;
        PG_CUDA(cub::DeviceSelect::Flagged(nullptr, tmp, idx, (const uint8_t*)fs.flags.p, (int64_t*)fs.rec.p, (int64_t*)d_n,
                                           (int64_t)len, ctx->stream));
        PG_TRY(fs.cub.ensure(tmp + 64));
        PG_TRY(pg_timed(ctx, marks.c_str(), [&] {
            cub::DeviceSelect::Flagged(fs.cub.p, tmp, idx, (const uint8_t*)fs.flags.p, (int64_t*)fs.rec.p, (int64_t*)d_n,
                                       (int64_t)len, ctx->stream);
        }));
    }
    ctx->launches += 2;
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    *n_rec = fs.n_rec;
    return PG_OK;
}

int pg_fa_starts(pg_ctx* ctx, PgFasta& fs, int64_t* starts) {
    if (fs.n_rec == 0) return PG_OK;
    PG_CUDA(cudaMemcpyAsync(starts, fs.rec.p, (size_t)fs.n_rec * 8, cudaMemcpyDeviceToHost, ctx->stream));
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    return PG_OK;
}

int pg_fa_index(pg_ctx* ctx, PgFasta& fs, int64_t n_rec, const int64_t* lo, const int64_t* hi, const char* tag,
                int64_t* rec_len) {
    const size_t len = fs.fa_len;
    PG_TRY(fs.scratch.ensure((size_t)n_rec * 24 + 64));
    int64_t* d_lo = (int64_t*)fs.scratch.p;
    int64_t* d_hi = d_lo + n_rec;
    unsigned long long* d_cnt = (unsigned long long*)(d_hi + n_rec);
    int64_t* d_n = (int64_t*)(d_cnt + n_rec);
    PG_CUDA(cudaMemcpyAsync(d_lo, lo, (size_t)n_rec * 8, cudaMemcpyHostToDevice, ctx->stream));
    PG_CUDA(cudaMemcpyAsync(d_hi, hi, (size_t)n_rec * 8, cudaMemcpyHostToDevice, ctx->stream));
    PG_CUDA(cudaMemsetAsync(d_cnt, 0, (size_t)n_rec * 8, ctx->stream));
    const size_t nb = (len + FA_BYTES - 1) / FA_BYTES;
    const unsigned grid = (unsigned)std::max<size_t>(1, std::min<size_t>((nb + 255) / 256, (size_t)ctx->sm_count * 16));
    PG_TRY(pg_timed(ctx, label(tag, "_fa_keep").c_str(), [&] {
        k_fa_keep<<<grid, 256, 0, ctx->stream>>>((const uint8_t*)fs.fa.p, len, d_lo, d_hi, n_rec, (uint8_t*)fs.flags.p,
                                                 d_cnt);
    }));
    std::vector<unsigned long long> cnt((size_t)n_rec);
    PG_CUDA(cudaMemcpyAsync(cnt.data(), d_cnt, (size_t)n_rec * 8, cudaMemcpyDeviceToHost, ctx->stream));
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    std::vector<int64_t> tab((size_t)n_rec * 2);        // rec_off [n_rec], rec_len [n_rec]
    int64_t total = 0;
    for (int64_t k = 0; k < n_rec; ++k) {
        tab[(size_t)k] = total;
        tab[(size_t)(n_rec + k)] = rec_len[k] = (int64_t)cnt[(size_t)k];
        total += (int64_t)cnt[(size_t)k];
    }
    PG_TRY(fs.seq.ensure((size_t)total + 64));
    size_t tmp = 0;
    PG_CUDA(cub::DeviceSelect::Flagged(nullptr, tmp, (const uint8_t*)fs.fa.p, (const uint8_t*)fs.flags.p, (uint8_t*)fs.seq.p,
                                       d_n, (int64_t)len, ctx->stream));
    PG_TRY(fs.cub.ensure(tmp + 64));
    PG_TRY(pg_timed(ctx, label(tag, "_fa_select").c_str(), [&] {
        cub::DeviceSelect::Flagged(fs.cub.p, tmp, (const uint8_t*)fs.fa.p, (const uint8_t*)fs.flags.p, (uint8_t*)fs.seq.p,
                                   d_n, (int64_t)len, ctx->stream);
    }));
    ctx->launches += 2;
    PG_TRY(fs.rec.ensure(tab.size() * 8 + 64));
    PG_CUDA(cudaMemcpyAsync(fs.rec.p, tab.data(), tab.size() * 8, cudaMemcpyHostToDevice, ctx->stream));
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    fs.fa.release();                                    // only the sequences stay resident
    fs.flags.release();
    fs.indexed = true;
    return PG_OK;
}
