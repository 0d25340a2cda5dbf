// mergeGeno.py on the device (mergeGeno.py:41-88): several .geno bodies joined by position in the order of the .fai's walk.
//
// The reference walks every position (scaffold, site) of the .fai and compares each file's current line with it: a line is
// consumed when it matches, and a file whose line never matches stalls there for good.  So a file's consumed lines are the
// longest prefix of its body whose lines each name a .fai scaffold, hold a canonical decimal site inside it and lie strictly
// after the line before in the walk.  With walk index key = offset(scaffold) + site - 1:
//   pg_merge_load  : one chunk of complete lines of one file.  k_merge_lines gives every physical line ONE WARP
//                    (pg_warp_fields): field count, scaffold id (hash table of the .fai names, exact byte compare), the site's
//                    canonical-decimal test, the key, the span of fields 2.. and its token bytes.  k_merge_stall flags every
//                    line that is invalid, not above the line before (carried across chunks) or refused (a byte >= 0x80, a
//                    lone '\r'); the first flag is the file's stall, and nothing from it on is merged.
//   pg_merge_rows  : the walk up to a bound hi.  Every file's waiting keys <= hi are gathered with (file, line) values and
//                    radix-sorted (stable, so a position's files stay in file order).  Sparse rule: the runs of equal keys
//                    are the positions some file matched; k_merge_len applies the write rule.  Dense rule (`all`, or `union`
//                    with unionMin <= 0, and no --mustIncludeFirst): every walk index in (previous hi, hi] is a row and finds
//                    its run by binary search.  k_merge_len writes each row's length, a CUB scan gives the offsets.
//   pg_merge_emit  : a slab of the rows, one warp per row: scaffold name, site digits, then every output file's genotypes —
//                    the matched line's tokens (copied as one span when they are single-tab separated and outSep is '\t',
//                    otherwise re-walked and joined with outSep) or its dummy genotypes.  A row may be cut between slabs.
// The host (cli/mergeGeno.py) picks the bounds: the smallest last loaded key over the files still reading, so that only the
// file(s) that set it load their next chunk and device memory holds about one chunk per file.
#include <algorithm>
#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>

#include "pgwin_internal.h"

namespace {

enum { MF_INVALID = 1, MF_BAD = 2, MF_SIMPLE = 4 };

struct LineRec {
    int64_t key;        // walk index, -1 when the line cannot match any position
    uint32_t f2;        // first byte of field 2 in the chunk
    uint32_t span;      // bytes from field 2's start to the end of the last field (0: no field 2)
    uint32_t ntok;      // fields 2..
    uint32_t toklen;    // their bytes
    uint32_t flags;     // MF_*
    uint32_t pad;
};

struct FileDev {
    const uint8_t* text;
    const LineRec* line;
    int64_t cursor, n_valid;    // lines [cursor, n_valid) of the chunk wait to be merged
    int64_t base;               // first entry of the file in the gather
    int32_t out;                // the file's columns are written
    int32_t pad;
    int64_t n_dummy;            // dummy genotypes of the file (its header's fields - 2, at least 0)
};

struct Scaf {
    const char* names;
    const int64_t* name_off;    // [n + 1]
    const int64_t* off;         // [n] walk offset
    const int64_t* len;         // [n]
    const int32_t* slot;        // [hmask + 1] hash table of the names, -1 empty
    uint64_t hmask;
    const int64_t* pos_off;     // [n_pos] walk offsets of the scaffolds of positive length, ascending
    const int32_t* pos_id;      // [n_pos]
    int32_t n_pos;
};

__host__ __device__ __forceinline__ uint64_t fnv1a(const uint8_t* s, int64_t n) {
    uint64_t h = 1469598103934665603ull;
    for (int64_t i = 0; i < n; ++i) h = (h ^ s[i]) * 1099511628211ull;
    return h;
}

__device__ __forceinline__ int digits(int64_t v) {
    int n = 1;
    while (v >= 10) v /= 10, ++n;
    return n;
}

__global__ void k_merge_hash(const char* __restrict__ names, const int64_t* __restrict__ name_off, int64_t n, int32_t* slot,
                             uint64_t hmask) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint64_t h = fnv1a((const uint8_t*)names + name_off[i], name_off[i + 1] - name_off[i]) & hmask;
    while (atomicCAS(&slot[h], -1, (int32_t)i) != -1) h = (h + 1) & hmask;
}

__global__ void k_merge_nl(const uint8_t* __restrict__ text, size_t len, uint8_t* __restrict__ flag) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < len; i += (size_t)gridDim.x * blockDim.x)
        flag[i] = text[i] == '\n';
}

// the .fai scaffold named by bytes [q, e) of the text, -1 when none
__device__ int32_t scaffold_of(const Scaf& sc, const uint8_t* t, size_t q, size_t e) {
    uint64_t h = fnv1a(t + q, (int64_t)(e - q)) & sc.hmask;
    for (;; h = (h + 1) & sc.hmask) {
        const int32_t s = sc.slot[h];
        if (s < 0) return -1;
        const int64_t a = sc.name_off[s], n = sc.name_off[s + 1] - a;
        if (n != (int64_t)(e - q)) continue;
        int64_t k = 0;
        while (k < n && (uint8_t)sc.names[a + k] == t[q + k]) ++k;
        if (k == n) return s;
    }
}

// one warp per physical line: line i is bytes [nl[i - 1] + 1, nl[i]) (the chunk's end for an unterminated last line)
__global__ void __launch_bounds__(256) k_merge_lines(const uint8_t* __restrict__ text, size_t len,
                                                     const uint32_t* __restrict__ nl, int64_t n_nl, int64_t n_lines,
                                                     const Scaf sc, LineRec* __restrict__ rec) {
    const int lane = threadIdx.x & 31;
    const int64_t i = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (i >= n_lines) return;
    const size_t l0 = i == 0 ? 0 : (size_t)nl[i - 1] + 1;
    const size_t le = i < n_nl ? (size_t)nl[i] : len;
    long long f0 = -1, f1 = -1, f2 = -1;
    bool hi = false, lone_cr = false;
    const unsigned nf = pg_warp_fields(text, len, l0, &hi, &lone_cr, [&](unsigned fidx, size_t q) {
        if (fidx == 0) f0 = (long long)q;
        else if (fidx == 1) f1 = (long long)q;
        else if (fidx == 2) f2 = (long long)q;
    });
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) {
        f0 = max(f0, __shfl_xor_sync(0xffffffffu, f0, d));
        f1 = max(f1, __shfl_xor_sync(0xffffffffu, f1, d));
        f2 = max(f2, __shfl_xor_sync(0xffffffffu, f2, d));
    }
    // fields 2..: token bytes and the end of the last token, then the blanks inside that are not single tabs
    uint32_t toklen = 0, last = 0, odd = 0;
    if (nf > 2) {
        const size_t s = (size_t)f2;
        unsigned cnt = 0;
        long long lastp = -1;
        for (size_t q = s + lane; q < le; q += 32)
            if (!pg_sblank(text[q])) ++cnt, lastp = (long long)q;
        for (int d = 16; d >= 1; d >>= 1) {
            cnt += __shfl_xor_sync(0xffffffffu, cnt, d);
            lastp = max(lastp, __shfl_xor_sync(0xffffffffu, lastp, d));
        }
        toklen = cnt;
        last = (uint32_t)(lastp + 1 - (long long)s);
        unsigned nt = 0;
        for (size_t q = s + lane; q < (size_t)lastp; q += 32) nt += text[q] != '\t' && pg_sblank(text[q]);
        for (int d = 16; d >= 1; d >>= 1) nt += __shfl_xor_sync(0xffffffffu, nt, d);
        odd = nt;
    }
    if (lane != 0) return;
    LineRec r;
    r.key = -1;
    r.f2 = nf > 2 ? (uint32_t)f2 : 0;
    r.span = nf > 2 ? last : 0;
    r.ntok = nf > 2 ? nf - 2 : 0;
    r.toklen = toklen;
    r.pad = 0;
    uint32_t flags = (hi || lone_cr) ? MF_BAD : 0;
    if (nf > 2 && odd == 0 && last - toklen == nf - 3) flags |= MF_SIMPLE;
    bool ok = nf >= 2 && !(flags & MF_BAD);
    int32_t s = -1;
    if (ok) {
        size_t e0 = (size_t)f0;
        while (e0 < le && !pg_sblank(text[e0])) ++e0;
        s = scaffold_of(sc, text, (size_t)f0, e0);
        ok = s >= 0;
    }
    int64_t n = 0;
    if (ok) {                                           // str(n) for 1 <= n <= the scaffold's length
        size_t q = (size_t)f1;
        ok = text[q] >= '1' && text[q] <= '9';
        int nd = 0;
        for (; ok && q < le && !pg_sblank(text[q]); ++q, ++nd) {
            const unsigned c = text[q];
            if (c < '0' || c > '9' || nd >= 19) ok = false;
            else n = n * 10 + (c - '0');
        }
        ok = ok && n <= sc.len[s];
    }
    if (ok) r.key = sc.off[s] + n - 1;
    else flags |= MF_INVALID;
    r.flags = flags;
    rec[i] = r;
}

// the first line that is refused, invalid or not above the line before (carry: the key before the chunk)
__global__ void k_merge_stall(const LineRec* __restrict__ rec, int64_t n, int64_t carry, unsigned long long* stall) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int64_t prev = i == 0 ? carry : rec[i - 1].key;
    if ((rec[i].flags & (MF_INVALID | MF_BAD)) || rec[i].key <= prev) atomicMin(stall, (unsigned long long)i);
}

// {stall line, its flags (0 none), key of the last line before it (carry when none)}
__global__ void k_merge_summary(const LineRec* __restrict__ rec, int64_t n, int64_t carry, const unsigned long long* stall,
                                int64_t* out) {
    const int64_t s = (int64_t)*stall;
    out[0] = s;
    out[1] = s < n ? rec[s].flags : 0;
    out[2] = s > 0 ? rec[s - 1].key : carry;
}

// per file: the waiting lines with key <= hi
__global__ void k_merge_count(const FileDev* __restrict__ fd, int nF, int64_t hi, int64_t* take) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    if (x >= nF) return;
    int64_t a = fd[x].cursor, z = fd[x].n_valid;        // first line with key > hi
    while (a < z) {
        const int64_t m = (a + z) >> 1;
        if (fd[x].line[m].key <= hi) a = m + 1;
        else z = m;
    }
    take[x] = a - fd[x].cursor;
}

__global__ void k_merge_gather(const FileDev* __restrict__ fd, int nF, int64_t N, uint64_t* __restrict__ key,
                               uint64_t* __restrict__ val) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= N) return;
    int a = 0, z = nF - 1;                              // the last file with base <= e
    while (a < z) {
        const int m = (a + z + 1) >> 1;
        if (fd[m].base <= e) a = m;
        else z = m - 1;
    }
    const int64_t line = fd[a].cursor + (e - fd[a].base);
    key[e] = (uint64_t)fd[a].line[line].key;
    val[e] = ((uint64_t)a << 32) | (uint64_t)line;
}

// dense rule: row r is walk index p0 + r, with the run of its entries in the sorted keys
__global__ void k_merge_dense(const uint64_t* __restrict__ key, int64_t N, int64_t p0, int64_t D, int nF,
                              int64_t* __restrict__ row_key, int32_t* __restrict__ row_start, int32_t* __restrict__ row_cnt) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= D) return;
    const uint64_t p = (uint64_t)(p0 + r);
    int64_t a = 0, z = N;
    while (a < z) {
        const int64_t m = (a + z) >> 1;
        if (key[m] < p) a = m + 1;
        else z = m;
    }
    int c = 0;
    while (c < nF && a + c < N && key[a + c] == p) ++c;
    row_key[r] = (int64_t)p;
    row_start[r] = (int32_t)a;
    row_cnt[r] = c;
}

struct RowParams {
    const FileDev* fd;
    int nF;
    const uint64_t* val;        // sorted entries: file << 32 | line
    const int64_t* row_key;
    const int32_t* row_start;
    const int32_t* row_cnt;
    int64_t R;
    int64_t* len;               // [R + 1]
    const int64_t* off;         // [R + 1]
    Scaf sc;
    const char* sep;
    const char* miss;
    int32_t sep_len, miss_len;
    int32_t dense, method, need_first, tab_sep;
    int64_t union_min;
    unsigned long long* written;
    // emission: output bytes [b0, b1) into out, rows [bounds[0], bounds[1])
    int64_t b0, b1;
    const int64_t* bounds;
    char* out;
};

__device__ __forceinline__ int scaf_of_key(const Scaf& sc, int64_t key) {
    int a = 0, z = sc.n_pos - 1;                        // the last positive-length scaffold with offset <= key
    while (a < z) {
        const int m = (a + z + 1) >> 1;
        if (sc.pos_off[m] <= key) a = m;
        else z = m - 1;
    }
    return sc.pos_id[a];
}

__global__ void k_merge_len(const __grid_constant__ RowParams p) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= p.R) return;
    const int64_t start = p.row_start[r];
    const int cnt = p.row_cnt[r];
    bool ok = true;
    if (!p.dense) {
        if (p.need_first > 0)
            ok = cnt >= p.need_first && (int)(p.val[start + p.need_first - 1] >> 32) == p.need_first - 1;
        if (p.method == 0) ok = ok && cnt == p.nF;
        else if (p.method == 1) ok = ok && cnt >= p.union_min;
    }
    if (!ok) {
        p.len[r] = 0;
        return;
    }
    const int64_t key = p.row_key[r];
    const int s = scaf_of_key(p.sc, key);
    int64_t n = p.sc.name_off[s + 1] - p.sc.name_off[s] + p.sep_len + digits(key - p.sc.off[s] + 1) + 1;
    int64_t j = start;
    for (int x = 0; x < p.nF; ++x) {
        const FileDev& f = p.fd[x];
        const bool hit = j < start + cnt && (int)(p.val[j] >> 32) == x;
        if (hit) {
            if (f.out) {
                const LineRec& L = f.line[p.val[j] & 0xffffffffu];
                n += (int64_t)L.ntok * p.sep_len + L.toklen;
            }
            ++j;
        } else if (f.out) {
            n += f.n_dummy * (p.sep_len + p.miss_len);
        }
    }
    p.len[r] = n;
    atomicAdd(p.written, 1ull);
}

// rows [bounds[0], bounds[1]) are the ones that overlap output bytes [b0, b1)
__global__ void k_merge_bounds(const int64_t* __restrict__ off, int64_t R, int64_t b0, int64_t b1, int64_t* bounds) {
    int64_t a = 0, z = R;                               // first row ending after b0: the last row with off <= b0
    while (a < z) {
        const int64_t m = (a + z) >> 1;
        if (off[m + 1] <= b0) a = m + 1;
        else z = m;
    }
    bounds[0] = a;
    z = R;                                              // first row starting at or after b1
    while (a < z) {
        const int64_t m = (a + z) >> 1;
        if (off[m] < b1) a = m + 1;
        else z = m;
    }
    bounds[1] = a;
}

struct Out {
    char* out;
    int64_t b0, b1;
    __device__ __forceinline__ void put(int64_t at, char c) const {
        if (at >= b0 && at < b1) out[at - b0] = c;
    }
    // the lanes' range of k in [0, n) whose byte o + k falls in the slab
    __device__ __forceinline__ int64_t lo(int64_t o) const { return max((int64_t)0, b0 - o); }
    __device__ __forceinline__ int64_t hi(int64_t o, int64_t n) const { return min(n, b1 - o); }
};

// the tokens of span [0, n) of t, each after the separator, by one warp
__device__ __forceinline__ void put_tokens(const Out& w, int64_t o, const uint8_t* t, int64_t n, const char* sep, int sl) {
    const int lane = threadIdx.x & 31;
    const unsigned lt = (1u << lane) - 1u;
    int64_t nonws = 0, starts = 0;
    bool prev_ws = true;
    for (int64_t base = 0; base < n; base += 32) {
        const int64_t i = base + lane;
        const unsigned c = i < n ? t[i] : ' ';
        const bool ws = pg_sblank(c);
        const unsigned m = __ballot_sync(0xffffffffu, !ws);
        const bool pws = lane == 0 ? prev_ws : !((m >> (lane - 1)) & 1u);
        const bool st = !ws && pws;
        const unsigned sm = __ballot_sync(0xffffffffu, st);
        if (!ws) {
            const int64_t at = o + nonws + __popc(m & lt) + (starts + __popc(sm & (lt | (1u << lane)))) * sl;
            w.put(at, (char)c);
            if (st)
                for (int k = 0; k < sl; ++k) w.put(at - sl + k, sep[k]);
        }
        nonws += __popc(m);
        starts += __popc(sm);
        prev_ws = !(m >> 31);
    }
}

__global__ void k_merge_emit(const __grid_constant__ RowParams p) {
    const int lane = threadIdx.x & 31;
    const int64_t r0 = p.bounds[0], r1 = p.bounds[1];
    const Out w{p.out, p.b0, p.b1};
    const int sl = p.sep_len;
    for (int64_t r = r0 + (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); r < r1;
         r += (int64_t)gridDim.x * (blockDim.x >> 5)) {
        if (p.len[r] == 0) continue;
        int64_t o = p.off[r];
        const int64_t key = p.row_key[r];
        const int s = scaf_of_key(p.sc, key);
        const int64_t na = p.sc.name_off[s], nn = p.sc.name_off[s + 1] - na;
        for (int64_t k = w.lo(o) + lane; k < w.hi(o, nn); k += 32) w.put(o + k, p.sc.names[na + k]);
        o += nn;
        for (int k = lane; k < sl; k += 32) w.put(o + k, p.sep[k]);
        o += sl;
        const int64_t site = key - p.sc.off[s] + 1;
        const int nd = digits(site);
        if (lane < nd) {
            int64_t v = site;
            for (int i = nd - 1; i > lane; --i) v /= 10;
            w.put(o + lane, (char)('0' + v % 10));
        }
        o += nd;
        const int64_t start = p.row_start[r];
        const int cnt = p.row_cnt[r];
        int64_t j = start;
        for (int x = 0; x < p.nF && o < p.b1; ++x) {
            const FileDev& f = p.fd[x];
            const bool hit = j < start + cnt && (int)(p.val[j] >> 32) == x;
            if (hit) {
                const uint64_t line = p.val[j] & 0xffffffffu;
                ++j;
                if (!f.out) continue;
                const LineRec L = f.line[line];
                const int64_t seg = (int64_t)L.ntok * sl + L.toklen;
                if (o + seg > p.b0 && L.ntok) {
                    const uint8_t* t = f.text + L.f2;
                    if (p.tab_sep && (L.flags & MF_SIMPLE)) {
                        if (lane == 0) w.put(o, '\t');
                        for (int64_t k = max((int64_t)0, p.b0 - o - 1) + lane; k < min((int64_t)L.span, p.b1 - o - 1); k += 32)
                            w.put(o + 1 + k, (char)t[k]);
                    } else {
                        put_tokens(w, o, t, L.span, p.sep, sl);
                    }
                }
                o += seg;
            } else if (f.out) {
                const int pl = sl + p.miss_len;
                const int64_t seg = f.n_dummy * pl;
                const int64_t k0 = w.lo(o) + lane;
                int q = (int)(k0 % pl);                 // the byte's place in sep + missing, stepped by 32
                for (int64_t k = k0; k < w.hi(o, seg); k += 32) {
                    w.put(o + k, q < sl ? p.sep[q] : p.miss[q - sl]);
                    for (q += 32; q >= pl; q -= pl) {}
                }
                o += seg;
            }
        }
        if (lane == 0) w.put(p.off[r] + p.len[r] - 1, '\n');
    }
}

struct FileHost {
    PgBuf text, line;
    int64_t cursor = 0, n_valid = 0, carry = -1, take = 0;
    int32_t out = 0;
    int64_t n_dummy = 0;
};

struct MergeState {
    bool ready = false;
    PgBuf scaf, flags, nl, misc, fd, keys, vals, keys2, vals2, rows, lens, cub;
    Scaf sc{};
    int64_t total = 0;          // walk length
    std::vector<FileHost> files;
    std::string sep, miss;
    int32_t method = 0, need_first = 0, dense = 0;
    int64_t union_min = 0;
    int64_t prev = -1;          // walk indices <= prev are merged
    int64_t R = 0, n_bytes = 0; // rows of the last pg_merge_rows and their bytes
    int64_t Rcap = 0;           // the row arrays' layout of the last pg_merge_rows
    const char *sep_dev = nullptr, *miss_dev = nullptr;
    int key_bits = 1;
};

MergeState* mstate(pg_ctx* ctx) {
    if (!ctx->merge_state) ctx->merge_state = new MergeState();
    return (MergeState*)ctx->merge_state;
}

int upload_files(pg_ctx* ctx, MergeState* ms, int64_t* bases) {
    const int nF = (int)ms->files.size();
    std::vector<FileDev> h((size_t)nF);
    for (int x = 0; x < nF; ++x) {
        const FileHost& F = ms->files[(size_t)x];
        h[(size_t)x] = FileDev{(const uint8_t*)F.text.p, (const LineRec*)F.line.p, F.cursor, F.n_valid,
                               bases ? bases[x] : 0, F.out, 0, F.n_dummy};
    }
    PG_TRY(ms->fd.ensure(h.size() * sizeof(FileDev) + 64));
    PG_CUDA(cudaMemcpyAsync(ms->fd.p, h.data(), h.size() * sizeof(FileDev), cudaMemcpyHostToDevice, ctx->stream));
    return PG_OK;
}

}  // namespace

void pg_merge_free(pg_ctx* ctx) {
    MergeState* ms = (MergeState*)ctx->merge_state;
    if (!ms) return;
    for (PgBuf* b : {&ms->scaf, &ms->flags, &ms->nl, &ms->misc, &ms->fd, &ms->keys, &ms->vals, &ms->keys2, &ms->vals2,
                     &ms->rows, &ms->lens, &ms->cub})
        b->release();
    for (FileHost& F : ms->files) {
        F.text.release();
        F.line.release();
    }
    delete ms;
    ctx->merge_state = nullptr;
}

extern "C" int pg_merge_setup(pg_ctx* ctx, int64_t n_scaf, const char* names, const int64_t* name_off, const int64_t* len,
                              int32_t n_files, const int32_t* out, const int64_t* n_dummy, const char* sep, int32_t sep_len,
                              const char* missing, int32_t miss_len, int32_t method, int64_t union_min,
                              int64_t must_include_first, int32_t* dense) {
    PG_CHECK(ctx && n_scaf >= 0 && (n_scaf == 0 || (names && name_off && len)) && n_files >= 1 && out && n_dummy &&
                 (sep_len == 0 || sep) && (miss_len == 0 || missing) && sep_len >= 0 && miss_len >= 0 && dense,
             "pg_merge_setup: null or negative argument");
    PG_CHECK(method >= 0 && method <= 2, "pg_merge_setup: method %d (0 intersect, 1 union, 2 all)", method);
    PG_CHECK(n_files < (1 << 24), "pg_merge_setup: %d files", n_files);
    pg_merge_free(ctx);
    MergeState* ms = mstate(ctx);
    PG_CUDA(cudaSetDevice(ctx->device));
    // the walk: offsets of every scaffold, and the scaffolds of positive length for decoding keys
    std::vector<int64_t> off((size_t)n_scaf), pos_off;
    std::vector<int32_t> pos_id;
    int64_t total = 0;
    for (int64_t s = 0; s < n_scaf; ++s) {
        PG_CHECK(name_off[s] >= 0 && name_off[s] <= name_off[s + 1], "pg_merge_setup: name %lld", (long long)s);
        off[(size_t)s] = total;
        if (len[s] > 0) {
            PG_CHECK(len[s] < ((int64_t)1 << 62) - total, "pg_merge_setup: the walk reaches 2^62 positions");
            pos_off.push_back(total);
            pos_id.push_back((int32_t)s);
            total += len[s];
        }
    }
    PG_CHECK(n_scaf < INT32_MAX / 2, "pg_merge_setup: %lld scaffolds", (long long)n_scaf);
    uint64_t hcap = 16;
    while (hcap < 2 * (uint64_t)n_scaf) hcap <<= 1;
    const int64_t nb = n_scaf ? name_off[n_scaf] : 0;
    const int64_t np = (int64_t)pos_off.size();
    // layout: name_off [n + 1], off [n], len [n], pos_off [np] (int64); slot [hcap], pos_id [np] (int32); names; sep; miss
    const size_t i64 = (size_t)(3 * n_scaf + 1 + np) * 8, i32 = (size_t)(hcap + np) * 4;
    PG_TRY(ms->scaf.ensure(i64 + i32 + (size_t)nb + (size_t)sep_len + (size_t)miss_len + 64));
    char* d = (char*)ms->scaf.p;
    int64_t* d_noff = (int64_t*)d;
    int64_t* d_off = d_noff + n_scaf + 1;
    int64_t* d_len = d_off + n_scaf;
    int64_t* d_pos_off = d_len + n_scaf;
    int32_t* d_slot = (int32_t*)(d + i64);
    int32_t* d_pos_id = d_slot + hcap;
    char* d_names = d + i64 + i32;
    char* d_sep = d_names + nb;
    char* d_miss = d_sep + sep_len;
    const int64_t zero = 0;
    PG_CUDA(cudaMemcpyAsync(d_noff, n_scaf ? name_off : &zero, (size_t)(n_scaf + 1) * 8, cudaMemcpyHostToDevice, ctx->stream));
    if (n_scaf) {
        PG_CUDA(cudaMemcpyAsync(d_off, off.data(), (size_t)n_scaf * 8, cudaMemcpyHostToDevice, ctx->stream));
        PG_CUDA(cudaMemcpyAsync(d_len, len, (size_t)n_scaf * 8, cudaMemcpyHostToDevice, ctx->stream));
    }
    if (np) {
        PG_CUDA(cudaMemcpyAsync(d_pos_off, pos_off.data(), (size_t)np * 8, cudaMemcpyHostToDevice, ctx->stream));
        PG_CUDA(cudaMemcpyAsync(d_pos_id, pos_id.data(), (size_t)np * 4, cudaMemcpyHostToDevice, ctx->stream));
    }
    if (nb) PG_CUDA(cudaMemcpyAsync(d_names, names, (size_t)nb, cudaMemcpyHostToDevice, ctx->stream));
    if (sep_len) PG_CUDA(cudaMemcpyAsync(d_sep, sep, (size_t)sep_len, cudaMemcpyHostToDevice, ctx->stream));
    if (miss_len) PG_CUDA(cudaMemcpyAsync(d_miss, missing, (size_t)miss_len, cudaMemcpyHostToDevice, ctx->stream));
    PG_CUDA(cudaMemsetAsync(d_slot, 0xff, (size_t)hcap * 4, ctx->stream));
    pg_timings_reset(ctx);
    if (n_scaf) {
        PG_TRY(pg_timed(ctx, "merge_hash", [&] {
            k_merge_hash<<<(unsigned)((n_scaf + 255) / 256), 256, 0, ctx->stream>>>(d_names, d_noff, n_scaf, d_slot, hcap - 1);
        }));
        ctx->launches += 1;
    }
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    ms->sc = Scaf{d_names, d_noff, d_off, d_len, d_slot, hcap - 1, d_pos_off, d_pos_id, (int32_t)np};
    ms->total = total;
    ms->files.assign((size_t)n_files, FileHost());
    for (int x = 0; x < n_files; ++x) {
        ms->files[(size_t)x].out = out[x] ? 1 : 0;
        ms->files[(size_t)x].n_dummy = std::max<int64_t>(0, n_dummy[x]);
    }
    ms->sep_dev = d_sep;
    ms->miss_dev = d_miss;
    ms->sep.assign(sep ? sep : "", (size_t)sep_len);
    ms->miss.assign(missing ? missing : "", (size_t)miss_len);
    ms->method = method;
    ms->need_first = (int32_t)std::min<int64_t>(std::max<int64_t>(must_include_first, 0), n_files);
    ms->union_min = std::max(union_min, must_include_first);
    ms->dense = (method == 2 || (method == 1 && ms->union_min <= 0)) && ms->need_first == 0;
    ms->prev = -1;
    ms->R = ms->n_bytes = 0;
    ms->key_bits = 1;
    while (ms->key_bits < 64 && (total >> ms->key_bits) != 0) ++ms->key_bits;
    ms->ready = true;
    *dense = ms->dense;
    return PG_OK;
}

extern "C" int pg_merge_load(pg_ctx* ctx, int32_t file, const char* text, size_t len, int64_t* info) {
    PG_CHECK(ctx && text && info, "pg_merge_load: null argument");
    MergeState* ms = mstate(ctx);
    PG_CHECK(ms->ready, "pg_merge_load: no pg_merge_setup");
    PG_CHECK(file >= 0 && file < (int32_t)ms->files.size(), "pg_merge_load: file %d of %zu", file, ms->files.size());
    PG_CHECK(len > 0 && len < UINT32_MAX, "pg_merge_load: a chunk of %zu bytes (1 .. 2^32 - 2)", len);
    FileHost& F = ms->files[(size_t)file];
    PG_CHECK(F.cursor == F.n_valid, "pg_merge_load: file %d still has %lld lines to merge", file,
             (long long)(F.n_valid - F.cursor));
    PG_CUDA(cudaSetDevice(ctx->device));
    pg_timings_reset(ctx);
    PG_TRY(F.text.ensure(len + 64));
    PG_TRY(ms->flags.ensure(len + 64));
    PG_TRY(ms->nl.ensure(len * 4 + 64));
    PG_TRY(ms->misc.ensure(64));
    PG_CUDA(cudaMemcpyAsync(F.text.p, text, len, cudaMemcpyHostToDevice, ctx->stream));
    const uint8_t* d_text = (const uint8_t*)F.text.p;
    const unsigned grid = (unsigned)std::min<size_t>((len + 255) / 256, (size_t)ctx->sm_count * 32);
    PG_TRY(pg_timed(ctx, "merge_nl", [&] {
        k_merge_nl<<<grid, 256, 0, ctx->stream>>>(d_text, len, (uint8_t*)ms->flags.p);
    }));
    int64_t* d_misc = (int64_t*)ms->misc.p;
    size_t tmp = 0;
    thrust::counting_iterator<uint32_t> idx(0);
    PG_CUDA(cub::DeviceSelect::Flagged(nullptr, tmp, idx, (const uint8_t*)ms->flags.p, (uint32_t*)ms->nl.p, d_misc, (int64_t)len,
                                       ctx->stream));
    PG_TRY(ms->cub.ensure(tmp + 64));
    PG_TRY(pg_timed(ctx, "merge_select", [&] {
        cub::DeviceSelect::Flagged(ms->cub.p, tmp, idx, (const uint8_t*)ms->flags.p, (uint32_t*)ms->nl.p, d_misc, (int64_t)len,
                                   ctx->stream);
    }));
    int64_t n_nl = 0;
    PG_CUDA(cudaMemcpyAsync(&n_nl, d_misc, 8, cudaMemcpyDeviceToHost, ctx->stream));
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    const int64_t n_lines = n_nl + (text[len - 1] != '\n' ? 1 : 0);
    PG_TRY(F.line.ensure((size_t)n_lines * sizeof(LineRec) + 64));
    LineRec* d_rec = (LineRec*)F.line.p;
    PG_TRY(pg_timed(ctx, "merge_lines", [&] {
        k_merge_lines<<<(unsigned)((n_lines + 7) / 8), 256, 0, ctx->stream>>>(d_text, len, (const uint32_t*)ms->nl.p, n_nl,
                                                                              n_lines, ms->sc, d_rec);
    }));
    unsigned long long* d_stall = (unsigned long long*)(d_misc + 1);
    const unsigned long long init = (unsigned long long)n_lines;
    PG_CUDA(cudaMemcpyAsync(d_stall, &init, 8, cudaMemcpyHostToDevice, ctx->stream));
    PG_TRY(pg_timed(ctx, "merge_stall", [&] {
        k_merge_stall<<<(unsigned)((n_lines + 255) / 256), 256, 0, ctx->stream>>>(d_rec, n_lines, F.carry, d_stall);
        k_merge_summary<<<1, 1, 0, ctx->stream>>>(d_rec, n_lines, F.carry, d_stall, d_misc + 2);
    }));
    ctx->launches += 5;
    int64_t sum[3];
    PG_CUDA(cudaMemcpyAsync(sum, d_misc + 2, sizeof(sum), cudaMemcpyDeviceToHost, ctx->stream));
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    const bool refused = sum[0] < n_lines && (sum[1] & MF_BAD);
    F.cursor = 0;
    F.n_valid = refused ? 0 : sum[0];
    F.carry = sum[2];
    info[0] = n_lines;
    info[1] = sum[0];
    info[2] = sum[0] < n_lines ? (refused ? 2 : 1) : 0;
    info[3] = sum[2];
    return PG_OK;
}

extern "C" int pg_merge_rows(pg_ctx* ctx, int64_t hi, int64_t* n_rows, int64_t* n_bytes) {
    PG_CHECK(ctx && n_rows && n_bytes, "pg_merge_rows: null argument");
    MergeState* ms = mstate(ctx);
    PG_CHECK(ms->ready, "pg_merge_rows: no pg_merge_setup");
    PG_CHECK(hi > ms->prev && hi < ms->total, "pg_merge_rows: bound %lld after %lld (walk of %lld)", (long long)hi,
             (long long)ms->prev, (long long)ms->total);
    const int64_t D = ms->dense ? hi - ms->prev : 0;
    PG_CHECK(D < INT32_MAX, "pg_merge_rows: %lld dense rows in one call", (long long)D);
    const int nF = (int)ms->files.size();
    PG_CUDA(cudaSetDevice(ctx->device));
    pg_timings_reset(ctx);
    // the waiting lines of every file up to hi
    PG_TRY(upload_files(ctx, ms, nullptr));
    PG_TRY(ms->misc.ensure((size_t)nF * 8 + 64));
    int64_t* d_take = (int64_t*)ms->misc.p;
    PG_TRY(pg_timed(ctx, "merge_count", [&] {
        k_merge_count<<<(unsigned)((nF + 127) / 128), 128, 0, ctx->stream>>>((const FileDev*)ms->fd.p, nF, hi, d_take);
    }));
    std::vector<int64_t> take((size_t)nF), base((size_t)nF);
    PG_CUDA(cudaMemcpyAsync(take.data(), d_take, (size_t)nF * 8, cudaMemcpyDeviceToHost, ctx->stream));
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    int64_t N = 0;
    for (int x = 0; x < nF; ++x) base[(size_t)x] = N, N += take[(size_t)x];
    PG_CHECK(N < INT32_MAX, "pg_merge_rows: %lld lines in one call", (long long)N);
    PG_TRY(upload_files(ctx, ms, base.data()));
    const size_t nN = (size_t)std::max<int64_t>(N, 1);
    PG_TRY(ms->keys.ensure(nN * 8));
    PG_TRY(ms->vals.ensure(nN * 8));
    PG_TRY(ms->keys2.ensure(nN * 8));
    PG_TRY(ms->vals2.ensure(nN * 8));
    uint64_t *k0 = (uint64_t*)ms->keys.p, *v0 = (uint64_t*)ms->vals.p, *k1 = (uint64_t*)ms->keys2.p,
             *v1 = (uint64_t*)ms->vals2.p;
    const int64_t Rcap = std::max<int64_t>(N, D);
    // rows: key [Rcap] int64, start [Rcap] int32, count [Rcap] int32, then the run count; lens / offsets [Rcap + 1] int64 each
    PG_TRY(ms->rows.ensure((size_t)Rcap * 16 + 64));
    PG_TRY(ms->lens.ensure((size_t)(Rcap + 1) * 16 + 64));
    int64_t* row_key = (int64_t*)ms->rows.p;
    int32_t* row_start = (int32_t*)(row_key + Rcap);
    int32_t* row_cnt = row_start + Rcap;
    int* d_nruns = (int*)(row_cnt + Rcap);
    int64_t* d_len = (int64_t*)ms->lens.p;
    int64_t* d_off = d_len + Rcap + 1;
    ms->Rcap = Rcap;
    int launches = 1;
    if (N) {
        PG_TRY(pg_timed(ctx, "merge_gather", [&] {
            k_merge_gather<<<(unsigned)((N + 255) / 256), 256, 0, ctx->stream>>>((const FileDev*)ms->fd.p, nF, N, k0, v0);
        }));
        size_t tmp = 0;
        PG_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmp, k0, k1, v0, v1, N, 0, ms->key_bits, ctx->stream));
        PG_TRY(ms->cub.ensure(tmp + 64));
        PG_TRY(pg_timed(ctx, "merge_sort", [&] {
            cub::DeviceRadixSort::SortPairs(ms->cub.p, tmp, k0, k1, v0, v1, N, 0, ms->key_bits, ctx->stream);
        }));
        launches += 2;
    }
    int64_t R = D;
    if (!ms->dense && N) {                              // the runs of equal keys: positions some file matched
        size_t tmp = 0;
        PG_CUDA(cub::DeviceRunLengthEncode::Encode(nullptr, tmp, k1, (uint64_t*)row_key, row_cnt, d_nruns, (int)N, ctx->stream));
        size_t tmp2 = 0;
        PG_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tmp2, row_cnt, row_start, (int)N, ctx->stream));
        PG_TRY(ms->cub.ensure(std::max(tmp, tmp2) + 64));
        PG_TRY(pg_timed(ctx, "merge_runs", [&] {
            cub::DeviceRunLengthEncode::Encode(ms->cub.p, tmp, k1, (uint64_t*)row_key, row_cnt, d_nruns, (int)N, ctx->stream);
        }));
        int nr = 0;
        PG_CUDA(cudaMemcpyAsync(&nr, d_nruns, 4, cudaMemcpyDeviceToHost, ctx->stream));
        PG_CUDA(cudaStreamSynchronize(ctx->stream));
        R = nr;
        PG_TRY(pg_timed(ctx, "merge_run_starts", [&] {
            cub::DeviceScan::ExclusiveSum(ms->cub.p, tmp2, row_cnt, row_start, (int)R, ctx->stream);
        }));
        launches += 2;
    } else if (!ms->dense) {
        R = 0;
    } else if (D) {
        PG_TRY(pg_timed(ctx, "merge_dense", [&] {
            k_merge_dense<<<(unsigned)((D + 255) / 256), 256, 0, ctx->stream>>>(k1, N, ms->prev + 1, D, nF, row_key, row_start,
                                                                                row_cnt);
        }));
        launches += 1;
    }
    unsigned long long* d_written = (unsigned long long*)d_take;
    PG_CUDA(cudaMemsetAsync(d_written, 0, 8, ctx->stream));
    PG_CUDA(cudaMemsetAsync(d_len + R, 0, 8, ctx->stream));
    RowParams p{};
    p.fd = (const FileDev*)ms->fd.p;
    p.nF = nF;
    p.val = v1;
    p.row_key = row_key;
    p.row_start = row_start;
    p.row_cnt = row_cnt;
    p.R = R;
    p.len = d_len;
    p.off = d_off;
    p.sc = ms->sc;
    p.sep_len = (int32_t)ms->sep.size();
    p.miss_len = (int32_t)ms->miss.size();
    p.dense = ms->dense;
    p.method = ms->method;
    p.need_first = ms->need_first;
    p.union_min = ms->union_min;
    p.sep = ms->sep_dev;
    p.miss = ms->miss_dev;
    p.written = d_written;
    if (R) {
        PG_TRY(pg_timed(ctx, "merge_len", [&] {
            k_merge_len<<<(unsigned)((R + 255) / 256), 256, 0, ctx->stream>>>(p);
        }));
        launches += 1;
    }
    size_t tmp = 0;
    PG_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tmp, d_len, d_off, (int)(R + 1), ctx->stream));
    PG_TRY(ms->cub.ensure(tmp + 64));
    PG_TRY(pg_timed(ctx, "merge_scan", [&] {
        cub::DeviceScan::ExclusiveSum(ms->cub.p, tmp, d_len, d_off, (int)(R + 1), ctx->stream);
    }));
    ctx->launches += launches + 1;
    int64_t res[2];
    PG_CUDA(cudaMemcpyAsync(&res[0], d_off + R, 8, cudaMemcpyDeviceToHost, ctx->stream));
    PG_CUDA(cudaMemcpyAsync(&res[1], d_written, 8, cudaMemcpyDeviceToHost, ctx->stream));
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    for (int x = 0; x < nF; ++x) ms->files[(size_t)x].cursor += take[(size_t)x];
    ms->prev = hi;
    ms->R = R;
    ms->n_bytes = res[0];
    *n_rows = res[1];
    *n_bytes = res[0];
    return PG_OK;
}

extern "C" int pg_merge_emit(pg_ctx* ctx, int64_t byte0, char* out, size_t cap, size_t* bytes) {
    PG_CHECK(ctx && out && bytes, "pg_merge_emit: null argument");
    MergeState* ms = mstate(ctx);
    PG_CHECK(ms->ready, "pg_merge_emit: no pg_merge_setup");
    PG_CHECK(byte0 >= 0 && byte0 <= ms->n_bytes && cap > 0, "pg_merge_emit: byte %lld of %lld", (long long)byte0,
             (long long)ms->n_bytes);
    *bytes = 0;
    if (byte0 == ms->n_bytes) return PG_OK;
    const int64_t b1 = std::min<int64_t>(ms->n_bytes, byte0 + (int64_t)cap);
    PG_CUDA(cudaSetDevice(ctx->device));
    pg_timings_reset(ctx);
    const int64_t Rcap = ms->Rcap;
    PG_TRY(ms->flags.ensure((size_t)(b1 - byte0) + 64));   // the slab (the line pass's flags are done with)
    PG_TRY(ms->misc.ensure(64));
    int64_t* d_bounds = (int64_t*)ms->misc.p;
    RowParams p{};
    p.fd = (const FileDev*)ms->fd.p;
    p.nF = (int)ms->files.size();
    p.val = (const uint64_t*)ms->vals2.p;
    p.row_key = (const int64_t*)ms->rows.p;
    p.row_start = (const int32_t*)(p.row_key + Rcap);
    p.row_cnt = p.row_start + Rcap;
    p.R = ms->R;
    p.len = (int64_t*)ms->lens.p;
    p.off = p.len + Rcap + 1;
    p.sc = ms->sc;
    p.sep = ms->sep_dev;
    p.miss = ms->miss_dev;
    p.sep_len = (int32_t)ms->sep.size();
    p.miss_len = (int32_t)ms->miss.size();
    p.tab_sep = ms->sep == "\t";
    p.b0 = byte0;
    p.b1 = b1;
    p.bounds = d_bounds;
    p.out = (char*)ms->flags.p;
    PG_TRY(pg_timed(ctx, "merge_emit", [&] {
        k_merge_bounds<<<1, 1, 0, ctx->stream>>>(p.off, p.R, byte0, b1, d_bounds);
        const unsigned grid = (unsigned)std::max<int64_t>(1, std::min<int64_t>((p.R + 7) / 8, (int64_t)ctx->sm_count * 16));
        k_merge_emit<<<grid, 256, 0, ctx->stream>>>(p);
    }));
    ctx->launches += 2;
    PG_CUDA(cudaMemcpyAsync(out, ms->flags.p, (size_t)(b1 - byte0), cudaMemcpyDeviceToHost, ctx->stream));
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    *bytes = (size_t)(b1 - byte0);
    return PG_OK;
}
