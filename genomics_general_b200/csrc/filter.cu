// filterGenotypes.py on the resident matrix of a strict text ingest (ingest.cu, pg_ingest_set_strict).
//
//   k_filter_sites : ONE WARP PER SITE; lanes take the selected samples, each reads its haplotypes' one-hot bytes and
//                    adds what genomics.siteTest reads (genomics.py:742-799): called samples (Genotype.isMissing), het
//                    samples (set of allele characters, 'N' included, 519-524), the A C G T counts, and per population the
//                    called samples and base counts (each population walks its member list; lists may overlap).  Lane 0
//                    evaluates the predicate in fp64.
//   k_filter_thin  : ONE THREAD PER POD (--thinDist; the reference restarts its lastScaf at every pod of --podSize lines,
//                    filterGenotypes.py:32-47, 55): folds the contig mask, the positions and the verdicts into the rows
//                    that are written.  Without --thinDist the same kernel is an elementwise AND.
//   k_filter_emit  : ONE WARP PER KEPT ROW; lane 0 finds the scaffold and position fields in the device copy of the text,
//                    the lanes format one sample each (GenomeSite.asList, 465-512) behind a warp scan of their lengths.
//                    Run twice: lengths (then a CUB exclusive scan gives every row's byte offset), then the bytes of a
//                    slab of rows that fits the caller's buffer.
#include <algorithm>
#include <cub/cub.cuh>

#include "pgwin_internal.h"

namespace {

constexpr int FL_TIE = 1, FL_PARTIAL = 2, FL_NOALLELE = 4;
constexpr int FILT_MAX_POPS = 64;

struct FiltState {
    int64_t S = -1;                 // sites of the last pg_filter
    int P = 0, n_samp = 0;
    int64_t n_kept = 0;
    int emit_fmt = -1, emit_order = -1;   // format the offsets were computed for
    std::vector<int64_t> off;       // [n_kept + 1] byte offset of every kept row
    size_t stats_bytes = 0;
    int p2m = 0;                    // --partialToMissing applies to the output too (genomics.py:347)
};

// layout of ctx->flt_stats for S sites and P populations
struct StatsView {
    int32_t* called;
    int32_t* het;
    int32_t* cnt;       // [S x 4]
    int32_t* pcalled;   // [S x P]
    uint8_t* pmask;     // [S x P]
    uint8_t* flags;
    uint8_t* keep;
    uint8_t* fin;
};

size_t stats_layout(void* base, int64_t S, int P, StatsView* v) {
    size_t o = 0;
    auto take = [&](size_t bytes) {
        const size_t at = o;
        o += (bytes + 255) & ~(size_t)255;
        return (char*)base + at;
    };
    StatsView t;
    t.called = (int32_t*)take((size_t)S * 4);
    t.het = (int32_t*)take((size_t)S * 4);
    t.cnt = (int32_t*)take((size_t)S * 16);
    t.pcalled = (int32_t*)take((size_t)S * P * 4);
    t.pmask = (uint8_t*)take((size_t)S * P);
    t.flags = (uint8_t*)take((size_t)S);
    t.keep = (uint8_t*)take((size_t)S);
    t.fin = (uint8_t*)take((size_t)S);
    if (v) *v = t;
    return o;
}

struct FiltParams {
    const uint8_t* geno;
    int pitch;
    int64_t S;
    int n_samp;
    const int32_t* hap0;
    const int8_t* pl;
    int P;
    const int32_t* pop_off;     // [P + 1] into pop_mem
    const int32_t* pop_mem;     // member sample indices of every population, in -p order
    const int32_t* mpc;         // nullptr: no --minPopCalls
    const int32_t* mpa;         // nullptr: no --minPopAlleles / --maxPopAlleles
    const int32_t* xpa;
    int min_calls, min_alleles, min_var_count, has_max_het, fixed, has_nfd, p2m, no_test;
    double max_alleles, max_het, min_freq, max_freq, nfd;
    StatsView st;
};

__device__ __forceinline__ int base_code(unsigned b) {
    return b == 0x01u ? 0 : (b == 0x04u ? 1 : (b == 0x10u ? 2 : (b == 0x40u ? 3 : -1)));
}

// one sample's alleles: the set of allele characters seen (bit 4 = 'N'), missing alleles, A C G T counts
// (--partialToMissing makes a sample with any missing allele all missing, genomics.py:347)
__device__ __forceinline__ void sample_geno(const uint8_t* row, int h0, int pl, int p2m, unsigned& seen, int& nmiss, int* sc) {
    seen = 0;
    nmiss = 0;
    sc[0] = sc[1] = sc[2] = sc[3] = 0;
    for (int a = 0; a < pl; ++a) {
        const int code = base_code(row[h0 + a]);
        if (code < 0) {
            ++nmiss;
            seen |= 16u;
        } else {
            ++sc[code];
            seen |= 1u << code;
        }
    }
    if (nmiss && p2m) {
        nmiss = pl;
        seen = 16u;
        sc[0] = sc[1] = sc[2] = sc[3] = 0;
    }
}

__device__ __forceinline__ int warp_sum(int v) {
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
    return v;
}

__global__ void __launch_bounds__(256) k_filter_sites(const __grid_constant__ FiltParams fp) {
    extern __shared__ int sm[];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    int* pc = sm + wid * fp.P * 5;      // [P] called samples, then [P x 4] base counts (written by lane 0)
    int* pk = pc + fp.P;
    for (int64_t s = (int64_t)blockIdx.x * 8 + wid; s < fp.S; s += (int64_t)gridDim.x * 8) {
        const uint8_t* row = fp.geno + s * fp.pitch;
        int called = 0, het = 0, c[4] = {0, 0, 0, 0};
        bool partial = false;
        for (int k = lane; k < fp.n_samp; k += 32) {
            unsigned seen;
            int nmiss, sc[4];
            sample_geno(row, fp.hap0[k], fp.pl[k], fp.p2m, seen, nmiss, sc);
            partial |= (nmiss > 0 && nmiss < fp.pl[k]);
            called += nmiss == 0;
            het += __popc(seen) > 1;
#pragma unroll
            for (int a = 0; a < 4; ++a) c[a] += sc[a];
        }
        // populations: each walks its own member list (a sample may be in several, genomics.py:774-796)
        for (int p = 0; p < fp.P; ++p) {
            int pcalled = 0, pcnt[4] = {0, 0, 0, 0};
            for (int j = fp.pop_off[p] + lane; j < fp.pop_off[p + 1]; j += 32) {
                const int k = fp.pop_mem[j];
                unsigned seen;
                int nmiss, sc[4];
                sample_geno(row, fp.hap0[k], fp.pl[k], fp.p2m, seen, nmiss, sc);
                pcalled += nmiss == 0;
#pragma unroll
                for (int a = 0; a < 4; ++a) pcnt[a] += sc[a];
            }
            pcalled = warp_sum(pcalled);
#pragma unroll
            for (int a = 0; a < 4; ++a) pcnt[a] = warp_sum(pcnt[a]);
            if (lane == 0) {
                pc[p] = pcalled;
#pragma unroll
                for (int a = 0; a < 4; ++a) pk[p * 4 + a] = pcnt[a];
            }
        }
        called = warp_sum(called);
        het = warp_sum(het);
#pragma unroll
        for (int a = 0; a < 4; ++a) c[a] = warp_sum(c[a]);
        partial = __any_sync(0xffffffffu, partial);
        __syncwarp();
        if (lane == 0) {
            unsigned smask = 0;
            int nal = 0, n = 0, first = 0, second = 0;
            for (int a = 0; a < 4; ++a) {
                if (c[a] > 0) {
                    smask |= 1u << a;
                    ++nal;
                }
                n += c[a];
                if (c[a] > first) {
                    second = first;
                    first = c[a];
                } else if (c[a] > second) {
                    second = c[a];
                }
            }
            bool tie = false;
            for (int a = 0; a < 4; ++a)
                for (int b = a + 1; b < 4; ++b) tie |= (c[a] > 0 && c[a] == c[b]);
            bool keep = true;
            if (called < fp.min_calls) keep = false;                                              // 747
            if (!(fp.min_alleles <= nal && (double)nal <= fp.max_alleles)) keep = false;          // 752-753
            if (nal > 1) {                                                                        // 755
                if (fp.min_var_count && second < fp.min_var_count) keep = false;                  // 757
                if (fp.has_max_het && (double)het / (double)called > fp.max_het) keep = false;    // 759
                const double f2 = (double)second / (double)n;
                if (fp.min_freq != 0.0 && !(fp.min_freq <= f2)) keep = false;                     // 761
                if (fp.max_freq != 0.0 && !(f2 <= fp.max_freq)) keep = false;                     // 762
            }
            if (fp.P > 0) {                                                                       // 773-799
                for (int p = 0; p < fp.P; ++p) {
                    unsigned m = 0;
                    for (int a = 0; a < 4; ++a) m |= (pk[p * 4 + a] > 0 ? 1u : 0u) << a;
                    if (fp.pop_off[p + 1] == fp.pop_off[p]) m = smask;       // an empty member list stands for every sample
                    fp.st.pmask[s * fp.P + p] = (uint8_t)m;
                    fp.st.pcalled[s * fp.P + p] = pc[p];
                    if (fp.mpc && pc[p] < fp.mpc[p]) keep = false;
                }
                if (fp.fixed) {
                    bool one = true;
                    unsigned all = 0;
                    for (int p = 0; p < fp.P; ++p) {
                        const unsigned m = fp.st.pmask[s * fp.P + p];
                        one &= (__popc(m) == 1);
                        all |= m;
                    }
                    if (!(one && __popc(all) > 1)) keep = false;
                }
                if (fp.mpa)
                    for (int p = 0; p < fp.P; ++p) {
                        const int na = __popc(fp.st.pmask[s * fp.P + p]);
                        if (!(fp.mpa[p] <= na && na <= fp.xpa[p])) keep = false;
                    }
                if (fp.has_nfd) {
                    bool any = false;
                    for (int i = 0; i < fp.P && !any; ++i)
                        for (int j = i + 1; j < fp.P && !any; ++j) {
                            const int* ci = fp.pop_off[i + 1] > fp.pop_off[i] ? pk + i * 4 : c;
                            const int* cj = fp.pop_off[j + 1] > fp.pop_off[j] ? pk + j * 4 : c;
                            const int ni = ci[0] + ci[1] + ci[2] + ci[3], nj = cj[0] + cj[1] + cj[2] + cj[3];
                            if (ni == 0 || nj == 0) continue;                 // nan frequencies never pass
                            for (int a = 0; a < 4; ++a)
                                any |= fabs((double)ci[a] / (double)ni - (double)cj[a] / (double)nj) >= fp.nfd;
                        }
                    if (!any) keep = false;
                }
            }
            fp.st.called[s] = called;
            fp.st.het[s] = het;
            for (int a = 0; a < 4; ++a) fp.st.cnt[s * 4 + a] = c[a];
            fp.st.flags[s] = (uint8_t)((tie ? FL_TIE : 0) | (partial ? FL_PARTIAL : 0) | (nal == 0 ? FL_NOALLELE : 0));
            fp.st.keep[s] = (uint8_t)(fp.no_test ? 1 : keep);
        }
        __syncwarp();
    }
}

// one thread per pod of pod_size sites (site 0 starts a pod); thin_dist == 0: every site is its own pod
__global__ void k_filter_thin(int64_t S, int pod_size, int thin_dist, const int32_t* __restrict__ pos,
                              const int32_t* __restrict__ scaf, const uint8_t* __restrict__ cmask, const uint8_t* __restrict__ keep,
                              const uint8_t* __restrict__ flags, uint8_t* __restrict__ fin, unsigned* __restrict__ flags_or) {
    const int64_t npods = (S + pod_size - 1) / pod_size;
    unsigned fo = 0;
    for (int64_t pod = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; pod < npods; pod += (int64_t)gridDim.x * blockDim.x) {
        const int64_t lo = pod * pod_size, hi = min(S, lo + pod_size);
        bool have = false;
        int32_t last_scaf = 0;
        long long last_pos = 0;
        for (int64_t s = lo; s < hi; ++s) {
            if (cmask && !cmask[s]) {               // filterGenotypes.py:37: before anything else
                fin[s] = 0;
                continue;
            }
            bool good = true;
            if (thin_dist) {                        // 41-47
                const long long p = pos[s];
                if (!have || scaf[s] != last_scaf) {
                    last_pos = p;
                    last_scaf = scaf[s];
                    have = true;
                    good = false;
                } else if (p - last_pos < thin_dist) {
                    good = false;
                }
            }
            good = good && keep[s];
            fin[s] = good ? 1 : 0;
            if (good) {
                if (thin_dist) last_pos = pos[s];   // 55
                fo |= flags[s];
            }
        }
    }
    if (fo) atomicOr(flags_or, fo);
}

__global__ void k_iota_flagged_prep(int64_t n, int64_t* __restrict__ idx) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) idx[i] = i;
}

struct EmitParams {
    const uint8_t* geno;
    int pitch;
    const uint8_t* text;
    const long long* starts;
    const uint8_t* aux;
    int H;
    int n_samp;
    const int32_t* hap0;
    const int8_t* pl;
    const int64_t* rows;        // site of every kept row
    int64_t row0, nrows;
    const int32_t* cnt;         // [S x 4]
    int fmt, freq_order, p2m;
    const int64_t* off;         // [n_kept + 1] (write pass)
    char* out;                  // write pass: bytes of rows [row0, row0 + nrows) from offset off[row0]
    int64_t* len;               // length pass: [n_kept]
};

__device__ __forceinline__ bool ws_or_nl(unsigned c) { return c == ' ' || c == '\t' || c == '\r' || c == '\v' || c == '\f' || c == '\n'; }

__device__ __forceinline__ char iupac(char a, char b) {     // genomics.py:358-360: diplo("".join(sorted(alleles)))
    if (a > b) {
        const char t = a;
        a = b;
        b = t;
    }
    if (a == b) return a;                                   // AA CC GG TT NN
    if (a == 'A') return b == 'C' ? 'M' : (b == 'G' ? 'R' : (b == 'T' ? 'W' : 'N'));
    if (a == 'C') return b == 'G' ? 'S' : (b == 'T' ? 'Y' : 'N');
    if (a == 'G') return b == 'T' ? 'K' : 'N';
    return 'N';                                             // a pair with one N: refused on the host (KeyError there)
}

__device__ __forceinline__ int code_of(char a) { return a == 'A' ? 0 : (a == 'C' ? 1 : (a == 'G' ? 2 : 3)); }

// bytes of one sample's field (without its leading tab); writes them at o when o != nullptr
__device__ int sample_field(const EmitParams& ep, const uint8_t* row, int64_t site, int k, const int* rank, int count_allele,
                            char* o) {
    const int h0 = ep.hap0[k], pl = ep.pl[k];
    char al[8];
    bool miss = false;
    for (int a = 0; a < pl; ++a) {
        const int code = base_code(row[h0 + a]);
        al[a] = code < 0 ? 'N' : "ACGT"[code];
        miss |= code < 0;
    }
    if (miss && ep.p2m)
        for (int a = 0; a < pl; ++a) al[a] = 'N';
    const char ph = ep.aux ? (char)ep.aux[site * ep.H + h0] : '/';
    const bool sorted = ep.freq_order && (ep.fmt == 2 || ep.fmt == 3);
    if (sorted)                                             // sorted(alleles, key=siteAlleles.index), 'N' last (468-478)
        for (int i = 1; i < pl; ++i)
            for (int j = i; j > 0; --j) {
                const int rj = al[j] == 'N' ? 4 : rank[code_of(al[j])];
                const int rp = al[j - 1] == 'N' ? 4 : rank[code_of(al[j - 1])];
                if (rp <= rj) break;
                const char t = al[j];
                al[j] = al[j - 1];
                al[j - 1] = t;
            }
    int n = 0;
    auto put = [&](char ch) {
        if (o) o[n] = ch;
        ++n;
    };
    switch (ep.fmt) {
        case 0:                                             // asPhased
            for (int a = 0; a < pl; ++a) {
                if (a) put(ph);
                put(al[a]);
            }
            break;
        case 1: put(iupac(al[0], al[1])); break;            // asDiplo
        case 2:                                             // bases: one column per allele
            for (int a = 0; a < pl; ++a) {
                if (a) put('\t');
                put(al[a]);
            }
            break;
        case 3:
            if (ep.freq_order) {
                for (int a = 0; a < pl; ++a) put(al[a]);
            } else {                                        // str(tuple)
                put('(');
                for (int a = 0; a < pl; ++a) {
                    if (a) {
                        put(',');
                        put(' ');
                    }
                    put('\'');
                    put(al[a]);
                    put('\'');
                }
                if (pl == 1) put(',');
                put(')');
            }
            break;
        case 4: {                                           // asCoded: rank in the frequency order, '.' when missing
            bool m = false;
            for (int a = 0; a < pl; ++a) m |= al[a] == 'N';
            for (int a = 0; a < pl; ++a) {
                if (a) put(ph);
                put(m ? '.' : (char)('0' + rank[code_of(al[a])]));
            }
            break;
        }
        default: {                                          // asCount of the last allele of the frequency order
            bool m = false;
            int cnt = 0;
            for (int a = 0; a < pl; ++a) {
                m |= al[a] == 'N';
                cnt += (al[a] != 'N' && code_of(al[a]) == count_allele);
            }
            if (m) {
                put('-');
                put('1');
            } else {
                put((char)('0' + cnt));
            }
            break;
        }
    }
    return n;
}

template <bool WRITE>
__global__ void __launch_bounds__(256) k_filter_emit(const __grid_constant__ EmitParams ep) {
    const int lane = threadIdx.x & 31;
    for (int64_t r = ep.row0 + (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5); r < ep.row0 + ep.nrows;
         r += (int64_t)gridDim.x * 8) {
        const int64_t site = ep.rows[r];
        const uint8_t* row = ep.geno + site * ep.pitch;
        // frequency order of the site's alleles: np.argsort(counts)[::-1] (genomics.py:556) as a stable sort gives it —
        // descending count, ties to the higher allele (flag 1 of pg_filter_stats marks the tied sites)
        int rank[4], count_allele = 0;
        {
            int c[4];
            for (int a = 0; a < 4; ++a) c[a] = ep.cnt[site * 4 + a];
            const int nr = pg_freq_order(c, rank);
            for (int a = 0; a < 4; ++a)
                if (rank[a] == nr - 1) count_allele = a;
        }
        // prefix: the scaffold and position fields as they are in the text (filterGenotypes.py:53 objects[:2]); a data line
        // may start with blanks (ingest.cu line_start_at), which line.split() drops
        long long l0 = 0, e0 = 0, b1 = 0, e1 = 0;
        if (lane == 0) {
            l0 = ep.starts[site];
            while (ep.text[l0] != '\n' && ws_or_nl(ep.text[l0])) ++l0;
            e0 = l0;
            while (!ws_or_nl(ep.text[e0])) ++e0;
            b1 = e0;
            while (ep.text[b1] != '\n' && ws_or_nl(ep.text[b1])) ++b1;
            e1 = b1;
            while (!ws_or_nl(ep.text[e1])) ++e1;
        }
        l0 = __shfl_sync(0xffffffffu, l0, 0);
        e0 = __shfl_sync(0xffffffffu, e0, 0);
        b1 = __shfl_sync(0xffffffffu, b1, 0);
        e1 = __shfl_sync(0xffffffffu, e1, 0);
        const int64_t plen = (e0 - l0) + 1 + (e1 - b1);
        char* o = nullptr;
        if (WRITE) {
            o = ep.out + (ep.off[r] - ep.off[ep.row0]);
            for (int64_t i = lane; i < plen; i += 32) {
                const int64_t a = e0 - l0;
                o[i] = i < a ? (char)ep.text[l0 + i] : (i == a ? '\t' : (char)ep.text[b1 + (i - a - 1)]);
            }
        }
        int64_t at = plen;
        for (int k0 = 0; k0 < ep.n_samp; k0 += 32) {
            const int k = k0 + lane;
            int n = k < ep.n_samp ? 1 + sample_field(ep, row, site, k, rank, count_allele, nullptr) : 0;
            int incl = n;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const int v = __shfl_up_sync(0xffffffffu, incl, d);
                if (lane >= d) incl += v;
            }
            if (WRITE && k < ep.n_samp) {
                char* q = o + at + (incl - n);
                q[0] = '\t';
                sample_field(ep, row, site, k, rank, count_allele, q + 1);
            }
            at += __shfl_sync(0xffffffffu, incl, 31);
        }
        if (lane == 0) {
            if (WRITE) o[at] = '\n';
            else ep.len[r] = at + 1;
        }
    }
}

FiltState* state(pg_ctx* ctx) {
    if (!ctx->flt_state) ctx->flt_state = new FiltState();
    return (FiltState*)ctx->flt_state;
}

int emit_params(pg_ctx* ctx, FiltState* fs, int fmt, int freq_order, EmitParams& ep) {
    ep.geno = (const uint8_t*)ctx->d_geno;
    ep.pitch = ctx->pitch;
    ep.text = (const uint8_t*)ctx->text.p;
    ep.starts = (const long long*)ctx->starts.p;
    ep.aux = ctx->ingest_fmt == 0 ? (const uint8_t*)ctx->flt_aux.p : nullptr;
    ep.H = ctx->H;
    ep.n_samp = fs->n_samp;
    ep.hap0 = (const int32_t*)ctx->flt_tab.p;
    ep.pl = (const int8_t*)(ep.hap0 + fs->n_samp);
    ep.rows = (const int64_t*)ctx->flt_rows.p;
    StatsView st;
    stats_layout(ctx->flt_stats.p, fs->S, fs->P, &st);
    ep.cnt = st.cnt;
    ep.fmt = fmt;
    ep.freq_order = freq_order;
    ep.off = nullptr;
    ep.out = nullptr;
    ep.len = nullptr;
    return PG_OK;
}

}  // namespace

void pg_filter_free(pg_ctx* ctx) {
    delete (FiltState*)ctx->flt_state;
    ctx->flt_state = nullptr;
}

extern "C" int pg_filter(pg_ctx* ctx, const pg_filter_spec* sp, const uint8_t* contig_mask, const int32_t* scaf_id,
                         int64_t* n_kept, uint8_t* flags_or) {
    PG_CHECK(ctx && sp && n_kept, "pg_filter: null argument");
    PG_CHECK(ctx->ingest_sites == ctx->S && ctx->ingest_strict == 1,
             "pg_filter: the resident sites must come from a text ingest with strict tokens (pg_ingest_set_strict)");
    const int64_t S = ctx->S;
    const int P = sp->P, ns = sp->n_samp;
    PG_CHECK(P >= 0 && P <= FILT_MAX_POPS, "pg_filter: %d populations (at most %d)", P, FILT_MAX_POPS);
    PG_CHECK(ns >= 1 && sp->samp_hap0 && sp->samp_ploidy, "pg_filter: no samples");
    PG_CHECK(P == 0 || (sp->pop_off && sp->pop_members), "pg_filter: populations without member lists");
    PG_CHECK((sp->min_pop_alleles == nullptr) == (sp->max_pop_alleles == nullptr),
             "pg_filter: min_pop_alleles and max_pop_alleles go together");
    PG_CHECK(!sp->thin_dist || scaf_id, "pg_filter: thinning needs the scaffold ids");
    PG_CHECK(sp->pod_size >= 1, "pg_filter: pod_size must be positive");
    for (int k = 0; k < ns; ++k)
        PG_CHECK(sp->samp_ploidy[k] >= 1 && sp->samp_ploidy[k] <= 8 && sp->samp_hap0[k] >= 0 &&
                     sp->samp_hap0[k] + sp->samp_ploidy[k] <= ctx->H,
                 "pg_filter: sample %d maps outside the %d haplotypes", k, ctx->H);
    const int n_mem = P ? sp->pop_off[P] : 0;
    if (P) {
        PG_CHECK(sp->pop_off[0] == 0, "pg_filter: pop_off[0] must be 0");
        for (int p = 0; p < P; ++p)
            PG_CHECK(sp->pop_off[p + 1] >= sp->pop_off[p], "pg_filter: pop_off must not decrease (population %d)", p);
        for (int j = 0; j < n_mem; ++j)
            PG_CHECK(sp->pop_members[j] >= 0 && sp->pop_members[j] < ns, "pg_filter: population member %d is sample %d", j,
                     sp->pop_members[j]);
    }
    PG_CUDA(cudaSetDevice(ctx->device));
    pg_timings_reset(ctx);
    FiltState* fs = state(ctx);
    fs->S = S;
    fs->P = P;
    fs->n_samp = ns;
    fs->p2m = sp->partial_to_missing ? 1 : 0;
    fs->n_kept = 0;
    fs->emit_fmt = -1;
    fs->off.clear();
    *n_kept = 0;
    if (flags_or) *flags_or = 0;
    // sample tables, one block after the other at 16-byte boundaries: hap0 [ns] with the ploidies right behind it (the emit
    // reads them so), the populations' member lists, the per-population settings, the flags word, scaffold ids, contig mask.
    // The layout is walked twice: once to size the staging buffer, once to fill it.
    const size_t pw = (size_t)std::max(P, 1) * 4;
    struct Block {
        const void* src;
        size_t bytes;
    };
    const Block blocks[] = {{nullptr, (size_t)ns * 5},                              // hap0 + ploidy, filled below
                            {P ? sp->pop_off : nullptr, (size_t)(P + 1) * 4},
                            {P ? sp->pop_members : nullptr, (size_t)std::max(n_mem, 1) * 4},
                            {sp->min_pop_calls, pw},
                            {sp->min_pop_alleles, pw},
                            {sp->max_pop_alleles, pw},
                            {nullptr, 16},                                          // OR of the kept sites' flags
                            {scaf_id, (size_t)S * 4},
                            {contig_mask, (size_t)S}};
    constexpr int NB = (int)(sizeof(blocks) / sizeof(blocks[0]));
    size_t at[NB];
    size_t o = 0;
    for (int i = 0; i < NB; ++i) {
        at[i] = o;
        o += (blocks[i].bytes + 15) & ~(size_t)15;
    }
    PG_TRY(ctx->flt_tab.ensure(o));
    std::vector<char> h(o, 0);
    for (int i = 0; i < NB; ++i)
        if (blocks[i].src) memcpy(h.data() + at[i], blocks[i].src, blocks[i].bytes);
    memcpy(h.data(), sp->samp_hap0, (size_t)ns * 4);
    memcpy(h.data() + (size_t)ns * 4, sp->samp_ploidy, (size_t)ns);
    const size_t o_off = at[1], o_mem = at[2], o_mpc = at[3], o_mpa = at[4], o_xpa = at[5], o_fo = at[6], o_scaf = at[7],
                 o_cm = at[8];
    char* d = (char*)ctx->flt_tab.p;
    PG_CUDA(cudaMemcpyAsync(d, h.data(), o, cudaMemcpyHostToDevice, ctx->stream));
    fs->stats_bytes = stats_layout(nullptr, S, P, nullptr);
    PG_TRY(ctx->flt_stats.ensure(fs->stats_bytes + 64));
    StatsView st;
    stats_layout(ctx->flt_stats.p, S, P, &st);
    if (S == 0) {
        PG_CUDA(cudaStreamSynchronize(ctx->stream));
        return PG_OK;
    }
    FiltParams fp;
    fp.geno = (const uint8_t*)ctx->d_geno;
    fp.pitch = ctx->pitch;
    fp.S = S;
    fp.n_samp = ns;
    fp.hap0 = (const int32_t*)d;
    fp.pl = (const int8_t*)(d + (size_t)ns * 4);
    fp.P = P;
    fp.pop_off = (const int32_t*)(d + o_off);
    fp.pop_mem = (const int32_t*)(d + o_mem);
    fp.mpc = sp->min_pop_calls && P ? (const int32_t*)(d + o_mpc) : nullptr;
    fp.mpa = sp->min_pop_alleles && P ? (const int32_t*)(d + o_mpa) : nullptr;
    fp.xpa = sp->max_pop_alleles && P ? (const int32_t*)(d + o_xpa) : nullptr;
    fp.min_calls = sp->min_calls;
    fp.min_alleles = sp->min_alleles;
    fp.min_var_count = sp->min_var_count;
    fp.has_max_het = sp->has_max_het;
    fp.fixed = sp->fixed_diffs;
    fp.has_nfd = sp->has_nearly_fixed;
    fp.p2m = sp->partial_to_missing;
    fp.no_test = sp->no_test;
    fp.max_alleles = sp->max_alleles;
    fp.max_het = sp->max_het;
    fp.min_freq = sp->min_freq;
    fp.max_freq = sp->max_freq;
    fp.nfd = sp->nearly_fixed_diff;
    fp.st = st;
    {
        const int ti = pg_time_begin(ctx, "filter_sites");
        const unsigned grid = (unsigned)std::min<int64_t>((S + 7) / 8, (int64_t)ctx->sm_count * 32);
        k_filter_sites<<<grid, 256, (size_t)8 * P * 5 * 4, ctx->stream>>>(fp);
        pg_time_end(ctx, ti);
        PG_CUDA(cudaGetLastError());
    }
    unsigned* d_fo = (unsigned*)(d + o_fo);
    {
        const int pod = sp->thin_dist ? sp->pod_size : 1;
        const int64_t npods = (S + pod - 1) / pod;
        const int ti = pg_time_begin(ctx, "filter_thin");
        k_filter_thin<<<(unsigned)std::min<int64_t>((npods + 255) / 256, 65535), 256, 0, ctx->stream>>>(
            S, pod, sp->thin_dist, ctx->d_pos, sp->thin_dist ? (const int32_t*)(d + o_scaf) : nullptr,
            contig_mask ? (const uint8_t*)(d + o_cm) : nullptr, st.keep, st.flags, st.fin, d_fo);
        pg_time_end(ctx, ti);
        PG_CUDA(cudaGetLastError());
    }
    // kept rows: site indices where fin = 1
    PG_TRY(ctx->flt_rows.ensure((size_t)S * 8 * 2 + 64));
    int64_t* d_idx = (int64_t*)ctx->flt_rows.p + S;
    int64_t* d_rows = (int64_t*)ctx->flt_rows.p;
    PG_TRY(ctx->flt_off.ensure(64));
    int64_t* d_nsel = (int64_t*)ctx->flt_off.p;
    k_iota_flagged_prep<<<(unsigned)std::min<int64_t>((S + 255) / 256, 4096), 256, 0, ctx->stream>>>(S, d_idx);
    PG_CUDA(cudaGetLastError());
    size_t tmp = 0;
    PG_CUDA(cub::DeviceSelect::Flagged(nullptr, tmp, d_idx, st.fin, d_rows, d_nsel, S, ctx->stream));
    PG_TRY(ctx->flt_cub.ensure(tmp + 64));
    PG_CUDA(cub::DeviceSelect::Flagged(ctx->flt_cub.p, tmp, d_idx, st.fin, d_rows, d_nsel, S, ctx->stream));
    ctx->launches += 3;
    int64_t nk = 0;
    unsigned fo = 0;
    PG_CUDA(cudaMemcpyAsync(&nk, d_nsel, 8, cudaMemcpyDeviceToHost, ctx->stream));
    PG_CUDA(cudaMemcpyAsync(&fo, d_fo, 4, cudaMemcpyDeviceToHost, ctx->stream));
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    fs->n_kept = nk;
    *n_kept = nk;
    if (flags_or) *flags_or = (uint8_t)fo;
    return PG_OK;
}

extern "C" int pg_filter_emit(pg_ctx* ctx, int32_t fmt, int32_t freq_order, int64_t row0, char* out, size_t cap, int64_t* rows,
                              size_t* bytes) {
    PG_CHECK(ctx && rows && bytes, "pg_filter_emit: null argument");
    PG_CHECK(fmt >= 0 && fmt <= 5, "pg_filter_emit: unknown format %d", fmt);
    FiltState* fs = state(ctx);
    PG_CHECK(fs->S == ctx->S && ctx->ingest_sites == ctx->S && ctx->text.p, "pg_filter_emit: no pg_filter on the current text");
    PG_CHECK(row0 >= 0 && row0 <= fs->n_kept, "pg_filter_emit: row %lld out of range", (long long)row0);
    *rows = 0;
    *bytes = 0;
    if (row0 == fs->n_kept) return PG_OK;
    PG_CUDA(cudaSetDevice(ctx->device));
    pg_timings_reset(ctx);
    const int64_t nk = fs->n_kept;
    PG_CHECK(nk < (int64_t)INT32_MAX, "pg_filter_emit: %lld kept rows in one call (at most %d): ingest smaller chunks",
             (long long)nk, INT32_MAX - 1);
    EmitParams ep;
    PG_TRY(emit_params(ctx, fs, fmt, freq_order ? 1 : 0, ep));
    ep.p2m = fs->p2m;
    if (fs->emit_fmt != fmt || fs->emit_order != (freq_order ? 1 : 0)) {
        PG_TRY(ctx->flt_off.ensure((size_t)(nk + 1) * 8 * 2 + 64));
        int64_t* d_len = (int64_t*)ctx->flt_off.p + (nk + 1);
        int64_t* d_off = (int64_t*)ctx->flt_off.p;
        PG_CUDA(cudaMemsetAsync(d_len + nk, 0, 8, ctx->stream));
        ep.row0 = 0;
        ep.nrows = nk;
        ep.len = d_len;
        const int ti = pg_time_begin(ctx, "filter_emit_len");
        k_filter_emit<false><<<(unsigned)std::min<int64_t>((nk + 7) / 8, (int64_t)ctx->sm_count * 32), 256, 0, ctx->stream>>>(ep);
        pg_time_end(ctx, ti);
        PG_CUDA(cudaGetLastError());
        size_t tmp = 0;
        PG_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tmp, d_len, d_off, (int)(nk + 1), ctx->stream));
        PG_TRY(ctx->flt_cub.ensure(tmp + 64));
        PG_CUDA(cub::DeviceScan::ExclusiveSum(ctx->flt_cub.p, tmp, d_len, d_off, (int)(nk + 1), ctx->stream));
        fs->off.resize((size_t)nk + 1);
        PG_CUDA(cudaMemcpyAsync(fs->off.data(), d_off, (size_t)(nk + 1) * 8, cudaMemcpyDeviceToHost, ctx->stream));
        PG_CUDA(cudaStreamSynchronize(ctx->stream));
        fs->emit_fmt = fmt;
        fs->emit_order = freq_order ? 1 : 0;
        ctx->launches += 2;
    }
    // rows that fit: off[row1] - off[row0] <= cap
    const int64_t base = fs->off[(size_t)row0];
    const int64_t row1 = (int64_t)(std::upper_bound(fs->off.begin() + row0, fs->off.end(), base + (int64_t)cap) - fs->off.begin()) - 1;
    PG_CHECK(row1 > row0, "pg_filter_emit: row %lld needs %lld bytes, more than the %zu of the buffer", (long long)row0,
             (long long)(fs->off[(size_t)row0 + 1] - base), cap);
    const size_t nb = (size_t)(fs->off[(size_t)row1] - base);
    PG_TRY(ctx->flt_out.ensure(nb + 64));
    ep.row0 = row0;
    ep.nrows = row1 - row0;
    ep.off = (const int64_t*)ctx->flt_off.p;
    ep.out = (char*)ctx->flt_out.p;
    {
        const int ti = pg_time_begin(ctx, "filter_emit");
        k_filter_emit<true><<<(unsigned)std::min<int64_t>((ep.nrows + 7) / 8, (int64_t)ctx->sm_count * 32), 256, 0, ctx->stream>>>(ep);
        pg_time_end(ctx, ti);
        PG_CUDA(cudaGetLastError());
    }
    ctx->launches += 1;
    PG_CUDA(cudaMemcpyAsync(out, ctx->flt_out.p, nb, cudaMemcpyDeviceToHost, ctx->stream));
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    *rows = row1 - row0;
    *bytes = nb;
    return PG_OK;
}

extern "C" int pg_filter_stats(pg_ctx* ctx, int64_t site0, int64_t n, int32_t* called, int32_t* het, int32_t* counts,
                               int32_t* pop_called, uint8_t* pop_mask, uint8_t* flags, uint8_t* keep, uint8_t* final_) {
    PG_CHECK(ctx != nullptr, "pg_filter_stats: null ctx");
    FiltState* fs = state(ctx);
    PG_CHECK(fs->S == ctx->S, "pg_filter_stats: no pg_filter on the resident sites");
    PG_CHECK(site0 >= 0 && n >= 0 && site0 + n <= fs->S, "pg_filter_stats: sites out of range");
    if (n == 0) return PG_OK;
    PG_CUDA(cudaSetDevice(ctx->device));
    StatsView st;
    stats_layout(ctx->flt_stats.p, fs->S, fs->P, &st);
    const int P = fs->P;
    auto get = [&](void* dst, const void* src, size_t bytes) {
        return dst ? (int)cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, ctx->stream) : 0;
    };
    int e = 0;
    e |= get(called, st.called + site0, (size_t)n * 4);
    e |= get(het, st.het + site0, (size_t)n * 4);
    e |= get(counts, st.cnt + site0 * 4, (size_t)n * 16);
    if (P) {
        e |= get(pop_called, st.pcalled + site0 * P, (size_t)n * P * 4);
        e |= get(pop_mask, st.pmask + site0 * P, (size_t)n * P);
    }
    e |= get(flags, st.flags + site0, (size_t)n);
    e |= get(keep, st.keep + site0, (size_t)n);
    e |= get(final_, st.fin + site0, (size_t)n);
    PG_CHECK(e == 0, "pg_filter_stats: device copy failed");
    PG_CUDA(cudaStreamSynchronize(ctx->stream));
    return PG_OK;
}
