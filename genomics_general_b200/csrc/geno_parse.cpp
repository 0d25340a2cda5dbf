// Host-side .geno text tokenizer -> int8 genotype matrix (multi-threaded, no CUDA).
//
// Replaces parseGenoLine / GenoFileReader (genomics.py:1884-1945) + splitSeq/haplo/forceHomo
// (genomics.py:390-396, 27, 407) + seqArrayToNumArray (genomics.py:74-77) for a whole file at once:
//   line   := scaffold WS position WS token (WS token)*        ('#' lines and blank lines are skipped)
//   phased : alleles are the characters 0,2,4.. of the token   ("A|T", "A/N", "G")
//   pairs  : two letters, no separator                          ("AT")
//   diplo  : one IUPAC letter -> two alleles via DIPLOTYPES/PAIRS (genomics.py:14-15)
//   haplo  : one letter
// Output haplotypes of sample k occupy columns hap_off[k] .. hap_off[k]+ploidy[k]-1 (file/sample order).
// Bases: A0 C1 G2 T3, anything else = missing (-1).  (The reference leaves non-ACGTN letters as
// uninitialised memory, genomics.py:75; here they are missing.)  A sample declared haploid keeps only
// homozygous calls (forceHomo, genomics.py:407 + HOMOTYPES).
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <string>
#include <thread>
#include <vector>

#include "../../include/pgwin.h"

void pg_set_error(const char* fmt, ...);

namespace {

inline bool is_ws(char c) { return c == ' ' || c == '\t' || c == '\r' || c == '\v' || c == '\f'; }

struct Lut {
    int8_t base[256];
    int8_t dip0[256], dip1[256];
    uint8_t ws[256];
    Lut() {
        for (int i = 0; i < 256; ++i) {
            base[i] = dip0[i] = dip1[i] = -1;
            ws[i] = is_ws((char)i) ? 1 : 0;
        }
        base[(int)'A'] = 0;
        base[(int)'C'] = 1;
        base[(int)'G'] = 2;
        base[(int)'T'] = 3;
        const char* d = "ACGKMNSRTWY";
        const char* p[] = {"AA", "CC", "GG", "GT", "AC", "NN", "CG", "AG", "TT", "AT", "CT"};
        for (int i = 0; d[i]; ++i) {
            dip0[(int)d[i]] = base[(int)p[i][0]];
            dip1[(int)d[i]] = base[(int)p[i][1]];
        }
    }
};
const Lut LUT;

// data lines start offsets inside [begin, end)
void index_lines(const char* buf, size_t begin, size_t end, std::vector<size_t>& starts) {
    size_t i = begin;
    while (i < end) {
        const char* nl = (const char*)memchr(buf + i, '\n', end - i);
        size_t e = nl ? (size_t)(nl - buf) : end;
        size_t j = i;
        while (j < e && is_ws(buf[j])) ++j;
        if (j < e && buf[i] != '#') starts.push_back(i);
        i = e + 1;
    }
}

// the same over the whole buffer with several threads: a line belongs to the thread whose byte range holds its first byte
void index_lines_parallel(const char* buf, size_t len, int n_threads, std::vector<size_t>& starts) {
    if (n_threads < 2 || len < ((size_t)1 << 22)) {
        index_lines(buf, 0, len, starts);
        return;
    }
    std::vector<std::vector<size_t>> part((size_t)n_threads);
    auto work = [&](int t) {
        size_t b = len * (size_t)t / (size_t)n_threads, e = len * (size_t)(t + 1) / (size_t)n_threads;
        if (t > 0 && buf[b - 1] != '\n') {            // the line that straddles the boundary belongs to the previous thread
            const char* nl = (const char*)memchr(buf + b, '\n', len - b);
            b = nl ? (size_t)(nl - buf) + 1 : len;
        }
        // index_lines stops at `end`; lines that START before e are wanted in full, so scan line by line here
        size_t i = b;
        while (i < e) {
            const char* nl = (const char*)memchr(buf + i, '\n', len - i);
            const size_t le = nl ? (size_t)(nl - buf) : len;
            size_t j = i;
            while (j < le && is_ws(buf[j])) ++j;
            if (j < le && buf[i] != '#') part[(size_t)t].push_back(i);
            i = le + 1;
        }
    };
    std::vector<std::thread> th;
    for (int t = 1; t < n_threads; ++t) th.emplace_back(work, t);
    work(0);
    for (auto& x : th) x.join();
    size_t total = 0;
    for (auto& v : part) total += v.size();
    starts.reserve(starts.size() + total);
    for (auto& v : part) starts.insert(starts.end(), v.begin(), v.end());
}

int default_threads() {
    const unsigned hc = std::thread::hardware_concurrency();
    return (int)std::max(1u, std::min(16u, hc / 2));
}

}  // namespace

extern "C" int pg_geno_count_lines(const char* buf, size_t len, int64_t* n) {
    if (!buf || !n) {
        pg_set_error("pg_geno_count_lines: null argument");
        return 1;
    }
    std::vector<size_t> st;
    index_lines_parallel(buf, len, default_threads(), st);
    *n = (int64_t)st.size();
    return 0;
}

// fmt: 0 phased, 1 diplo, 2 pairs, 3 haplo
extern "C" int pg_geno_parse(const char* buf, size_t len, int32_t fmt, int32_t n_out, const int32_t* col_take,
                             const int8_t* ploidy, int32_t H_out, int64_t n_lines, int8_t* geno, int32_t* pos,
                             int8_t* new_scaffold, int64_t* line_off, int32_t n_threads) {
    if (!buf || !col_take || !ploidy || !geno || !pos || !new_scaffold || !line_off) {
        pg_set_error("pg_geno_parse: null argument");
        return 1;
    }
    if (fmt < 0 || fmt > 3) {
        pg_set_error("pg_geno_parse: unknown format %d", fmt);
        return 1;
    }
    std::vector<size_t> starts;
    starts.reserve((size_t)n_lines + 1);
    index_lines_parallel(buf, len, n_threads > 0 ? n_threads : default_threads(), starts);
    if ((int64_t)starts.size() != n_lines) {
        pg_set_error("pg_geno_parse: buffer holds %lld data lines, caller allocated %lld", (long long)starts.size(),
                     (long long)n_lines);
        return 1;
    }
    int max_col = -1;
    std::vector<int32_t> hap_off(n_out, 0);
    {
        int off = 0;
        for (int k = 0; k < n_out; ++k) {
            hap_off[k] = off;
            off += ploidy[k];
            if (col_take[k] > max_col) max_col = col_take[k];
            if (ploidy[k] < 1 || ploidy[k] > 8) {
                pg_set_error("pg_geno_parse: ploidy %d of sample %d unsupported", (int)ploidy[k], k);
                return 1;
            }
        }
        if (off != H_out) {
            pg_set_error("pg_geno_parse: ploidies sum to %d, H_out is %d", off, H_out);
            return 1;
        }
    }
    // file column -> list of outputs (a column may be requested once)
    std::vector<int32_t> col_to_out(max_col + 1, -1);
    for (int k = 0; k < n_out; ++k) {
        if (col_take[k] < 0) {
            pg_set_error("pg_geno_parse: negative column index");
            return 1;
        }
        col_to_out[col_take[k]] = k;
    }
    int uniform_ploidy = n_out > 0 ? ploidy[0] : 0;     // 0 = mixed
    for (int k = 1; k < n_out; ++k)
        if (ploidy[k] != uniform_ploidy) uniform_ploidy = 0;
    if (n_threads < 1) n_threads = 1;
    if ((int64_t)n_threads > n_lines) n_threads = (int)(n_lines > 0 ? n_lines : 1);
    std::atomic<int> failed(0);
    std::string err;
    std::vector<std::string> errs(n_threads);

    auto work = [&](int t) {
        const int64_t l0 = n_lines * t / n_threads, l1 = n_lines * (t + 1) / n_threads;
        for (int64_t l = l0; l < l1 && !failed.load(std::memory_order_relaxed); ++l) {
            const char* p = buf + starts[l];
            const char* e = (const char*)memchr(p, '\n', len - starts[l]);
            if (!e) e = buf + len;
            line_off[l] = (int64_t)starts[l];
            while (p < e && is_ws(*p)) ++p;
            const char* sc0 = p;
            while (p < e && !is_ws(*p)) ++p;
            const char* sc1 = p;
            // new scaffold flag: compare with the previous data line's first field
            if (l == 0) new_scaffold[l] = 1;
            else {
                const char* q = buf + starts[l - 1];
                while (is_ws(*q)) ++q;
                const char* q1 = q;
                while (!is_ws(*q1) && *q1 != '\n') ++q1;
                new_scaffold[l] = ((q1 - q) != (sc1 - sc0) || memcmp(q, sc0, (size_t)(sc1 - sc0)) != 0) ? 1 : 0;
            }
            while (p < e && is_ws(*p)) ++p;
            if (p >= e) {
                char b[160];
                snprintf(b, sizeof(b), "data line %lld: no position field", (long long)l + 1);
                errs[t] = b;
                failed.store(1);
                return;
            }
            // position: an optional sign and leading digits (the rest of the field is skipped); it must fit in int32
            bool neg = false;
            if (*p == '-' || *p == '+') {
                neg = (*p == '-');
                ++p;
            }
            if (p >= e || *p < '0' || *p > '9') {
                char b[160];
                snprintf(b, sizeof(b), "data line %lld: position is not an integer", (long long)l + 1);
                errs[t] = b;
                failed.store(1);
                return;
            }
            int64_t v = 0;
            while (p < e && *p >= '0' && *p <= '9') {
                if (v <= ((int64_t)1 << 31)) v = v * 10 + (*p - '0');    // past the limit the value stays out of range
                ++p;
            }
            if (v > ((int64_t)1 << 31) - (neg ? 0 : 1)) {
                char b[160];
                snprintf(b, sizeof(b), "data line %lld: position outside the int32 range", (long long)l + 1);
                errs[t] = b;
                failed.store(1);
                return;
            }
            while (p < e && !is_ws(*p)) ++p;
            pos[l] = (int32_t)(neg ? -v : v);
            int8_t* grow = geno + (size_t)l * H_out;
            int col = 0, found = 0;
            // fast path: every token has the same width and is followed by one blank (the normal layout of .geno files)
            // -> address the requested columns directly instead of tokenising the whole line
            {
                const char* q = p;
                while (q < e && is_ws(*q)) ++q;
                const char* e2 = e;
                while (e2 > q && is_ws(e2[-1])) --e2;
                const int tokw = (fmt == 0) ? 3 : (fmt == 2 ? 2 : 1);
                const long rem = (long)(e2 - q);
                bool fast = uniform_ploidy == ((fmt == 0 || fmt == 1 || fmt == 2) ? 2 : 1) && rem > 0 && ((rem + 1) % (tokw + 1)) == 0;
                if (fmt == 1 && uniform_ploidy == 1) fast = false;
                long ncols = fast ? (rem + 1) / (tokw + 1) : 0;
                if (fast && max_col >= ncols) fast = false;
                if (fast) {
                    // the grid is the whitespace split only when every separator is one blank and no token byte is blank
                    // (branch-free over the line: one table load per byte)
                    const unsigned char* u = (const unsigned char*)q;
                    unsigned bad = 0;
                    for (long c2 = 0; c2 < ncols; ++c2, u += tokw + 1) {
                        for (int j = 0; j < tokw; ++j) bad |= LUT.ws[u[j]];
                        if (c2 + 1 < ncols) bad |= LUT.ws[u[tokw]] ^ 1u;
                    }
                    fast = bad == 0;
                }
                if (fast) {
                    for (int k = 0; k < n_out; ++k) {
                        const char* t0 = q + (long)col_take[k] * (tokw + 1);
                        int8_t* o = grow + hap_off[k];
                        if (fmt == 0) {
                            o[0] = LUT.base[(unsigned char)t0[0]];
                            o[1] = LUT.base[(unsigned char)t0[2]];
                        } else if (fmt == 2) {
                            o[0] = LUT.base[(unsigned char)t0[0]];
                            o[1] = LUT.base[(unsigned char)t0[1]];
                        } else if (fmt == 1) {
                            o[0] = LUT.dip0[(unsigned char)t0[0]];
                            o[1] = LUT.dip1[(unsigned char)t0[0]];
                        } else {
                            o[0] = LUT.base[(unsigned char)t0[0]];
                        }
                    }
                    continue;
                }
            }
            while (p < e) {
                while (p < e && is_ws(*p)) ++p;
                if (p >= e) break;
                const char* t0 = p;
                while (p < e && !is_ws(*p)) ++p;
                const int tl = (int)(p - t0);
                if (col <= max_col && col_to_out[col] >= 0) {
                    const int k = col_to_out[col];
                    const int pl = ploidy[k];
                    int8_t* o = grow + hap_off[k];
                    // alleles in the token: every other character (phased), every character (pairs), two (diplo), one (haplo)
                    const int nall = fmt == 0 ? (tl + 1) / 2 : (fmt == 2 ? tl : (fmt == 1 ? 2 : 1));
                    if (pl == 1 && fmt == 1) {
                        // forceHomo (genomics.py:407): keep homozygous calls only
                        const int8_t a0 = LUT.dip0[(unsigned char)t0[0]], a1 = LUT.dip1[(unsigned char)t0[0]];
                        o[0] = (a0 == a1) ? a0 : (int8_t)-1;
                    } else if (nall != pl) {
                        char b[200];
                        snprintf(b, sizeof(b), "data line %lld, genotype column %d: token has %d alleles, sample ploidy is %d "
                                 "(genomics.py:1111 asserts the same)", (long long)l + 1, col + 1, nall, pl);
                        errs[t] = b;
                        failed.store(1);
                        return;
                    } else {
                        for (int a = 0; a < pl; ++a) {
                            const unsigned char c = (unsigned char)t0[fmt == 0 ? 2 * a : (fmt == 2 ? a : 0)];
                            o[a] = fmt == 1 ? (a == 0 ? LUT.dip0[c] : LUT.dip1[c]) : LUT.base[c];
                        }
                    }
                    ++found;
                }
                ++col;
            }
            if (found != n_out) {
                char b[160];
                snprintf(b, sizeof(b), "data line %lld: %d genotype columns, %d requested samples found", (long long)l + 1,
                         col, found);
                errs[t] = b;
                failed.store(1);
                return;
            }
        }
    };
    if (n_threads == 1) work(0);
    else {
        std::vector<std::thread> th;
        for (int t = 0; t < n_threads; ++t) th.emplace_back(work, t);
        for (auto& x : th) x.join();
    }
    if (failed.load()) {
        for (auto& s : errs)
            if (!s.empty()) {
                pg_set_error("pg_geno_parse: %s", s.c_str());
                break;
            }
        return 1;
    }
    return 0;
}
