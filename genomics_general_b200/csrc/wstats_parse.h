// windowStats' decimal parser: one token of ASCII text -> binary64, correctly rounded, under Python's float() grammar
//   [+-]? ( inf | infinity | nan )                          (any case)
//   [+-]? ( digits [ . [digits] ] | . digits ) [ (e|E) [+-]? digits ]
//   digits := [0-9] ( _? [0-9] )*                          (PEP 515 underscores: single, between two digits)
// The significand's first 19 significant digits become w (exact in uint64) and the decimal exponent q.  Two exact paths:
//   Clinger (1990): w <= 2^53 and |q| <= 22 -> one IEEE multiplication or division of exact operands;
//   Eisel-Lemire (Lemire 2021): w normalised to 64 bits times the 128 leading bits of 5^q (pow5_128.h, truncated), the top 54
//   bits rounded to 53.  It gives up (PG_WS_HOST) where the truncated product cannot decide: the 9 bits below the kept ones
//   all ones with a carry possible, a result that is subnormal, or a possible exact halfway case (q in [-27, 23] only).
// More than 19 significant digits: w and w + 1 bracket the value, and a result stands only when both give the same double.
// Tokens neither path settles are resolved on the host with float(); the count is small and reported under --timing.
#pragma once
#include <stdint.h>
#include <string.h>

#include "pow5_128.h"

#ifndef __CUDACC__
#define __host__
#define __device__
#define __forceinline__ inline
#endif

enum { PG_WS_OK = 0, PG_WS_BAD = 1, PG_WS_HOST = 2 };

namespace pgws {

__host__ __device__ __forceinline__ void mul64(uint64_t a, uint64_t b, uint64_t* hi, uint64_t* lo) {
#ifdef __CUDA_ARCH__
    *lo = a * b;
    *hi = __umul64hi(a, b);
#else
    const unsigned __int128 p = (unsigned __int128)a * b;
    *lo = (uint64_t)p;
    *hi = (uint64_t)(p >> 64);
#endif
}

__host__ __device__ __forceinline__ int clz64(uint64_t x) {
#ifdef __CUDA_ARCH__
    return __clzll((long long)x);
#else
    return __builtin_clzll(x);
#endif
}

__host__ __device__ __forceinline__ double from_bits(uint64_t b) {
    double d;
    memcpy(&d, &b, 8);
    return d;
}

// w * 10^q, w != 0: the double's bits, or -1 when the product cannot decide
__host__ __device__ __forceinline__ int64_t eisel_lemire(uint64_t w, int q, const uint64_t (*pow5)[2]) {
    if (q < PG_POW5_QMIN) return 0;                                  // below half the least subnormal
    if (q > PG_POW5_QMAX) return (int64_t)0x7ff0000000000000ll;      // inf
    const int l = clz64(w);
    w <<= l;
    const uint64_t thi = pow5[q - PG_POW5_QMIN][0], tlo = pow5[q - PG_POW5_QMIN][1];
    uint64_t zh, zl, yh, yl;
    mul64(w, thi, &zh, &zl);
    mul64(w, tlo, &yh, &yl);
    zl += yh;
    zh += zl < yh;
    // z <= the exact product < z + w (units of z): a carry into the kept bits is possible only through 9 bits of ones
    if ((zh & 0x1ff) == 0x1ff && zl + w < zl) return -1;
    const int upper = (int)(zh >> 63);
    uint64_t m = zh >> (upper + 9);                                  // 54 bits: 53 and the rounding bit
    const int e2 = ((q * 217706) >> 16) + upper + 10 - l;            // floor(q log2 10) + ...: the value is ~ m * 2^e2
    int be = e2 + 1076;                                              // biased exponent of the rounded 53-bit significand
    if (be <= 0) return -1;                                          // subnormal: the host decides
    if ((m & 1) && zl == 0 && (zh & ((1ull << (upper + 9)) - 1)) == 0 && q >= -27 && q <= 23) return -1;   // maybe a tie
    m = (m + 1) >> 1;
    if (m >> 53) {
        m >>= 1;
        ++be;
    }
    if (be >= 2047) return (int64_t)0x7ff0000000000000ll;
    return (int64_t)(((uint64_t)be << 52) | (m & ((1ull << 52) - 1)));
}

// bytes [t, t + n) -> *out; PG_WS_OK, PG_WS_BAD (float() raises) or PG_WS_HOST (valid, the host rounds it)
__host__ __device__ __forceinline__ int parse_double(const uint8_t* t, int n, const uint64_t (*pow5)[2], double* out) {
    int i = 0;
    bool neg = false;
    *out = 0.0;
    if (i < n && (t[i] == '+' || t[i] == '-')) neg = t[i++] == '-';
    if (i < n && !(t[i] >= '0' && t[i] <= '9') && t[i] != '.') {     // inf, infinity, nan
        const char* words[3] = {"inf", "infinity", "nan"};
        const int lens[3] = {3, 8, 3};
        for (int k = 0; k < 3; ++k) {
            if (n - i != lens[k]) continue;
            bool eq = true;
            for (int j = 0; j < lens[k]; ++j) eq &= (t[i + j] | 0x20u) == (unsigned)words[k][j];
            if (eq) {
                *out = k < 2 ? (neg ? -1.0 : 1.0) * from_bits(0x7ff0000000000000ull) : from_bits(0x7ff8000000000000ull);
                return PG_WS_OK;
            }
        }
        return PG_WS_BAD;
    }
    uint64_t w = 0;
    int nd = 0;                      // significant digits taken into w (at most 19)
    int64_t drop = 0;                // significant digits after the first 19 (each scales by 10)
    int64_t frac = 0;                // digits of w that lie after the point
    bool more = false;               // a nonzero digit was dropped
    bool any = false;
    for (int part = 0; part < 2; ++part) {                           // integer part, then fraction
        bool prev_digit = false;
        while (i < n) {
            const unsigned c = t[i];
            if (c >= '0' && c <= '9') {
                any = true;
                prev_digit = true;
                if (nd == 0 && c == '0') {
                    if (part == 1) ++frac;                           // a leading zero after the point
                } else if (nd < 19) {
                    w = w * 10 + (c - '0');
                    ++nd;
                    if (part == 1) ++frac;
                } else {
                    if (part == 0) ++drop;
                    more |= c != '0';
                }
                ++i;
            } else if (c == '_') {
                if (!prev_digit || i + 1 >= n || !(t[i + 1] >= '0' && t[i + 1] <= '9')) return PG_WS_BAD;
                prev_digit = false;
                ++i;
            } else {
                break;
            }
        }
        if (part == 0) {
            if (i < n && t[i] == '.') ++i;
            else break;
        }
    }
    if (!any) return PG_WS_BAD;
    int64_t ex = 0;
    if (i < n && (t[i] == 'e' || t[i] == 'E')) {
        ++i;
        bool eneg = false;
        if (i < n && (t[i] == '+' || t[i] == '-')) eneg = t[i++] == '-';
        bool ed = false, prev_digit = false;
        while (i < n) {
            const unsigned c = t[i];
            if (c >= '0' && c <= '9') {
                if (ex < 100000000) ex = ex * 10 + (c - '0');
                ed = prev_digit = true;
                ++i;
            } else if (c == '_' && prev_digit && i + 1 < n && t[i + 1] >= '0' && t[i + 1] <= '9') {
                prev_digit = false;
                ++i;
            } else {
                break;
            }
        }
        if (!ed) return PG_WS_BAD;
        if (eneg) ex = -ex;
    }
    if (i != n) return PG_WS_BAD;
    const double sgn = neg ? -1.0 : 1.0;
    if (w == 0) {
        *out = sgn * 0.0;
        return PG_WS_OK;
    }
    int64_t q64 = ex - frac + drop;
    if (q64 < -100000) q64 = -100000;
    if (q64 > 100000) q64 = 100000;
    const int q = (int)q64;
    if (!more && w <= (1ull << 53) && q >= -22 && q <= 22) {        // Clinger's fast path
        const double p10[23] = {1e0, 1e1, 1e2, 1e3, 1e4, 1e5, 1e6, 1e7, 1e8, 1e9, 1e10, 1e11, 1e12, 1e13, 1e14, 1e15, 1e16,
                                1e17, 1e18, 1e19, 1e20, 1e21, 1e22};
        const double d = (double)w;
        *out = sgn * (q >= 0 ? d * p10[q] : d / p10[-q]);
        return PG_WS_OK;
    }
    const int64_t b = eisel_lemire(w, q, pow5);
    if (b < 0) return PG_WS_HOST;
    if (more) {                                                      // the value lies in (w, w + 1) * 10^q
        const int64_t b1 = eisel_lemire(w + 1, q, pow5);
        if (b1 != b) return PG_WS_HOST;
    }
    *out = sgn * from_bits((uint64_t)b);
    return PG_WS_OK;
}

}  // namespace pgws
