// csv_format.cuh -- the text of one field of the CSV writer (k_csv_write.cu; the rules are in include/b200df.h):
// integers in plain decimal, booleans as true / false, floats as Rust's Display prints them -- the shortest digit string that
// reads back to the same value in its own type (the closest to the exact value among several), written positionally.
//
// Shortest digits: Schubfach (R. Giulietti, "The Schubfach way to render doubles", 2020; PAPERS.md).  With the value
// v = c * 2^q and k = floor(log10(2^q)) (floor(log10(3/4 * 2^q)) at the closer lower neighbour of a power of two), the rounding
// interval R of v is narrower than 10^(k+1) and wider than 10^k, so its shortest decimal is either the one multiple of 10^(k+1)
// inside R or one of s * 10^k, (s + 1) * 10^k with s = floor(v / 10^k).  v / 10^k and both interval ends are computed with
// one 64x128-bit product each (rop) against the table g ~ 10^-k of gen_csv_pow5.py, which decides every membership exactly.
// Giulietti's Java code asks for at least two digits (4.9E-324); Display wants the shortest (5e-324), so the multiple of
// 10^(k+1) is tried whenever s has two digits or more, and tiny subnormals need no scaling by 10.
// Everything here is plain integer arithmetic: compiled by a host compiler (with __device__ defined empty) it gives the same text,
// which is how it can be checked against Python on a machine without a GPU.
#pragma once

#include <stdint.h>

#include "csv_pow5.cuh"

namespace bdf {

#if defined(__CUDACC__)
#define CSVF __device__ __forceinline__
#else
#define CSVF inline
#endif

CSVF uint64_t csvf_mulhi(uint64_t a, uint64_t b) {
#if defined(__CUDACC__)
    return __umul64hi(a, b);
#else
    return (uint64_t)(((unsigned __int128)a * b) >> 64);
#endif
}
CSVF uint64_t csvf_g(int i) {
#if defined(__CUDACC__)
    return __ldg(kPow10G + i);
#else
    return kPow10G[i];
#endif
}

// floor(log10(2^q)), floor(log10(3/4 * 2^q)), floor(log2(10^e)): exact for |q| <= 1200 and |e| <= 400 (checked with integers)
CSVF int csvf_flog10pow2(int q) { return (int)(((int64_t)q * 661971961083LL) >> 41); }
CSVF int csvf_flog10tq(int q) { return (int)(((int64_t)q * 661971961083LL - 274743187321LL) >> 41); }
CSVF int csvf_flog2pow10(int e) { return (int)(((int64_t)e * 913124641741LL) >> 38); }

struct CsvDec { uint64_t f; int e; };   // f * 10^e

// Round to odd of g * cp / 2^127 (g = g1 2^63 + g0): the integer part with a sticky bit for any nonzero remainder.
CSVF uint64_t csvf_rop64(uint64_t g1, uint64_t g0, uint64_t cp) {
    const uint64_t x1 = csvf_mulhi(g0, cp);
    const uint64_t y0 = g1 * cp, y1 = csvf_mulhi(g1, cp);
    const uint64_t z = (y0 >> 1) + x1;
    const uint64_t vbp = y1 + (z >> 63);
    return vbp | (((z & 0x7fffffffffffffffull) + 0x7fffffffffffffffull) >> 63);
}
CSVF uint32_t csvf_rop32(uint64_t g, uint64_t cp) {
    const uint64_t x1 = csvf_mulhi(g, cp);
    return (uint32_t)((x1 >> 31) | (((x1 & 0xffffffffull) + 0xffffffffull) >> 32));
}

// The decision shared by both widths: vb, vbl, vbr are 4 v / 10^k and the interval ends, rounded to odd; out = 1 when the
// ends are excluded (odd c: round half to even reads them back to the neighbours).
template <typename U>
CSVF CsvDec csvf_choose(U vb, U vbl, U vbr, U out, int k) {
    const U s = vb >> 2;
    if (s >= 10) {
        const U sp10 = 10 * (s / 10), tp10 = sp10 + 10;
        const bool upin = vbl + out <= sp10 << 2, wpin = (tp10 << 2) + out <= vbr;
        if (upin != wpin) return CsvDec{upin ? (uint64_t)sp10 : (uint64_t)tp10, k};
    }
    const U t = s + 1;
    const bool uin = vbl + out <= s << 2, win = (t << 2) + out <= vbr;
    if (uin != win) return CsvDec{uin ? (uint64_t)s : (uint64_t)t, k};
    const U mid = (s + t) << 1;   // both inside: the closer, ties to even
    return CsvDec{(vb < mid || (vb == mid && (s & 1) == 0)) ? (uint64_t)s : (uint64_t)t, k};
}

// Shortest digits of a finite nonzero Float64 (the sign is ignored).
CSVF CsvDec csvf_shortest64(uint64_t bits) {
    const int bq = (int)((bits >> 52) & 0x7ff);
    const uint64_t frac = bits & ((1ull << 52) - 1);
    const int q = bq ? bq - 1075 : -1074;
    const uint64_t c = bq ? frac | (1ull << 52) : frac;
    const uint64_t out = c & 1, cb = c << 2, cbr = cb + 2;
    uint64_t cbl;
    int k;
    if (c != (1ull << 52) || bq == 1) { cbl = cb - 2; k = csvf_flog10pow2(q); }
    else { cbl = cb - 1; k = csvf_flog10tq(q); }   // a power of two: the lower neighbour is half as far
    const int h = q + csvf_flog2pow10(-k) + 2;
    const int i = 2 * (-k - kPow10GMinE);
    const uint64_t g1 = csvf_g(i), g0 = csvf_g(i + 1);
    return csvf_choose<uint64_t>(csvf_rop64(g1, g0, cb << h), csvf_rop64(g1, g0, cbl << h), csvf_rop64(g1, g0, cbr << h), out, k);
}

// Shortest digits of a finite nonzero Float32, as a Float32 (never through Float64).
CSVF CsvDec csvf_shortest32(uint32_t bits) {
    const int bq = (int)((bits >> 23) & 0xff);
    const uint32_t frac = bits & ((1u << 23) - 1);
    const int q = bq ? bq - 150 : -149;
    const uint64_t c = bq ? frac | (1u << 23) : frac;
    const uint32_t out = (uint32_t)(c & 1);
    const uint64_t cb = c << 2, cbr = cb + 2;
    uint64_t cbl;
    int k;
    if (c != (1u << 23) || bq == 1) { cbl = cb - 2; k = csvf_flog10pow2(q); }
    else { cbl = cb - 1; k = csvf_flog10tq(q); }
    const int h = q + csvf_flog2pow10(-k) + 33;
    const uint64_t g = csvf_g(2 * (-k - kPow10GMinE)) + 1;
    return csvf_choose<uint32_t>(csvf_rop32(g, cb << h), csvf_rop32(g, cbl << h), csvf_rop32(g, cbr << h), out, k);
}

CSVF int csvf_digits(uint64_t f) {   // decimal digits of f (1 for 0)
    int n = 1;
    uint64_t p = 10;
    while (n < 20 && f >= p) { n++; p *= 10; }
    return n;
}

// n digits of f ending at p + n, two at a time (a division by the constant 100 is a multiply-high and a shift).
CSVF void csvf_put_digits(char* p, uint64_t f, int n) {
    char* q = p + n;
    while (f >= 100) {
        const uint64_t d = f / 100;
        const uint32_t r = (uint32_t)(f - d * 100), hi = r / 10;
        q -= 2;
        q[0] = (char)('0' + hi);
        q[1] = (char)('0' + (r - hi * 10));
        f = d;
    }
    if (f >= 10) {
        const uint32_t r = (uint32_t)f, hi = r / 10;
        q -= 2;
        q[0] = (char)('0' + hi);
        q[1] = (char)('0' + (r - hi * 10));
    } else {
        q[-1] = (char)('0' + f);
    }
}

// A float field: NaN (any sign or payload), inf, -inf, 0, -0, or [-]digits positionally.
struct CsvFloat { uint64_t f; int e, n; bool neg; int special; };   // special: 0 number, 1 NaN, 2 inf, 3 zero

CSVF int csvf_float_len(const CsvFloat& x) {
    if (x.special == 1) return 3;
    if (x.special == 2) return 3 + x.neg;
    if (x.special == 3) return 1 + x.neg;
    const int d = x.n + x.e;   // digits before the point
    const int body = x.e >= 0 ? d : d > 0 ? x.n + 1 : 2 - d + x.n;
    return body + x.neg;
}

CSVF CsvFloat csvf_from_dec(CsvDec dd, bool neg) {
    uint64_t f = dd.f;
    int e = dd.e;
    while (f % 100000000 == 0) { f /= 100000000; e += 8; }
    if (f % 10000 == 0) { f /= 10000; e += 4; }
    if (f % 100 == 0) { f /= 100; e += 2; }
    if (f % 10 == 0) { f /= 10; e += 1; }
    return CsvFloat{f, e, csvf_digits(f), neg, 0};
}

CSVF CsvFloat csvf_f64(uint64_t bits) {
    const bool neg = bits >> 63;
    const uint64_t mag = bits & 0x7fffffffffffffffull;
    if (mag >= 0x7ff0000000000000ull) return CsvFloat{0, 0, 0, neg, mag == 0x7ff0000000000000ull ? 2 : 1};
    if (mag == 0) return CsvFloat{0, 0, 0, neg, 3};
    return csvf_from_dec(csvf_shortest64(mag), neg);
}
CSVF CsvFloat csvf_f32(uint32_t bits) {
    const bool neg = bits >> 31;
    const uint32_t mag = bits & 0x7fffffffu;
    if (mag >= 0x7f800000u) return CsvFloat{0, 0, 0, neg, mag == 0x7f800000u ? 2 : 1};
    if (mag == 0) return CsvFloat{0, 0, 0, neg, 3};
    return csvf_from_dec(csvf_shortest32(mag), neg);
}

// Writes csvf_float_len(x) bytes at p.
CSVF void csvf_float_put(const CsvFloat& x, char* p) {
    if (x.special == 1) { p[0] = 'N'; p[1] = 'a'; p[2] = 'N'; return; }
    if (x.neg) *p++ = '-';
    if (x.special == 2) { p[0] = 'i'; p[1] = 'n'; p[2] = 'f'; return; }
    if (x.special == 3) { p[0] = '0'; return; }
    const int d = x.n + x.e;
    if (x.e >= 0) {
        csvf_put_digits(p, x.f, x.n);
        for (int j = x.n; j < d; j++) p[j] = '0';
    } else if (d > 0) {   // the point inside the digits: write them, then open the gap
        csvf_put_digits(p, x.f, x.n);
        for (int j = x.n; j > d; j--) p[j] = p[j - 1];
        p[d] = '.';
    } else {
        p[0] = '0';
        p[1] = '.';
        for (int j = 0; j < -d; j++) p[2 + j] = '0';
        csvf_put_digits(p + 2 - d, x.f, x.n);
    }
}

// An integer field: [-]digits.
CSVF int csvf_int_len(uint64_t mag, bool neg) { return csvf_digits(mag) + neg; }
CSVF void csvf_int_put(uint64_t mag, bool neg, char* p) {
    if (neg) *p++ = '-';
    csvf_put_digits(p, mag, csvf_digits(mag));
}

}  // namespace bdf
