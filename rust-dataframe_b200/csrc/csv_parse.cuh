// csv_parse.cuh -- field-level rules of the CSV reader (k_csv.cu): unquoting, schema classification, and the integer, float and
// boolean grammars with their conversions.  Device code in the library; the same source compiles as plain C++ so the conversions
// can be checked against the C library on the host.
//
// Floats: a field is lexed into (sign, w, q, ...) with w the first 19 significant digits and value = w * 10^q when nothing
// non-zero was dropped.  Eisel-Lemire (a 128-bit product with the powers of five of csv_pow5.cuh) then rounds w * 10^q to the
// target format directly -- float32 is never rounded through float64.  It reports failure where the truncated product cannot
// decide the rounding; with more than 19 significant digits, w and w + 1 must round alike.  Undecided fields go to the exact
// slow path of the caller.
#pragma once
#include <stdint.h>

#include "csv_pow5.cuh"

#ifdef __CUDACC__
#define CSV_FN __device__ __forceinline__
#else
#define CSV_FN inline
#endif

namespace csv {

// Raw field bytes [p, e) (no delimiter or terminator) -> the bytes of the field value.  A field that starts with '"' is
// quoted: "" inside it is one '"', a lone '"' closes it, and whatever follows the close up to the end is appended literally
// ("ab"cd -> abcd).  Any other field is literal, quotes included.
struct Unquote {
    const uint8_t* p;
    const uint8_t* e;
    int st;   // 0 literal, 1 inside quotes, 2 just after a quote inside quotes
    CSV_FN Unquote(const uint8_t* b, const uint8_t* end) : p(b), e(end), st(0) {
        if (p < e && *p == '"') { st = 1; p++; }
    }
    CSV_FN int next() {
        while (p < e) {
            const uint8_t b = *p++;
            if (st == 0) return b;
            if (st == 1) {
                if (b == '"') { st = 2; continue; }
                return b;
            }
            if (b == '"') { st = 1; return '"'; }
            st = 0;
            return b;
        }
        return -1;
    }
};

// inference classes (bits, OR-ed per column)
enum { kEmpty = 1, kBool = 2, kInt = 4, kDec = 8, kOther = 16 };

CSV_FN int lower(int c) { return (c >= 'A' && c <= 'Z') ? c + 32 : c; }

// The class of one field: empty (a null), then `starts with "` -> Utf8, (?i)^(true|false)$, ^-?\d+\.\d+$, ^-?\d+$, else Utf8.
// \d is ASCII 0-9 here (Rust's regex \d is Unicode-aware: a documented departure).
CSV_FN int classify(Unquote u) {
    int c = u.next();
    if (c < 0) return kEmpty;
    if (c == '"') return kOther;
    char b[5];   // the first five characters, lower-cased
    int n = 0;
    int num = 0;   // 0 start, 1 after '-', 2 integer digits, 3 after '.', 4 fraction digits, 5 no number
    for (; c >= 0; c = u.next()) {
        if (n < 5) b[n] = (char)lower(c);
        n++;
        const bool d = c >= '0' && c <= '9';
        switch (num) {
            case 0: num = c == '-' ? 1 : d ? 2 : 5; break;
            case 1: num = d ? 2 : 5; break;
            case 2: num = d ? 2 : c == '.' ? 3 : 5; break;
            case 3: case 4: num = d ? 4 : 5; break;
            default: break;
        }
        if (num == 5 && n > 5) return kOther;
    }
    if (n == 4 && b[0] == 't' && b[1] == 'r' && b[2] == 'u' && b[3] == 'e') return kBool;
    if (n == 5 && b[0] == 'f' && b[1] == 'a' && b[2] == 'l' && b[3] == 's' && b[4] == 'e') return kBool;
    return num == 4 ? kDec : num == 2 ? kInt : kOther;
}

// ---- integers: [+-]?[0-9]+ (Rust FromStr); unsigned types refuse '-' (even -0); overflow is an error -----------------------
// dtype: 0 i8, 1 i16, 2 i32, 3 i64, 4 u8, 5 u16, 6 u32, 7 u64.  Returns false on a syntax error or overflow.
CSV_FN bool parse_int(Unquote u, int dtype, uint64_t* out) {
    int c = u.next();
    bool neg = false;
    if (c == '+' || c == '-') { neg = c == '-'; c = u.next(); }
    if (c < 0) return false;
    const bool is_unsigned = dtype >= 4;
    if (neg && is_unsigned) return false;
    uint64_t mag = 0;
    bool over = false;
    for (; c >= 0; c = u.next()) {
        if (c < '0' || c > '9') return false;
        const uint64_t d = (uint64_t)(c - '0');
        if (mag > (0xffffffffffffffffull - d) / 10) over = true;
        else mag = mag * 10 + d;
    }
    if (over) return false;
    const int bits = 8 << (dtype & 3);
    if (is_unsigned) {
        if (bits < 64 && mag > ((1ull << bits) - 1)) return false;
        *out = mag;
        return true;
    }
    const uint64_t lim = 1ull << (bits - 1);   // |min|
    if (neg ? mag > lim : mag > lim - 1) return false;
    *out = neg ? (uint64_t)0 - mag : mag;
    return true;
}

// ---- booleans: to_lowercase() == "true" / "false" ---------------------------------------------------------------------------
CSV_FN bool parse_bool(Unquote u, bool* out) {
    char b[6];
    int n = 0;
    for (int c = u.next(); c >= 0; c = u.next()) {
        if (n == 5) return false;
        b[n++] = (char)lower(c);
    }
    if (n == 4 && b[0] == 't' && b[1] == 'r' && b[2] == 'u' && b[3] == 'e') { *out = true; return true; }
    if (n == 5 && b[0] == 'f' && b[1] == 'a' && b[2] == 'l' && b[3] == 's' && b[4] == 'e') { *out = false; return true; }
    return false;
}

// ---- floats --------------------------------------------------------------------------------------------------------------
struct FloatFormat {
    int mbits, min_exp, inf_pow, min_rte, max_rte, min_p10, max_p10;
};
#define CSV_F64 ::csv::FloatFormat{52, -1023, 0x7FF, -4, 23, -342, 308}
#define CSV_F32 ::csv::FloatFormat{23, -127, 0xFF, -17, 10, -65, 38}

struct U128 { uint64_t hi, lo; };

CSV_FN U128 mul64(uint64_t a, uint64_t b) {
#ifdef __CUDA_ARCH__
    return U128{__umul64hi(a, b), a * b};
#else
    const unsigned __int128 p = (unsigned __int128)a * b;
    return U128{(uint64_t)(p >> 64), (uint64_t)p};
#endif
}

CSV_FN int clz64(uint64_t x) {
#ifdef __CUDA_ARCH__
    return __clzll((long long)x);
#else
    return __builtin_clzll(x);
#endif
}

// w * 10^q rounded to nearest-even in format F: biased exponent in *power2 and the explicit mantissa bits; false = undecided.
CSV_FN bool eisel_lemire(const FloatFormat F, int64_t q, uint64_t w, uint64_t* mant, int* power2) {
    if (w == 0 || q < F.min_p10) { *mant = 0; *power2 = 0; return true; }
    if (q > F.max_p10) { *mant = 0; *power2 = F.inf_pow; return true; }
    const int lz = clz64(w);
    w <<= lz;
    const int idx = 2 * (int)(q - kPow5MinQ);
    U128 p = mul64(w, kPow5Table[idx]);
    const uint64_t mask = 0xffffffffffffffffull >> (F.mbits + 3);
    if ((p.hi & mask) == mask) {   // the low bits of the high word are all ones: the second word can carry into them
        const U128 p2 = mul64(w, kPow5Table[idx + 1]);
        p.lo += p2.hi;
        if (p2.hi > p.lo) p.hi++;
    }
    if (p.lo == 0xffffffffffffffffull && (q < -27 || q > 55)) return false;   // the truncated product cannot decide
    const int upper = (int)(p.hi >> 63);
    const int shift = upper + 64 - F.mbits - 3;
    uint64_t m = p.hi >> shift;
    int e = (int)(((((152170 + 65536) * (int32_t)q) >> 16) + 63) + upper - lz - F.min_exp);
    if (e <= 0) {   // subnormal (or rounds up to the smallest normal)
        if (-e + 1 >= 64) { *mant = 0; *power2 = 0; return true; }
        m >>= -e + 1;
        m += m & 1;
        m >>= 1;
        *power2 = m < (1ull << F.mbits) ? 0 : 1;
        *mant = m & ((1ull << F.mbits) - 1);
        return true;
    }
    // exactly halfway between two floats (only possible where 5^q fits the product exactly): round to even
    if (p.lo <= 1 && q >= F.min_rte && q <= F.max_rte && (m & 3) == 1 && (m << shift) == p.hi) m &= ~1ull;
    m += m & 1;
    m >>= 1;
    if (m >= (2ull << F.mbits)) { m = 1ull << F.mbits; e++; }
    m &= ~(1ull << F.mbits);
    if (e >= F.inf_pow) { m = 0; e = F.inf_pow; }
    *mant = m;
    *power2 = e;
    return true;
}

enum { kFloatOk = 0, kFloatBad = 1, kFloatSlow = 2 };

// Rust's f32 / f64 FromStr grammar: [+-]? (digits [. digits?] | . digits) ([eE] [+-]? digits)?, or inf / infinity / nan in any
// case.  Returns kFloatOk with the bits, kFloatBad for a syntax error, kFloatSlow when the rounding must be decided exactly.
CSV_FN int parse_float(Unquote u, const FloatFormat F, uint64_t* bits) {
    const int sign_shift = F.mbits == 52 ? 63 : 31;
    int c = u.next();
    uint64_t neg = 0;
    if (c == '+' || c == '-') { neg = c == '-'; c = u.next(); }
    if (c < 0) return kFloatBad;
    const int l0 = lower(c);
    if (l0 == 'i' || l0 == 'n') {   // inf, infinity, nan
        char b[9];
        int n = 0;
        for (; c >= 0; c = u.next()) {
            if (n == 8) return kFloatBad;
            b[n++] = (char)lower(c);
        }
        const bool inf3 = n >= 3 && b[0] == 'i' && b[1] == 'n' && b[2] == 'f';
        const bool inf8 = n == 8 && inf3 && b[3] == 'i' && b[4] == 'n' && b[5] == 'i' && b[6] == 't' && b[7] == 'y';
        const bool nan = n == 3 && b[0] == 'n' && b[1] == 'a' && b[2] == 'n';
        if (!((inf3 && n == 3) || inf8 || nan)) return kFloatBad;
        const uint64_t exp_all = (uint64_t)F.inf_pow << F.mbits;
        *bits = (neg << sign_shift) | exp_all | (nan ? 1ull << (F.mbits - 1) : 0);
        return kFloatOk;
    }
    uint64_t w = 0;
    int nd = 0;             // significant digits kept in w (at most 19)
    int64_t q = 0;          // value = w * 10^q (+ the dropped digits)
    bool dropped = false;   // a non-zero digit did not fit in w
    int digits = 0;         // digits of the mantissa, significant or not
    for (; c >= '0' && c <= '9'; c = u.next(), digits++) {
        const int d = c - '0';
        if (w == 0 && d == 0) continue;
        if (nd < 19) { w = w * 10 + d; nd++; }
        else { q++; dropped |= d != 0; }
    }
    if (c == '.') {
        c = u.next();
        for (; c >= '0' && c <= '9'; c = u.next(), digits++) {
            const int d = c - '0';
            if (w == 0 && d == 0) { q--; continue; }
            if (nd < 19) { w = w * 10 + d; nd++; q--; }
            else dropped |= d != 0;
        }
    }
    if (digits == 0) return kFloatBad;
    if (c == 'e' || c == 'E') {
        c = u.next();
        bool eneg = false;
        if (c == '+' || c == '-') { eneg = c == '-'; c = u.next(); }
        if (!(c >= '0' && c <= '9')) return kFloatBad;
        int64_t ev = 0;
        for (; c >= '0' && c <= '9'; c = u.next()) ev = ev < 100000000 ? ev * 10 + (c - '0') : ev;   // saturates far out of range
        q += eneg ? -ev : ev;
    }
    if (c >= 0) return kFloatBad;
    if (q < -100000000) q = -100000000;
    if (q > 100000000) q = 100000000;
    uint64_t m;
    int e;
    if (!eisel_lemire(F, q, w, &m, &e)) return kFloatSlow;
    if (dropped) {   // the exact value lies strictly between w and w + 1 (times 10^q): both must round alike
        uint64_t m2;
        int e2;
        if (!eisel_lemire(F, q, w + 1, &m2, &e2) || m2 != m || e2 != e) return kFloatSlow;
    }
    *bits = (neg << sign_shift) | ((uint64_t)e << F.mbits) | m;
    return kFloatOk;
}

}  // namespace csv
