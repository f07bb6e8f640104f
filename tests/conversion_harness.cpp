// conversion_harness.cpp -- the CSV / JSON readers' float and integer parser (csv_parse.cuh) and the CSV writer's float formatter
// (csv_format.cuh), compiled for the host and driven through ctypes by tests/test_conversions.py.  Both headers are written to
// compile as plain C++ with __device__ defined empty, so their decisions can be checked here without a GPU.
//
// The checks of formatted text use nothing from the headers: glibc's strtof_l / strtod_l for the round trip (correctly rounded
// and independent of this code) and exact integer comparisons (Big below) for "shortest" and "closest".
#include <locale.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include <atomic>
#include <mutex>
#include <thread>
#include <vector>

#include "csv_format.cuh"
#include "csv_parse.cuh"

namespace {

locale_t c_locale() {
    static locale_t loc = newlocale(LC_ALL_MASK, "C", (locale_t)0);
    return loc;
}

// ---- exact comparison of d * 10^e10 with c * 2^e2 -------------------------------------------------------------------------
// N 64-bit limbs, little-endian.  Float32's operands stay below 2^210 (4 limbs), Float64's below 2^1200 (20 limbs).
template <int N>
struct Big {
    uint64_t w[N];
    void set(uint64_t x) {
        w[0] = x;
        for (int i = 1; i < N; i++) w[i] = 0;
    }
    void mul(uint64_t x) {
        unsigned __int128 carry = 0;
        for (int i = 0; i < N; i++) {
            const unsigned __int128 p = (unsigned __int128)w[i] * x + carry;
            w[i] = (uint64_t)p;
            carry = p >> 64;
        }
        if (carry) abort();   // an operand outgrew the limbs: a harness bug, never a finding
    }
    void shl(int k) {
        const int limbs = k / 64, bits = k % 64;
        if (limbs) {
            for (int i = N - limbs; i < N; i++)
                if (w[i]) abort();
            for (int i = N - 1; i >= 0; i--) w[i] = i >= limbs ? w[i - limbs] : 0;
        }
        if (bits) {
            if (w[N - 1] >> (64 - bits)) abort();
            for (int i = N - 1; i > 0; i--) w[i] = (w[i] << bits) | (w[i - 1] >> (64 - bits));
            w[0] <<= bits;
        }
    }
    int cmp(const Big& o) const {
        for (int i = N - 1; i >= 0; i--)
            if (w[i] != o.w[i]) return w[i] < o.w[i] ? -1 : 1;
        return 0;
    }
};

template <int N>
struct Pow10Table {
    std::vector<Big<N>> p;
    explicit Pow10Table(int max_e) : p((size_t)max_e + 1) {
        p[0].set(1);
        for (int e = 1; e <= max_e; e++) { p[(size_t)e] = p[(size_t)e - 1]; p[(size_t)e].mul(10); }
    }
};

template <int N>
const Pow10Table<N>& pow10_table() {
    static const Pow10Table<N> t(N == 4 ? 60 : 360);
    return t;
}

// sign of d * 10^e10 - c * 2^e2
template <int N>
int cmp_dec_bin(uint64_t d, int e10, uint64_t c, int e2) {
    const Pow10Table<N>& t = pow10_table<N>();
    Big<N> l, r;
    if (e10 >= 0) { l = t.p[(size_t)e10]; l.mul(d); r.set(c); }
    else { l.set(d); r = t.p[(size_t)-e10]; r.mul(c); }
    if (e2 >= 0) r.shl(e2);
    else l.shl(-e2);
    return l.cmp(r);
}

struct Width {
    int mbits, bias;
};
constexpr Width kW32{23, 127}, kW64{52, 1023};

// The rounding interval of a finite nonzero magnitude c * 2^q as two boundaries num * 2^exp, and whether they belong to it
// (round half to even: they do when c is even).
struct Interval {
    uint64_t lo, hi;
    int lo_e, hi_e;
    bool closed;
};

Interval interval(const Width W, uint64_t mag) {
    const int be = (int)(mag >> W.mbits);
    const uint64_t frac = mag & ((1ull << W.mbits) - 1);
    const int q = be ? be - W.bias - W.mbits : 1 - W.bias - W.mbits;
    const uint64_t c = be ? frac | (1ull << W.mbits) : frac;
    Interval I{2 * c - 1, 2 * c + 1, q - 1, q - 1, (c & 1) == 0};
    if (frac == 0 && be > 1) { I.lo = 4 * c - 1; I.lo_e = q - 2; }   // a power of two: the lower neighbour is half as far
    return I;
}

template <int N>
bool above_lo(const Interval& I, uint64_t d, int e) {
    const int s = cmp_dec_bin<N>(d, e, I.lo, I.lo_e);
    return s > 0 || (s == 0 && I.closed);
}
template <int N>
bool below_hi(const Interval& I, uint64_t d, int e) {
    const int s = cmp_dec_bin<N>(d, e, I.hi, I.hi_e);
    return s < 0 || (s == 0 && I.closed);
}
template <int N>
bool rounds_to(const Interval& I, uint64_t d, int e) { return d != 0 && above_lo<N>(I, d, e) && below_hi<N>(I, d, e); }

// The text's digits as d * 10^e with no trailing zeros in d; false when it is not [-]digits[.digits].
bool text_decimal(const char* s, uint64_t* d, int* e) {
    if (*s == '-') s++;
    uint64_t v = 0;
    int ex = 0, nd = 0, zeros = 0;   // zeros: a run of zeros after a nonzero digit, not yet in v
    bool point = false, any = false;
    for (; *s; s++) {
        if (*s == '.') {
            if (point) return false;
            point = true;
            continue;
        }
        if (*s < '0' || *s > '9') return false;
        any = true;
        if (point) ex--;
        if (*s == '0') { if (v) zeros++; continue; }
        nd += zeros + 1;
        if (nd > 19) return false;
        for (; zeros; zeros--) v *= 10;
        v = v * 10 + (uint64_t)(*s - '0');
    }
    if (!any || v == 0) return false;
    ex += zeros;
    *d = v;
    *e = ex;
    return true;
}

int format_bits(int width, uint64_t bits, char* out) {
    const bdf::CsvFloat x = width == 32 ? bdf::csvf_f32((uint32_t)bits) : bdf::csvf_f64(bits);
    const int n = bdf::csvf_float_len(x);
    bdf::csvf_float_put(x, out);
    out[n] = 0;
    return n;
}

enum { kChecked, kRoundTrip, kDigits, kShortest, kClosest, kParse, kCounts };

// Every check of one pattern; returns the first check that failed (kChecked when none did).
template <int N>
int check_one(int width, uint64_t bits) {
    const Width W = width == 32 ? kW32 : kW64;
    const uint64_t sign = 1ull << (width - 1), mag = bits & (sign - 1);
    char text[400];
    const int n = format_bits(width, bits, text);
    // 1. the round trip through glibc
    uint64_t back;
    if (width == 32) {
        const float f = strtof_l(text, nullptr, c_locale());
        uint32_t b;
        memcpy(&b, &f, 4);
        back = b;
    } else {
        const double f = strtod_l(text, nullptr, c_locale());
        memcpy(&back, &f, 8);
    }
    if (back != bits) return kRoundTrip;
    // 2. the parser of the same library reads the text back to the same bits, never through its exact fallback
    uint64_t parsed = 0;
    const int st = csv::parse_float(csv::Unquote((const uint8_t*)text, (const uint8_t*)text + n), width == 32 ? CSV_F32 : CSV_F64, &parsed);
    if (st != csv::kFloatOk || parsed != bits) return kParse;
    if (mag == 0 || (mag >> W.mbits) == (uint64_t)(2 * W.bias + 1)) return kChecked;   // zero and inf have one spelling
    // 3. the digits written are the digits chosen, and they lie in the rounding interval
    uint64_t d;
    int e;
    if (!text_decimal(text, &d, &e)) return kDigits;
    const Interval I = interval(W, mag);
    if (!rounds_to<N>(I, d, e)) return kDigits;
    // 4. shortest: no multiple of 10^(e+1) lies in the interval (the interval is convex and holds d * 10^e, so the multiples
    //    just below and just above it are the only ones to try)
    const uint64_t t = d / 10;
    if ((t != 0 && above_lo<N>(I, t, e + 1)) || below_hi<N>(I, t + 1, e + 1)) return kShortest;
    // 5. closest: a neighbour d - 1 or d + 1 that also reads back is no closer to the exact value c * 2^q = num * 2^(q-1)
    const uint64_t num = I.lo + 1;   // 2c, or 4c at a power of two
    const int num_e = I.lo_e;
    if (cmp_dec_bin<N>(2 * d + 1, e, num, num_e + 1) < 0 && rounds_to<N>(I, d + 1, e)) return kClosest;   // v > (d + 1/2) 10^e
    if (cmp_dec_bin<N>(2 * d - 1, e, num, num_e + 1) > 0 && rounds_to<N>(I, d - 1, e)) return kClosest;   // v < (d - 1/2) 10^e
    return kChecked;
}

struct Tally {
    std::atomic<int64_t> counts[kCounts];
    std::mutex mu;
    std::vector<uint64_t> first_bad;   // (pattern, failed check) pairs
    int max_bad;
    explicit Tally(int m) : max_bad(m) {
        for (auto& c : counts) c = 0;
    }
    void add(int64_t checked, const int64_t* fails, const std::vector<uint64_t>& bad) {
        counts[kChecked] += checked;
        for (int k = 1; k < kCounts; k++) counts[k] += fails[k];
        std::lock_guard<std::mutex> g(mu);
        for (size_t i = 0; i < bad.size() && (int)first_bad.size() < 2 * max_bad; i++) first_bad.push_back(bad[i]);
    }
    void out(int64_t* counts_out, uint64_t* bad_out, int* n_bad) {
        for (int k = 0; k < kCounts; k++) counts_out[k] = counts[k];
        *n_bad = (int)first_bad.size() / 2;
        for (size_t i = 0; i < first_bad.size(); i++) bad_out[i] = first_bad[i];
    }
};

template <typename Next>
void run_threads(int threads, int width, Tally& tally, Next next) {
    std::vector<std::thread> pool;
    for (int t = 0; t < threads; t++) {
        pool.emplace_back([&, t]() {
            int64_t fails[kCounts] = {0}, checked = 0;
            std::vector<uint64_t> bad;
            uint64_t lo, hi;
            while (next(&lo, &hi)) {
                for (uint64_t b = lo; b < hi; b++) {
                    uint64_t bits;
                    if (!next.pattern(b, &bits)) continue;
                    const int r = width == 32 ? check_one<4>(32, bits) : check_one<20>(64, bits);
                    checked++;
                    if (r != kChecked) {
                        fails[r]++;
                        if ((int)bad.size() < 2 * tally.max_bad) { bad.push_back(bits); bad.push_back((uint64_t)r); }
                    }
                }
            }
            tally.add(checked, fails, bad);
        });
    }
    for (auto& th : pool) th.join();
}

}  // namespace

extern "C" {

// Parses n fields (field i is buf[off[i], off[i + 1])) as Float32 (width 32) or Float64: status kFloatOk / kFloatBad / kFloatSlow.
void h_parse_float(const char* buf, const int64_t* off, int64_t n, int width, uint64_t* bits, int32_t* status) {
    for (int64_t i = 0; i < n; i++) {
        const uint8_t* s = (const uint8_t*)buf + off[i];
        const uint8_t* e = (const uint8_t*)buf + off[i + 1];
        uint64_t b = 0;
        status[i] = csv::parse_float(csv::Unquote(s, e), width == 32 ? CSV_F32 : CSV_F64, &b);
        bits[i] = b;
    }
}

// parse_int of n fields as dtype (0 i8 .. 7 u64): ok[i] = 1 with the value's bits, or 0.
void h_parse_int(const char* buf, const int64_t* off, int64_t n, int dtype, uint64_t* out, int32_t* ok) {
    for (int64_t i = 0; i < n; i++) {
        uint64_t v = 0;
        ok[i] = csv::parse_int(csv::Unquote((const uint8_t*)buf + off[i], (const uint8_t*)buf + off[i + 1]), dtype, &v);
        out[i] = v;
    }
}

// The formatter's integer logarithms: kind 0 floor(log10(2^x)), 1 floor(log10(3/4 * 2^x)), 2 floor(log2(10^x)).
int h_flog(int kind, int x) {
    return kind == 0 ? bdf::csvf_flog10pow2(x) : kind == 1 ? bdf::csvf_flog10tq(x) : bdf::csvf_flog2pow10(x);
}

// The writer's text of n patterns, NUL-terminated, one per `slot` bytes of out.
void h_format(const uint64_t* bits, int64_t n, int width, char* out, int64_t slot) {
    for (int64_t i = 0; i < n; i++) format_bits(width, bits[i], out + i * slot);
}

// The writer's text of n patterns, one line each ("\n"-terminated), into out (cap bytes); returns the length or -1 if it overflows.
int64_t h_format_lines(const uint64_t* bits, int64_t n, int width, char* out, int64_t cap) {
    int64_t len = 0;
    for (int64_t i = 0; i < n; i++) {
        if (len + 400 > cap) return -1;
        len += format_bits(width, bits[i], out + len);
        out[len++] = '\n';
    }
    return len;
}

// Every check of check_one over n given patterns.  counts: checked, then failures per check; bad: up to max_bad (pattern, check).
void h_check_list(const uint64_t* bits, int64_t n, int width, int threads, int64_t* counts, uint64_t* bad, int max_bad, int* n_bad) {
    Tally tally(max_bad);
    std::atomic<int64_t> pos{0};
    struct Next {
        std::atomic<int64_t>* pos;
        int64_t n;
        const uint64_t* bits;
        bool operator()(uint64_t* lo, uint64_t* hi) const {
            const int64_t s = pos->fetch_add(4096);
            if (s >= n) return false;
            *lo = (uint64_t)s;
            *hi = (uint64_t)(s + 4096 < n ? s + 4096 : n);
            return true;
        }
        bool pattern(uint64_t i, uint64_t* b) const { *b = bits[i]; return true; }
    } next{&pos, n, bits};
    run_threads(threads, width, tally, next);
    tally.out(counts, bad, n_bad);
}

// Float32 patterns but the NaNs, in blocks of 2^16 handed out to `threads` threads: every multiple of `stride`, and with a stride
// above one also the first and last 4096 patterns of every biased exponent of both signs (those not already a multiple).
void h_check_f32(uint32_t stride, int threads, int64_t* counts, uint64_t* bad, int max_bad, int* n_bad) {
    Tally tally(max_bad);
    std::atomic<uint64_t> pos{0};
    struct Next {
        std::atomic<uint64_t>* pos;
        uint64_t stride, strided, total;
        bool operator()(uint64_t* lo, uint64_t* hi) const {
            const uint64_t s = pos->fetch_add(1ull << 16);
            if (s >= total) return false;
            *lo = s;
            *hi = s + (1ull << 16) < total ? s + (1ull << 16) : total;
            return true;
        }
        bool pattern(uint64_t i, uint64_t* b) const {
            if (i < strided) {
                *b = i * stride;
            } else {   // boundary item j of exponent (sign, be)
                const uint64_t k = i - strided, j = k % 8192, be = (k / 8192) % 256, sign = k / (8192 * 256);
                *b = (sign << 31) | (be << 23) | (j < 4096 ? j : (1u << 23) - 8192 + j);
                if (*b % stride == 0) return false;
            }
            return (*b & 0x7fffffffu) <= 0x7f800000u;   // not NaN
        }
    } next{&pos, stride, ((1ull << 32) + stride - 1) / stride, 0};
    next.total = next.strided + (stride > 1 ? 2 * 256 * 8192 : 0);
    run_threads(threads, 32, tally, next);
    tally.out(counts, bad, n_bad);
}

}  // extern "C"
