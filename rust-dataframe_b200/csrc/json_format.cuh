// json_format.cuh -- the text of one value of the JSON writer (k_json_write.cu; the rules are in include/b200df.h "line-delimited
// JSON files straight from the device"):
//   floats     the shortest digits of csv_format.cuh (Float32 as an f32) in ryu's "pretty" layout (RECALLED: the ryu crate's
//              format64 / format32, which serde_json prints with): with kk the decimal exponent of the first digit plus one,
//              integral values as digits and ".0" while kk <= 16 (Float32: 13), the point inside the digits for 0 < kk <= 16 (13),
//              0.000ddd for -5 < kk <= 0 (-6 < kk), else d.ddde[-]x.  Only finite values: NaN and inf are written as null by the caller.
//   integers   plain decimal (csvf_int_put); Booleans true / false.
//   temporal   a JSON string: "YYYY-MM-DD", "YYYY-MM-DDTHH:MM:SS[.fff]<suffix>" or "HH:MM:SS[.fff]", the year as chrono's %Y writes it
//              (4 digits for 0..9999, '+' and the digits above, '-' and at least 4 digits below 0).
// Like csv_format.cuh it is plain integer arithmetic that a host compiler (with __device__ defined empty) compiles to the same text.
#pragma once

#include <stdint.h>

#include "civil.cuh"
#include "csv_format.cuh"

namespace bdf {

// ---- floats: x is finite (special 0 or 3) ----

CSVF int jsonf_exp_len(int e) {
    const int a = e < 0 ? -e : e;
    return (e < 0) + (a >= 100 ? 3 : a >= 10 ? 2 : 1);
}

CSVF int jsonf_float_len(const CsvFloat& x, bool f32) {
    if (x.special == 3) return 3 + x.neg;   // 0.0, -0.0
    const int kk = x.n + x.e, top = f32 ? 13 : 16, low = f32 ? -6 : -5;
    int body;
    if (x.e >= 0 && kk <= top) body = kk + 2;
    else if (kk > 0 && kk <= top) body = x.n + 1;
    else if (kk > low && kk <= 0) body = 2 - kk + x.n;
    else body = x.n + (x.n > 1) + 1 + jsonf_exp_len(kk - 1);
    return body + x.neg;
}

// Writes jsonf_float_len(x, f32) bytes at p.
CSVF void jsonf_float_put(const CsvFloat& x, bool f32, char* p) {
    if (x.neg) *p++ = '-';
    if (x.special == 3) { p[0] = '0'; p[1] = '.'; p[2] = '0'; return; }
    const int kk = x.n + x.e, top = f32 ? 13 : 16, low = f32 ? -6 : -5;
    if (x.e >= 0 && kk <= top) {
        csvf_put_digits(p, x.f, x.n);
        for (int j = x.n; j < kk; j++) p[j] = '0';
        p[kk] = '.';
        p[kk + 1] = '0';
    } else if (kk > 0 && kk <= top) {   // the point inside the digits: write them, then open the gap
        csvf_put_digits(p, x.f, x.n);
        for (int j = x.n; j > kk; j--) p[j] = p[j - 1];
        p[kk] = '.';
    } else if (kk > low && kk <= 0) {
        p[0] = '0';
        p[1] = '.';
        for (int j = 0; j < -kk; j++) p[2 + j] = '0';
        csvf_put_digits(p + 2 - kk, x.f, x.n);
    } else {
        int at = 1;
        if (x.n > 1) {   // d.ddd
            csvf_put_digits(p + 1, x.f, x.n);
            p[0] = p[1];
            p[1] = '.';
            at = x.n + 1;
        } else {
            p[0] = (char)('0' + x.f);
        }
        p[at++] = 'e';
        int ex = kk - 1;
        if (ex < 0) { p[at++] = '-'; ex = -ex; }
        csvf_put_digits(p + at, (uint64_t)ex, csvf_digits((uint64_t)ex));
    }
}

// ---- temporal values ----
// kind: JT_DATE (the floor day of a Date32 / Date64 / date-only value), JT_TIMESTAMP, JT_TIME (a time of day, already checked to
// lie in [0, upd)).  upd / ups: units per day / per second; off: the fixed tz offset in units (|off| < upd); frac: 0, 3, 6 or 9
// fraction digits; the suffix ("Z", "+05:30" or none) is written after the fraction.  Dates are checked to lie in chrono's range.
enum : int { JT_NONE = 0, JT_DATE, JT_TIMESTAMP, JT_TIME };

// (days, time of day) of v by floor division, then the offset applied (as split_local of k_temporal.cu).
CIVILF void jsonf_split(int64_t v, int kind, int64_t upd, int64_t off, int64_t& days, int64_t& tod) {
    if (kind == JT_TIME) { days = 0; tod = v; return; }
    days = v / upd;
    tod = v - days * upd;
    if (tod < 0) { tod += upd; days -= 1; }
    tod += off;
    if (tod >= upd) { tod -= upd; days += 1; }
    else if (tod < 0) { tod += upd; days -= 1; }
}

CSVF int jsonf_year_len(int32_t y) {
    if (y >= 0 && y <= 9999) return 4;
    if (y > 9999) return 1 + csvf_digits((uint64_t)y);
    const int d = csvf_digits((uint64_t)(-(int64_t)y));
    return 1 + (d < 4 ? 4 : d);
}

CSVF void jsonf_pad(char* p, uint64_t v, int n) {   // v in n digits, zero-padded
    for (int j = n - 1; j >= 0; j--) { p[j] = (char)('0' + v % 10); v /= 10; }
}

CSVF int jsonf_time_len(int64_t v, int kind, int64_t upd, int64_t off, int frac, int suffix_len) {
    int n = 2;   // the quotes
    if (kind != JT_TIME) {
        int64_t days, tod;
        jsonf_split(v, kind, upd, off, days, tod);
        if (days >= -719528 && days < 2932897) n += 4;   // 0000-01-01 .. 9999-12-31
        else {
            int32_t y; uint32_t m, d;
            civil_from_days((int32_t)days, y, m, d);
            n += jsonf_year_len(y);
        }
        n += 6;   // -MM-DD
    }
    if (kind != JT_DATE) n += 8 + (frac ? frac + 1 : 0);
    if (kind == JT_TIMESTAMP) n += 1 + suffix_len;   // 'T'
    return n;
}

// Writes jsonf_time_len(...) bytes at p.
CSVF void jsonf_time_put(int64_t v, int kind, int64_t upd, int64_t ups, int64_t off, int frac, int suffix_len, const char* suffix, char* p) {
    int64_t days, tod;
    jsonf_split(v, kind, upd, off, days, tod);
    *p++ = '"';
    if (kind != JT_TIME) {
        int32_t y; uint32_t m, d;
        civil_from_days((int32_t)days, y, m, d);
        const int yl = jsonf_year_len(y);
        if (y > 9999) { p[0] = '+'; jsonf_pad(p + 1, (uint64_t)y, yl - 1); }
        else if (y < 0) { p[0] = '-'; jsonf_pad(p + 1, (uint64_t)(-(int64_t)y), yl - 1); }
        else jsonf_pad(p, (uint64_t)y, 4);
        p += yl;
        p[0] = '-'; jsonf_pad(p + 1, m, 2);
        p[3] = '-'; jsonf_pad(p + 4, d, 2);
        p += 6;
        if (kind == JT_TIMESTAMP) *p++ = 'T';
    }
    if (kind != JT_DATE) {
        const int64_t secs = tod / ups, sub = tod - secs * ups;
        jsonf_pad(p, (uint64_t)(secs / 3600), 2);
        p[2] = ':'; jsonf_pad(p + 3, (uint64_t)((secs / 60) % 60), 2);
        p[5] = ':'; jsonf_pad(p + 6, (uint64_t)(secs % 60), 2);
        p += 8;
        if (frac) { p[0] = '.'; jsonf_pad(p + 1, (uint64_t)sub, frac); p += frac + 1; }
        if (kind == JT_TIMESTAMP)
            for (int j = 0; j < suffix_len; j++) *p++ = suffix[j];
    }
    *p = '"';
}

}  // namespace bdf
