// json_parse.cuh -- the record grammar and value rules of the line-delimited JSON reader (k_json.cu).  Device code in the library;
// the same source compiles as plain C++, so the host walks a bad record with exactly the device's rules to name the error.
//
// A record is one line.  The walker checks the whole record against JSON's grammar (RFC 8259: objects, arrays, strings with their
// escapes, numbers, true / false / null), with nesting limited to 128 levels, and reports every member of the top-level object:
// its key's raw bytes, its value's bytes and the value's class.  The numbers' conversions are csv_parse.cuh's: JSON's number
// grammar is a subset of the one they read, and a JSON number never starts with '"', so csv::Unquote passes its bytes through.
#pragma once
#include <stdint.h>

#include "csv_parse.cuh"

#ifdef __CUDACC__
#define JSON_FN __host__ __device__ __forceinline__
#else
#define JSON_FN inline
#endif

namespace json {

// what a line is
enum { kBad = -1, kBlank = 0, kRecord = 1 };

// value classes (bits, OR-ed per column by the inference); a list is classified by its direct elements
enum {
    kNull = 1, kBool = 2, kInt = 4, kFloat = 8, kStr = 16, kObj = 32,
    kListInt = 64,      // every typed element is an integer literal in i64 range
    kListFloat = 128,   // numbers, at least one of them not such an integer
    kListOther = 256,   // an element that is a Boolean, a string, an object or an array
    kListEmpty = 512,   // no element other than null
    kMissing = 1024,    // inference only: a record without the key
};

// what went wrong (runtime.cu turns the code into text)
enum { eNone = 0, eNotObject, eExpectKey, eExpectColon, eExpectValue, eExpectCommaOrClose, eUnterminated, eEscape, eControl, eNumber,
       eLiteral, eTrailing, eDepth };

constexpr int kMaxDepth = 128;   // serde_json's recursion limit: the record's object is level 1

struct Cursor {
    const uint8_t* p;
    const uint8_t* e;
    int err;
    const uint8_t* at;   // where the error was found
};

JSON_FN bool is_ws(uint8_t c) { return c == ' ' || c == '\t' || c == '\r' || c == '\n'; }
JSON_FN bool is_digit(uint8_t c) { return c >= '0' && c <= '9'; }
JSON_FN bool is_hex(uint8_t c) { return is_digit(c) || (c >= 'a' && c <= 'f') || (c >= 'A' && c <= 'F'); }
JSON_FN bool fail(Cursor& c, int code, const uint8_t* at) { c.err = code; c.at = at; return false; }
JSON_FN void skip_ws(Cursor& c) { while (c.p < c.e && is_ws(*c.p)) c.p++; }
JSON_FN bool at(const Cursor& c, uint8_t b) { return c.p < c.e && *c.p == b; }

// A string at c.p == '"'; after it c.p is past the closing quote.  *escaped: it contains a backslash.
JSON_FN bool string(Cursor& c, bool* escaped) {
    const uint8_t* open = c.p++;
    while (c.p < c.e) {
        const uint8_t b = *c.p;
        if (b == '"') { c.p++; return true; }
        if (b < 0x20) return fail(c, eControl, c.p);
        if (b == '\\') {
            *escaped = true;
            const uint8_t* esc = c.p++;
            if (c.p >= c.e) return fail(c, eEscape, esc);
            const uint8_t x = *c.p;
            if (x == 'u') {
                for (int k = 1; k <= 4; k++)
                    if (c.p + k >= c.e || !is_hex(c.p[k])) return fail(c, eEscape, esc);
                c.p += 5;
                continue;
            }
            if (!(x == '"' || x == '\\' || x == '/' || x == 'b' || x == 'f' || x == 'n' || x == 'r' || x == 't')) return fail(c, eEscape, esc);
        }
        c.p++;
    }
    return fail(c, eUnterminated, open);
}

// -? (0 | [1-9][0-9]*) (. [0-9]+)? ([eE] [+-]? [0-9]+)?   *cls: kInt for an integer literal in i64 range, else kFloat.
JSON_FN bool number(Cursor& c, int* cls) {
    const uint8_t* s = c.p;
    bool neg = false;
    if (*c.p == '-') { neg = true; c.p++; }
    if (!(c.p < c.e && is_digit(*c.p))) return fail(c, eNumber, s);
    uint64_t mag = 0;
    bool over = false, integral = true;
    if (*c.p == '0') {
        c.p++;
        if (c.p < c.e && is_digit(*c.p)) return fail(c, eNumber, s);   // a leading zero
    } else {
        for (; c.p < c.e && is_digit(*c.p); c.p++) {
            const uint64_t d = (uint64_t)(*c.p - '0');
            if (mag > (0xffffffffffffffffull - d) / 10) over = true;
            else mag = mag * 10 + d;
        }
    }
    if (at(c, '.')) {
        integral = false;
        c.p++;
        if (!(c.p < c.e && is_digit(*c.p))) return fail(c, eNumber, s);
        while (c.p < c.e && is_digit(*c.p)) c.p++;
    }
    if (at(c, 'e') || at(c, 'E')) {
        integral = false;
        c.p++;
        if (at(c, '+') || at(c, '-')) c.p++;
        if (!(c.p < c.e && is_digit(*c.p))) return fail(c, eNumber, s);
        while (c.p < c.e && is_digit(*c.p)) c.p++;
    }
    *cls = integral && !over && (neg ? mag <= (1ull << 63) : mag < (1ull << 63)) ? kInt : kFloat;
    return true;
}

JSON_FN bool literal(Cursor& c, const char* w, int n) {
    if (c.e - c.p < n) return fail(c, eLiteral, c.p);
    for (int k = 0; k < n; k++)
        if (c.p[k] != (uint8_t)w[k]) return fail(c, eLiteral, c.p);
    c.p += n;
    return true;
}

// A value that is not an array or object.
JSON_FN bool scalar(Cursor& c, int* cls) {
    if (c.p >= c.e) return fail(c, eExpectValue, c.p);
    const uint8_t b = *c.p;
    if (b == '"') { bool esc = false; *cls = kStr; return string(c, &esc); }
    if (b == 't') { *cls = kBool; return literal(c, "true", 4); }
    if (b == 'f') { *cls = kBool; return literal(c, "false", 5); }
    if (b == 'n') { *cls = kNull; return literal(c, "null", 4); }
    if (b == '-' || is_digit(b)) return number(c, cls);
    return fail(c, eExpectValue, c.p);
}

// Any value at c.p (whitespace skipped), `depth` levels below the top.  Containers are walked with an explicit stack (one bit per
// level: array or object), not by recursion.
JSON_FN bool value(Cursor& c, int depth, int* cls) {
    if (!(at(c, '[') || at(c, '{'))) return scalar(c, cls);
    const bool outer_array = *c.p == '[';
    uint64_t lo = 0, hi = 0;   // the stack: bit d set when level d is an array (two words, so it stays in registers)
    int d = 0, elems = 0;   // elems: the classes of the outer array's direct elements
    int state = 0;          // 0 at an opening bracket, 1 at a member or element, 2 after one
    for (;;) {
        if (state == 0) {
            if (depth + d >= kMaxDepth) return fail(c, eDepth, c.p);
            const bool arr = *c.p == '[';
            const uint64_t bit = 1ull << (d & 63);
            uint64_t& w = d < 64 ? lo : hi;
            w = arr ? (w | bit) : (w & ~bit);
            d++;
            c.p++;
            skip_ws(c);
            if (at(c, arr ? ']' : '}')) {
                c.p++;
                if (--d == 0) break;
                state = 2;
            } else {
                state = 1;
            }
            continue;
        }
        const bool top_arr = (((d - 1) < 64 ? lo : hi) >> ((d - 1) & 63)) & 1u;
        if (state == 1) {
            if (!top_arr) {
                if (!at(c, '"')) return fail(c, eExpectKey, c.p);
                bool esc = false;
                if (!string(c, &esc)) return false;
                skip_ws(c);
                if (!at(c, ':')) return fail(c, eExpectColon, c.p);
                c.p++;
                skip_ws(c);
            }
            if (at(c, '[') || at(c, '{')) {
                if (d == 1) elems |= kObj;
                state = 0;
                continue;
            }
            int sc = 0;
            if (!scalar(c, &sc)) return false;
            if (d == 1) elems |= sc;
            state = 2;
            continue;
        }
        skip_ws(c);
        if (at(c, ',')) {
            c.p++;
            skip_ws(c);
            state = 1;
        } else if (at(c, top_arr ? ']' : '}')) {
            c.p++;
            if (--d == 0) break;
        } else {
            return fail(c, eExpectCommaOrClose, c.p);
        }
    }
    if (!outer_array) *cls = kObj;
    else if (elems & (kBool | kStr | kObj)) *cls = kListOther;
    else if (elems & kFloat) *cls = kListFloat;
    else if (elems & kInt) *cls = kListInt;
    else *cls = kListEmpty;
    return true;
}

// One line [p, e) (without its '\n'): kBlank, kBad (c.err, c.at) or kRecord, with v.member(key_begin, key_end, value_begin,
// value_end, class, key_escaped) for every member of the object in order.
template <class V>
JSON_FN int record(Cursor& c, V& v) {
    skip_ws(c);
    if (c.p >= c.e) return kBlank;
    if (*c.p != '{') { fail(c, eNotObject, c.p); return kBad; }
    c.p++;
    skip_ws(c);
    if (at(c, '}')) {
        c.p++;
    } else {
        for (;;) {
            if (!at(c, '"')) { fail(c, eExpectKey, c.p); return kBad; }
            const uint8_t* k0 = c.p;
            bool esc = false;
            if (!string(c, &esc)) return kBad;
            const uint8_t* k1 = c.p;
            skip_ws(c);
            if (!at(c, ':')) { fail(c, eExpectColon, c.p); return kBad; }
            c.p++;
            skip_ws(c);
            const uint8_t* v0 = c.p;
            int cls = 0;
            if (!value(c, 1, &cls)) return kBad;
            v.member(k0 + 1, k1 - 1, v0, c.p, cls, esc);
            skip_ws(c);
            if (at(c, ',')) { c.p++; skip_ws(c); continue; }
            if (at(c, '}')) { c.p++; break; }
            fail(c, eExpectCommaOrClose, c.p);
            return kBad;
        }
    }
    skip_ws(c);
    if (c.p < c.e) { fail(c, eTrailing, c.p); return kBad; }
    return kRecord;
}

// The direct elements of a valid array value [p, e): f(index, begin, end) for each; returns their number.
template <class F>
JSON_FN int64_t elements(const uint8_t* p, const uint8_t* e, F& f) {
    Cursor c{p + 1, e, 0, nullptr};
    skip_ws(c);
    if (at(c, ']')) return 0;
    int64_t n = 0;
    for (;;) {
        const uint8_t* s = c.p;
        int cls = 0;
        value(c, 2, &cls);
        f(n, s, c.p);
        n++;
        skip_ws(c);
        if (!at(c, ',')) return n;
        c.p++;
        skip_ws(c);
    }
}

enum { kConvNull = 0, kConvOk = 1, kConvSlow = 2 };

// The value bytes [s, e) as a scalar of dtype 0..9 or 10 (Boolean): kConvOk with the bits, kConvNull when it does not convert
// (null, a value of another kind, an integer out of range or not integral), kConvSlow for a float the caller rounds exactly.
CSV_FN int convert(const uint8_t* s, const uint8_t* e, int dtype, uint64_t* bits) {
    const uint8_t b = *s;
    if (dtype == 10) {
        if (b == 't') { *bits = 1; return kConvOk; }
        if (b == 'f') { *bits = 0; return kConvOk; }
        return kConvNull;
    }
    if (!(b == '-' || is_digit(b))) return kConvNull;
    const csv::Unquote u(s, e);
    uint64_t v = 0;
    int r;
    if (dtype == 8 || dtype == 9) {   // one inlined copy of the float path, the format chosen at run time
        const int f = csv::parse_float(u, dtype == 9 ? CSV_F64 : CSV_F32, &v);
        r = f == csv::kFloatOk ? kConvOk : f == csv::kFloatSlow ? kConvSlow : kConvNull;
    } else {
        r = csv::parse_int(u, dtype, &v) ? kConvOk : kConvNull;
    }
    *bits = v;
    return r;
}

// FNV-1a over the key's raw bytes, seeded with its length; never ~0 (the empty slot of the key table).
JSON_FN uint64_t key_hash(const uint8_t* s, const uint8_t* e) {
    uint64_t h = 0xcbf29ce484222325ull ^ (uint64_t)(e - s);
    for (; s < e; s++) h = (h ^ *s) * 0x100000001b3ull;
    return h == ~0ull ? 1 : h;
}

}  // namespace json
