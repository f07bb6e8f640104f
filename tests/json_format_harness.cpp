// json_format_harness.cpp -- the JSON writer's value formatter (json_format.cuh) compiled for the host and driven through ctypes by
// tests/test_json_write.py, which compares its text with tests/json_write_oracle.py.  The header compiles as plain C++ with
// __device__ defined empty, so its text can be checked here without a GPU.
#include <stdint.h>
#include <string.h>

#include "json_format.cuh"

extern "C" {

// The text of n Float32 (width 32) or Float64 patterns, one line each ("null" for NaN and inf), into out (cap bytes); returns the
// length, or -1 if it overflows.
int64_t jh_format_floats(const uint64_t* bits, int64_t n, int width, char* out, int64_t cap) {
    int64_t len = 0;
    for (int64_t i = 0; i < n; i++) {
        if (len + 64 > cap) return -1;
        const bdf::CsvFloat x = width == 32 ? bdf::csvf_f32((uint32_t)bits[i]) : bdf::csvf_f64(bits[i]);
        if (x.special == 1 || x.special == 2) {
            memcpy(out + len, "null", 4);
            len += 4;
        } else {
            bdf::jsonf_float_put(x, width == 32, out + len);
            len += bdf::jsonf_float_len(x, width == 32);
        }
        out[len++] = '\n';
    }
    return len;
}

// The Date32 text of days first .. first + n - 1, each in a zero-padded slot of 16 bytes.
void jh_format_dates(int32_t first, int64_t n, char* out) {
    memset(out, 0, (size_t)n * 16);
    for (int64_t i = 0; i < n; i++) {
        const int64_t v = first + i;
        char* p = out + i * 16;
        const int len = bdf::jsonf_time_len(v, bdf::JT_DATE, 1, 0, 0, 0);
        if (len > 16) continue;   // cannot happen in chrono's range; the comparison then fails
        bdf::jsonf_time_put(v, bdf::JT_DATE, 1, 1, 0, 0, 0, "", p);
    }
}

// The temporal text of n values of one column, one line each: kind (json_format.cuh's JT_*), units per day and second, the tz
// offset in units, fraction digits and suffix.  Returns the length, or -1 if it overflows.
int64_t jh_format_temporal(const int64_t* v, int64_t n, int kind, int64_t upd, int64_t ups, int64_t off, int frac, const char* suffix,
                           char* out, int64_t cap) {
    const int sl = (int)strlen(suffix);
    int64_t len = 0;
    for (int64_t i = 0; i < n; i++) {
        const int l = bdf::jsonf_time_len(v[i], kind, upd, off, frac, sl);
        if (len + l + 1 > cap) return -1;
        bdf::jsonf_time_put(v[i], kind, upd, ups, off, frac, sl, suffix, out + len);
        len += l;
        out[len++] = '\n';
    }
    return len;
}

}  // extern "C"
