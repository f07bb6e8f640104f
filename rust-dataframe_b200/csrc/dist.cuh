// dist.cuh -- the scalar rules of the column distributions (include/b200df.h "distributions"), shared by the host (whole-column
// percentile, histogram edges and density) and the device (per-group median), so both paths compute the same bits.
#pragma once

#include <math.h>
#include <stdint.h>
#include <string.h>

namespace bdf {

#if defined(__CUDA_ARCH__)
#define BDF_DIST_HD __host__ __device__
__device__ __forceinline__ double dist_add(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double dist_sub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double dist_mul(double a, double b) { return __dmul_rn(a, b); }
#else
#if defined(__CUDACC__)
#define BDF_DIST_HD __host__ __device__
#else
#define BDF_DIST_HD
#endif
// volatile: one rounding per operation on the host too (no contraction into an FMA)
inline double dist_add(double a, double b) { volatile double r = a + b; return r; }
inline double dist_sub(double a, double b) { volatile double r = a - b; return r; }
inline double dist_mul(double a, double b) { volatile double r = a * b; return r; }
#endif

constexpr uint64_t kDistNaN = 0x7ff8000000000000ull;   // the positive quiet NaN every NaN result is returned as

BDF_DIST_HD inline double dist_quiet_nan(double x) {
    if (x != x) {
        const uint64_t q = kDistNaN;
        memcpy(&x, &q, sizeof x);
    }
    return x;
}

// What a key stands for: every NaN is the positive quiet NaN, -0.0 is +0.0.
BDF_DIST_HD inline double dist_canonical(double x) { return x == 0.0 ? 0.0 : dist_quiet_nan(x); }

// The percentile of a and b, the lo-th and hi-th valid values in key order (read as f64), at pos = (n - 1) * p: exactly this
// sequence of IEEE operations; a NaN result is the positive quiet NaN.
BDF_DIST_HD inline double dist_interp(double a, double b, double pos, double lo, double hi) {
    a = dist_canonical(a);
    b = dist_canonical(b);
    double r = a;
    if (!(lo == hi || a == b)) r = dist_add(dist_mul(dist_sub(hi, pos), a), dist_mul(dist_sub(pos, lo), b));
    return dist_quiet_nan(r);
}

}  // namespace bdf
