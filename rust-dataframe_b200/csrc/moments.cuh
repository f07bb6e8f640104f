// moments.cuh -- the moment record of a column (count, mean and the central sums m2, m3, m4), the pairwise merge of two records
// and the statistics derived from one (include/b200df.h "statistical aggregates").
//
// One module knows the formulas: the in-CTA tree and the finish of k_moments.cu, the group fold (group_acc.cuh), the rank-order
// combine of a communicator or a multi-GPU context (runtime.cu) and the context-free bdf_moments_stat / bdf_moments_merge all call
// the functions below, on the device or on the host.  Every operation is one IEEE double operation rounded once (no FMA
// contraction on either side), so the host and the device compute the same bits.
#pragma once

#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

namespace bdf {

struct Moments {   // the layout of bdf_moments
    long long count;
    double mean, m2, m3, m4;
};

// Rounded-once operations.  On the host the result goes through a volatile so that no compiler contracts a product into an add.
__host__ __device__ __forceinline__ double mo_add(double a, double b) {
#ifdef __CUDA_ARCH__
    return __dadd_rn(a, b);
#else
    volatile double r = a + b;
    return r;
#endif
}
__host__ __device__ __forceinline__ double mo_sub(double a, double b) {
#ifdef __CUDA_ARCH__
    return __dsub_rn(a, b);
#else
    volatile double r = a - b;
    return r;
#endif
}
__host__ __device__ __forceinline__ double mo_mul(double a, double b) {
#ifdef __CUDA_ARCH__
    return __dmul_rn(a, b);
#else
    volatile double r = a * b;
    return r;
#endif
}
__host__ __device__ __forceinline__ double mo_div(double a, double b) {
#ifdef __CUDA_ARCH__
    return __ddiv_rn(a, b);
#else
    volatile double r = a / b;
    return r;
#endif
}
__host__ __device__ __forceinline__ double mo_sqrt(double a) {
#ifdef __CUDA_ARCH__
    return __dsqrt_rn(a);
#else
    volatile double r = sqrt(a);
    return r;
#endif
}

// The record of one value: a non-finite value makes every moment NaN (and NaN sticks through every merge).
__host__ __device__ __forceinline__ Moments moments_one(double x) {
    const bool finite = isfinite(x);
    const double nan = (double)NAN;
    return Moments{1, finite ? x : nan, finite ? 0.0 : nan, finite ? 0.0 : nan, finite ? 0.0 : nan};
}

// Chan's update for the mean and m2, Pébay's for m3 and m4, with one division: f = delta / n.
//   mean = ma + f nb
//   m2   = m2a + m2b + t                                     t = delta f (na nb)        (= delta^2 na nb / n)
//   m3   = m3a + m3b + t f (na - nb) + 3 f (na m2b - nb m2a)
//   m4   = m4a + m4b + t f^2 (na^2 - na nb + nb^2) + 6 f^2 (na^2 m2b + nb^2 m2a) + 4 f (na m3b - nb m3a)
// Each line is evaluated left to right as written.  An empty side returns the other unchanged; two records with the same mean merge
// to exactly that mean with m2 = m3 = m4 = 0 when both are constant (delta = 0).
__host__ __device__ __forceinline__ Moments moments_merge(const Moments& a, const Moments& b) {
    if (b.count == 0) return a;
    if (a.count == 0) return b;
    Moments r;
    r.count = a.count + b.count;
    const double n = (double)r.count, na = (double)a.count, nb = (double)b.count;
    const double delta = mo_sub(b.mean, a.mean);
    const double f = mo_div(delta, n);
    r.mean = mo_add(a.mean, mo_mul(f, nb));
    const double t = mo_mul(mo_mul(delta, f), mo_mul(na, nb));
    r.m2 = mo_add(mo_add(a.m2, b.m2), t);
    const double m3_cross = mo_mul(mo_mul(t, f), mo_sub(na, nb));
    const double m3_lin = mo_mul(mo_mul(3.0, f), mo_sub(mo_mul(na, b.m2), mo_mul(nb, a.m2)));
    r.m3 = mo_add(mo_add(mo_add(a.m3, b.m3), m3_cross), m3_lin);
    const double f2 = mo_mul(f, f);
    const double poly = mo_add(mo_sub(mo_mul(na, na), mo_mul(na, nb)), mo_mul(nb, nb));
    const double m4_cross = mo_mul(mo_mul(t, f2), poly);
    const double m4_sq = mo_mul(mo_mul(6.0, f2), mo_add(mo_mul(mo_mul(na, na), b.m2), mo_mul(mo_mul(nb, nb), a.m2)));
    const double m4_lin = mo_mul(mo_mul(4.0, f), mo_sub(mo_mul(na, b.m3), mo_mul(nb, a.m3)));
    r.m4 = mo_add(mo_add(mo_add(mo_add(a.m4, b.m4), m4_cross), m4_sq), m4_lin);
    return r;
}

enum : int { STAT_VARIANCE = 0, STAT_VAR_POP, STAT_STDDEV, STAT_STDDEV_POP, STAT_SKEWNESS, STAT_KURTOSIS, STAT_N };

// The statistic of a record; false = None (count 0; count 1 for the sample forms; m2 == 0 for skewness and kurtosis).
__host__ __device__ __forceinline__ bool moments_stat(const Moments& m, int stat, double* out) {
    if (m.count == 0) return false;
    const double n = (double)m.count;
    switch (stat) {
        case STAT_VARIANCE:
            if (m.count == 1) return false;
            *out = mo_div(m.m2, mo_sub(n, 1.0));
            return true;
        case STAT_VAR_POP: *out = mo_div(m.m2, n); return true;
        case STAT_STDDEV:
            if (m.count == 1) return false;
            *out = mo_sqrt(mo_div(m.m2, mo_sub(n, 1.0)));
            return true;
        case STAT_STDDEV_POP: *out = mo_sqrt(mo_div(m.m2, n)); return true;
        case STAT_SKEWNESS:
            if (m.m2 == 0.0) return false;
            *out = mo_div(mo_mul(mo_sqrt(n), m.m3), mo_mul(m.m2, mo_sqrt(m.m2)));
            return true;
        case STAT_KURTOSIS:
            if (m.m2 == 0.0) return false;
            *out = mo_sub(mo_div(mo_mul(n, m.m4), mo_mul(m.m2, m.m2)), 3.0);
            return true;
        default: return false;
    }
}

}  // namespace bdf
