// group_acc.cuh -- the per-group accumulators of the group-by fold (k_group.cu), shared with the window functions' segmented scan
// (k_window.cu): a running SUM / MIN / MAX / AVG over a window frame must give exactly the group-by's answer for the same rows,
// so both fold with this code (float min/max order, NaN rules, integer wrapping, double sums).
#pragma once

#include "common.cuh"
#include "moments.cuh"

namespace bdf {

// The accumulator of the EXTRA instantiations (FusedAgg<T> itself stays as K4/K5 use it).  Integers: FusedAgg's wrapping sum
// and min/max keys plus a double sum for avg.  Floats: FusedAgg's double sum (which is also avg's numerator) plus min/max
// over order-preserving unsigned keys of the IEEE totalOrder with every NaN made the positive quiet NaN.
template <typename T> struct FloatKey;
template <> struct FloatKey<float> {
    static __device__ __forceinline__ unsigned long long key(float x) {
        const unsigned int u = x != x ? 0x7fc00000u : __float_as_uint(x);
        return (unsigned long long)((u & 0x80000000u) ? ~u : (u | 0x80000000u));
    }
    static __device__ __forceinline__ float value(unsigned long long k) {
        const unsigned int u = (unsigned int)k;
        return __uint_as_float((u & 0x80000000u) ? (u ^ 0x80000000u) : ~u);
    }
};
template <> struct FloatKey<double> {
    static __device__ __forceinline__ unsigned long long key(double x) {
        const unsigned long long u = x != x ? 0x7ff8000000000000ull : (unsigned long long)__double_as_longlong(x);
        return (u >> 63) ? ~u : (u | (1ull << 63));
    }
    static __device__ __forceinline__ double value(unsigned long long k) {
        return __longlong_as_double((long long)((k >> 63) ? (k ^ (1ull << 63)) : ~k));
    }
};

template <typename T, bool F = IsFloat<T>::value> struct GroupAggX;
template <typename T> struct GroupAggX<T, false> {
    FusedAgg<T> a;
    double dsum;
    __device__ __forceinline__ void init() { a.init(); dsum = 0.0; }
    __device__ __forceinline__ void add(T x, bool valid, unsigned long long flip) { a.add(x, valid, flip); dsum = __dadd_rn(dsum, valid ? (double)x : 0.0); }
    __device__ __forceinline__ void merge_shfl(int o) { a.merge_shfl(o); dsum = __dadd_rn(dsum, __shfl_xor_sync(0xffffffffu, dsum, o)); }
    __device__ __forceinline__ void merge(const GroupAggX& o) { a.merge(o.a); dsum = __dadd_rn(dsum, o.dsum); }
};
template <typename T> struct GroupAggX<T, true> {
    double sum;
    unsigned long long kmin, kmax;
    __device__ __forceinline__ void init() { sum = 0.0; kmin = ~0ull; kmax = 0; }
    __device__ __forceinline__ void add(T x, bool valid, unsigned long long) {
        sum = __dadd_rn(sum, valid ? (double)x : 0.0);
        if (valid) { const unsigned long long k = FloatKey<T>::key(x); kmin = k < kmin ? k : kmin; kmax = k > kmax ? k : kmax; }
    }
    __device__ __forceinline__ void merge_shfl(int o) {
        const double s2 = __shfl_xor_sync(0xffffffffu, sum, o);
        const unsigned long long a2 = __shfl_xor_sync(0xffffffffu, kmin, o), b2 = __shfl_xor_sync(0xffffffffu, kmax, o);
        sum = __dadd_rn(sum, s2); kmin = a2 < kmin ? a2 : kmin; kmax = b2 > kmax ? b2 : kmax;
    }
    __device__ __forceinline__ void merge(const GroupAggX& o) { sum = __dadd_rn(sum, o.sum); kmin = o.kmin < kmin ? o.kmin : kmin; kmax = o.kmax > kmax ? o.kmax : kmax; }
};

// The moments accumulator (variance, stddev, skewness, kurtosis): every valid value is read `as f64` and merged into the record as
// a one-value record, in the fold order of the other accumulators (moments.cuh).  It carries its own count.
template <typename T> struct GroupMoments {
    Moments m;
    __device__ __forceinline__ void init() { m = Moments{0, 0.0, 0.0, 0.0, 0.0}; }
    __device__ __forceinline__ void add(T x, bool valid, unsigned long long) {
        if (valid) m = moments_merge(m, moments_one((double)x));
    }
    __device__ __forceinline__ void merge_shfl(int o) {
        Moments b;
        b.count = __shfl_xor_sync(0xffffffffu, m.count, o);
        b.mean = __shfl_xor_sync(0xffffffffu, m.mean, o);
        b.m2 = __shfl_xor_sync(0xffffffffu, m.m2, o);
        b.m3 = __shfl_xor_sync(0xffffffffu, m.m3, o);
        b.m4 = __shfl_xor_sync(0xffffffffu, m.m4, o);
        m = moments_merge(m, b);
    }
    __device__ __forceinline__ void merge(const GroupMoments& o) { m = moments_merge(m, o.m); }
};

template <typename T> struct GroupFlip {
    static constexpr unsigned long long value = IsFloat<T>::value ? 0ull : (((T)-1 < (T)0) ? (1ull << (8 * sizeof(T) - 1)) : 0ull);
};

}  // namespace bdf
