// math_exact.cuh -- the few float functions whose CUDA libm result misses an exactly representable true value.
//
// CUDA documents these functions to 1-2 ulp, and that holds, but a user expects log2(2^k) == k, log10(1e9) == 9 and
// hypot(x, tiny) == x, as glibc (the reference's libm) returns them.  On sm_90a (CUDA 12.9) log2(2^k) is 1 ulp away
// from k for part of the powers of two (2^-126, 2^-500, 2^500, ...), log10f(1e9f) = 9.000001f, and hypot(x, y) can be
// 1 ulp above x when y is negligible next to x -- which overflows hypot(DBL_MAX, 1) to +inf.  Each wrapper returns the
// exact result at those inputs and CUDA's everywhere else (bit for bit), selected after both are computed so that lanes
// do not diverge.  Shared by the unfused kernels (k_unary.cu, k_binary.cu) and the fused one (k_expr.cu), so both
// paths agree bit for bit.
#pragma once

namespace bdf {

// log2 of a double: x = 2^k (normal or subnormal) -> k exactly.  CUDA's log2 is within 1 ulp of k there, so rint
// gives k.  The check reads the bits with 32-bit integer instructions only: log2 f64 runs at the HBM rate without it,
// and costs 4.5% more with it (1e8 rows: 0.553 -> 0.578 ms on an H100 80GB HBM3 at 400 W), where frexp or 64-bit bit
// tests cost 9% and 13%.  An empty significand also matches +-0, +-inf and the negative powers of two, where
// rint(log2(x)) = log2(x) (-inf, +inf, NaN).
__device__ __forceinline__ double log2_exact(double x) {
    const double y = log2(x);
    const int hi = __double2hiint(x);
    const unsigned lo = (unsigned)__double2loint(x);
    const bool empty_significand = (lo | ((unsigned)hi & 0xfffffu)) == 0u;
    const bool one_bit_subnormal = (hi >> 20) == 0 && __popc(hi) + __popc(lo) == 1;
    return (empty_significand || one_bit_subnormal) ? rint(y) : y;
}

// log10 of a float: x = 10^k (k = 0..10, every power of ten a float holds exactly) -> k exactly.
__device__ __forceinline__ float log10_exact(float x) {
    const float y = log10f(x);
    const float k = rintf(y);
    const int n = (int)k;
    float p = 1.0f, b = 10.0f;   // p = 10^n by squaring: every factor and partial product is exact for n <= 10
#pragma unroll
    for (int i = 0; i < 4; i++) {
        if (n & (1 << i)) p = __fmul_rn(p, b);
        b = __fmul_rn(b, b);
    }
    return (k >= 0.0f && k <= 10.0f && x == p) ? k : y;
}

// hypot of doubles: with s = min(|a|, |b|) <= t * 2^-27, t = max(|a|, |b|), the true value t (1 + (s/t)^2 / 2 + ...)
// is within a quarter ulp of t, so t is the correctly rounded result.  A NaN operand never takes this path (the
// comparisons are false), so hypot(+-inf, NaN) = +inf and hypot(NaN, y) = NaN stay CUDA's.
__device__ __forceinline__ double hypot_exact(double a, double b) {
    const double h = hypot(a, b);
    const double x = fabs(a), y = fabs(b);
    const double t = x > y ? x : y, s = x > y ? y : x;
    return s <= t * 0x1p-27 ? t : h;
}

}  // namespace bdf
